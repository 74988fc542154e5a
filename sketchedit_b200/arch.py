"""Layer tables of the two generator networks on the hot path.

This is the single source of truth for layer names (== state_dict key prefixes),
shapes and gating activations. It restates the constructors of the reference
networks:

  * netM = MDGenerator          (reference models/networks/editline2_g.py:14-43)
  * netG = DeepFillC2Generator  (reference models/networks/editline_g.py:25-100)

and the gated-conv contract of reference models/networks/utils.py:9-51
(``gen_conv`` pads by ``rate*(k-1)/2``; ``gen_deconv`` = nearest x2 + 3x3 conv;
a layer whose cout is 3 or whose activation is None returns the raw conv).
"""
from collections import namedtuple

CNUM = 48

# kind: "conv" | "deconv" (nearest x2 upsample first);  act: "elu" | "relu" | None (raw)
LayerSpec = namedtuple("LayerSpec", "name cin cout k stride rate kind act")


def _c(name, cin, cout, k=3, stride=1, rate=1, act="elu"):
    if cout == 3:          # reference utils.py:27 -- cout==3 short-circuits the gate
        act = None
    return LayerSpec(name, cin, cout, k, stride, rate, "conv", act)


def _d(name, cin, cout):
    return LayerSpec(name, cin, cout, 3, 1, 1, "deconv", "elu")


def _encoder(prefix, cin0, c=CNUM):
    """conv1..conv10_atrous trunk shared by netM.conv*, netG.conv*, netG.wconv*."""
    return [
        _c(prefix + "conv1", cin0, c, 5),
        _c(prefix + "conv2_downsample", c // 2, 2 * c, 3, 2),
        _c(prefix + "conv3", c, 2 * c),
        _c(prefix + "conv4_downsample", c, 4 * c, 3, 2),
        _c(prefix + "conv5", 2 * c, 4 * c),
        _c(prefix + "conv6", 2 * c, 4 * c),
        _c(prefix + "conv7_atrous", 2 * c, 4 * c, rate=2),
        _c(prefix + "conv8_atrous", 2 * c, 4 * c, rate=4),
        _c(prefix + "conv9_atrous", 2 * c, 4 * c, rate=8),
        _c(prefix + "conv10_atrous", 2 * c, 4 * c, rate=16),
    ]


def _decoder(prefix, cin11, cout17, c=CNUM):
    """convNN11..17 decoder; prefix is 'conv', 'conv_mask_' or 'allconv'."""
    return [
        _c(prefix + "11", cin11, 4 * c),
        _c(prefix + "12", 2 * c, 4 * c),
        _d(prefix + "13_upsample_conv", 2 * c, 2 * c),
        _c(prefix + "14", c, 2 * c),
        _d(prefix + "15_upsample_conv", c, c),
        _c(prefix + "16", c // 2, c // 2),
        _c(prefix + "17", c // 4, cout17, act=None),
    ]


def netM_layers():
    c = CNUM
    return _encoder("", 4) + _decoder("conv", 2 * c, 3) + _decoder("conv_mask_", 2 * c, 1)


def netG_layers():
    c = CNUM
    ls = _encoder("", 5) + _decoder("conv", 4 * c, 3) + _encoder("w", 5)
    ls += [
        _c("xconv1", 3, c, 5),
        _c("xconv2_downsample", c // 2, c, 3, 2),
        _c("xconv3", c // 2, 2 * c),
        _c("xconv4_downsample", c, 2 * c, 3, 2),
        _c("xconv5", c, 4 * c),
        _c("xconv6", 2 * c, 4 * c),
        _c("xconv7_atrous", 2 * c, 4 * c, rate=2),
        _c("xconv8_atrous", 2 * c, 4 * c, rate=4),
        _c("xconv9_atrous", 2 * c, 4 * c, rate=8),
        _c("xconv10_atrous", 2 * c, 4 * c, rate=16),
        _c("pmconv1", 3, c, 5),
        _c("pmconv2_downsample", c // 2, c, 3, 2),
        _c("pmconv3", c // 2, 2 * c),
        _c("pmconv4_downsample", c, 4 * c, 3, 2),
        _c("pmconv5", 2 * c, 4 * c),
        _c("pmconv6", 2 * c, 4 * c, act="relu"),   # editline_g.py:89-90
        _c("pmconv9", 2 * c, 4 * c),
        _c("pmconv10", 2 * c, 4 * c),
    ]
    ls += _decoder("allconv", 4 * c, 3)
    return ls


NET_LAYERS = {"M": netM_layers(), "G": netG_layers()}


def layer_map(net):
    return {l.name: l for l in NET_LAYERS[net]}


def out_channels_after_gate(l):
    return l.cout if l.act is None else l.cout // 2


def conv_flops_per_image(H, W):
    """2*MAC over all 76 convs, full pre-gate cout (SURVEY.md section 8d convention)."""
    total = 0
    for net in ("M", "G"):
        for l in NET_LAYERS[net]:
            h, w = _out_hw(l.name, H, W)
            total += 2 * h * w * l.cout * l.cin * l.k * l.k
    return total


def dead_flops_per_image(H, W):
    """2*MAC of netM's image decoder conv11-17: computed by the reference but unused by mode='inference'
    (reference models/editline2_model.py:128-133 drops mask_image), skipped here."""
    total = 0
    for l in NET_LAYERS["M"]:
        if l.name.startswith("conv1") and l.name[4:6] in ("11", "12", "13", "14", "15", "16", "17"):
            h, w = _out_hw(l.name, H, W)
            total += 2 * h * w * l.cout * l.cin * l.k * l.k
    return total


def cam_flops_per_image(H, W, c=2 * CNUM, patch=4, stride=2):
    """QK^T + AV of the contextual attention (SURVEY.md section 8d): 4*L*N*d."""
    h, w = H // 4, W // 4
    hs, ws = (h - patch) // stride + 1, (w - patch) // stride + 1
    L = hs * ws
    return 4 * L * L * c * patch * patch


def _out_hw(name, H, W):
    import re
    return _out_hw_at_index(int(re.search(r"(\d+)", name).group(1)), H, W)


def in_hw(name, H, W):
    """input size of layer `name` in an H x W forward: the output size of the layer before it."""
    import re
    idx = int(re.search(r"(\d+)", name).group(1))
    return (H, W) if idx == 1 else _out_hw_at_index(idx - 1, H, W)


def _out_hw_at_index(idx, H, W):
    """output size of the layers numbered idx (conv<idx>, xconv<idx>, conv_mask_<idx>, ...) in an H x W forward."""
    if idx == 1:
        return H, W
    if idx in (2, 3):
        return H // 2, W // 2
    if 4 <= idx <= 12:
        return H // 4, W // 4
    if idx in (13, 14):
        return H // 2, W // 2
    return H, W

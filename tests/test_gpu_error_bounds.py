"""Kernels against float64 with per-element error bounds (tests/util_bounds.py), at the inputs, shapes and masks where they
go wrong; and forward call forms against the oracle.

* Gated convolutions, every layer of test_gpu_ops.py LAYER_CASES in bf16, split-half fp32 and fp32_direct: at the map the
  layer sees in a 16 x 16 forward, on an output one tile high and one narrower than a tile, with pre-activations near 0
  (ELU's polynomial branch), O(1), saturated, an all-zero input (y = act(b_f) sigmoid(b_g)) and, split-half only, inputs
  up to +-1000; and the many-tile shapes of test_gpu_c8_many_tiles.py.
* Contextual attention in its three kernels (split-half GEMMs, fp32 CUDA cores with the attention map, bf16 wgmma) on
  maps with one key, one patch row or column, L = 128 k +- 1 keys, and masks that are all hole, all valid, one valid
  key, valid fractions 25/256 and 26/256 either side of the 0.1 threshold, and different per image.
* Forward call forms at 16 x 16, 16 x 256, 256 x 16 and 24 x 40, every reference-golden flag set in bf16, netG with
  different x / x2 and mask / mask2, and guide=None in bf16 (tolerances and flip rules of test_gpu_forward.py).

Each bound check reports max |y - Y| / bound.
"""
import glob
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from tests import util_bounds as UB
from tests.test_gpu_c8_many_tiles import MANY_TILE_CASES
from tests.test_gpu_forward import TOL, _golden_inputs
from tests.test_gpu_ops import LAYER_CASES
from tests.util_attention import contextual_attention_at
from tests.util_parity import engine, maxdiff, weights

pytestmark = pytest.mark.gpu
PRECS = ["bf16", "fp32", "fp32_direct"]


def _conv_ratio(net, name, x, prec):
    y = engine().gated_conv(net, name, x.cuda(), precision=prec).cpu()
    r = UB.reference(net, name, x, prec)
    assert y.shape == r["Y"].shape, (y.shape, r["Y"].shape)
    if prec == "fp32":
        assert float(x.abs().max()) <= UB.SPLIT_MAX and float(r["Y"].abs().max()) <= UB.SPLIT_MAX   # inside the split range
    return UB.max_ratio(y, r["Y"], UB.gated_bound(r, prec))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("net,name", [(n, l) for n, l, _, _ in LAYER_CASES])
def test_gated_conv_within_bound(net, name, prec):
    worst = (0.0, None)
    for label, B, H, W in UB.conv_sizes(net, name):
        for regime in UB.conv_regimes(prec, label, UB.layer(net, name)[0]):
            x = UB.conv_input(net, name, B, H, W, regime, UB.stable_seed(net, name, label, regime))
            worst = max(worst, (_conv_ratio(net, name, x, prec), (label, H, W, regime)))
    print("bound %s %s.%s: max ratio %.3g at %s" % (prec, net, name, worst[0], worst[1]))
    assert worst[0] <= 1.0, (net, name, prec, worst)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("net,name,H,W", MANY_TILE_CASES)
def test_gated_conv_many_tiles_within_bound(net, name, H, W, prec):
    x = UB.conv_input(net, name, 3, H, W, "unit", UB.stable_seed(net, name, H, W))
    q = _conv_ratio(net, name, x, prec)
    print("bound %s %s.%s many tiles: max ratio %.3g" % (prec, net, name, q))
    assert q <= 1.0, (net, name, prec, q)


# --------------------------------------------------------------------------------------------- contextual attention
# feature maps (h, w): L = 1 (4 x 4), one patch row / column, L = 127, 129, 255, 257
CAM_MAPS = [(4, 4), (4, 64), (64, 4), (256, 4), (88, 8), (32, 36), (516, 4)]
CAM_MASKS = ["hole", "valid", "one_key", "frac25_26", "rect"]


def _mask_s(kind, B, h, w):
    """mask_s (hole fraction per cell) of the attention."""
    m = torch.zeros(B, 1, h, w)
    if kind == "hole":
        m[:] = 1.0                                  # every key masked: every logit is 0
    elif kind == "one_key":
        m[:] = 1.0
        m[:, :, :2, :2] = 0.0                       # key (0, 0) sees 4 of 16 valid cells; its neighbours none
    elif kind == "frac25_26":
        m[:] = 1.0 - 25.0 / 256                     # valid fraction 25/256 < 0.1: masked
        m[..., w // 2:] = 1.0 - 26.0 / 256          # 26/256 > 0.1: valid
    elif kind == "rect":
        m[:, :, h // 4:3 * h // 4, w // 4:w // 2 + 2] = 1.0
    return m


def _feat(kind, B, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "zero":
        return torch.zeros(B, 96, h, w)
    f = F.relu(torch.randn(B, 96, h, w, generator=g))            # pmconv6 outputs are ReLU-gated: non-negative
    if kind == "zero_plane":
        f[:, 5] = 0.0                                            # rnorm of that plane = 1 / sqrt(1e-8)
        return f * 0.5
    return f * float(kind)


CAM_CASES = [(h, w, 1, m, "0.15") for h, w in CAM_MAPS for m in CAM_MASKS]
CAM_CASES += [(32, 36, 1, m, f) for m in ("rect", "valid") for f in ("1e-3", "1", "5", "zero", "zero_plane")]
CAM_CASES += [(32, 32, 2, "per_image", "0.15")]


def _cam_inputs(h, w, B, mkind, fkind):
    feat = _feat(fkind, B, h, w, seed=UB.stable_seed(h, w, B, mkind, fkind))
    if mkind == "per_image":                                     # image 0 all hole, image 1 one rectangle
        mask_s = torch.cat([_mask_s("hole", 1, h, w), _mask_s("rect", 1, h, w)])
    else:
        mask_s = _mask_s(mkind, B, h, w)
    return feat, mask_s


@pytest.mark.parametrize("mode", ["fp32", "fp32_attn", "bf16"])
@pytest.mark.parametrize("h,w,B,mkind,fkind", CAM_CASES)
def test_contextual_attention_within_bound(h, w, B, mkind, fkind, mode):
    from sketchedit_b200.engine import contextual_attention
    feat, mask_s = _cam_inputs(h, w, B, mkind, fkind)
    prec = "fp32_direct" if mode == "fp32_attn" else mode       # the attention-map form runs the fp32 CUDA-core kernels
    if mode == "fp32_attn":
        out, attn = contextual_attention(feat.cuda(), mask_s.cuda(), precision="fp32", want_attn=True)
    else:
        out = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec)
    out = out.cpu().double()
    if prec == "bf16":
        ref, bound = UB.attention_bf16_reference(feat, mask_s)
        q = UB.max_ratio(out, ref, bound)
        print("bound attention %s %dx%d B%d %s feat %s: max ratio %.3g" % (mode, h, w, B, mkind, fkind, q))
        assert q <= 1.0, q
        return
    px = [(b, y, x) for b in range(B) for y in range(h) for x in range(w)]
    err = UB.attention_err(prec, 96, h, w)
    ref, t = contextual_attention_at(feat, mask_s, px, err=err)
    got = torch.stack([out[b, :, y, x] for b, y, x in px])
    q = UB.max_ratio(got, ref, UB.attention_out_bound(t["bound"], ref, err["out"]))
    print("bound attention %s %dx%d B%d %s feat %s: max ratio %.3g" % (mode, h, w, B, mkind, fkind, q))
    assert q <= 1.0, q
    if mode == "fp32_attn":
        # the attention map against fp64: P_l moves by at most P_l (exp(2 delta_n) - 1 + rel)
        A, bA = UB.attention_fp32_map(feat, mask_s)
        qa = UB.max_ratio(attn.cpu(), A, bA)
        print("bound attention map %dx%d %s feat %s: max ratio %.3g" % (h, w, mkind, fkind, qa))
        assert qa <= 1.0, qa


# --------------------------------------------------------------------------------------------- forward call forms
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("H,W", [(16, 16), (16, 256), (256, 16), (24, 40)])
def test_inference_small_and_thin_inputs(prec, H, W):
    WM, WG = weights()
    img, sk = synth.synth_inputs(1, H, W, seed=H * 7 + W)
    composed, mask, ex = engine().inference(img.cuda(), sk.cuda(), precision=prec, want=("coarse", "fine", "mask_bin"))
    ours_bin = ex["mask_bin"].cpu()
    flips = int((ours_bin != O.inference(WM, WG, img, sk)["mask_bin"]).sum())
    assert flips <= (0 if prec.startswith("fp32") else 0.02 * ours_bin.numel()), flips
    ref = O.inference(WM, WG, img, sk, mask_bin_override=ours_bin)
    assert maxdiff(mask.cpu(), ref["mask"]) <= TOL[prec]
    for k, t in (("coarse", ex["coarse"]), ("fine", ex["fine"]), ("composed", composed)):
        assert maxdiff(t.cpu(), ref[k]) <= TOL[prec], (k, maxdiff(t.cpu(), ref[k]))


GOLDEN = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


@pytest.mark.parametrize("name", GOLDEN)
def test_bf16_golden_flags_vs_oracle(name, golden_dir):
    """every flag set of the reference goldens (avg pool, use_cam=False, no_mask_cc, no_mask_coarse, joint_train_inp=False)
    in bf16, against the oracle run with the same flags on our binarised mask; at most 2 % threshold flips."""
    WM, WG = weights()
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    image, sketch = _golden_inputs(z)
    flags = dict(eval(str(z["flags"])))
    composed, mask, ex = engine(**flags).inference(image.cuda(), sketch.cuda(), precision="bf16", want=("coarse", "fine", "mask_bin"))
    ours_bin = ex["mask_bin"].cpu()
    flips = int((ours_bin != O.inference(WM, WG, image, sketch, **flags)["mask_bin"]).sum())
    assert flips <= 0.02 * ours_bin.numel(), flips
    ref = O.inference(WM, WG, image, sketch, mask_bin_override=ours_bin, **flags)
    assert maxdiff(mask.cpu(), ref["mask"]) <= TOL["bf16"]
    for k, t in (("coarse", ex["coarse"]), ("fine", ex["fine"]), ("composed", composed)):
        assert maxdiff(t.cpu(), ref[k]) <= TOL["bf16"], (k, maxdiff(t.cpu(), ref[k]))


def _netG_inputs():
    """x2 is a black and white checkerboard (inside the image range [-1, 1]) and mask2 covers most of the image: the style
    branch's global max pool damps x2, and a smooth x2 would change the outputs by less than the bf16 tolerance."""
    img, sk = synth.synth_inputs(2, 64, 64, seed=31)
    yy, xx = torch.meshgrid(torch.arange(64), torch.arange(64), indexing="ij")
    img2 = (((yy // 8 + xx // 8) % 2) * 2 - 1).float().expand(2, 3, 64, 64).contiguous()
    mask = torch.zeros(2, 1, 64, 64)
    mask[0, :, 16:40, 8:50] = 1
    mask[1, :, 30:60, 20:44] = 1
    mask2 = torch.ones(2, 1, 64, 64)
    mask2[0, :, 40:, :] = 0
    mask2[1, :, :, 48:] = 0
    return img, img2, mask, mask2, sk


@pytest.mark.parametrize("prec", PRECS)
def test_netG_unpaired_inputs(prec):
    """x != x2 and mask != mask2, passed as separate tensors: reading the wrong one of a pair changes the output."""
    _, WG = weights()
    img, img2, mask, mask2, sk = _netG_inputs()
    s1, s2 = engine().netG(img.cuda(), img2.cuda(), mask.cuda(), mask2.cuda(), sk.cuda(), precision=prec)
    r1, r2 = O.netG_forward(WG, img, img2, mask, mask2, sk)
    assert maxdiff(s1.cpu(), r1) <= TOL[prec], maxdiff(s1.cpu(), r1)
    assert maxdiff(s2.cpu(), r2) <= TOL[prec], maxdiff(s2.cpu(), r2)
    # reading x for x2, or mask for mask2, would move the outputs by more than the tolerance
    for wrong in ((img, img, mask, mask2, sk), (img, img2, mask, mask, sk)):
        w1, w2 = O.netG_forward(WG, *wrong)
        assert max(maxdiff(r1, w1), maxdiff(r2, w2)) > 3 * TOL[prec]


def test_netG_without_guide_bf16():
    _, WG = weights()
    img, img2, mask, mask2, _ = _netG_inputs()
    s1, s2 = engine().netG(img.cuda(), img2.cuda(), mask.cuda(), mask2.cuda(), None, precision="bf16")
    r1, r2 = O.netG_forward(WG, img, img2, mask, mask2, None)
    assert maxdiff(s1.cpu(), r1) <= TOL["bf16"], maxdiff(s1.cpu(), r1)
    assert maxdiff(s2.cpu(), r2) <= TOL["bf16"], maxdiff(s2.cpu(), r2)

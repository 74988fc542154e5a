"""CPU oracle for the SketchEdit generator forward pass  --  TEST INFRASTRUCTURE ONLY.

This file is the checker, never the product: only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may import it. The shipped
path (``sketchedit_b200`` + ``models``) never does, and fails loudly without its CUDA
library.

It is an independent fp32 restatement (plain torch-CPU functional ops, no nn.Module,
weights passed as a ``{name: tensor}`` dict in the reference's state_dict format) of

  * gated conv / nearest-x2 deconv      reference models/networks/utils.py:9-51
  * contextual attention P1 + P2       reference models/networks/splitcam.py:37-108,132-174
                                        (+ batch_conv2d / batch_transposeconv2d, utils.py:72-128)
    written here in attention form  A = softmax_l(10 * (Q K^T) * m_l),  out = fold_sum(A V)
  * MDGenerator.forward  (netM)        reference models/networks/editline2_g.py:59-94
  * DeepFillC2Generator.forward (netG) reference models/networks/editline_g.py:119-221
  * EditLine2Model inference           reference models/editline2_model.py:128-133,338-370

Pinning: the reference ships no tests or golden vectors for this path (SURVEY.md section 4)
and no checkpoints, so the oracle is pinned against OUTPUTS OF THE REFERENCE ITSELF:
``oracle/make_golden.py`` imports the unmodified reference from the reference checkout (SKETCHEDIT_REFERENCE) where it is
container, runs it on seeded synthetic checkpoints (``oracle/synth.py``) and commits the
results under ``tests/golden/``; ``tests/test_oracle_golden.py`` checks this file against
them (fp32, max-abs <= 2e-5).
"""
import torch
import torch.nn.functional as F

from sketchedit_b200.arch import NET_LAYERS, layer_map

_LM = {"M": layer_map("M"), "G": layer_map("G")}


# ----------------------------------------------------------------------------- gated conv
def gated_conv(x, w, b, spec):
    """reference utils.py:25-33 (gen_conv.forward) and :48-51 (gen_deconv.forward)."""
    if spec.kind == "deconv":
        x = F.interpolate(x, scale_factor=2, mode="nearest")       # utils.py:49
    pad = int(spec.rate * (spec.k - 1) / 2)                       # utils.py:21
    y = F.conv2d(x, w, b, stride=spec.stride, padding=pad, dilation=spec.rate)
    if spec.act is None:                                          # utils.py:27
        return y
    half = spec.cout // 2
    f, g = y[:, :half], y[:, half:]
    f = F.elu(f) if spec.act == "elu" else F.relu(f)
    return f * torch.sigmoid(g)


def _run(net, W, name, x):
    spec = _LM[net][name]
    return gated_conv(x, W[name + ".weight"], W[name + ".bias"], spec)


def _chain(net, W, names, x, taps=None):
    for n in names:
        x = _run(net, W, n, x)
        if taps is not None:
            taps[("net" + net + "." + n)] = x
    return x


# ----------------------------------------------------------------------------- attention
def patches(x, k=4, s=2):
    """F.unfold order (c, u, v) -> [B, L, C*k*k]   (splitcam.py:42-44)."""
    return F.unfold(x, kernel_size=k, stride=s).transpose(1, 2)


def contextual_attention(feat, mask_s, patch=4, stride=2, th=0.1, scale=10.0):
    """cam_1 + cam_2 of netG with the constructor arguments of editline_g.py:35-42.

    feat   [B, C, h, w]  query, key and value source (cam_1(x, x, mask_s); cam_2(.., x, ..))
    mask_s [B, 1, h, w]  fraction of hole per cell (avg_pool2d(mask, 4, 4))
    Returns (out [B, C, h, w], attn [B, L, N]).
    """
    B, C, h, w = feat.shape
    valid = 1.0 - mask_s                                                    # splitcam.py:62-63
    # keys: plane-normalised per (batch, channel)                           splitcam.py:39-40
    fn = feat / torch.sqrt((feat ** 2).sum(3, keepdim=True).sum(2, keepdim=True) + 1e-8)
    K = patches(fn, patch, stride)                                          # [B, L, d]
    Q = patches(feat, patch, stride)                                        # [B, N, d] (unnormalised, :68-69)
    V = Q                                                                   # mk=False, raw values :137-141
    mmk = patches(valid, patch, stride).mean(2)                             # [B, L]    :49-53
    m = (mmk > th).to(feat.dtype)                                           # is_th     :89-90
    S = torch.einsum("bnd,bld->bln", Q, K)                                  # scores[b, l, n]
    S = S * m[:, :, None]                                                   # masked logits -> 0 (not -inf) :104
    A = torch.softmax(S * scale, dim=1)                                     # over keys l   :105
    O = torch.einsum("bln,bld->bnd", A, V)                                  # [B, N, d]
    out = F.fold(O.transpose(1, 2), output_size=(h, w), kernel_size=patch, stride=stride)   # fold-SUM :152
    return out, A


# ----------------------------------------------------------------------------- netM
def netM_forward(W, x, guide, taps=None):
    """MDGenerator.forward, editline2_g.py:59-94.  Returns (mask1, x_stage1)."""
    z = torch.cat([x, guide], 1)
    enc = ["conv1", "conv2_downsample", "conv3", "conv4_downsample", "conv5", "conv6",
           "conv7_atrous", "conv8_atrous", "conv9_atrous"]
    z9 = _chain("M", W, enc, z, taps)
    bneck = _run("M", W, "conv10_atrous", z9)
    if taps is not None:
        taps["netM.conv10_atrous"] = bneck
    # NOTE editline2_g.py:76-77: conv11 consumes the conv9 output, NOT the bottleneck
    img = _chain("M", W, ["conv11", "conv12", "conv13_upsample_conv", "conv14",
                          "conv15_upsample_conv", "conv16", "conv17"], z9, taps)
    x_stage1 = torch.tanh(img)
    mk = _chain("M", W, ["conv_mask_11", "conv_mask_12", "conv_mask_13_upsample_conv", "conv_mask_14",
                         "conv_mask_15_upsample_conv", "conv_mask_16", "conv_mask_17"], bneck, taps)
    return torch.sigmoid(mk), x_stage1


# ----------------------------------------------------------------------------- netG
def netG_forward(W, x, x2, mask, mask2, guide, use_cam=True, pool_type="max",
                 no_mask_cc=False, no_mask_coarse=False, joint_train_inp=True, taps=None):
    """DeepFillC2Generator.forward, editline_g.py:119-221.  Returns (x_stage1, x_stage2)."""
    if not no_mask_cc:
        x2 = x2 * mask2
    x = x * (1 - mask)
    xin = x
    ones_x = torch.ones_like(mask) if guide is None else guide
    x = torch.cat([x, ones_x, mask], 1)
    x2 = torch.cat([x2, ones_x * 0 if joint_train_inp else ones_x, mask2], 1)
    trunk = ["conv1", "conv2_downsample", "conv3", "conv4_downsample", "conv5", "conv6",
             "conv7_atrous", "conv8_atrous", "conv9_atrous", "conv10_atrous"]
    x = _chain("G", W, trunk, x, taps)
    x2 = _chain("G", W, ["w" + n for n in trunk], x2, taps)
    hs, ws = x2.shape[2:]
    if pool_type == "avg":
        x2 = x2.mean(3).mean(2)[..., None, None]
    elif pool_type == "max":
        x2 = F.max_pool2d(x2, kernel_size=(hs, ws))
    else:
        raise NotImplementedError(pool_type)
    x2 = x2.expand(-1, -1, hs, ws)                                 # nearest 1x1 -> hs x ws (:166)
    x = torch.cat((x, x2), 1)
    x = _chain("G", W, ["conv11", "conv12", "conv13_upsample_conv", "conv14",
                        "conv15_upsample_conv", "conv16", "conv17"], x, taps)
    x_stage1 = torch.tanh(x)
    x = x_stage1
    if not no_mask_coarse:
        x = x * mask + xin[:, 0:3] * (1.0 - mask)
    xnow = x
    xh = _chain("G", W, ["x" + n for n in trunk], xnow, taps)
    pm = _chain("G", W, ["pmconv1", "pmconv2_downsample", "pmconv3", "pmconv4_downsample",
                         "pmconv5", "pmconv6"], xnow, taps)
    if use_cam:
        mask_s = F.avg_pool2d(mask, kernel_size=4, stride=4)
        pm, _ = contextual_attention(pm, mask_s)
        if taps is not None:
            taps["netG.cam"] = pm
    pm = _chain("G", W, ["pmconv9", "pmconv10"], pm, taps)
    x = torch.cat([xh, pm], 1)
    x = _chain("G", W, ["allconv11", "allconv12", "allconv13_upsample_conv", "allconv14",
                        "allconv15_upsample_conv", "allconv16", "allconv17"], x, taps)
    return x_stage1, torch.tanh(x)


# ----------------------------------------------------------------------------- model
def inference(WM, WG, image, sketch, mask_bin_override=None, taps=None, **flags):
    """EditLine2Model.forward(data, mode='inference'), editline2_model.py:128-133 + 338-370.

    Returns dict(composed, mask, mask_bin, coarse, fine, mask_image).
    ``mask_bin_override`` lets a parity test feed an externally binarised mask into netG
    (the threshold at editline2_model.py:347 is discontinuous, SURVEY.md section 7.3-2).
    """
    with torch.no_grad():
        mask, mask_image = netM_forward(WM, image, sketch, taps)
        mask_bin = (mask > 0.5).float() if mask_bin_override is None else mask_bin_override
        coarse, fine = netG_forward(WG, image, image, mask_bin, mask_bin, sketch, taps=taps, **flags)
        composed = fine * mask + image * (1 - mask)                 # SOFT mask, :132
    return dict(composed=composed, mask=mask, mask_bin=mask_bin, coarse=coarse, fine=fine,
                mask_image=mask_image)


def to_uint8_outputs(composed, mask):
    """test.py:25-27 output conversion (truncation, no clamp, no rounding)."""
    import numpy as np
    m = (mask * 255).cpu().numpy().astype(np.uint8)[:, 0]
    g = ((composed + 1) / 2 * 255).cpu().numpy().astype(np.uint8)
    return g, m

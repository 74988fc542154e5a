"""The per-element error bounds of tests/util_bounds.py are tight enough to catch subtly wrong kernels (CPU only).

torch-CPU emulations restate the arithmetic of each mode: bf16 operands with fp32 accumulation and a bf16 output; the
split-half mode as three fp16 products per tap (x_hi w_hi + x_hi w_lo + x_lo w_hi, conv by unfold, fp32 accumulation, as in
test_split_half_math.py) with gate_one_exact's ELU / sigmoid in fp32 and a re-split output; fp32 FMA chains for
fp32_direct. On the inputs the GPU tests use (tests/test_gpu_error_bounds.py), every unmutated emulation satisfies its
bound, and each of the mutations below violates it (max |y - Y| / bound > 1), each one a plausible kernel bug that the
per-layer tolerances of test_gpu_ops.py (1e-4 for the fp32 modes, 2^-8 max|y| + 1e-3 for bf16) pass or only just fail.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import util_bounds as UB
from tests.test_gpu_ops import LAYER_CASES
from tests.util_parity import oracle_layer

LAYERS = [(net, name) for net, name, _, _ in LAYER_CASES]


def conv_unfold(x, w, bias=None, stride=1, padding=0, dilation=1):
    """F.conv2d as one fp32 matmul over unfolded patches (the GEMM form of the kernels)."""
    B, _, H, W = x.shape
    Co, _, kh, kw = w.shape
    cols = F.unfold(x, (kh, kw), dilation=dilation, padding=padding, stride=stride)
    Ho = (H + 2 * padding - dilation * (kh - 1) - 1) // stride + 1
    Wo = (W + 2 * padding - dilation * (kw - 1) - 1) // stride + 1
    return (w.reshape(Co, -1) @ cols).view(B, Co, Ho, Wo)


def split(v, scale):
    """hi / lo fp16 halves (as fp32) of scale * v, saturated like se_common.cuh kSplitActMax."""
    s = (v * scale).clamp(-65000.0, 65000.0)
    hi = UB.f16(s)
    return hi, UB.f16(s - hi)


def expm1_poly(f, c3=1.0 / 6.0):
    """gate_one_exact's degree-5 Taylor polynomial of expm1 (Horner, fp32)."""
    return f * (((((f / 120.0 + 1.0 / 24.0) * f + c3) * f + 0.5) * f) + 1.0)


def gate_exact(f, g, spec, c3=1.0 / 6.0):
    """gate_one_exact in fp32 (ex2 / rcp approximations replaced by fp32 exp / divide)."""
    if spec.act == "elu":
        a = torch.where(f > 0, f, torch.where(f > -0.0625, expm1_poly(f, c3), torch.exp(f) - 1.0))
    else:
        a = torch.relu(f)
    return a * (1.0 / (1.0 + torch.exp(-g)))


def packed_weights(spec, w, round_bf16=False, per_tap_round=False):
    """weights as packed: gate rows x 0.5, deconvs folded into their sub-pixel classes."""
    w = w.float().clone()
    if not UB.is_head(spec):
        w[spec.cout // 2:] *= 0.5
    if spec.kind == "deconv":
        return UB.folded_deconv_weights(w, round_bf16=round_bf16, per_tap_round=per_tap_round)
    return UB.bf16(w) if round_bf16 else w


def emulate(net, name, x, prec, mutation=None):
    spec, w, b = UB.layer(net, name)
    b = b.float()[None, :, None, None]
    conv = lambda xx, ww: UB.conv_nobias(xx, ww, spec, conv_unfold)
    if UB.is_head(spec):                                     # heads: fp32 FMA on the CUDA cores (bf16: on bf16(x))
        xx = UB.bf16(x) if prec == "bf16" else x
        return conv(xx, w.float()) + b
    h = spec.cout // 2
    if prec == "bf16":
        wp = packed_weights(spec, w, round_bf16=True, per_tap_round=mutation == "deconv_round_per_tap")
        z = conv(UB.bf16(x), wp)
        f, g = z[:, :h] + b[:, :h], 2 * z[:, h:] + b[:, h:]
        y = (F.elu(f) if spec.act == "elu" else F.relu(f)) * torch.sigmoid(g)
        if mutation == "bf16_truncate":
            return (y.view(torch.int32) & -65536).view(torch.float32)
        return UB.bf16(y)
    if prec == "fp32_direct":
        z = conv(x, packed_weights(spec, w))
        f, g = z[:, :h] + b[:, :h], 2 * z[:, h:] + b[:, h:]
        return (F.elu(f) if spec.act == "elu" else F.relu(f)) * torch.sigmoid(g)
    # split-half
    s_act = 1.0 if mutation == "act_scale_1" else UB.ACT_SCALE
    s_w = UB.split_weight_scale(spec, w)
    wp = packed_weights(spec, w)
    ws = {k: split(v, s_w) for k, v in wp.items()} if isinstance(wp, dict) else split(wp, s_w)
    w_hi = {k: v[0] for k, v in ws.items()} if isinstance(ws, dict) else ws[0]
    w_lo = {k: v[1] for k, v in ws.items()} if isinstance(ws, dict) else ws[1]
    x_hi, x_lo = split(x, s_act)
    x_lo_w_hi = x_lo.clone()
    if mutation == "drop_xlo_whi_block":
        x_lo_w_hi[:, :8] = 0.0                             # the x_lo * w_hi product of channel block 0 is skipped
    acc = conv(x_hi, w_hi) + conv(x_hi, w_lo) + conv(x_lo_w_hi, w_hi)
    inv = 1.0 / (s_act * s_w)
    f, g = acc[:, :h] * inv + b[:, :h], 2 * (acc[:, h:] * inv) + b[:, h:]
    y = gate_exact(f, g, spec, c3=0.17 if mutation == "poly_coeff" else 1.0 / 6.0)
    y_hi, y_lo = split(y, s_act)
    if mutation == "hi_only_output":
        y_lo = torch.zeros_like(y_lo)
    return (y_hi + y_lo) / s_act


def todays_tolerance_passes(net, name, x, y, prec):
    """the per-layer check of test_gpu_ops.py applied to y."""
    spec = UB.layer(net, name)[0]
    if prec == "bf16":          # that test feeds bf16-representable inputs
        ref = oracle_layer(net, name, UB.bf16(x), bf16_weights=not UB.is_head(spec))
        tol = float(ref.abs().max()) * 2.0 ** -8 + 1e-3
        if spec.kind == "deconv":
            tol *= 2
    else:
        ref = oracle_layer(net, name, x, bf16_weights=False)
        tol = 1e-4
    return float((y - ref).abs().max()) <= tol


def check_ratio(net, name, x, prec, mutation=None):
    r = UB.reference(net, name, x, prec)
    y = emulate(net, name, x, prec, mutation)
    assert y.shape == r["Y"].shape
    return UB.max_ratio(y, r["Y"], UB.gated_bound(r, prec))


# --------------------------------------------------------------------------------------------- reference plumbing
@pytest.mark.parametrize("net,name", [("M", "conv13_upsample_conv"), ("M", "conv15_upsample_conv")])
def test_subpixel_classes_equal_nearest_upsample_conv(net, name):
    spec, w, _ = UB.layer(net, name)
    x = torch.randn(2, spec.cin, 5, 7, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    folded = {k: v.double() for k, v in UB.folded_deconv_weights(w.double(), round_bf16=False).items()}
    want = UB.conv_nobias(x, w.double(), spec)
    got = UB.subpixel_conv(x, folded)
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())   # the fold itself runs in fp32


# --------------------------------------------------------------------------------------------- unmutated: within the bounds
@pytest.mark.parametrize("prec", ["bf16", "fp32", "fp32_direct"])
@pytest.mark.parametrize("net,name", LAYERS)
def test_emulation_within_bound(net, name, prec):
    worst = (0.0, None)
    for label, B, H, W in UB.conv_sizes(net, name):
        for regime in UB.conv_regimes(prec):
            x = UB.conv_input(net, name, B, H, W, regime, UB.stable_seed(net, name, label, regime))
            q = check_ratio(net, name, x, prec)
            worst = max(worst, (q, (label, regime)))
    print("%s.%s %s: max bound ratio %.3g at %s" % (net, name, prec, worst[0], worst[1]))
    assert worst[0] <= 1.0, (name, prec, worst)


# --------------------------------------------------------------------------------------------- mutations: outside the bounds
# (mutation, precision, layers, regime): each is checked on layers where it applies, on the GPU tests' inputs
MUTATIONS = [
    ("drop_xlo_whi_block", "fp32", [("G", "conv1"), ("M", "conv16"), ("M", "conv3"), ("M", "conv5")], "unit"),
    ("poly_coeff", "fp32", [("M", "conv16"), ("M", "conv5"), ("G", "conv11")], "small"),
    ("hi_only_output", "fp32", [("M", "conv1"), ("M", "conv16"), ("M", "conv5"), ("G", "pmconv6")], "unit"),
    ("act_scale_1", "fp32", [("M", "conv16"), ("M", "conv5"), ("G", "conv11")], "small"),
    ("bf16_truncate", "bf16", [("M", "conv1"), ("M", "conv16"), ("M", "conv5"), ("G", "pmconv6")], "unit"),
    ("deconv_round_per_tap", "bf16", [("M", "conv13_upsample_conv"), ("M", "conv15_upsample_conv")], "unit"),
]


@pytest.mark.parametrize("mutation,prec,layers,regime", MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_mutation_violates_bound(mutation, prec, layers, regime):
    for net, name in layers:
        label, B, H, W = UB.conv_sizes(net, name)[1]          # the thin map: 8 x 56 outputs
        x = UB.conv_input(net, name, B, H, W, regime, UB.stable_seed(net, name, label, regime))
        q = check_ratio(net, name, x, prec, mutation)
        passes = todays_tolerance_passes(net, name, x, emulate(net, name, x, prec, mutation), prec)
        print("%s on %s.%s (%s): max bound ratio %.3g; the test_gpu_ops.py tolerance %s it"
              % (mutation, net, name, regime, q, "passes" if passes else "fails"))
        assert q > 1.0, (mutation, name, q)


# --------------------------------------------------------------------------------------------- bf16 contextual attention
def emulate_attention_bf16(feat, mask_s, mutation=None):
    """se_cam.cu in fp32: bf16 map, keys bf16(f * rnorm), fp32 logits and softmax, bf16 P, fp32 P V and fold, bf16 output."""
    f = UB.bf16(feat.float())
    B, C, h, w = f.shape
    rn = 1.0 / torch.sqrt((f ** 2).sum((2, 3), keepdim=True) + 1e-8)
    K, Q = F.unfold(UB.bf16(f * rn), 4, stride=2), F.unfold(f, 4, stride=2)
    valid = (F.unfold(1 - mask_s, 4, stride=2).mean(1) > 0.1).float()
    scale = 9.9 if mutation == "logit_scale_9.9" else 10.0
    P = UB.bf16(torch.softmax(scale * valid[:, :, None] * torch.einsum("bdl,bdn->bln", K, Q), 1))
    out = F.fold(torch.einsum("bln,bdl->bdn", P, Q), (h, w), 4, stride=2)
    if mutation == "output_x0.99":
        out = out * 0.99
    elif mutation == "zero_output":
        out = torch.zeros_like(out)
    return UB.bf16(out)


def _cam_case_ids():
    from tests.test_gpu_error_bounds import CAM_CASES
    return CAM_CASES


@pytest.mark.parametrize("h,w,B,mkind,fkind", _cam_case_ids())
def test_attention_bf16_bound(h, w, B, mkind, fkind):
    """the emulation satisfies the bound; an output 1 % small or zero exceeds it wherever the map is not all zero, and
    logits scaled by 9.9 instead of 10 exceed it on the mask sweep wherever a valid key exists (L > 1)."""
    from tests.test_gpu_error_bounds import _cam_inputs
    feat, mask_s = _cam_inputs(h, w, B, mkind, fkind)
    Y, bound = UB.attention_bf16_reference(feat, mask_s)
    q = {m: UB.max_ratio(emulate_attention_bf16(feat, mask_s, m), Y, bound)
         for m in (None, "output_x0.99", "zero_output", "logit_scale_9.9")}
    print("attention bf16 %dx%d B%d %s feat %s: max bound ratios %s" % (h, w, B, mkind, fkind, q))
    assert q[None] <= 1.0, q
    if fkind != "zero":
        assert q["output_x0.99"] > 1.0 and q["zero_output"] > 1.0, q
    has_key = bool((F.unfold(1 - mask_s, 4, stride=2).mean(1) > 0.1).any())
    if fkind == "0.15" and has_key and Y.shape[-1] * Y.shape[-2] > 16:
        assert q["logit_scale_9.9"] > 1.0, q

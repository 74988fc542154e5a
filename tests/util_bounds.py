"""float64 references of the gated convolutions and the contextual attention, with per-element error bounds of each
arithmetic mode (test infrastructure, like oracle/sketchedit_oracle.py).

A check is |y - Y| <= bound elementwise, where Y is the fp64 result on the operands the kernel really multiplies and the
bound is derived from the arithmetic of the mode (DESIGN.md section 3):

  bf16          operands bf16(x) and bf16(w) (gate columns pre-multiplied by 0.5: exact); deconv classes use the packer's
                folded sub-pixel weights (taps summed in fp32, rounded to bf16 once). Heads: bf16(x), fp32 weights.
  fp32 (split)  operands are the fp32 x and w; the split-half representation error goes into the bound.
  fp32_direct   operands are the fp32 x and w; fp32 FMA chains on the CUDA cores.

Pre-activation errors dz are propagated through the gate act(f) * sigmoid(g) with the mean-value bounds
|d/df| <= sigmoid(g + dg) and |d/dg| <= (|act(f)| + df) * sigmoid'(max(|g| - dg, 0)), then the epilogue's own rounding
and the output rounding are added. Every check reports max(|y - Y| / bound).
"""
import math

import torch
import torch.nn.functional as F

from sketchedit_b200.arch import in_hw, layer_map
from tests.util_parity import weights

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
U16 = 2.0 ** -11          # unit roundoff of fp16 (11 significant bits)
UBF = 2.0 ** -8           # unit roundoff of bf16 (8 significant bits)
U_SPLIT = 2.0 ** -22      # hi + lo split-half pair: |lo - (v - hi)| <= U16 * |v - hi| <= U16 * U16 * |v|
ACT_SCALE = 64.0          # se_common.cuh kSplitActScale
SPLIT_MAX = 65000.0 / ACT_SCALE   # se_common.cuh kSplitActMax: split-half values saturate beyond |v| = 1015.6
LOG2E = 1.4426950408889634

# Accumulation on the tensor cores. Products of bf16 / fp16 operands are exact in fp32; the fp32 accumulator of wgmma is
# not specified (earlier tensor cores align and truncate), so each k16 step is charged one truncating add, 2^-23 of the
# partial sum, and the partial sums are bounded by A = sum |x||w|. The steps' errors are taken to add like a random walk
# (probabilistic bound lambda * sqrt(n) * u of Higham and Mary) with lambda = 4: a constant chosen with margin, not derived.
LAMBDA_ACC = 4.0


def c_acc(n_add):
    """relative (to A) error of an fp32 tensor-core accumulation over n_add wgmma k16 steps (see LAMBDA_ACC)."""
    return LAMBDA_ACC * math.sqrt(n_add) * 2.0 ** -23


def bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def f16(t):
    return t.to(torch.float16).to(t.dtype)


def layer(net, name):
    WM, WG = weights()
    W = WM if net == "M" else WG
    return layer_map(net)[name], W[name + ".weight"], W[name + ".bias"]


def is_head(spec):
    return spec.act is None


# --------------------------------------------------------------------------------------------- operands of the kernels
# se_engine.cu pack_layer: nearest x2 + 3x3 == four sub-pixel 2x2 convolutions. Output row 2i + py reads input rows i + dy with
# kernel rows summed per (py, a); columns the same.
DECONV_ROWS = {(0, 0): [0], (0, 1): [1, 2], (1, 0): [0, 1], (1, 1): [2]}


def folded_deconv_weights(w, round_bf16, per_tap_round=False):
    """{(py, px): [Co, Ci, 2, 2]} of pack_class: the taps of each sub-pixel weight summed in fp32 in the packer's order
    (rows outer, columns inner, from 0), then rounded to bf16 once. per_tap_round rounds every tap before the sum (the
    oracle's arithmetic, not the kernel's)."""
    w = w.float()
    src = bf16(w) if per_tap_round else w
    out = {}
    for py in (0, 1):
        for px in (0, 1):
            wc = torch.zeros(w.shape[0], w.shape[1], 2, 2)
            for a in (0, 1):
                for b in (0, 1):
                    acc = torch.zeros(w.shape[0], w.shape[1])
                    for r in DECONV_ROWS[py, a]:
                        for c in DECONV_ROWS[px, b]:
                            acc = acc + src[:, :, r, c]
                    wc[:, :, a, b] = acc
            out[py, px] = bf16(wc) if round_bf16 else wc
    return out


def subpixel_conv(x, wcls, conv2d=F.conv2d):
    """conv of the nearest-x2 upsampled x through its four sub-pixel classes (no bias); dtype of x."""
    B, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = None
    for (py, px), wc in wcls.items():
        z = conv2d(xp, wc.to(x.dtype))                          # [B, Co, H + 1, W + 1]
        if out is None:
            out = x.new_zeros(B, wc.shape[0], 2 * H, 2 * W)
        out[:, :, py::2, px::2] = z[:, :, py:py + H, px:px + W]
    return out


def conv_nobias(x, w, spec, conv2d=F.conv2d):
    """the layer's convolution without bias (x, w of one dtype); w may be the folded classes of a deconv."""
    if isinstance(w, dict):
        return subpixel_conv(x, w, conv2d)
    if spec.kind == "deconv":
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    pad = spec.rate * (spec.k - 1) // 2
    return conv2d(x, w.to(x.dtype), None, stride=spec.stride, padding=pad, dilation=spec.rate)


def kernel_operands(spec, w, x, prec):
    """(x, w) as the kernel of `prec` multiplies them (fp32 tensors; w a dict of classes for bf16 deconvs)."""
    x = x.float()
    if prec == "bf16":
        if is_head(spec):
            return bf16(x), w.float()
        if spec.kind == "deconv":
            return bf16(x), folded_deconv_weights(w, round_bf16=True)
        return bf16(x), bf16(w.float())
    return x, w.float()


def abs_w(w):
    return {k: v.abs() for k, v in w.items()} if isinstance(w, dict) else w.abs()


def k_terms(spec):
    """products summed per output element: taps x input channels as the kernels run them (deconv: 4 folded taps; stem:
    5 kernel rows x 64 packed channels on the tensor cores, 25 taps x cin on the CUDA cores)."""
    if spec.kind == "deconv":
        return 4 * spec.cin
    return spec.k * spec.k * spec.cin


def tc_steps(spec):
    """wgmma k16 steps per accumulator (channels padded to blocks of 8, stems as 5 rows of 64 packed channels)."""
    if spec.k == 5:
        return 5 * 64 // 16
    taps = 4 if spec.kind == "deconv" else spec.k * spec.k
    return taps * math.ceil(spec.cin / 16)


def split_weight_scale(spec, w):
    """ClassW::s_wscale of pack_class: 2^kw bringing the largest packed weight (gates x 0.5) to [8192, 16384)."""
    wm = w.float().clone()
    if not is_head(spec):
        wm[spec.cout // 2:] *= 0.5
    if spec.kind == "deconv":
        wmax = max(float(v.abs().max()) for v in folded_deconv_weights(wm, round_bf16=False).values())
    else:
        wmax = float(wm.abs().max())
    kw = min(24, max(0, 13 - math.floor(math.log2(wmax)))) if wmax > 0 else 0
    return 2.0 ** kw


# --------------------------------------------------------------------------------------------- reference and bound
def sigmoid_prime(g):
    return torch.sigmoid(g) * torch.sigmoid(-g)          # s (1 - s) without cancelling to 0 at large |g|


def act64(f, spec):
    return F.elu(f) if spec.act == "elu" else F.relu(f)


def reference(net, name, x, prec):
    """fp64 reference of one layer on the kernel's operands: dict(Y, z, A, spec, ...). z includes the bias."""
    spec, w, b = layer(net, name)
    xo, wo = kernel_operands(spec, w, x, prec)
    x64 = xo.double()
    w64 = {k: v.double() for k, v in wo.items()} if isinstance(wo, dict) else wo.double()
    z = conv_nobias(x64, w64, spec) + b.double()[None, :, None, None]
    A = conv_nobias(x64.abs(), abs_w(w64), spec)
    r = dict(spec=spec, z=z, A=A, x=xo, w=w, b=b)
    if prec == "fp32":
        # floors of the split-half representation: |x| per window (weights' floor) and sum |w| per window (inputs' floor)
        r["X1"] = conv_nobias(x64.abs(), torch.ones_like(w64), spec)
        r["W1"] = conv_nobias(torch.ones_like(x64), abs_w(w64), spec)
        r["s_w"] = split_weight_scale(spec, w)
    if is_head(spec):
        r["Y"] = z
    else:
        h = spec.cout // 2
        r["Y"] = act64(z[:, :h], spec) * torch.sigmoid(z[:, h:])
    return r


def preact_error(r, prec):
    """bound on |z_kernel - z| (before the activation), same shape as z."""
    spec, z, A = r["spec"], r["z"], r["A"]
    if prec == "fp32_direct" or is_head(spec):
        # a chain of n fp32 FMAs (and the bias add): gamma_n = n u (first order); deconv folds add <= 3 fp32 roundings per weight
        dz = k_terms(spec) * U32 * A + U32 * z.abs()
        if spec.kind == "deconv":
            dz = dz + 3 * U32 * A
        return dz
    if prec == "bf16":
        # exact bf16 products, fp32 tensor-core accumulation, fp32 bias add
        return c_acc(tc_steps(spec)) * A + U32 * z.abs()
    # split-half: each of x and w carries U_SPLIT of itself, the dropped lo*lo product is <= U16^2 |x||w|; lo halves below fp16's
    # normal range (activations |v| < 2^-9, weights below 2^-9 of the class's largest) are rounded to the subnormal quantum 2^-24:
    # half of it, unscaled, per operand (the x floor meets sum |w|, the w floor meets sum |x|); three wgmma per k16 step
    floor_x = 2.0 ** -25 / ACT_SCALE
    floor_w = 2.0 ** -25 / r["s_w"]
    dz = (3 * U_SPLIT + c_acc(3 * tc_steps(spec))) * A + floor_x * r["W1"] + floor_w * r["X1"] + U32 * z.abs()
    if spec.kind == "deconv":
        dz = dz + 3 * U32 * A                                   # the fold's fp32 sums before the split
    return dz


def gated_bound(r, prec):
    """per-element bound on |y - Y| of a layer's output (r = reference(...))."""
    spec, z, Y = r["spec"], r["z"], r["Y"]
    dz = preact_error(r, prec)
    if is_head(spec):
        return dz + U32 * Y.abs()                                # fp32 output
    h = spec.cout // 2
    f, g, df, dg = z[:, :h], z[:, h:], dz[:, :h], dz[:, h:]
    a = act64(f, spec)
    s = torch.sigmoid(g)
    # first-order propagation through the gate, with the derivatives bounded over [z - dz, z + dz]
    prop = df * torch.sigmoid(g + dg) + (a.abs() + df) * sigmoid_prime(torch.clamp(g.abs() - dg, min=0)) * dg
    elu = spec.act == "elu"
    neg = (f <= 0).double() if elu else torch.zeros_like(f)
    ef = torch.exp(torch.clamp(f, max=0))
    if prec == "bf16":
        # gate_one: ELU's exp as ex2.approx.ftz (PTX ISA: 2^-22 relative; its argument fma(f, log2 e, b log2 e) rounds to
        # u (|f| + |b|) log2 e, i.e. u (|f| + |b|) relative after the exp) minus 1 (2^-25 absolute)
        bf = r["b"].double()[:h][None, :, None, None].abs()
        da = neg * (ef * (2.0 ** -22 + 2 * U32 * (f.abs() + 2 * bf)) + 2.0 ** -25)
        # sigmoid = 0.5 tanh.approx(g / 2) + 0.5 (PTX ISA: tanh.approx.f32 is good to 2^-10.987 relative), so y = (a / 2)(1 + t)
        # carries (|a| / 2) 2^-10.987 |t|; the final fma rounds to u |y|
        epi = da * s + a.abs() * 0.5 * 2.0 ** -10.987 * torch.tanh(g / 2).abs() + U32 * Y.abs()
        pre = prop + epi
        # half an ulp of the bf16 output, taken at the largest magnitude the fp32 result can have
        return pre + bf16_half_ulp(Y.abs() + pre)
    # fp32 modes: exp(-g) overflows fp32 below g = -88.7 and the sigmoid becomes 0 (the true y is below 1e-38 |a|); results
    # below fp32's normal range (2^-126) are flushed (.ftz) or rounded to the subnormal quantum
    under = a.abs() * s * (g < -80).double() + 2.0 ** -126
    if prec == "fp32":
        # gate_one_exact: ELU below -1/16 as ex2.approx(f log2 e) - 1 (2^-22 relative, argument rounding u |f| log2 e, the
        # subtraction 2^-25), above it the degree-5 Taylor polynomial (remainder |f|^6 / 720, Horner's 5 fma: 6u of |a|)
        big = ef * (2.0 ** -22 + 2 * U32 * f.abs()) + 2.0 ** -25
        small = f.abs() ** 6 / 720 + 6 * U32 * a.abs()
        da = neg * torch.where(f > -0.0625, small, big)
        # sigmoid = rcp.approx(1 + ex2.approx(-g log2 e)): 2^-22 (rcp) + (1 - s)(2^-22 + 2u |g|) (ex2 and its argument) + u (add)
        ds_rel = 2.0 ** -22 + torch.sigmoid(-g) * (2.0 ** -22 + 2 * U32 * g.abs()) + 2 * U32
        epi = da * s + a.abs() * s * ds_rel + U32 * Y.abs() + under
        pre = prop + epi
        # the output is re-split (hi + lo of 64 y): U_SPLIT relative, and its lo half's subnormal floor (2^-25 / 64)
        return pre + U_SPLIT * (Y.abs() + pre) + 2.0 ** -25 / ACT_SCALE
    # fp32_direct: expm1f (1 ulp), expf (2 ulp), the IEEE divide and the product (u each)
    da = neg * 2 * U32 * a.abs()
    ds_rel = torch.sigmoid(-g) * 4 * U32 + 2 * U32
    return prop + da * s + a.abs() * s * ds_rel + U32 * Y.abs() * 2 + under


def bf16_half_ulp(v):
    """half an ulp of bf16 at magnitude v (>= 0): 2^(floor(log2 v) - 8); bf16 keeps fp32's exponent range."""
    v = torch.clamp(v, min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(v)) - 8)


def ratio(y, Y, bound):
    """elementwise |y - Y| / bound (bound 0 demands equality)."""
    err = (y.double() - Y).abs()
    return torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                       torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))


def max_ratio(y, Y, bound):
    return float(ratio(y, Y, bound).max())


# --------------------------------------------------------------------------------------------- inputs
TARGET_STD = {"small": 0.01, "unit": 1.0, "sat": 25.0}   # std of the pre-activations without bias


def input_scale(net, name, target):
    """input std that gives pre-activations (without bias) of std `target` for i.i.d. inputs: target / rms_c ||w_c||."""
    spec, w, _ = layer(net, name)
    if spec.kind == "deconv":
        w = torch.stack([v for v in folded_deconv_weights(w, round_bf16=False).values()], 0)[0]
    rms = float(w.double().flatten(1).norm(dim=1).pow(2).mean().sqrt())
    return target / rms


def conv_input(net, name, B, H, W, regime, seed):
    """fp32 input of a layer. Regimes: 'small' (|f| within b_f +- ~0.03: the ELU polynomial branch and near-zero outputs
    where |b_f| < 1/16), 'unit' (O(1) pre-activations), 'sat' (pre-activations of std 25: f < -10, |g| > 20 at many
    elements), 'zero' (all-zero input: y = act(b_f) sigmoid(b_g)), 'big' (split-half only: sparse values up to +-1000,
    inside the saturation-free range |v| <= 65000 / 64 of inputs and outputs). The non-zero regimes also carry an
    all-zero quadrant in image 0 and are not bf16-representable (the lo halves of the split-half mode matter)."""
    spec = layer_map(net)[name]
    g = torch.Generator().manual_seed(seed)
    shape = (B, spec.cin, H, W)
    if regime == "zero":
        return torch.zeros(shape)
    if regime == "big":
        # O(1) inputs with every 509th element replaced by a value up to +-1000 (exactly 1000 and -1000 at the ends):
        # sparse enough that the layer's outputs stay inside the range too
        x = torch.randn(shape, generator=g) * input_scale(net, name, 1.0)
        big = (torch.rand(shape, generator=g) * 2 - 1) * 1000.0
        big.view(-1)[0], big.view(-1)[-1] = 1000.0, -1000.0
        x.view(-1)[::509] = big.view(-1)[::509]
        x.view(-1)[-1] = -1000.0
        return x
    x = torch.randn(shape, generator=g) * input_scale(net, name, TARGET_STD[regime])
    x[0, :, :(H + 1) // 2, :(W + 1) // 2] = 0.0
    return x


def thin_input(spec, Ho, Wo):
    """input H, W that gives a Ho x Wo output."""
    if spec.kind == "deconv":
        return Ho // 2, Wo // 2
    return Ho * spec.stride, Wo * spec.stride


def stable_seed(*parts):
    import zlib
    return zlib.crc32(repr(parts).encode()) % 100000


def conv_sizes(net, name):
    """(label, B, H, W) of a layer's input. Output tiles are 16 rows x 8 columns (se_conv_c8.cu C8_TH x C8_TW). Entries:
    the map the layer sees in a 16 x 16 forward; an output 8 rows high (half a tile: partial rows) and 56 wide (seven
    whole column tiles); 56 rows high (three tiles and a half) and 8 wide (exactly one whole column tile); and 24 x 13,
    whose last column tile holds 5 columns (a deconv's output width is even: 12, a last tile of 4)."""
    spec = layer_map(net)[name]
    H, W = in_hw(name, 16, 16)
    return [("fwd16", 2, H, W), ("thin", 2) + thin_input(spec, 8, 56), ("tall", 2) + thin_input(spec, 56, 8),
            ("partcols", 2) + thin_input(spec, 24, 13)]


def conv_regimes(prec, label=None, spec=None):
    """input regimes of a conv_sizes entry (label) of a layer (spec). On the GPU the 192-input-channel layer skips
    split-half's sparse +-1000 inputs at the partial-column entry. On them its tensor-core accumulation exceeds the
    probabilistic bound (LAMBDA_ACC) by 1-2 % at interior pixels, and at some seeds it does so on other entries too
    (DESIGN.md 5.1, an open finding). That says nothing about the tile's columns. The CPU emulations keep every regime."""
    big = prec == "fp32" and not (label == "partcols" and spec is not None and spec.cin == 192)
    return ["small", "unit", "sat", "zero"] + (["big"] if big else [])


# --------------------------------------------------------------------------------------------- contextual attention
def attention_err(prec, C, h, w):
    """error model of contextual_attention(precision=prec), prec "fp32" or "fp32_direct", for tests/util_attention.py contextual_attention_at(err=...):
    logits good to logit_rel * |scale m q| . |k| + logit_abs, softmax-weighted sums good to rel * sum P |V| + abs."""
    hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
    L, d = hs * ws, 16 * C
    norm = h * w * U32 + 3 * U32                  # plane norm: an fp32 sum of h w squares, sqrt and reciprocal
    if prec == "fp32":
        # split-half GEMMs: three products (3 U_SPLIT + the dropped lo lo), q scaled by 64 and k by 2^15: subnormal floors of
        # 2^-25 / scale per element against |k| <= 1 and |q| < 2^9
        logit_rel = 3 * U_SPLIT + norm + c_acc(3 * d // 16)
        logit_abs = 10.0 * d * (2.0 ** -25 / 64 + 2.0 ** 9 * 2.0 ** -25 / 2 ** 15)
        # expf (2 ulp), the lane-strided row sum (L / 32 + 5 adds), P split (x 2^14) and V split, P V over 3 L / 16 truncating
        # steps of non-negative terms, the fold of <= 4 terms
        rel = 4 * U32 + (L / 32 + 5) * U32 + 3 * U_SPLIT + (3 * L / 16 + 1) * 2.0 ** -23 + 4 * U32
        abs_ = L * 2.0 ** -25 / 2 ** 14 * 2.0 ** 9 + 2.0 ** -25 / 64
        return dict(logit_rel=logit_rel, logit_abs=logit_abs, rel=rel, abs=abs_, out="fp32")
    # fp32_direct: fp32 FMA chains of d (logits) and L (P V) terms, expf, the row sum and the fold
    return dict(logit_rel=d * U32 + norm + 2 * U32, logit_abs=0.0, rel=4 * U32 + 2 * L * U32 + 8 * U32, abs=0.0, out="fp32")


def attention_out_bound(pre, y_ref, mode):
    """adds the rounding of the stored output to the bound `pre` of the fp32 result."""
    if mode == "bf16":
        return pre + bf16_half_ulp(y_ref.abs() + pre)
    return pre + U32 * (y_ref.abs() + pre) + 2.0 ** -126


def attention_fp32_map(feat, mask_s):
    """fp64 softmax weights P [B, L keys, L queries] of the attention on feat and the per-element bound of the fp32 CUDA-core
    map (contextual_attention(precision="fp32" or "fp32_direct", want_attn=True), and the fp32_direct forward's export):
    logits off by at most delta_n (attention_err("fp32_direct")) move P_l by at most P_l (exp(2 delta_n) - 1 + rel), and
    the stored fp32 value adds u. Runs on the device of feat."""
    f = feat.double()
    B, C, h, w = f.shape
    err = attention_err("fp32_direct", C, h, w)
    Q = F.unfold(f, 4, stride=2)                                                   # [B, d, L]
    K = F.unfold(f / torch.sqrt((f ** 2).sum((2, 3), keepdim=True) + 1e-8), 4, stride=2)
    valid = (F.unfold(1 - mask_s.double(), 4, stride=2).mean(1) > 0.1).double()   # [B, L]
    P = torch.softmax(10.0 * valid[:, :, None] * torch.einsum("bdl,bdn->bln", K, Q), dim=1)
    qk = torch.einsum("bdl,bdn->bln", K.abs(), Q.abs()) * valid[:, :, None] * 10.0  # [B, keys, queries]
    d_n = err["logit_rel"] * qk.max(1).values + err["logit_abs"]                     # [B, N]
    return P, P * (torch.expm1(2 * d_n)[:, None, :] + err["rel"]) + U32 * P + 2.0 ** -126


def attention_bf16_map(feat, mask_s):
    """fp64 reference and per-element bound of the bf16 attention's stored probabilities (se_cam.cu; the map that
    contextual_attention(precision="bf16", want_attn=True) and the bf16 export forward return): Pb = bf16(P) of the exact
    softmax on the kernels' operands, and Wp, how far the stored value may be from Pb (see attention_bf16_reference).
    Returns (Pb, Wp), both [B, L keys, L queries]; runs on the device of feat."""
    return _attention_bf16_probs(feat, mask_s)[:2]


def _attention_bf16_probs(feat, mask_s):
    """(Pb, Wp, Q, h, w) of attention_bf16_reference."""
    f = bf16(feat.float()).double()
    B, C, h, w = f.shape
    hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
    L, d = hs * ws, 16 * C
    # cam_norm_kernel: per thread an fp32 sum of h w / 256 squares, a 5-level shuffle tree and 8 adds; rnorm = 1 / sqrt(s +
    # 1e-8) carries half of the sum's relative error plus sqrt, reciprocal and the f * rnorm product
    eps_r = (math.ceil(h * w / 256) + 13) * U32 / 2 + 3 * U32
    kv = f / torch.sqrt((f ** 2).sum((2, 3), keepdim=True) + 1e-8)
    k_mid = bf16(kv)
    dk = torch.maximum((bf16(kv * (1 + eps_r)) - k_mid).abs(), (bf16(kv * (1 - eps_r)) - k_mid).abs())
    Q = F.unfold(f, 4, stride=2)                                                   # [B, d, L] queries = values
    K, dK = F.unfold(k_mid, 4, stride=2), F.unfold(dk, 4, stride=2)
    valid = (F.unfold(1 - mask_s.double(), 4, stride=2).mean(1) > 0.1).double()   # [B, L]; masked keys: logit exactly 0
    S = 10.0 * valid[:, :, None] * torch.einsum("bdl,bdn->bln", K, Q)              # [B, keys, queries]
    # logit error per (key, query): flipped key elements, d-term tensor-core accumulation (96 k16 steps), and the fp32
    # scaling by 10 log2 e, the subtraction of the row maximum and ex2's argument (4 u of |S| + max |S|)
    Qa = Q.abs()
    D = 10.0 * valid[:, :, None] * (torch.einsum("bdl,bdn->bln", dK, Qa) + c_acc(d // 16) * torch.einsum("bdl,bdn->bln", K.abs() + dK, Qa))
    D = D + 4 * U32 * (S.abs() + S.abs().amax(1, keepdim=True))
    P = torch.softmax(S, dim=1)
    # softmax: log(P'_l / P_l) = -log sum_m P_m exp(dS_m - dS_l), so |log(P'_l / P_l)| <= E_l = sum_{m != l} P_m (exp(D_m + D_l) - 1)
    # (upper side: log(1 + t) <= t; lower side: Jensen); the top weight of a peaked softmax is then nearly exact
    eD = torch.exp(D)
    E = eD * (P * eD).sum(1, keepdim=True) - 1 - P * (eD * eD - 1)
    # the kernel's own softmax arithmetic: ex2.approx (2^-22) per exponential, per-lane fp32 row sums of about L / 4 terms with
    # one ex2 rescale per key tile, 1 / sum and the product (u each)
    eps_c = 2.0 ** -22 + (L / 4 + 8) * U32 + (L / 128 + 2) * 2.0 ** -22 + 2 * U32
    Pb = bf16(P)
    # (+ 2^-126: ex2.approx.ftz flushes probabilities below fp32's normal range to 0)
    Wp = torch.maximum((bf16(P * torch.exp(E) * (1 + eps_c)) - Pb).abs(), (bf16(P * torch.exp(-E) * (1 - eps_c)) - Pb).abs()) + 2.0 ** -126
    return Pb, Wp, Q, h, w


def attention_bf16_reference(feat, mask_s):
    """fp64 reference and per-element bound of contextual_attention(precision="bf16") (se_cam.cu), whole map at once.

    The reference runs on what the kernels multiply: queries and values bf16(feat), keys bf16(f * rnorm) and the
    probabilities rounded to bf16, Y = fold(sum_l bf16(P_l) V_l). The bound covers what can still differ: a key element
    whose fp32 rnorm moves it across a bf16 rounding boundary (one ulp), the fp32 accumulation of the logits, the softmax
    statistics, a P_l that lands on the other side of a bf16 rounding boundary, the P V accumulation and the bf16 output.
    Returns (Y [B, C, h, w], bound [B, C, h, w])."""
    Pb, Wp, Q, h, w = _attention_bf16_probs(feat, mask_s)
    L = Pb.shape[1]
    Qa = Q.abs()
    O = torch.einsum("bln,bdl->bdn", Pb, Q)
    Ow = torch.einsum("bln,bdl->bdn", Wp, Qa)
    Oa = torch.einsum("bln,bdl->bdn", Pb + Wp, Qa)
    # P V (cam_pv_kernel): a pixel sums <= 4 patches x L keys of non-negative-weight terms in 4 L / 16 + 4 k16 steps. Each step
    # is charged two truncations, 2^-22 of the sum of |terms| (aligning its products, adding them): set by measurement, on an
    # H100 one step-truncation per step (2^-23) fell just short at L = 127 and 257
    pre = Ow + (4 * L / 16 + 4) * 2.0 ** -22 * Oa
    fold = lambda t: F.fold(t, output_size=(h, w), kernel_size=4, stride=2)
    Y, pre = fold(O), fold(pre)
    return Y, pre + bf16_half_ulp(Y.abs() + pre) + 2.0 ** -126

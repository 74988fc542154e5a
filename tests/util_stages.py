"""Stage checks of a whole forward (test infrastructure): every edge of the graph is checked as "the consumer's input, as
stored, equals f(the producer's input, as stored) within f's bound", on the engine's own stored operands (activation taps
decoded by tests/util_taps.py). Nothing is propagated through the network, so the per-element bounds of
tests/util_bounds.py apply to every layer of a real forward as they do to a single operator call.

Each check returns max |y - Y| / bound (<= 1 passes; a bound of 0 demands equality). A dict of taps maps a tap name to the
decoded fp32 NCHW tensor (packed stem rows: all 8 channels); `pads` maps a packed tap to its pad values.
"""
import math

import torch
import torch.nn.functional as F

from tests import util_bounds as UB
from tests.util_attention import contextual_attention_at, sample_pixels

U32 = UB.U32
TINY = 2.0 ** -126

ENC = ["conv1", "conv2_downsample", "conv3", "conv4_downsample", "conv5", "conv6", "conv7_atrous", "conv8_atrous",
       "conv9_atrous", "conv10_atrous"]
DEC = ["11", "12", "13_upsample_conv", "14", "15_upsample_conv", "16", "17"]
PM = ["pmconv1", "pmconv2_downsample", "pmconv3", "pmconv4_downsample", "pmconv5", "pmconv6"]


# --------------------------------------------------------------------------------------------- storage of each mode
def store(v, prec):
    """v (fp32) as the activation storage of `prec` holds it: bf16 round to nearest even, the split-half pair of
    se_common.cuh split_half (64 v clamped to +-65000, hi = fp16, lo = fp16 of the rest), or fp32."""
    v = v.float()
    if prec == "bf16":
        return UB.bf16(v)
    if prec == "fp32":
        s = (v * UB.ACT_SCALE).clamp(-65000.0, 65000.0)
        hi = UB.f16(s)
        return (hi + UB.f16(s - hi)) / UB.ACT_SCALE
    return v


def store_error(a, prec):
    """bound on |store(v) - v| for |v| <= a: half a bf16 ulp; the split-half pair's 2^-22 relative plus the lo half's
    subnormal quantum (2^-24 / 2, unscaled by 64); nothing in fp32."""
    if prec == "bf16":
        return UB.bf16_half_ulp(a)
    if prec == "fp32":
        return UB.U_SPLIT * a + 2.0 ** -25 / UB.ACT_SCALE
    return torch.zeros_like(a)


def exact_ratio(y, Y):
    """0 when y == Y everywhere, inf otherwise."""
    return 0.0 if torch.equal(y.float(), Y.float()) else float("inf")


# --------------------------------------------------------------------------------------------- graph edges
def conv_edges(net, flags, mask_image=False):
    """[(producer, consumer tap, channel slice)] of every non-stem gated layer: its output is (a slice of) that tap."""
    e = []
    if net == "M":
        e += [(ENC[i], "in:M." + ENC[i + 1], None) for i in range(1, 9)]
        if mask_image:
            e += [("conv9_atrous", "in:M.conv11", None)]
            e += [("conv" + DEC[i], "in:M.conv" + DEC[i + 1], None) for i in range(6)]
        e += [("conv10_atrous", "in:M.conv_mask_11", None)]
        e += [("conv_mask_" + DEC[i], "in:M.conv_mask_" + DEC[i + 1], None) for i in range(6)]
        return e
    for p in ("", "w", "x"):
        e += [(p + ENC[i], "in:G." + p + ENC[i + 1], None) for i in range(1, 9)]
    e += [("conv10_atrous", "in:G.conv11", slice(0, 96)), ("wconv10_atrous", "in:G.pool", None),
          ("xconv10_atrous", "in:G.allconv11", slice(0, 96))]
    for p in ("conv", "allconv"):
        e += [(p + DEC[i], "in:G." + p + DEC[i + 1], None) for i in range(6)]
    e += [(PM[i], "in:G." + PM[i + 1], None) for i in range(1, 5)]
    e += [("pmconv6", "in:G.cam" if flags.get("use_cam", True) else "in:G.pmconv9", None),
          ("pmconv9", "in:G.pmconv10", None), ("pmconv10", "in:G.allconv11", slice(96, 192))]
    return e


def conv_ratio(net, name, x, y, prec):
    r = UB.reference(net, name, x, prec)
    assert y.shape == r["Y"].shape, (name, y.shape, r["Y"].shape)
    return UB.max_ratio(y, r["Y"], UB.gated_bound(r, prec))


def check_convs(T, net, prec, flags, mask_image=False):
    """{producer: ratio} of every non-stem gated conv / deconv of the net."""
    out = {}
    for name, cons, sl in conv_edges(net, flags, mask_image):
        y = T[cons] if sl is None else T[cons][:, sl]
        out[name] = conv_ratio(net, name, T["in:%s.%s" % (net, name)], y, prec)
    return out


# --------------------------------------------------------------------------------------------- inputs of the stems
def stem_inputs(io, flags):
    """{(net, stem): fp32 input} as the oracle builds it from the public inputs (oracle netM_forward / netG_forward)."""
    x, x2, m, m2, g = io["x"], io["x2"], io["mask"], io["mask2"], io["guide"]
    out = {}
    if io.get("netM"):
        out["M", "conv1"] = torch.cat([x, g], 1)
    ones = torch.ones_like(m) if g is None else g
    out["G", "conv1"] = torch.cat([x * (1 - m), ones, m], 1)
    out["G", "wconv1"] = torch.cat([x2 if flags.get("no_mask_cc") else x2 * m2,
                                    ones * 0 if flags.get("joint_train_inp", True) else ones, m2], 1)
    return out


def packed_expect(io, flags, name):
    """the fp32 8 channels pack8 writes for packed tap `name` (se_misc.cu pack8_kernel)."""
    x, x2, m, m2, g = io["x"], io["x2"], io["mask"], io["mask2"], io["guide"]
    ones = torch.ones_like(m) if g is None else g
    z1, z3 = torch.zeros_like(m), torch.zeros_like(x)
    style = x if flags.get("no_mask_cc") else x * m
    if name == "in:M.conv1":
        return torch.cat([x, g, z1, z3], 1)
    if name == "in:G.conv1+wconv1":
        return torch.cat([x * (1 - m), ones * 1.0, m, style], 1)
    if name == "in:G.conv1":
        return torch.cat([x * (1 - m), ones * 1.0, m, z3], 1)
    assert name == "in:G.wconv1", name
    style2 = x2 if flags.get("no_mask_cc") else x2 * m2
    return torch.cat([style2, ones * (0.0 if flags.get("joint_train_inp", True) else 1.0), m2, z3], 1)


def check_pack8(T, pads, io, flags, prec):
    """the packed network inputs equal the storage rounding of pack8's fp32 formula bit for bit; pad pixels are zero."""
    out = {}
    for name in ("in:M.conv1", "in:G.conv1+wconv1", "in:G.conv1", "in:G.wconv1"):
        if name in T and (name != "in:M.conv1" or io.get("netM")):
            q = exact_ratio(T[name], store(packed_expect(io, flags, name), prec))
            out[name] = max(q, exact_ratio(pads[name], torch.zeros_like(pads[name])))
    return out


def xnow_tap(T):
    return T["in:G.xconv1+pmconv1"] if "in:G.xconv1+pmconv1" in T else T["in:G.xconv1"]


def check_xnow(T, pads, io, flags, prec):
    """the packed stage-2 input against the blend of the public coarse output (se_misc.cu HEAD_COARSE: t m + (x (1 - m))
    (1 - m), or t under no_mask_coarse) in fp64: the blend's fp32 rounding (two products, 1 - m and the sum, contracted or
    not: 3 u of the terms) plus the storage rounding. Channels 3-7 and the pad pixels are zero."""
    name = "in:G.xconv1+pmconv1" if "in:G.xconv1+pmconv1" in T else "in:G.xconv1"
    t, x, m = io["coarse"].double(), io["x"].double(), io["mask"].double()
    if flags.get("no_mask_coarse"):
        V, pre = t, torch.zeros_like(t)
    else:
        a, b = t * m, x * (1 - m) * (1 - m)
        V, pre = a + b, 3 * U32 * (a.abs() + b.abs())
    got = T[name]
    q = UB.max_ratio(got[:, :3], V, pre + store_error(V.abs() + pre, prec) + TINY)
    q = max(q, exact_ratio(got[:, 3:], torch.zeros_like(got[:, 3:])), exact_ratio(pads[name], torch.zeros_like(pads[name])))
    if "in:G.xconv1" in T and "in:G.pmconv1" in T:
        q = max(q, exact_ratio(T["in:G.xconv1"], T["in:G.pmconv1"]))
    return q


def check_stems(T, io, flags, prec):
    """each stem's output against the float64 reference of its input built from the public inputs (the stem pair's two
    halves against their own layers: checks make_stem_pair's channel maps and the zeroed sketch weight independently)."""
    out = {}
    for (net, name), x in stem_inputs(io, flags).items():
        out[net + "." + name] = conv_ratio(net, name, x, T["in:%s.%s" % (net, name.replace("conv1", "conv2_downsample"))], prec)
    xn = xnow_tap(T)[:, :3]
    for name in ("xconv1", "pmconv1"):
        out["G." + name] = conv_ratio("G", name, xn, T["in:G." + name.replace("conv1", "conv2_downsample")], prec)
    return out


# --------------------------------------------------------------------------------------------- heads
def head_pre(net, name, x, prec):
    """fp64 pre-activation z of a head on its stored input and the bound on the kernel's z: an fp32 FMA chain of
    9 x 12 = 108 products started at (or ended with) the bias, gamma_109 of sum |x||w| + |b|."""
    spec, w, b = UB.layer(net, name)
    xo = UB.bf16(x.float()) if prec == "bf16" else x.float()
    x64 = xo.double()
    z = F.conv2d(x64, w.double(), b.double(), padding=1)
    A = F.conv2d(x64.abs(), w.double().abs(), b.double().abs(), padding=1)
    return z, 109 * U32 * A


def tanh_bound(z, dz):
    """(tanh z, bound on |tanhf(z') - tanh z| for |z' - z| <= dz): the slope sech^2 at the nearest point of the interval to 0,
    plus tanhf's 2 ulp (4 u relative)."""
    t = torch.tanh(z)
    prop = (1 - torch.tanh(torch.clamp(z.abs() - dz, min=0)) ** 2) * dz
    return t, prop + 4 * U32 * (t.abs() + prop) + TINY


def sigmoid_bound(z, dz):
    """(sigmoid z, bound of 1 / (1 + expf(-z'))): the slope, expf's 2 ulp (4 u of e = exp(-z), so (1 - s) 4 u of s), the
    add and the IEEE divide (u each)."""
    s = torch.sigmoid(z)
    prop = UB.sigmoid_prime(torch.clamp(z.abs() - dz, min=0)) * dz
    return s, prop + (s + prop) * ((1 - s) * 4 * U32 + 2 * U32) + TINY


def check_threshold(soft, mask_bin):
    """the binarised mask is exactly (soft mask > 0.5) (reference editline2_model.py:347)."""
    return exact_ratio(mask_bin, (soft > 0.5).float())


def check_heads(T, io, flags, prec):
    """every public output against float64 from its head's stored input."""
    out = {}
    if io.get("netM"):
        z, dz = head_pre("M", "conv_mask_17", T["in:M.conv_mask_17"], prec)
        S, bS = sigmoid_bound(z, dz)
        out["mask"] = UB.max_ratio(io["soft"], S, bS)
        if io.get("mask_bin") is not None:
            out["mask_bin"] = check_threshold(io["soft"], io["mask_bin"])
        if io.get("mask_image") is not None:
            z, dz = head_pre("M", "conv17", T["in:M.conv17"], prec)
            out["mask_image"] = UB.max_ratio(io["mask_image"], *tanh_bound(z, dz))
    z, dz = head_pre("G", "conv17", T["in:G.conv17"], prec)
    out["coarse"] = UB.max_ratio(io["coarse"], *tanh_bound(z, dz))
    z, dz = head_pre("G", "allconv17", T["in:G.allconv17"], prec)
    Tf, bT = tanh_bound(z, dz)
    out["fine"] = UB.max_ratio(io["fine"], Tf, bT)
    if io.get("composed") is not None:
        # composed = t m + img (1 - m) in fp32 on the soft mask: |m| times the fine bound, plus two products, 1 - m and the sum
        m, img = io["soft"].double(), io["x"].double()
        a, b = Tf * m, img * (1 - m)
        out["composed"] = UB.max_ratio(io["composed"], a + b, m.abs() * bT + 3 * U32 * (a.abs() + b.abs()) + TINY)
    return out


# --------------------------------------------------------------------------------------------- pooling, attention
def check_pool(T, flags, prec):
    """every pixel of the concat's blocks 12-23 equals the storage rounding of the global pool of the stored style map: max is
    exact, avg carries an fp32 sum of h w terms in any order ((h w) u of sum |v|) and the divide (u)."""
    v = T["in:G.pool"].double()
    got = T["in:G.conv11"][:, 96:]
    if flags.get("pool_type", "max") == "max":
        P = v.amax((2, 3), keepdim=True).expand_as(got)
        return exact_ratio(got, store(P.float(), prec))
    hw = v.shape[2] * v.shape[3]
    P = v.mean((2, 3), keepdim=True)
    pre = hw * U32 * v.abs().mean((2, 3), keepdim=True) + U32 * P.abs()
    return UB.max_ratio(got, P.expand_as(got), (pre + store_error(P.abs() + pre, prec)).expand_as(got) + TINY)


def check_attention(T, io, prec, max_pixels=2048):
    """{"mask_s": the pooled mask equals avg_pool2d(mask, 4) exactly, "attention": the attention output (pmconv9's input)
    against float64 of the stored feature map and mask}. The fp32 modes are checked at every pixel up to max_pixels, at a
    sample of pixels beyond."""
    out = {}
    mask_s = T["in:G.cam.mask_s"]
    out["mask_s"] = exact_ratio(mask_s, F.avg_pool2d(io["mask"].float(), 4))
    feat, y = T["in:G.cam"], T["in:G.pmconv9"].double()
    B, C, h, w = feat.shape
    if prec == "bf16":
        Y, bound = UB.attention_bf16_reference(feat, mask_s)
        out["attention"] = UB.max_ratio(y, Y, bound)
        return out
    if prec == "fp32":
        # the split-half mode runs the attention in fp32 between two conversions (se_misc.cu act_to_f32 and
        # f32_to_act): the fp32 map equals the stored one, and the stored result is the re-split of the fp32 one
        out["attention_glue"] = max(exact_ratio(T["in:G.cam.f32"], feat), exact_ratio(y.float(), store(T["out:G.cam.f32"], prec)))
        y = T["out:G.cam.f32"].double()
    err = UB.attention_err(prec, C, h, w)
    if B * h * w <= max_pixels:
        px = [(b, yy, xx) for b in range(B) for yy in range(h) for xx in range(w)]
    else:
        px = sample_pixels(B, h, w, max_pixels // 16, seed=h * 1000 + w)
    ref, t = contextual_attention_at(feat, mask_s, px, err=err)
    got = torch.stack([y[b, :, yy, xx] for b, yy, xx in px])
    out["attention"] = UB.max_ratio(got, ref, UB.attention_out_bound(t["bound"], ref, "fp32"))
    return out


def check_forward(T, pads, io, flags, prec, raw=None):
    """every stage check of one forward: {"conv:<net>.<layer>" / "stem:.." / "pack8:.." / "head:.." / "xnow" / "pool" /
    "attention" / "mask_s" / "conv9_fanout": max ratio}."""
    res = {}
    if io.get("netM"):
        res.update({"conv:M." + k: v for k, v in check_convs(T, "M", prec, flags, io.get("mask_image") is not None).items()})
        if raw is not None and "in:M.conv11" in raw:
            # netM's conv9 output feeds conv10_atrous and the image decoder's conv11: one buffer, the same bytes
            res["conv9_fanout"] = 0.0 if torch.equal(raw["in:M.conv10_atrous"], raw["in:M.conv11"]) else float("inf")
    res.update({"conv:G." + k: v for k, v in check_convs(T, "G", prec, flags).items()})
    res.update({"stem:" + k: v for k, v in check_stems(T, io, flags, prec).items()})
    res.update({"pack8:" + k: v for k, v in check_pack8(T, pads, io, flags, prec).items()})
    res["xnow"] = check_xnow(T, pads, io, flags, prec)
    res.update({"head:" + k: v for k, v in check_heads(T, io, flags, prec).items()})
    res["pool"] = check_pool(T, flags, prec)
    if flags.get("use_cam", True):
        res.update(check_attention(T, io, prec))
    return res


def summary(res):
    """max ratio per stage class."""
    cls = {}
    for k, v in res.items():
        c = k.split(":")[0]
        cls[c] = max(cls.get(c, 0.0), v)
    return cls

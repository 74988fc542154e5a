"""The index arithmetic of the attention's three P V forms, restated from the kernels and run in float64 (no GPU needed).

* bf16, cam_pv_kernel (se_cam.cu): the 64-key chunk walk (j = c >> 2, kyc, kx0) over the S kernel's key tiles, one stage
  per chunk as the TMA boxes fill it (P window of 8 key blocks x 9 x 9 query positions, value windows of the four
  parities, out-of-bounds zeros), the wgmma operands read through their descriptors (poff, voff, LBO, SBO) and the
  epilogue's (yy, xx) and class mapping. P is laid out as cam_s_kernel writes it: key (ky, kx) in block
  j * 32 + ky % 32, j = (ky / 32) tk_x + kx / 8, element kx % 8; padding keys (ky >= hs or kx >= ws) hold 0.
* fp32, cam_split_fold_kernel (se_gemm_split.cu): O [Mp, 16 C] of the split P V GEMM folded over (ny, nx, u, v) with row
  stride ws.
* fp32_direct (se_misc.cu, se_engine.cu run_cam): softmax_rows_kernel in its in-register form (L <= 4096) and its
  re-reading form, cam_pack_v_direct_kernel's sub-pixel values and the four classes' 2 x 2 direct convolutions over P.

At every map of tests/test_gpu_attention_output.py the correct walks reproduce the float64 attention to 1e-12. Each mutant
(a plausible index bug) must exceed the per-element bound the GPU test holds the kernels to (tests/util_bounds.py) at
some element. Its report line also says whether the tolerances the suite used before would catch it: 2e-2 max|y| (bf16,
test_gpu_ops.py), 2e-4 max|y| (fp32, test_gpu_ops.py) and 1e-3 relative (test_attention_bands.py), each on max(1, .).
The emulation runs C = 8 channels (one channel block); the walks do not depend on the channel count.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import util_bounds as UB
from tests.test_gpu_error_bounds import _feat, _mask_s
from tests.util_attention import contextual_attention_at

C, CB = 8, 1
# (h, w) feature maps -> patch grid (hs, ws): the maps of tests/test_gpu_attention_output.py
MAPS = [(66, 18), (68, 20), (132, 36), (68, 100), (128, 128), (130, 130), (132, 132), (36, 484)]

# se_cam.cu stage layout in bf16 elements (bytes / 2)
WR = 9                                   # CAM_WR: window width of the P and value boxes
PPLANE = 9 * 9 * 8                       # CAM_PPLANE: one key block of the P window (LBO of A)
PW = 8 * PPLANE                          # CAM_PW_TX
ROW = WR * 8                             # CAM_ROW: one window row (SBO of A)
VPLANE = 9 * 9 * 8                       # CAM_VPLANE: one channel block of a value window (SBO of B)
V_PITCH = (2 * CB * VPLANE + 127) // 128 * 128 // 2
STAGE = (2 * (PW + 4 * V_PITCH) + 1023) // 1024 * 1024 // 2


def v_off(par):
    return PW + par * V_PITCH


def geometry(h, w):
    Hs, Ws = h // 2, w // 2
    hs, ws = Hs - 1, Ws - 1
    tk_x = -(-ws // 8)
    KT = tk_x * -(-hs // 32)
    return dict(h=h, w=w, Hs=Hs, Ws=Ws, hs=hs, ws=ws, L=hs * ws, tk_x=tk_x, KT=KT, KB=32 * KT, to_x=-(-Ws // 8))


def inputs(h, w, mkind="rect"):
    """bf16-representable features (the bf16 kernels' queries and values are then the features themselves) and a mask."""
    feat = UB.bf16(_feat("0.15", 1, h, w, seed=UB.stable_seed("walk", h, w))[:, :C]).double()
    return feat, _mask_s(mkind, 1, h, w).double()


def logits(feat, mask_s):
    """float64 logits S [L keys, L queries] (10 m_l <k_l, q_n>, masked keys 0) and the query patches Q [16 C, L]."""
    f = feat.double()
    Q = F.unfold(f, 4, stride=2)[0]
    K = F.unfold(f / torch.sqrt((f ** 2).sum((2, 3), keepdim=True) + 1e-8), 4, stride=2)[0]
    valid = (F.unfold(1 - mask_s.double(), 4, stride=2).mean(1)[0] > 0.1).double()
    return 10.0 * valid[:, None] * (K.T @ Q), Q


def fold(Q, P, g):
    """the float64 attention output [C, h, w]: fold-sum of the patches sum_l P[l, n] Q[:, l]."""
    return F.fold((Q @ P)[None], (g["h"], g["w"]), 4, stride=2)[0]


# --------------------------------------------------------------------------------------------- bf16: cam_pv_kernel
def p_buffer(P, g, pad=None):
    """P [L keys, L queries] in the S kernel's layout [KB][hs][ws][8]; padding keys get pad [L queries] (default 0)."""
    hs, ws, tk_x = g["hs"], g["ws"], g["tk_x"]
    buf = torch.zeros(g["KB"], 8, hs * ws, dtype=torch.float64)
    if pad is not None:
        buf[:] = pad
    ky, kx = torch.div(torch.arange(g["L"]), ws, rounding_mode="floor"), torch.arange(g["L"]) % ws
    j = (ky // 32) * tk_x + kx // 8
    buf[j * 32 + ky % 32, kx % 8] = P
    return buf.view(g["KB"], 8, hs, ws).permute(0, 2, 3, 1).contiguous()


def box(t, y0, x0, rows, cols):
    """a TMA box [..., rows, cols, 8] of t [..., H, W, 8] at (y0, x0); elements outside t are 0."""
    H, W = t.shape[-3], t.shape[-2]
    out = t.new_zeros(t.shape[:-3] + (rows, cols, 8))
    ya, yb, xa, xb = max(y0, 0), min(y0 + rows, H), max(x0, 0), min(x0 + cols, W)
    if ya < yb and xa < xb:
        out[..., ya - y0:yb - y0, xa - x0:xb - x0, :] = t[..., ya:yb, xa:xb, :]
    return out


def s2d(feat):
    """the space-to-depth value planes [4 parities x CB][Hs][Ws][8] (parity 2 (y & 1) + (x & 1), se_misc.cu LAYOUT_S2D)."""
    f = feat[0]
    planes = [f[:, py::2, px::2].reshape(CB, 8, f.shape[1] // 2, f.shape[2] // 2).permute(0, 2, 3, 1) for py in (0, 1) for px in (0, 1)]
    return torch.cat(planes, 0)


def operand_addresses(poff_col=0):
    """element addresses in a stage of the A (P, K-major) and B (values, MN-major) operands of every (tap, k2) wgmma:
    A [4, 4, 64 M, 16 K], B [4 classes, 4, 4, 16 K, C N]."""
    m, k, n = torch.arange(64), torch.arange(16), torch.arange(C)
    A = torch.zeros(4, 4, 64, 16, dtype=torch.long)
    B = torch.zeros(4, 4, 4, 16, C, dtype=torch.long)
    for tap in range(4):
        a, b = tap >> 1, tap & 1
        poff = ((1 - a) * WR + (1 - b) + poff_col) * 8         # query (yy - a, xx - b) inside the 9 x 9 window
        voff = (a * 9 + b) * 8                                 # value pixel (ky + a, kx + b) inside the 9 x 9 window
        for k2 in range(4):
            A[tap, k2] = 2 * k2 * PPLANE + poff + ((m % 8) * 8 + (m // 8) * ROW)[:, None] + ((k % 8) + (k // 8) * PPLANE)[None, :]
            for cls in range(4):                               # accumulator q of warpgroup wg: class 2 wg + q, values of that parity
                B[cls, tap, k2] = v_off(cls) + 2 * k2 * 9 * 8 + voff + ((k % 8) * 8 + (k // 8) * 9 * 8)[:, None] + ((n % 8) + (n // 8) * VPLANE)[None, :]
    return A, B


def pv_walk(Pbuf, V, g, drop_last_chunk=False, tkx_plus1=False, v_row_down=False, poff_col=0):
    """cam_pv_kernel on one image, one band: out [C, h, w]. The flags are the mutants."""
    n_chunks = g["KB"] // 8 - (1 if drop_last_chunk else 0)
    last_row = g["KT"] // g["tk_x"] - 1
    # value part of each chunk's stage: it does not depend on the output tile
    vst = torch.zeros(n_chunks, STAGE, dtype=torch.float64)
    for c in range(n_chunks):
        j = c >> 2
        kyc = (j // (g["tk_x"] + (1 if tkx_plus1 else 0))) * 32 + (c & 3) * 8
        kx0 = (j % g["tk_x"]) * 8
        if v_row_down and j // g["tk_x"] == last_row:
            kyc += 1
        for par in range(4):
            vst[c, v_off(par):v_off(par) + CB * VPLANE] = box(V[par * CB:(par + 1) * CB], kyc, kx0, 9, 9).reshape(-1)
    A_addr, B_addr = operand_addresses(poff_col)
    out = torch.zeros(C, g["h"], g["w"], dtype=torch.float64)
    Hs, Ws = g["Hs"], g["Ws"]
    for yy0 in range(0, Hs, 8):
        for xx0 in range(0, Ws, 8):
            st = vst.clone()
            pw = box(Pbuf, yy0 - 1, xx0 - 1, 9, 9)             # [KB, 9, 9, 8]: one row / column before the tile
            st[:, :PW] = pw[:n_chunks * 8].reshape(n_chunks, PW)
            A = st[:, A_addr]                                   # [chunks, tap, k2, 64, 16]
            for cls in range(4):
                acc = torch.einsum("ctsmk,ctskn->mn", A, st[:, B_addr[cls]]).view(8, 8, C)
                ny, nx = min(8, Hs - yy0), min(8, Ws - xx0)     # epilogue: yy < y1 = Hs, xx < Ws
                py, px = cls >> 1, cls & 1
                out[:, 2 * yy0 + py:2 * (yy0 + ny) + py:2, 2 * xx0 + px:2 * (xx0 + nx) + px:2] = acc[:ny, :nx].permute(2, 0, 1)
    return out


# --------------------------------------------------------------------------------------------- fp32: cam_split_fold_kernel
def split_fold(P, Q, g, row_stride=None):
    """O = P^T Q as the split P V GEMM writes it ([Mp, 16 C], column (u 4 + v) C + c), then the fold kernel's loop."""
    L, hs, ws, h, w = g["L"], g["hs"], g["ws"], g["h"], g["w"]
    Mp = -(-L // 256) * 256
    stride = ws if row_stride is None else row_stride
    O = torch.zeros(Mp + hs * 2 + 2, 16 * C, dtype=torch.float64)   # rows past Mp read as 0
    O[:L] = P.T @ Q.view(C, 16, L).permute(2, 1, 0).reshape(L, 16 * C)
    out = torch.zeros(C, h, w, dtype=torch.float64)
    ny, nx = torch.arange(hs), torch.arange(ws)
    for u in range(4):
        for v in range(4):
            rows = O[(ny[:, None] * stride + nx[None, :]).reshape(-1)][:, (u * 4 + v) * C:(u * 4 + v + 1) * C]
            out[:, u:u + 2 * hs:2, v:v + 2 * ws:2] += rows.view(hs, ws, C).permute(2, 0, 1)
    return out


# --------------------------------------------------------------------------------------------- fp32_direct
def softmax_rows(S, L, ldp, sum_to_ldp=False):
    """softmax_rows_kernel on rows S [rows, Lpad] -> P [rows, ldp]: registers for L <= 256 x 16, else re-reading S."""
    i = torch.arange(ldp)
    if L <= 256 * 16:
        v = torch.where(i < L, S[:, :ldp], torch.full_like(S[:, :ldp], -float("inf")))
        mx = v.max(1, keepdim=True).values
        e = torch.exp(v - mx)
        return torch.where(i < L, e / e.sum(1, keepdim=True), torch.zeros_like(e))
    mx = S[:, :L].max(1, keepdim=True).values
    s = torch.exp(S[:, :ldp if sum_to_ldp else L] - mx).sum(1, keepdim=True)
    return torch.where(i < L, torch.exp(S[:, :ldp] - mx) / s, torch.zeros_like(S[:, :ldp]))


def direct(S, feat, g, sum_to_ldp=False):
    """run_cam: softmax_rows over the logits [L queries, Lpad] (the direct conv writes columns < L only; the others are
    taken as 0 here), cam_pack_v_direct_kernel's values [class][tap][Lpad][C] and the classes' 2 x 2 convolutions."""
    L, hs, ws, Hs, Ws = g["L"], g["hs"], g["ws"], g["Hs"], g["Ws"]
    Lpad = -(-L // 128) * 128
    P = softmax_rows(S, L, Lpad, sum_to_ldp)
    f = feat[0]
    l = torch.arange(L)
    ly, lx = torch.div(l, ws, rounding_mode="floor"), l % ws
    vbuf = torch.zeros(4, 4, Lpad, C, dtype=torch.float64)
    for pc in range(4):
        for tap in range(4):
            py, px, a, bb = pc // 2, pc % 2, tap // 2, tap % 2
            vbuf[pc, tap, :L] = f[:, 2 * ly + py + 2 * a, 2 * lx + px + 2 * bb].T
    Pg = F.pad(P.view(hs, ws, Lpad), (0, 0, 1, 1, 1, 1))     # query rows / columns -1 and hs / ws are the conv's zero padding
    out = torch.zeros(C, g["h"], g["w"], dtype=torch.float64)
    for pc in range(4):
        for tap in range(4):
            a, bb = tap // 2, tap % 2                            # dy = -a, dx = -bb
            z = Pg[1 - a:1 - a + Hs, 1 - bb:1 - bb + Ws] @ vbuf[pc, tap]
            out[:, pc // 2::2, pc % 2::2] += z.permute(2, 0, 1)
    return out


def padded_logits(S, g):
    Lpad = -(-g["L"] // 128) * 128
    return F.pad(S.T, (0, Lpad - g["L"]))                         # [queries, Lpad]


# --------------------------------------------------------------------------------------------- correct walks
@pytest.mark.parametrize("h,w", MAPS)
def test_correct_walks_reproduce_float64(h, w):
    g = geometry(h, w)
    feat, mask_s = inputs(h, w)
    S, Q = logits(feat, mask_s)
    P = torch.softmax(S, 0)
    Y = fold(Q, P, g)
    scale = float(Y.abs().max())
    assert scale > 0
    got = {"bf16 cam_pv_kernel": pv_walk(p_buffer(P, g), s2d(feat), g),
           "fp32 cam_split_fold_kernel": split_fold(P, Q, g),
           "fp32_direct softmax_rows + pack_v": direct(padded_logits(S, g), feat, g)}
    for name, y in got.items():
        d = float((y - Y).abs().max())
        assert d <= 1e-12 * scale, (name, h, w, d)
    # the pointwise reference the GPU test uses agrees with this one
    px = [(0, 0, 0), (0, h - 1, w - 1), (0, h // 2, w // 3), (0, h - 3, w - 2)]
    ref = contextual_attention_at(feat, mask_s, px)
    assert float((ref - torch.stack([Y[:, y, x] for _, y, x in px])).abs().max()) <= 1e-12 * scale


# --------------------------------------------------------------------------------------------- mutants
def old_tolerances(y, Y):
    """which of the suite's earlier tolerances the deviation y - Y exceeds."""
    err = (y - Y).abs()
    top = max(1.0, float(Y.abs().max()))
    return {"2e-2 max": float(err.max()) > 2e-2 * top, "2e-4 max": float(err.max()) > 2e-4 * top,
            "1e-3 rel": bool((err > 1e-3 * Y.abs().clamp(min=1.0)).any())}


def _report(capsys, name, h, w, q, y, Y):
    old = old_tolerances(y, Y)
    if q > 1:
        verdict = "caught"
    else:
        verdict = "missed" if float((y - Y).abs().max()) > 0 else "no effect at this map"
    with capsys.disabled():
        print("\n[mutant %s at %dx%d] bound max ratio %.3g (%s); old tolerances: %s" % (
            name, h, w, q, verdict, ", ".join("%s %s" % (k, "caught" if v else "missed") for k, v in old.items())))
    return q > 1


def bf16_mutant(name, feat, mask_s, g):
    """the mutant's bf16 output from the S kernel's bf16 probabilities (attention_bf16_map) and bf16 values."""
    Pb = UB.attention_bf16_map(feat, mask_s)[0][0]
    V = s2d(feat)
    if name == "padding keys with nonzero P":
        # colscale without its -1: padding keys take part in the softmax with logit 0, as masked keys do
        S, _ = logits(feat, mask_s)
        n_pad = g["KB"] * 8 - g["L"]
        m = torch.clamp(S.max(0).values, min=0.0)
        e = torch.exp(S - m)
        s = e.sum(0) + n_pad * torch.exp(-m)
        return pv_walk(p_buffer(UB.bf16(e / s), g, pad=UB.bf16(torch.exp(-m) / s)), V, g)
    flags = {"last chunk dropped": dict(drop_last_chunk=True), "tk_x + 1 in kyc": dict(tkx_plus1=True),
             "value window one row down in the last key-tile row": dict(v_row_down=True),
             "poff one column off": dict(poff_col=1)}[name]
    return pv_walk(p_buffer(Pb, g), V, g, **flags)


BF16_MUTANTS = ["last chunk dropped", "tk_x + 1 in kyc", "value window one row down in the last key-tile row", "poff one column off",
                "padding keys with nonzero P"]
# the small maps of the table, where the bf16 bound's [L, L] float64 tensors stay small on the CPU; the last chunk holds
# real keys only where hs % 32 is 0 or above 24, so it also runs at the 512^2 working map (its last chunk: 56 of 3969 keys)
BF16_MUTANT_MAPS = [(66, 18), (68, 20), (132, 36), (68, 100)]


@pytest.mark.parametrize("name", BF16_MUTANTS)
def test_bf16_mutant_exceeds_the_bound(name, capsys):
    caught = []
    for h, w in BF16_MUTANT_MAPS + ([(128, 128)] if name == "last chunk dropped" else []):
        g = geometry(h, w)
        if name == "padding keys with nonzero P" and g["KB"] * 8 == g["L"]:
            continue                                            # no padding keys at this map
        feat, mask_s = inputs(h, w)
        Y, bound = UB.attention_bf16_reference(feat, mask_s)
        assert float((pv_walk(p_buffer(UB.attention_bf16_map(feat, mask_s)[0][0], g), s2d(feat), g) - Y[0]).abs().max()) <= 1e-12
        y = bf16_mutant(name, feat, mask_s, g)
        caught.append(_report(capsys, name, h, w, UB.max_ratio(y, Y[0], bound[0]), y, Y[0]))
    assert any(caught), name


def _fp32_ratio(y, Y, feat, mask_s, prec, g, n=64):
    """max |y - Y| / bound over the n pixels where the mutant moves the output most, with the bound of the fp32 modes
    (contextual_attention_at with attention_err, as tests/test_gpu_attention_output.py)."""
    err = (y - Y).abs().amax(0).view(-1)
    idx = torch.topk(err, n).indices
    px = [(0, int(i) // g["w"], int(i) % g["w"]) for i in idx]
    e = UB.attention_err(prec, C, g["h"], g["w"])
    ref, t = contextual_attention_at(feat, mask_s, px, err=e)
    assert float((ref - torch.stack([Y[:, yy, xx] for _, yy, xx in px])).abs().max()) <= 1e-12 * max(1.0, float(Y.abs().max()))
    got = torch.stack([y[:, yy, xx] for _, yy, xx in px])
    return UB.max_ratio(got, ref, UB.attention_out_bound(t["bound"], ref, "fp32"))


@pytest.mark.parametrize("h,w", [(68, 20), (132, 36)])
def test_fold_row_stride_mutant_exceeds_the_bound(h, w, capsys):
    g = geometry(h, w)
    feat, mask_s = inputs(h, w)
    S, Q = logits(feat, mask_s)
    P = torch.softmax(S, 0)
    Y = fold(Q, P, g)
    y = split_fold(P, Q, g, row_stride=g["ws"] + 1)
    assert _report(capsys, "fold row stride ws + 1", h, w, _fp32_ratio(y, Y, feat, mask_s, "fp32", g), y, Y)


@pytest.mark.parametrize("h,w", [(132, 132), (36, 484)])
@pytest.mark.parametrize("mkind", ["valid", "rect"])
def test_softmax_reread_sum_mutant_exceeds_the_bound(h, w, mkind, capsys):
    """L = 4225 and 4097: past softmax_rows' 4096 keys in registers; the mutant sums the row's Lpad - L padding logits too."""
    g = geometry(h, w)
    assert g["L"] > 4096
    feat, mask_s = inputs(h, w, mkind)
    S, Q = logits(feat, mask_s)
    Y = fold(Q, torch.softmax(S, 0), g)
    y = direct(padded_logits(S, g), feat, g, sum_to_ldp=True)
    assert _report(capsys, "softmax re-read sum over ldp (%s mask)" % mkind, h, w, _fp32_ratio(y, Y, feat, mask_s, "fp32_direct", g), y, Y)

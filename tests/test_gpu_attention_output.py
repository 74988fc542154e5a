"""The attention output (pmconv9's input) against float64 with per-element bounds (tests/util_bounds.py) where the P V step
walks several key tiles, output tiles and bands: cam_pv_kernel (bf16), the split-half P V GEMM and cam_split_fold_kernel
(fp32), cam_pack_v_direct_kernel with the direct convolution and softmax_rows_kernel (fp32_direct).

Feature maps (h, w) -> patch grid (hs, ws), L keys, chosen from the kernel constants (16 x 8 query tiles, 32 x 8 key tiles,
8 x 8 PV output tiles, 64-key chunks, 128 / 256 split GEMM tiles, softmax_rows' 4096 keys in registers):
  66 x 18   32 x 8, 256     exactly one key tile; a one-column last PV output tile; L = one split N tile
  68 x 20   33 x 9, 297     a second key-tile row and column holding one key each
  132 x 36  65 x 17, 1105   three key-tile rows, the last one a single row
  68 x 100  33 x 49, 1617   seven key-tile columns, the last one a single column
  128 x 128 63 x 63, 3969   the 512^2 working map: two key-tile rows, chunk row 3 of the second partial
  130 x 130 64 x 64, 4096   softmax_rows at its in-register limit
  132 x 132 65 x 65, 4225   one past it (the re-reading path); Mp = 4352
  36 x 484  17 x 241, 4097  one key past the limit; 31 key-tile and 31 PV output-tile columns
with masks that are one rectangle, all valid, valid fractions 25/256 | 26/256 and one valid key, and per image at B = 2.
bf16 is checked at every pixel (the float64 reference on the GPU, one image at a time); the fp32 modes at the pixels of
every class row and column on a chunk, key-tile or output-tile boundary (class rows 8k - 1, 8k, 32k - 1, 32k, Hs - 1 and
the same columns) where they cross, each boundary row and column at random places, every pixel of the last two class rows
and columns, and random 2 x 2 blocks. Also: a persistent walk (128 x 128 at B = 5: 320 PV and 160 S tiles, so CTAs run a
second tile across an image boundary), every map with hs >= 33 in bands under workspace limits, and the forward's own
attention at 512 x 512 and 512 x 408 (B = 2). Each check prints max |y - Y| / bound.
"""
import random

import pytest
import torch

from sketchedit_b200 import synth
from sketchedit_b200.engine import contextual_attention
from tests import util_bounds as UB
from tests import util_stages as US
from tests.test_attention_bands import _grid, attention_limit, bf16_row_bytes, direct_row_bytes, forced_limits, split_row_bytes  # noqa: F401
from tests.test_gpu_error_bounds import _feat, _mask_s
from tests.test_gpu_forward_stages import _inference
from tests.util_attention import contextual_attention_at, sample_pixels

pytestmark = pytest.mark.gpu
PRECS = ["bf16", "fp32", "fp32_direct"]
MAPS = [(66, 18), (68, 20), (132, 36), (68, 100), (128, 128), (130, 130), (132, 132), (36, 484)]
MASKS = ["rect", "valid", "frac25_26", "one_key", "per_image"]


def _inputs(h, w, mkind, B=1):
    if mkind == "per_image":                    # B = 2: image 0 one rectangle, image 1 the 25/256 | 26/256 split
        feat = _feat("0.15", 2, h, w, seed=UB.stable_seed("out", h, w, mkind))
        return feat, torch.cat([_mask_s("rect", 1, h, w), _mask_s("frac25_26", 1, h, w)])
    return _feat("0.15", B, h, w, seed=UB.stable_seed("out", h, w, mkind, B)), _mask_s(mkind, B, h, w)


def _boundaries(n):
    """class rows (or columns) 8k - 1, 8k, 32k - 1, 32k and n - 1 below n: chunk, key-tile and output-tile edges."""
    s = {n - 1}
    for k in range(1, n // 8 + 1):
        s |= {8 * k - 1, 8 * k}
    return sorted(v for v in s if v < n)


def boundary_pixels(B, h, w, seed):
    """(b, y, x) of the classes (yy, xx) where boundary rows and columns cross, of each boundary row and column at four
    random places, of the last two class rows and columns, plus sample_pixels' corners and 16 random 2 x 2 blocks."""
    Hs, Ws = h // 2, w // 2
    rows, cols = _boundaries(Hs), _boundaries(Ws)
    rnd = random.Random(seed)
    cls = {(y, x) for y in rows for x in cols}
    cls |= {(y, rnd.randrange(Ws)) for y in rows for _ in range(4)} | {(rnd.randrange(Hs), x) for x in cols for _ in range(4)}
    cls |= {(y, x) for y in (Hs - 2, Hs - 1) for x in range(Ws)} | {(y, x) for y in range(Hs) for x in (Ws - 2, Ws - 1)}
    px = [(b, 2 * y + py, 2 * x + px) for b in range(B) for y, x in sorted(cls) for py in (0, 1) for px in (0, 1)]
    return sample_pixels(B, h, w, 16, seed, extra=px)


_REF = {}


def reference(prec, h, w, mkind, feat, mask_s):
    """(pixels or None, Y, bound) of the inputs, cached for the banded runs of the same case."""
    key = (prec, h, w, mkind, feat.shape[0])
    if key not in _REF:
        if prec == "bf16":
            parts = [UB.attention_bf16_reference(feat[b:b + 1].cuda(), mask_s[b:b + 1].cuda()) for b in range(feat.shape[0])]
            _REF[key] = (None, torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]))
        else:
            px = boundary_pixels(feat.shape[0], h, w, seed=UB.stable_seed(h, w, mkind))
            ref, t = contextual_attention_at(feat, mask_s, px, err=UB.attention_err(prec, feat.shape[1], h, w))
            _REF[key] = (px, ref, UB.attention_out_bound(t["bound"], ref, "fp32"))
    return _REF[key]


def ratio(out, ref):
    px, Y, bound = ref
    if px is None:
        return UB.max_ratio(out.cuda().double(), Y, bound)
    o = out.cpu()
    return UB.max_ratio(torch.stack([o[b, :, y, x] for b, y, x in px]), Y, bound)


def _print(capsys, msg):
    with capsys.disabled():
        print("\n[attention output %s" % msg)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("mkind", MASKS)
@pytest.mark.parametrize("h,w", MAPS)
def test_attention_output_within_bound(h, w, mkind, prec, capsys):
    feat, mask_s = _inputs(h, w, mkind)
    out = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec)
    ref = reference(prec, h, w, mkind, feat, mask_s)
    q = ratio(out, ref)
    hs, ws = _grid(h, w)
    npx = "all" if ref[0] is None else len(ref[0])
    _print(capsys, "%s %dx%d -> %dx%d L %d B%d %s, %s pixels] max ratio %.3g" % (prec, h, w, hs, ws, hs * ws, feat.shape[0], mkind, npx, q))
    assert q <= 1.0, q


def test_persistent_walk_b5(capsys):
    """128 x 128 at B = 5: 320 PV output tiles and 160 S query tiles on 132 SMs, so CTAs take a second tile, and that tile
    lies in another image. Images 0, 2 and 4 are bounded and equal their B = 1 runs bit for bit."""
    h, w, B = 128, 128, 5
    feat = torch.cat([_feat("0.15", 1, h, w, seed=UB.stable_seed("walk5", b)) for b in range(B)])
    kinds = ["rect", "valid", "frac25_26", "one_key", "rect"]
    mask_s = torch.cat([_mask_s(k, 1, h, w) for k in kinds])
    out = contextual_attention(feat.cuda(), mask_s.cuda(), precision="bf16")
    for b in (0, 2, 4):
        one = contextual_attention(feat[b:b + 1].cuda(), mask_s[b:b + 1].cuda(), precision="bf16")
        assert torch.equal(out[b:b + 1], one), b
        Y, bound = UB.attention_bf16_reference(feat[b:b + 1].cuda(), mask_s[b:b + 1].cuda())
        q = UB.max_ratio(out[b:b + 1].double(), Y, bound)
        _print(capsys, "bf16 %dx%d B%d image %d %s] max ratio %.3g" % (h, w, B, b, kinds[b], q))
        assert q <= 1.0, (b, q)


def band_plan(prec, B, h, w, limit):
    """bands of the workspace limit, mirrored from the plans (se_cam.cu cam_plan, se_gemm_split.cu cam_split_plan,
    se_engine.cu run_cam): (rows per band, bands)."""
    hs, ws = _grid(h, w)
    if prec == "bf16":
        band = min(limit // bf16_row_bytes(B, h, w) - 1, hs) // 16 * 16
        return band, -(-hs // band)
    if prec == "fp32":
        Mp = -(-hs * ws // 256) * 256
        band = limit // split_row_bytes(B, h, w) // 128 * 128
        return band, -(-Mp // band)
    R = limit // direct_row_bytes(B, h, w) - 1
    return R, -(-(h // 2) // R)


BAND_MAPS = [(h, w) for h, w in MAPS if _grid(h, w)[0] >= 33]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("h,w", BAND_MAPS)
def test_bands_within_bound(h, w, prec, attention_limit, capsys):
    """workspace limits that force three bands or more; in bf16 always 16-row bands too, whose edges fall inside a key-tile
    row and whose carried query row is used twice or more. Each result is bounded and equals the single band."""
    feat, mask_s = _inputs(h, w, "rect")
    attention_limit(0)
    one = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec)
    ref = reference(prec, h, w, "rect", feat, mask_s)
    limits = forced_limits(prec, 1, h, w)
    if prec == "bf16":
        limits = sorted({bf16_row_bytes(1, h, w) * 17, bf16_row_bytes(1, h, w) * 33} | set(limits))
    limits = [lim for lim in limits if band_plan(prec, 1, h, w, lim)[1] >= 3]
    assert limits and (prec != "bf16" or band_plan(prec, 1, h, w, limits[0])[0] == 16), limits
    for lim in limits:
        attention_limit(lim)
        banded = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec)
        q = ratio(banded, ref)
        band, n = band_plan(prec, 1, h, w, lim)
        _print(capsys, "%s %dx%d rect, %d bands of %d] max ratio %.3g" % (prec, h, w, n, band, q))
        assert q <= 1.0, (lim, q)
        assert torch.equal(banded, one), (lim, float((banded - one).abs().max()))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("B,H,W", [(1, 512, 512), (2, 512, 408)])
def test_forward_attention_within_bound(B, H, W, prec, capsys):
    """util_stages.check_attention on a tapped forward at the 512^2 working size and the Places shape: pmconv9's input
    against float64 of the forward's own stored feature map and pooled mask (bf16: the reference on the GPU)."""
    img, sk = synth.synth_inputs(B, H, W, seed=H + W + B)
    T, _, _, io = _inference(prec, img, sk, {})
    if prec == "bf16":
        T = {k: T[k].cuda() for k in ("in:G.cam", "in:G.cam.mask_s", "in:G.pmconv9")}
        io = dict(mask=io["mask"].cuda())
    res = US.check_attention(T, io, prec)
    _print(capsys, "forward %s %dx%dx%d] %s" % (prec, B, H, W, ", ".join("%s max ratio %.3g" % kv for kv in sorted(res.items()))))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad

"""CPU side of tests/test_gpu_attention_map.py and tests/test_gpu_detail_float64.py: the vectorised float64 fold is the loop's,
the boxes and holes those tests use have the geometry they claim, and each check fails on a CPU emulation of a plausible
bug: an attention export that swaps two key tiles or drops the key-tile row term, a map with hs and ws transposed, a detail
plane read one footprint column off, one box's detail computed with another box's attention, and the plane added to the
paste mask instead of to the colour."""
import numpy as np
import pytest
import torch
from PIL import Image

from sketchedit_b200.serving import feather_mask
from tests import util_bounds as UB
from tests import util_detail as U
from tests.test_gpu_detail_float64 import HOLES, _boxes, _hole, _min_side, _weights
from tests.test_gpu_error_bounds import _feat, _mask_s


def _case(bh, bw, Hn, Wn, hole_kind, seed):
    rs = np.random.RandomState(seed)
    crop = rs.randint(0, 256, (bh, bw, 3), dtype=np.uint8)
    hole = (_hole(hole_kind, Hn, Wn) >= 128).astype(np.uint8)
    return crop, U.low_of(crop, Hn, Wn), hole, _weights("dominant", hole, rs).numpy()


@pytest.mark.parametrize("hole_kind", HOLES)
@pytest.mark.parametrize("bh,bw,Hn,Wn", [(152, 120, 64, 48), (40, 61, 48, 64), (7, 5, 64, 48), (64, 48, 64, 48), (5, 3, 16, 16),
                                          (130, 97, 32, 24)])
def test_vectorised_fold_is_the_loop(bh, bw, Hn, Wn, hole_kind):
    crop, low, hole, P = _case(bh, bw, Hn, Wn, hole_kind, bh * bw)
    A, D, inh = U.aggregate(crop, low, hole, P)
    Av, Dv, inhv = U.aggregate_vec(crop, low, hole, P)
    assert np.array_equal(inh, inhv) and np.array_equal(D, Dv)
    assert np.abs(A - Av).max(initial=0.0) <= 1e-9 * 255
    assert not U.violations(Av, Dv, A, D, inh, P.shape[0])


def test_box_and_hole_geometry():
    for Hn, Wn in [(192, 320), (320, 192), (272, 200), (512, 512), (64, 48), (16, 16)]:
        boxes = _boxes(Hn, Wn)
        sizes = [(b[2] - b[0]) * (b[3] - b[1]) for b in boxes]
        assert sizes[0] > sizes[1] < sizes[4]                        # large -> small -> large: the scratch changes size
        assert U.footprint(_min_side(Wn), Wn) == 3 and U.footprint(_min_side(Hn), Hn) == 3
        assert any(b[2] - b[0] == Wn and b[3] - b[1] != Hn for b in boxes)
        assert max(b[2] for b in boxes) == 2600 and max(b[3] for b in boxes) == 2200       # flush with the photo's edges
        edges = _hole("edges", Hn, Wn) >= 128
        assert edges[0].any() and edges[-1].any() and edges[:, 0].any() and edges[:, -1].any()
        assert (_hole("line", Hn, Wn) >= 128).sum(0).max() == 1
    assert (_boxes(16, 16)[0][2] - _boxes(16, 16)[0][0]) / 16 >= 8 and (_boxes(64, 48)[0][2] - _boxes(64, 48)[0][0]) / 48 >= 8


# --------------------------------------------------------------------------------------------- the attention map's check
def export_emulation(Pb, hs, ws, mutation=None):
    """cam_attn_export_kernel on CPU: Pb [B, keys, queries] written in the S kernel's key-tile order (key (ky, kx) in row
    j * 32 + ky % 32 of key block j = (ky / 32) tk_x + kx / 8, lane kx % 8), then read back as the kernel decodes it."""
    B, L, _ = Pb.shape
    tk_x = (ws + 7) // 8
    KB = tk_x * ((hs + 31) // 32) * 32
    ky, kx = np.divmod(np.arange(L), ws)

    def rows(j):
        return (j * 32 + ky % 32) * 8 + kx % 8

    buf = torch.zeros(B, KB * 8, L, dtype=Pb.dtype)
    buf[:, rows((ky // 32) * tk_x + kx // 8)] = Pb
    j = (ky // 32) * tk_x + kx // 8
    if mutation == "drop_tile_row":
        j = kx // 8
    elif mutation == "swap_tiles":
        j = np.where(j == 0, 1, np.where(j == 1, 0, j))
    return buf[:, rows(j)]


@pytest.mark.parametrize("h,w", [(68, 20), (132, 36)])
def test_attention_map_check_catches_export_bugs(h, w):
    """hs = 33 and 65: two and three key-tile rows, so the tile-row term and the tile order matter."""
    feat, mask_s = _feat("0.15", 1, h, w, seed=5), _mask_s("rect", 1, h, w)
    hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
    Pb, Wp = UB.attention_bf16_map(feat, mask_s)
    q = {m: UB.max_ratio(export_emulation(Pb, hs, ws, m), Pb, Wp) for m in (None, "drop_tile_row", "swap_tiles")}
    transposed = Pb.view(1, hs, ws, hs, ws).permute(0, 2, 1, 4, 3).reshape(Pb.shape)
    q["transposed"] = UB.max_ratio(transposed, Pb, Wp)
    print("attention map %dx%d: max bound ratios %s" % (h, w, q))
    assert q[None] == 0.0 and min(q["drop_tile_row"], q["swap_tiles"], q["transposed"]) > 1.0, q


def test_fp32_map_check_catches_a_transposed_map():
    feat, mask_s = _feat("0.15", 1, 68, 20, seed=6), _mask_s("rect", 1, 68, 20)
    P, bound = UB.attention_fp32_map(feat, mask_s)
    assert UB.max_ratio(P.float(), P, bound) <= 1.0
    assert UB.max_ratio(P.view(1, 33, 9, 33, 9).permute(0, 2, 1, 4, 3).reshape(P.shape).float(), P, bound) > 1.0


# --------------------------------------------------------------------------------------------- the detail checks
def fold_shifted(crop, low, hole, P, shift):
    """aggregate() with the fold reading each patch sum `shift` footprint columns right of its own (clamped)."""
    bh, bw = crop.shape[:2]
    Hn, Wn = hole.shape
    ws = Wn // 8 - 1
    ax, ay = U.anchors(bw, Wn), U.anchors(bh, Hn)
    fw, fh = U.footprint(bw, Wn), U.footprint(bh, Hn)
    R, inh = U.residual(crop, low, hole)
    ky, kx = np.divmod(np.arange(P.shape[0]), ws)
    sy = np.minimum(ay[ky][:, None] + np.arange(fh)[None], bh - 1)
    sx = np.minimum(ax[kx][:, None] + np.arange(fw)[None], bw - 1)
    C = (P.astype(np.float64).T @ R[sy[:, :, None], sx[:, None, :]].reshape(P.shape[0], -1)).reshape(-1, fh, fw, 3)
    A = np.zeros((bh, bw, 3))
    u, v = U.work_of(np.arange(bw), bw, Wn), U.work_of(np.arange(bh), bh, Hn)
    for y, x in zip(*np.nonzero(inh)):
        qs = [(py, px) for py in U.covering(v[y], Hn) for px in U.covering(u[x], Wn)]
        A[y, x] = sum(C[py * ws + px, y - ay[py], min(x - ax[px] + shift, fw - 1)] for py, px in qs) / len(qs)
    D = np.where(inh[..., None], np.sign(A) * np.floor(np.abs(A) + 0.5), 0).astype(np.int64)
    return A, D


def test_detail_check_catches_a_plane_one_column_off():
    crop, low, hole, P = _case(152, 120, 64, 48, "rect", 3)
    A64, D64, inh = U.aggregate(crop, low, hole, P)
    assert not U.violations(*fold_shifted(crop, low, hole, P, 0), A64, D64, inh, P.shape[0])
    v = U.violations(*fold_shifted(crop, low, hole, P, 1), A64, D64, inh, P.shape[0])
    assert "|A - A64| > bound" in v and "|D - D64| > 1" in v, v


def test_detail_check_catches_another_boxs_attention():
    crop, low, hole, P = _case(152, 120, 64, 48, "rect", 4)
    P0 = _case(152, 120, 64, 48, "rect", 5)[3]
    A64, D64, inh = U.aggregate(crop, low, hole, P)
    A, D, _ = U.aggregate(crop, low, hole, P0)
    v = U.violations(A, D, A64, D64, inh, P.shape[0])
    assert "|A - A64| > bound" in v and "|D - D64| > 1" in v, v


def test_paste_check_catches_the_plane_on_the_mask():
    """The paste test compares bytes: the plane added to the paste mask instead of the colour changes them."""
    rs = np.random.RandomState(8)
    canvas = Image.fromarray(rs.randint(0, 256, (60, 70, 3), dtype=np.uint8))
    up = rs.randint(0, 256, (40, 50, 3)).astype(np.int64)
    m = feather_mask(rs.randint(0, 256, (40, 50), dtype=np.uint8), (3, 0, 5, 2))
    d = rs.randint(-40, 41, (40, 50, 3))
    right, wrong = canvas.copy(), canvas.copy()
    right.paste(Image.fromarray(np.clip(up + d, 0, 255).astype(np.uint8)), (7, 9), Image.fromarray(m))
    wrong.paste(Image.fromarray(up.astype(np.uint8)), (7, 9), Image.fromarray(np.clip(m + d[..., 0], 0, 255).astype(np.uint8)))
    assert not np.array_equal(np.asarray(right), np.asarray(wrong))

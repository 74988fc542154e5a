"""Previews on the CPU: Pillow 12.2's Image.thumbnail restated in numpy (tests/util_thumbnail.py) and pinned against Pillow
(the size rule, Image.reduce over every cell sum and every partial-cell remainder, the whole thumbnail on random and
photo-like images across factors and the tall branch), EditSession.image/jpeg/png(size=...) in the host flow after edits
and undo, the argument checks, the host checks of se_resize_reducing_u8, and the registers of se_thumbnail.cu."""
import ctypes
import io
import os
import re
import shutil
import subprocess

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build, engine
from tests import util_thumbnail as U
from tests.test_edit_session import _chain, _FakeProcessor, _NoForward, _photo

PHOTOS = [(4000, 2667), (2667, 4000), (1000, 667), (640, 427), (1, 1), (1, 500), (500, 1), (3, 5000), (17, 2001), (333, 777),
          (100, 100), (30, 20000)]
BOUNDS = [(640, 640), (256, 256), (1280, 1280), (1, 1), (1, 1000), (1000, 1), (4000, 10), (10, 4000), (639, 427), (640, 426),
          (5000, 5000), (100, 3), (5, 5000), (999, 20000)]


def test_thumbnail_size_is_pillows():
    """Every photo size and bound: no-op, 1-pixel sides, extreme aspect ratios, a bound larger on one axis only."""
    for w, h in PHOTOS:
        for size in BOUNDS:
            im = Image.new("1", (w, h))              # the size rule does not depend on the mode
            im.thumbnail(size)
            got = engine.thumbnail_size(w, h, size)
            assert (got or (w, h)) == im.size, ((w, h), size, got, im.size)
            assert got is None or got != (w, h)
    assert engine.thumbnail_size(4000, 2667, (640, 640)) == (640, 427)
    assert engine.thumbnail_size(640, 427, (640, 427)) is None


def _cells_with_sums(fx, fy, sums):
    """An RGB image of fx x fy cells whose channel sums are `sums` (3 per cell, the last cell's padded with its last sum):
    a cell with sum s has s % n pixels of s // n + 1 and the rest of s // n."""
    n = fx * fy
    s = np.concatenate([sums, np.full((-len(sums)) % 3, sums[-1])]).reshape(-1, 3)
    k = len(s)
    cols = int(np.ceil(np.sqrt(k)))
    rows = -(-k // cols)
    s = np.concatenate([s, np.zeros((rows * cols - k, 3), s.dtype)])
    q, r = s // n, s % n
    pix = (q[:, None, :] + (np.arange(n)[None, :, None] < r[:, None, :])).astype(np.uint8)     # [cells, n, 3]
    img = pix.reshape(rows, cols, fy, fx, 3).transpose(0, 2, 1, 3, 4).reshape(rows * fy, cols * fx, 3)
    return np.ascontiguousarray(img)


def _reduce_matches(a, fx, fy):
    want = np.array(Image.fromarray(a).reduce((fx, fy)))
    got = U.reduce(a, fx, fy)
    return got.shape == want.shape and np.array_equal(got, want), int((got != want).sum()) if got.shape == want.shape else -1


@pytest.mark.parametrize("fy", range(1, 17))
def test_reduce_every_cell_sum(fy):
    """Every sum 0 .. 255 n of a full cell, for every factor pair up to 16 x 16 (Pillow has its own loops for small ones)."""
    for fx in range(1, 17):
        n = fx * fy
        ok, nbad = _reduce_matches(_cells_with_sums(fx, fy, np.arange(255 * n + 1)), fx, fy)
        assert ok, (fx, fy, nbad, PIL.__version__)


@pytest.mark.parametrize("fx, fy", [(1, 200), (200, 1), (37, 2), (2, 37), (25, 3), (64, 64)])
def test_reduce_every_cell_sum_of_asymmetric_factors(fx, fy):
    n = fx * fy
    sums = np.arange(255 * n + 1) if n <= 256 else np.unique(np.concatenate([np.arange(0, 255 * n + 1, 97),
                                                                                np.arange(255 * n - 3000, 255 * n + 1)]))
    ok, nbad = _reduce_matches(_cells_with_sums(fx, fy, sums), fx, fy)
    assert ok, (fx, fy, nbad)


def test_reduce_partial_cells_every_remainder():
    """Images whose right and bottom cells hold every remainder of the factors up to 9 (and a few larger ones), with random,
    255-filled and near-255 content: a partial cell averages over its own pixel count."""
    rs = np.random.RandomState(3)
    pairs = [(fx, fy) for fx in range(1, 10) for fy in range(1, 10)] + [(1, 200), (37, 2), (16, 13)]
    for fx, fy in pairs:
        for rx in range(fx):
            for ry in range(fy):
                h, w = 2 * fy + ry, 3 * fx + rx
                for kind in range(3):
                    if kind == 0:
                        a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
                    elif kind == 1:
                        a = np.full((h, w, 3), 255, np.uint8)
                    else:
                        a = (255 - rs.randint(0, 3, (h, w, 3))).astype(np.uint8)
                    ok, nbad = _reduce_matches(a, fx, fy)
                    assert ok, (fx, fy, rx, ry, kind, nbad)


def _random(h, w, seed):
    a = np.random.RandomState(seed).randint(0, 256, (h, w, 3), dtype=np.uint8)
    a[: h // 3] = 255                        # flat regions and hard edges next to the noise: every clamp is reached
    a[h // 3: h // 2] = 0
    return a


# ((h, w), bound): factors 1 to 31 and 2000 x 1333, one axis reduced, the tall branch with and without a reduce
THUMBS = [((2667, 4000), (640, 640)), ((2667, 4000), (64, 64)), ((2667, 4000), (1, 1)), ((667, 1000), (640, 640)),
          ((667, 1000), (256, 256)), ((1001, 999), (71, 99)), ((5000, 3), (1, 100)), ((3000, 20), (10, 30)),
          ((2001, 17), (16, 2000)), ((5000, 3), (1, 1000)), ((20000, 30), (5, 5000)), ((100, 100), (3, 100)),
          ((7, 1000), (50, 50)), ((333, 777), (31, 31)), ((2000, 5), (2, 50)), ((200, 1), (1, 10)), ((50, 60), (49, 100)),
          ((1200, 1000), (19, 19)), ((427, 640), (640, 640))]


@pytest.mark.parametrize("hw, size", THUMBS)
def test_thumbnail_is_pillow(hw, size):
    """The whole restatement equals Image.thumbnail byte for byte on random and photo-like content."""
    for a in (_random(*hw, seed=hw[0] + hw[1]), U.photo_like(*hw, seed=7)):
        im = Image.fromarray(a)
        im.thumbnail(size)
        want = np.asarray(im)
        got = U.thumbnail(a, size)
        assert got.shape == want.shape and np.array_equal(got, want), (hw, size, PIL.__version__)


def test_the_tall_branch_changes_bytes():
    """Where Pillow resamples vertically first, horizontal-first gives other bytes: the order matters."""
    for hw, size in (((2001, 17), (16, 2000)), ((20000, 30), (5, 5000))):
        a = _random(*hw, seed=1)
        ts = engine.thumbnail_size(hw[1], hw[0], size)
        fx, fy = U.factors(hw, (ts[1], ts[0]))
        r = U.reduce(a, fx, fy) if fx > 1 or fy > 1 else a
        assert r.shape[0] > 100 * r.shape[1]
        in1_w, in1_h = hw[1] / fx, hw[0] / fy
        hv = U.resample(U.resample(r, 1, in1_w, ts[0]), 0, in1_h, ts[1])
        assert not np.array_equal(hv, U.thumbnail(a, size)), hw


# ---------------------------------------------------------------------------------------------------- sessions (host)
@pytest.fixture
def proc():
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    yield p
    p.close()


def _jpeg(img, **kw):
    buf = io.BytesIO()
    img.save(buf, "JPEG", **kw)
    return buf.getvalue()


def _png(img):
    import cv2
    return cv2.imencode(".png", np.ascontiguousarray(np.asarray(img)[:, :, ::-1]))[1].tobytes()


def check_previews(s, box, size):
    """s.image/jpeg/png(size=...) against the Pillow statements on s.image(); the session's photo is left as it was."""
    before = np.asarray(s.image())
    full = s.image()
    img = full.crop(box) if box is not None else full.copy()
    img.thumbnail(size)
    if box is None:
        assert np.array_equal(np.asarray(s.image(size=size)), np.asarray(img)), size
    for q, sub, opt, prog in ((75, 2, False, False), (90, 0, True, False), (75, 2, False, True)):
        try:
            want = _jpeg(img, quality=q, subsampling=sub, optimize=opt, progressive=prog)
        except OSError:                  # Pillow refuses optimized files past its buffer (noise at quality 90, 4:4:4)
            with pytest.raises(OSError):
                s.jpeg(q, sub, box=box, size=size, optimize=opt, progressive=prog)
            continue
        assert s.jpeg(q, sub, box=box, size=size, optimize=opt, progressive=prog) == want, (box, size, q, sub, opt, prog)
    assert s.png(box, size=size) == _png(img)
    assert np.array_equal(np.asarray(s.image()), before)


def test_host_session_previews_after_edits_and_undo(proc):
    s = proc.open_session(_photo())
    check_previews(s, None, (64, 64))
    for k, (mask, em, region) in enumerate(_chain()[:5]):
        r = s.edit(mask, em, region=region)
        check_previews(s, None, [(64, 64), (299, 5), (1, 1), (300, 200)][k % 4])
        check_previews(s, r.boxes[0], (16, 16))
    s.undo()
    check_previews(s, None, (100, 100))
    check_previews(s, (10, 20, 290, 190), (np.int64(70), np.int32(70)))
    s.undo()
    check_previews(s, None, (33, 200))


def test_a_size_that_fits_gives_todays_bytes(proc):
    s = proc.open_session(_photo())
    for size in ((300, 200), (5000, 200), (300, 4000)):
        assert np.array_equal(np.asarray(s.image(size=size)), np.asarray(s.image()))
        assert s.jpeg(size=size) == s.jpeg()
        assert s.png(size=size) == s.png()
        assert s.png((3, 4, 50, 60), size=(47, 56)) == s.png((3, 4, 50, 60))


BAD_SIZES = [(0, 5), (5, 0), (-1, 5), (5,), (1, 2, 3), (True, 5), (5, False), (5.0, 5), (5, np.float32(5)), "ab", 7, {1: 2},
             (None, 5)]


def test_size_validation(proc):
    s = proc.open_session(_photo())
    for bad in BAD_SIZES:
        for call in (lambda: s.image(size=bad), lambda: s.jpeg(size=bad), lambda: s.png(size=bad),
                     lambda: engine.thumbnail_u8([], bad)):
            with pytest.raises(ValueError, match="size must be"):
                call()
    assert engine.check_thumbnail_size([np.int64(3), 2]) == (3, 2)


# ---------------------------------------------------------------------------------------------------- the C entry's host side
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _query(lib, src_hw, dst_hw, pitch=None, n=1):
    L = ctypes.c_longlong
    need = L(-1)
    k = max(n, 1)
    rc = lib.se_resize_reducing_u8(None, (L * k)(*([pitch or 3 * src_hw[1]] * k)), (ctypes.c_int * (2 * k))(*(src_hw * k)),
                                   None, (L * k)(*([0] * k)), (ctypes.c_int * (2 * k))(*(dst_hw * k)), n, None, ctypes.byref(need),
                                   None)
    return rc, need.value


def test_entry_scratch_query_and_checks(lib):
    r256 = lambda b: (b + 255) // 256 * 256
    assert _query(lib, (2667, 4000), (427, 640)) == (0, r256(889 * 1334 * 3) + r256(889 * 640 * 3))   # reduced + intermediate
    assert _query(lib, (667, 1000), (427, 640)) == (0, r256(667 * 640 * 3))                            # no reduce
    assert _query(lib, (667, 1000), (667, 640)) == (0, 0)                                              # one pass, no reduce
    assert _query(lib, (667, 1000), (667, 1000)) == (0, 0)                                             # a copy
    assert _query(lib, (2001, 17), (1883, 16)) == (0, r256(1883 * 17 * 3))                             # vertical first
    assert _query(lib, (20000, 30), (3333, 5)) == (0, r256(6667 * 10 * 3) + r256(3333 * 10 * 3))
    assert _query(lib, (2667, 4000), (427, 640), n=32)[0] == 0
    assert _query(lib, (2667, 4000), (427, 640), n=33)[0] != 0
    assert _query(lib, (2667, 4000), (427, 640), pitch=11999)[0] != 0
    assert b"narrower" in lib.se_last_error()
    assert _query(lib, (2667, 4000), (0, 640))[0] != 0
    assert _query(lib, (65535, 65535), (1, 1))[0] != 0                                                # cells of 2^30 pixels
    assert b"2^24" in lib.se_last_error()
    assert _query(lib, (8000, 8000), (1, 1))[0] == 0                                                  # 4000 x 4000 cells


def test_thumbnail_kernels_do_not_spill(tmp_path):
    """se_thumbnail.cu compiled for sm_90a with the library's flags: its one kernel keeps everything in registers."""
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    flags = [f for f in build.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "se_thumbnail.cu"), "-o", str(tmp_path / "t.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout[-3000:]
    assert "se_thumbnail.cu" in build.SOURCES
    lines = out.stdout.splitlines()
    entries = [i for i, ln in enumerate(lines) if re.search(r"Compiling entry function '\w+'", ln)]
    names = [re.search(r"'(\w+)'", lines[i]).group(1) for i in entries]
    assert len(names) == 1 and "reduce_kernel" in names[0], names
    m = next(s for s in (re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
                         for ln in lines[entries[0]:]) if s)
    assert m.groups() == ("0", "0", "0"), lines[entries[0]:entries[0] + 4]

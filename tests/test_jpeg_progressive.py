"""Progressive JPEG, CPU side: tests/util_jpeg_progressive.py (the numpy restatement se_jpeg_prog.cu follows) writes Pillow's
``progressive=True`` bytes over the sizes, contents and qualities of the baseline and optimize tests at both subsamplings,
at 4:2:0 sizes whose MCUs end in right-edge, bottom-edge and corner dummy blocks, and on content whose EOB runs are cut at
0x7FFF blocks and at the correction-bit limit; the files stay within se_jpeg_progressive_max_bytes; and
se_jpeg_encode_progressive_u8 checks its arguments on the host before anything runs. Needs no GPU."""
import ctypes
import io

import numpy as np
import PIL
import pytest
from PIL import Image, ImageFile, features

from sketchedit_b200 import _lib, build
from tests import test_jpeg as TJ
from tests import test_jpeg_optimize as TO
from tests import util_jpeg as J
from tests import util_jpeg_progressive as P
from tests.test_jpeg import CONTENTS, content

PILLOW, LIBJPEG_TURBO = "12.2", "3.1"
# (h, w) at 4:2:0: h % 16 and w % 16 in 1..8 give a dummy luma row / column, 9..15 none
EDGE_SIZES = [(32, 23), (16, 40), (23, 32), (40, 16), (23, 23), (17, 40), (41, 25), (25, 41), (30, 45)]


def _env():
    return "Pillow %s, libjpeg-turbo %s" % (PIL.__version__, features.version("libjpeg_turbo"))


def pillow_jpeg_prog(a, quality=75, subsampling=2, optimize=False):
    """Pillow's progressive=True file. Pillow fails on a file larger than its buffer, as with optimize=True
    (tests/test_jpeg_optimize.py, pillow_jpeg_opt); a larger buffer writes the same bytes, so it is raised here."""
    buf = io.BytesIO()
    old, ImageFile.MAXBLOCK = ImageFile.MAXBLOCK, max(ImageFile.MAXBLOCK, 8 * a.shape[0] * a.shape[1] + 4096)
    try:
        Image.fromarray(a).save(buf, "JPEG", quality=quality, subsampling=subsampling, optimize=optimize, progressive=True)
    finally:
        ImageFile.MAXBLOCK = old
    return buf.getvalue()


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def test_environment_is_the_restated_one():
    """The restatement follows jcphuff.c as Pillow 12.2 bundles it."""
    assert PIL.__version__.startswith(PILLOW) and (features.version("libjpeg_turbo") or "").startswith(LIBJPEG_TURBO), _env()


def _matrix(hw, subsampling, qualities, lib):
    rs = np.random.RandomState(hw[0] * 1000 + hw[1])
    bound = lib.se_jpeg_progressive_max_bytes(hw[0], hw[1], subsampling)
    for kind in CONTENTS:
        a = content(kind, *hw, rs)
        for q in qualities:
            got = P.encode(a, q, subsampling)
            assert got == pillow_jpeg_prog(a, q, subsampling), (hw, kind, q, subsampling, _env())
            assert len(got) <= bound


@pytest.mark.parametrize("subsampling", [0, 2])
@pytest.mark.parametrize("hw", TO.SIZES)
def test_numpy_progressive_is_pillow_optimize_matrix(lib, hw, subsampling):
    _matrix(hw, subsampling, TO.QUALITIES, lib)


@pytest.mark.parametrize("subsampling", [0, 2])
@pytest.mark.parametrize("hw", TJ.SIZES)
def test_numpy_progressive_is_pillow_baseline_matrix(lib, hw, subsampling):
    _matrix(hw, subsampling, TJ.QUALITIES, lib)


@pytest.mark.parametrize("hw", EDGE_SIZES)
def test_dummy_blocks_at_the_right_bottom_and_corner(lib, hw):
    _matrix(hw, 2, (50, 75, 100), lib)


def test_edge_sizes_cover_each_dummy_kind():
    right = [hw for hw in EDGE_SIZES if -(-hw[1] // 8) % 2 and not -(-hw[0] // 8) % 2]
    bottom = [hw for hw in EDGE_SIZES if -(-hw[0] // 8) % 2 and not -(-hw[1] // 8) % 2]
    corner = [hw for hw in EDGE_SIZES if -(-hw[0] // 8) % 2 and -(-hw[1] // 8) % 2]
    assert right and bottom and corner
    rem = {v % 16 for hw in EDGE_SIZES for v in hw}
    assert rem & set(range(1, 9)) and rem & set(range(9, 16))


def test_optimize_makes_no_difference():
    a = content("places_11_512x408.npz", 67, 93, np.random.RandomState(2))
    for sub in (0, 2):
        assert pillow_jpeg_prog(a, 80, sub, optimize=True) == pillow_jpeg_prog(a, 80, sub, optimize=False) == P.encode(a, 80, sub)


def corr_limit_image(h=64, w=256, seed=0, ncoef=63):
    """A grey image at quality 100 whose luma blocks hold their first ``ncoef`` AC coefficients at a magnitude of 4..9 and
    the rest at 0: the last refinement scan codes no coefficient for the first time, so each block adds ``ncoef``
    correction bits to one long EOB run."""
    rs = np.random.RandomState(seed)
    n = np.arange(8)
    c = np.where(n == 0, np.sqrt(0.5), 1.0)
    basis = c[:, None] * np.cos((2 * n[None, :] + 1) * n[:, None] * np.pi / 16) / 2
    blocks = []
    for _ in range((h // 8) * (w // 8)):
        v = rs.randint(4, 10, 64) * rs.choice([-1, 1], 64)
        v[0] = 0
        v[ncoef + 1:] = 0
        blk = 128 + np.einsum("uv,ux,vy->xy", _natural(v), basis, basis)
        blocks.append(np.rint(blk))
    b = np.array(blocks).reshape(h // 8, w // 8, 8, 8).transpose(0, 2, 1, 3).reshape(h, w)
    return np.repeat(np.clip(b, 0, 255).astype(np.uint8)[..., None], 3, -1)


def _natural(v):
    """zigzag-ordered coefficients as an 8x8 array in natural order"""
    out = np.zeros(64)
    out[J.ZIGZAG] = v
    return out.reshape(8, 8)


def test_refinement_runs_are_cut_at_the_correction_bit_limit():
    a = corr_limit_image()
    for sub in (0, 2):
        coef, per = J.coefficients(a, 100, sub)
        y = P.component_blocks(coef, per, *a.shape[:2], 0)
        assert (np.abs(y[:, 1:]) != 1).mean() > 0.99                        # hardly any luma coefficient is first coded last
        stats = {}
        got = P.encode(a, 100, sub, stats)
        assert stats["corr_limit"] >= 10, stats
        assert got == pillow_jpeg_prog(a, 100, sub), (sub, _env())


def test_runs_are_cut_at_0x7fff_blocks():
    """A flat image of 2^15 luma blocks: every AC scan is one EOB run, cut once at 0x7FFF blocks in each scan with that
    many blocks: the four luma AC scans, and at 4:4:4 the four chroma ones."""
    a = np.full((1024, 2048, 3), (90, 120, 200), np.uint8)
    for sub in (0, 2):
        stats = {}
        got = P.encode(a, 75, sub, stats)
        assert stats["max_run"] == (8 if sub == 0 else 4), stats
        assert got == pillow_jpeg_prog(a, 75, sub), (sub, _env())


@pytest.mark.parametrize("subsampling", [0, 2])
def test_noise_at_quality_100_is_within_the_bound(lib, subsampling):
    """A progressive file can be larger than the optimized one (64x64 noise at quality 100, 4:4:4), so it has its own
    bound; noise at quality 100 stays within it."""
    rs = np.random.RandomState(12)
    for h, w in ((8, 8), (17, 33), (64, 64), (200, 120)):
        a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        got = P.encode(a, 100, subsampling)
        assert got == pillow_jpeg_prog(a, 100, subsampling)
        assert len(got) <= lib.se_jpeg_progressive_max_bytes(h, w, subsampling)
        assert lib.se_jpeg_progressive_max_bytes(h, w, subsampling) >= lib.se_jpeg_max_bytes(h, w, subsampling)


def test_pillow_refuses_large_progressive_files():
    a = np.random.RandomState(1).randint(0, 256, (300, 400, 3), dtype=np.uint8)
    with pytest.raises(OSError):
        Image.fromarray(a).save(io.BytesIO(), "JPEG", quality=90, subsampling=0, progressive=True)


def _call(lib, hw, pitch, n=1, quality=75, subsampling=2, scratch=None, need=None, src=None, out=None, out_bytes=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    hw_a = (ctypes.c_int * (2 * k))(*(list(hw) * k))
    p_a = (ctypes.c_longlong * k)(*([pitch] * k))
    o_a = (ctypes.c_longlong * k)(*([0] * k))
    rc = lib.se_jpeg_encode_progressive_u8(src, p_a, hw_a, n, quality, subsampling, out, o_a, out_bytes, scratch,
                                           ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    rc, need1, _ = _call(lib, (2667, 4000), 12000)
    rc0, base, _ = TO._call(lib, (2667, 4000), 12000, optimize=1)
    assert rc == 0 and rc0 == 0 and base < need1 < 3 * base
    rc, need2, _ = _call(lib, (2667, 4000), 12000, n=2)
    assert rc == 0 and need2 > need1
    assert _call(lib, (2667, 4000), 12000, n=0)[:2] == (0, 256)
    for kw, msg in [(dict(quality=0), "quality must be in"), (dict(subsampling=1), "subsampling must be 0"), (dict(n=33), "n must be in")]:
        rc, _, err = _call(lib, (10, 10), 30, **kw)
        assert rc != 0 and msg in err, (kw, err)
    for hw, pitch, msg in [((0, 10), 30, "sizes must be in"), ((10, 10), 29, "narrower than its row of 30 bytes")]:
        rc, _, err = _call(lib, hw, pitch)
        assert rc != 0 and msg in err, (hw, pitch, err)
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes" in err
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1 << 30))
    assert rc != 0 and "null src / out / out_bytes" in err
    assert lib.se_jpeg_progressive_max_bytes(0, 5, 2) == -1 and lib.se_jpeg_progressive_max_bytes(5, 5, 1) == -1


def test_python_checks(lib):
    import torch

    from sketchedit_b200.engine import _check_jpeg_args, jpeg_encode_u8, jpeg_encode_u8_packed, jpeg_max_bytes
    t = torch.empty(300, dtype=torch.uint8)
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(ValueError, match="progressive must be a bool"):
            jpeg_encode_u8([t], progressive=bad)
        with pytest.raises(ValueError, match="progressive must be a bool"):
            jpeg_encode_u8_packed(t, [0], [30], [(10, 10)], progressive=bad)
    assert _check_jpeg_args(75, 2, False, np.bool_(True)) == (75, 2)
    assert jpeg_encode_u8([], progressive=True) == []
    assert jpeg_max_bytes(2667, 4000, 2, progressive=True) == lib.se_jpeg_progressive_max_bytes(2667, 4000, 2)
    assert jpeg_max_bytes(2667, 4000, 2) == lib.se_jpeg_max_bytes(2667, 4000, 2)

"""JPEG with optimal Huffman tables, CPU side: tests/util_jpeg_optimize.py (the numpy restatement se_jpeg_opt.cu follows)
writes Pillow's ``optimize=True`` bytes over sizes, qualities, both subsamplings and contents, including 4:2:0 MCUs with dummy
blocks, a 4000x2667 photo-like image and a histogram whose unlimited code lengths pass 16 bits; the files stay within
se_jpeg_max_bytes; and se_jpeg_encode_opt_u8 checks its arguments on the host before anything runs. Needs no GPU."""
import ctypes
import io
import os
import re
import subprocess

import numpy as np
import PIL
import pytest
from PIL import Image, ImageFile, features

from sketchedit_b200 import _lib, build
from tests import util_jpeg as J
from tests import util_jpeg_optimize as O
from tests.test_jpeg import CONTENTS, content

SIZES = [(1, 1), (7, 9), (8, 8), (16, 17), (17, 23), (255, 257)]   # (h, w); 17x23 at 4:2:0 ends in MCUs with dummy blocks
QUALITIES = [1, 50, 75, 95, 100]
PILLOW, LIBJPEG_TURBO = "12.2", "3.1"


def _env():
    return "Pillow %s, libjpeg-turbo %s" % (PIL.__version__, features.version("libjpeg_turbo"))


def pillow_jpeg_opt(a, quality=75, subsampling=2):
    """Pillow's optimize=True file. Pillow gives libjpeg an output buffer of max(64 KiB, h w) bytes (2 h w from quality 95)
    and fails on a larger optimized file; a larger buffer writes the same bytes, so it is raised here for noise."""
    buf = io.BytesIO()
    old, ImageFile.MAXBLOCK = ImageFile.MAXBLOCK, max(ImageFile.MAXBLOCK, 8 * a.shape[0] * a.shape[1] + 4096)
    try:
        Image.fromarray(a).save(buf, "JPEG", quality=quality, subsampling=subsampling, optimize=True)
    finally:
        ImageFile.MAXBLOCK = old
    return buf.getvalue()


def test_environment_is_the_restated_one():
    """The encoder restates libjpeg-turbo's optimize_coding as Pillow 12.2 bundles it."""
    assert PIL.__version__.startswith(PILLOW) and (features.version("libjpeg_turbo") or "").startswith(LIBJPEG_TURBO), _env()


@pytest.mark.parametrize("subsampling", [0, 2])
@pytest.mark.parametrize("hw", SIZES)
def test_numpy_optimize_is_pillow(hw, subsampling):
    rs = np.random.RandomState(hw[0] * 1000 + hw[1])
    for kind in CONTENTS:
        a = content(kind, *hw, rs)
        for q in QUALITIES:
            got = O.encode(a, q, subsampling)
            assert got == pillow_jpeg_opt(a, q, subsampling), (hw, kind, q, subsampling, _env())
            assert len(got) <= J.max_bytes(*hw, subsampling)


def test_the_odd_size_has_dummy_blocks():
    h, w = 17, 23
    assert -(-h // 8) % 2 == 1 and -(-w // 8) % 2 == 1      # the last MCU row and column hold luma blocks outside the image


def test_numpy_optimize_is_pillow_at_12mp():
    """The 4000x2667 photo-like image of tests/test_jpeg.py at quality 75, 4:2:0."""
    rs = np.random.RandomState(5)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "places_11_512x408.npz"))["image_u8"]
    a = np.asarray(Image.fromarray(g).resize((4000, 2667))).astype(np.int16) + rs.randint(-8, 9, (2667, 4000, 3))
    a = np.clip(a, 0, 255).astype(np.uint8)
    got = O.encode(a)
    assert got == pillow_jpeg_opt(a), _env()
    assert len(got) < len(J.encode(a))


def test_flat_image_codes_only_dc_0_and_eob():
    """Mid grey: every DC is 0 after the level shift, so each table holds one symbol (DC category 0, EOB)."""
    a = np.full((40, 56, 3), 128, np.uint8)
    for sub in (0, 2):
        coef, per = J.coefficients(a, 75, sub)
        hist = O.histograms(coef, per)
        assert (hist[:, 1:] == 0).all() and (hist[:, 0] > 0).all()
        tabs = O.tables(coef, per)
        assert all(t == ([1] + [0] * 15, b"\x00") for t in tabs), tabs
        assert O.encode(a, 75, sub) == pillow_jpeg_opt(a, 75, sub)


def _fibonacci_image():
    """A grey image at quality 50, 4:4:4, whose 8x8 blocks each hold one AC coefficient, chosen so that the AC luma counts
    are Fibonacci numbers: the Huffman tree is a chain, 20 levels deep before Annex K.3 limits it."""
    q = J.quant_table(50, J.LUMA_Q).reshape(8, 8)
    n = np.arange(8)
    c = np.where(n == 0, np.sqrt(0.5), 1.0)
    basis = c[:, None] * np.cos((2 * n[None, :] + 1) * n[:, None] * np.pi / 16) / 2     # basis[u, x], orthonormal
    fib, blocks = [1, 1], []
    while len(fib) < 21:
        fib.append(fib[-1] + fib[-2])
    for s, count in enumerate(fib[1:]):                      # symbol s: zigzag position 1 + s // 2, value 1 or 2
        k, v = 1 + s // 2, 1 + s % 2
        u, x = divmod(int(J.ZIGZAG[k]), 8)
        blk = 128 + v * q[u, x] * np.outer(basis[u], basis[x])
        blocks += [np.rint(blk)] * count
    cols = 256
    blocks += [np.full((8, 8), 128.0)] * (-len(blocks) % cols)
    b = np.array(blocks).reshape(-1, cols, 8, 8).transpose(0, 2, 1, 3).reshape(-1, cols * 8)
    return np.repeat(np.clip(b, 0, 255).astype(np.uint8)[..., None], 3, -1)


def test_code_lengths_past_16_bits_are_limited_as_pillow_does():
    a = _fibonacci_image()
    coef, per = J.coefficients(a, 50, 0)
    hist = O.histograms(coef, per)
    assert np.count_nonzero(hist[2]) >= 21                 # 20 AC symbols and EOB
    sizes = O.code_lengths(hist[2])
    assert max(sizes) > 16, max(sizes)                     # the unlimited tree is deeper than a JPEG code may be
    counts, syms = O.optimal_table(hist[2])
    assert sum(counts) == len(syms) == np.count_nonzero(hist[2]) and counts[15] > 0
    got = O.encode(a, 50, 0)
    assert got == pillow_jpeg_opt(a, 50, 0), _env()
    assert len(got) <= J.max_bytes(*a.shape[:2], 0)


@pytest.mark.parametrize("subsampling", [0, 2])
def test_noise_at_quality_100_is_within_the_bound(subsampling):
    """The widest AC alphabets: optimal tables make the file smaller, never past se_jpeg_max_bytes, and their header is no
    longer than the Annex K one."""
    rs = np.random.RandomState(11)
    for h, w in ((8, 8), (17, 33), (64, 48), (200, 120)):
        a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        a[::2, ::2] = 255 - a[::2, ::2] // 8
        got = O.encode(a, 100, subsampling)
        assert got == pillow_jpeg_opt(a, 100, subsampling)
        assert len(got) <= len(J.encode(a, 100, subsampling)) <= J.max_bytes(h, w, subsampling)
        coef, per = J.coefficients(a, 100, subsampling)
        assert len(O.header(h, w, 100, subsampling, O.tables(coef, per))) <= J.HEADER_BYTES


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _call(lib, hw, pitch, n=1, quality=75, subsampling=2, optimize=1, scratch=None, need=None, src=None, out=None,
          out_bytes=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    hw_a = (ctypes.c_int * (2 * k))(*(list(hw) * k))
    p_a = (ctypes.c_longlong * k)(*([pitch] * k))
    o_a = (ctypes.c_longlong * k)(*([0] * k))
    rc = lib.se_jpeg_encode_opt_u8(src, p_a, hw_a, n, quality, subsampling, optimize, out, o_a, out_bytes, scratch,
                                   ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    base = ctypes.c_longlong(0)
    hw_a, p_a, o_a = (ctypes.c_int * 2)(2667, 4000), (ctypes.c_longlong * 1)(12000), (ctypes.c_longlong * 1)(0)
    assert lib.se_jpeg_encode_u8(None, p_a, hw_a, 1, 75, 2, None, o_a, None, None, ctypes.byref(base), None) == 0
    rc, need0, _ = _call(lib, (2667, 4000), 12000, optimize=0)
    assert rc == 0 and need0 == base.value                       # se_jpeg_encode_u8 is the entry with optimize = 0
    rc, need1, _ = _call(lib, (2667, 4000), 12000)
    assert rc == 0 and 0 < need1 - need0 <= 13 * 1024             # histograms, tables and the header length
    rc, need2, _ = _call(lib, (2667, 4000), 12000, n=2)
    assert rc == 0 and need2 > need1
    assert _call(lib, (2667, 4000), 12000, n=0)[:2] == (0, 256)
    for kw, msg in [(dict(optimize=2), "optimize must be 0 or 1"), (dict(optimize=-1), "optimize must be 0 or 1"),
                    (dict(quality=0), "quality must be in"), (dict(subsampling=1), "subsampling must be 0"),
                    (dict(n=33), "n must be in")]:
        rc, _, err = _call(lib, (10, 10), 30, **kw)
        assert rc != 0 and msg in err, (kw, err)
    for hw, pitch, msg in [((0, 10), 30, "sizes must be in"), ((10, 10), 29, "narrower than its row of 30 bytes")]:
        rc, _, err = _call(lib, hw, pitch)
        assert rc != 0 and msg in err, (hw, pitch, err)
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes" in err
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1 << 30))
    assert rc != 0 and "null src / out / out_bytes" in err


def test_python_checks(lib):
    import torch

    from sketchedit_b200.engine import _check_jpeg_args, jpeg_encode_u8, jpeg_encode_u8_packed
    t = torch.empty(300, dtype=torch.uint8)
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(ValueError, match="optimize must be a bool"):
            jpeg_encode_u8([t], optimize=bad)
        with pytest.raises(ValueError, match="optimize must be a bool"):
            jpeg_encode_u8_packed(t, [0], [30], [(10, 10)], optimize=bad)
    assert _check_jpeg_args(75, 2, True) == (75, 2) and _check_jpeg_args(75, 2, np.bool_(False)) == (75, 2)
    assert jpeg_encode_u8([], optimize=True) == []


def test_opt_kernels_do_not_spill(tmp_path):
    """Every kernel of se_jpeg_opt.cu, compiled for sm_90a with the library's flags, keeps everything in registers."""
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    if not os.path.exists(nvcc) and not any(os.access(os.path.join(p, nvcc), os.X_OK) for p in os.environ["PATH"].split(":")):
        pytest.skip("nvcc not available")
    flags = [f for f in build.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "se_jpeg_opt.cu"), "-o", str(tmp_path / "j.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    lines = out.stdout.splitlines()
    entries = [i for i, ln in enumerate(lines) if re.search(r"Compiling entry function '\w+'", ln)]
    names = [re.search(r"'(\w+)'", lines[i]).group(1) for i in entries]
    assert len(entries) == 4 and all(any(k in n for n in names) for k in ("hist", "table", "opt_header", "opt_bits")), names
    for i in entries:
        m = next(s for s in (re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
                             for ln in lines[i:]) if s)
        assert m.groups() == ("0", "0", "0"), lines[i:i + 4]

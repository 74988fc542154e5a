"""JPEG encoding, CPU side: tests/util_jpeg.py (the numpy restatement se_jpeg.cu follows) writes Pillow's bytes over sizes,
qualities, both subsamplings and contents from flat colour to noise; the header's quantisation tables follow Pillow's rule at
every quality; se_jpeg_max_bytes bounds the worst file; and se_jpeg_encode_u8 checks its arguments on the host before
anything runs. Needs no GPU."""
import ctypes
import io
import os
import re
import subprocess

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from tests import util_jpeg as J

SIZES = [(1, 1), (7, 9), (15, 17), (16, 16), (17, 33), (641, 481)]   # (h, w)
QUALITIES = [1, 10, 49, 50, 75, 90, 95, 100]


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def pillow_jpeg(a, quality=75, subsampling=2):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "JPEG", quality=quality, subsampling=subsampling)
    return buf.getvalue()


def content(kind, h, w, rs):
    """noise: long codes and many 0xFF bytes; flat: EOB and ZRL runs; gradient: smooth ramps; golden: photos (tiled)."""
    if kind == "noise":
        return rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), (30, 140, 220), np.uint8)
    if kind == "gradient":
        y, x = np.mgrid[:h, :w]
        return np.stack([(x * 7) % 256, (y * 3) % 256, (x + y) % 256], -1).astype(np.uint8)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", kind))["image_u8"]
    return np.tile(g, (-(-h // g.shape[0]), -(-w // g.shape[1]), 1))[:h, :w]


CONTENTS = ["noise", "flat", "gradient", "face_602_256x256.npz", "places_11_512x408.npz"]


@pytest.mark.parametrize("subsampling", [0, 2])
@pytest.mark.parametrize("hw", SIZES)
def test_numpy_encoder_is_pillow(hw, subsampling):
    rs = np.random.RandomState(hw[0] * 1000 + hw[1])
    for kind in CONTENTS:
        a = content(kind, *hw, rs)
        for q in QUALITIES:
            assert J.encode(a, q, subsampling) == pillow_jpeg(a, q, subsampling), (hw, kind, q, subsampling, PIL.__version__)


def test_numpy_encoder_is_pillow_at_12mp():
    """A 4000x2667 photo-like image (a golden image upscaled, plus noise) at Pillow's defaults."""
    rs = np.random.RandomState(5)
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "places_11_512x408.npz"))["image_u8"]
    a = np.asarray(Image.fromarray(g).resize((4000, 2667))).astype(np.int16) + rs.randint(-8, 9, (2667, 4000, 3))
    a = np.clip(a, 0, 255).astype(np.uint8)
    assert J.encode(a) == pillow_jpeg(a)


def _segments(data):
    """(marker, body) of each segment up to SOS."""
    out, i = [], 2
    while True:
        m, n = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        out.append((m, data[i + 4:i + 2 + n]))
        if m == 0xDA:
            return out
        i += 2 + n


def test_header_layout_and_quality_tables():
    """SOI, APP0, DQT, DQT, SOF0, 4 DHT, SOS, as Pillow writes them, and the DQT tables of all 100 qualities."""
    a = np.zeros((9, 11, 3), np.uint8)
    for q in range(1, 101):
        for s in (0, 2):
            data = pillow_jpeg(a, q, s)
            assert data[:J.HEADER_BYTES] == J.header(9, 11, q, s), (q, s)
            segs = _segments(data)
            assert [m for m, _ in segs] == [0xE0, 0xDB, 0xDB, 0xC0, 0xC4, 0xC4, 0xC4, 0xC4, 0xDA]
            for t, base in ((1, J.LUMA_Q), (2, J.CHROMA_Q)):
                assert list(segs[t][1][1:]) == list(J.quant_table(q, base)[J.ZIGZAG]), (q, t)


def test_reciprocals_divide_like_libjpeg():
    """The reciprocal quantiser is round-half-up division of |x| by 8 q for every DCT magnitude and quantiser."""
    x = np.arange(0, 8 * 1024 + 1)
    for q in range(1, 256):
        recip, corr, shift = J.reciprocal(8 * q)
        assert recip < 65536 and corr < 65536
        assert np.array_equal(((x + corr) * recip) >> shift, (x + 4 * q) // (8 * q)), q


@pytest.mark.parametrize("subsampling", [0, 2])
def test_noise_at_quality_100_is_within_the_bound(lib, subsampling):
    rs = np.random.RandomState(11)
    for h, w in ((8, 8), (17, 33), (64, 48)):
        a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        a[::2, ::2] = 255 - a[::2, ::2] // 8                 # high contrast between neighbours: the largest AC values
        n = len(pillow_jpeg(a, 100, subsampling))
        bound = lib.se_jpeg_max_bytes(h, w, subsampling)
        assert bound == J.max_bytes(h, w, subsampling) and n <= bound, (h, w, n, bound)


def _call(lib, hw, pitch, n=1, quality=75, subsampling=2, scratch=None, need=None, src=None, out=None, out_bytes=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    hw_a = (ctypes.c_int * (2 * k))(*(list(hw) * k))
    p_a = (ctypes.c_longlong * k)(*([pitch] * k))
    o_a = (ctypes.c_longlong * k)(*([0] * k))
    rc = lib.se_jpeg_encode_u8(src, p_a, hw_a, n, quality, subsampling, out, o_a, out_bytes, scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    rc, need, _ = _call(lib, (2667, 4000), 12000)
    assert rc == 0 and need > 0
    rc, need444, _ = _call(lib, (2667, 4000), 12000, subsampling=0)
    assert rc == 0 and need444 > need                       # 4:4:4 has twice the chroma blocks
    rc, need2, _ = _call(lib, (2667, 4000), 12000, n=2)
    assert rc == 0 and need2 > need
    assert _call(lib, (2667, 4000), 12000, n=0)[:2] == (0, 256)
    for kw, msg in [(dict(quality=0), "quality must be in"), (dict(quality=101), "quality must be in"),
                    (dict(subsampling=1), "subsampling must be 0"), (dict(subsampling=4), "subsampling must be 0"),
                    (dict(n=33), "n must be in"), (dict(n=-1), "n must be in")]:
        rc, _, err = _call(lib, (10, 10), 30, **kw)
        assert rc != 0 and msg in err, (kw, err)
    for hw, pitch, msg in [((0, 10), 30, "sizes must be in"), ((10, 65536), 3 * 65536, "sizes must be in"),
                           ((10, 10), 29, "narrower than its row of 30 bytes")]:
        rc, _, err = _call(lib, hw, pitch)
        assert rc != 0 and msg in err, (hw, pitch, err)
    # past the query: scratch too small, then null pointers, all refused before anything is enqueued
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes" in err
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(1 << 30))
    assert rc != 0 and "null src / out / out_bytes" in err
    assert lib.se_jpeg_max_bytes(0, 5, 2) == -1 and lib.se_jpeg_max_bytes(5, 5, 1) == -1
    assert lib.se_jpeg_max_bytes(65535, 65535, 0) == J.max_bytes(65535, 65535, 0)


def test_python_checks(lib):
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8, jpeg_encode_u8_packed, jpeg_max_bytes
    t = torch.empty(300, dtype=torch.uint8)
    for q, s in [(0, 2), (101, 2), (75, 1), (75.0, 2), (True, 2)]:
        with pytest.raises(ValueError):
            jpeg_encode_u8([t], q, s)
    with pytest.raises(_lib.SketchEditB200Error, match="CUDA uint8"):
        jpeg_encode_u8([t.view(10, 10, 3)])
    with pytest.raises(_lib.SketchEditB200Error, match="CUDA uint8"):
        jpeg_encode_u8_packed(t, [0], [30], [(10, 10)])
    with pytest.raises(_lib.SketchEditB200Error, match="same length"):
        jpeg_encode_u8_packed([t, t], [0], [30], [(10, 10)])
    assert jpeg_encode_u8([]) == []
    from sketchedit_b200.engine import _check_jpeg_args, _is_int
    got = _check_jpeg_args(np.int64(75), np.int32(2))           # numpy integers are integers, as in a session's box
    assert got == (75, 2) and all(type(v) is int for v in got)
    assert _is_int(np.uint16(3)) and _is_int(7) and not _is_int(True) and not _is_int(np.bool_(True)) and not _is_int(3.0)
    assert jpeg_max_bytes(16, 16, 2) == J.max_bytes(16, 16, 2)
    with pytest.raises(ValueError):
        jpeg_max_bytes(16, 16, 1)


def test_jpeg_kernels_do_not_spill(tmp_path):
    """Every kernel of se_jpeg.cu, compiled for sm_90a with the library's flags, keeps everything in registers."""
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    if not os.path.exists(nvcc) and not any(os.access(os.path.join(p, nvcc), os.X_OK) for p in os.environ["PATH"].split(":")):
        pytest.skip("nvcc not available")
    flags = [f for f in build.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "se_jpeg.cu"), "-o", str(tmp_path / "j.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    lines = out.stdout.splitlines()
    entries = [i for i, ln in enumerate(lines) if re.search(r"Compiling entry function '\w+'", ln)]
    names = [re.search(r"'(\w+)'", lines[i]).group(1) for i in entries]
    assert len(entries) == 9 and any("jpeg_dct_kernel" in n for n in names), names
    for i in entries:
        m = next(s for s in (re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
                             for ln in lines[i:]) if s)
        assert m.groups() == ("0", "0", "0"), lines[i:i + 4]

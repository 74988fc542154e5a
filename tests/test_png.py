"""tests/util_png.py is cv2's PNG encoder: its files equal ``cv2.imencode(".png", img)`` and ``cv2.imwrite`` over sizes at every
zlib window step, both channel counts and the contents that reach each of zlib's block forms, plus constructed blocks (an
empty final block, the 15-bit length repair, static trees, stored data). One test pins the environment the encoder restates,
and one that se_png_encode_u8 checks its arguments on the host before anything runs."""
import ctypes
import os
import re
import zlib

import cv2
import numpy as np
import pytest

from sketchedit_b200 import _lib, build
from tests import util_png as P

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
PHOTOS = ("face_602_256x256.npz", "places_11_512x408.npz")


def window_steps():
    """(h, w) pairs whose filtered size lies on each side of every CMF window step (2^k, k = 8..14), for 1 and 3 channels."""
    out = []
    for k in range(8, 15):
        for c in (1, 3):
            w = (2 ** k - 1) // c
            out += [(1, w, c), (1, w + 1, c)]
    return out


SIZES = [(1, 1), (1, 9), (13, 1), (2, 2), (37, 61), (256, 256), (512, 408)]
CONTENTS = ("noise", "flat", "mask", "gradient") + PHOTOS


def content(kind, h, w, channels, rs):
    """A BGR [h, w, 3] or grey [h, w] uint8 image of the given kind."""
    if kind == "noise":
        a = rs.randint(0, 256, (h, w, 3))
    elif kind == "flat":
        a = np.full((h, w, 3), (200, 31, 7))
    elif kind == "mask":
        a = np.repeat(((rs.rand(h // 4 + 1, w // 4 + 1) > 0.5) * 255)[:, :, None], 3, 2).repeat(4, 0).repeat(4, 1)[:h, :w]
    elif kind == "gradient":
        y, x = np.mgrid[:h, :w]
        a = np.stack([(x + y) % 256, (2 * x) % 256, (y // 3) % 256], 2)
    else:
        img = np.load(os.path.join(GOLDEN, kind))["image_u8"][:, :, ::-1]   # RGB -> BGR
        reps = (-(-h // img.shape[0]), -(-w // img.shape[1]), 1)
        a = np.tile(img, reps)[:h, :w]
    a = np.ascontiguousarray(a.astype(np.uint8))
    return a if channels == 3 else np.ascontiguousarray(cv2.cvtColor(a, cv2.COLOR_BGR2GRAY) if kind in PHOTOS else a[:, :, 1])


def cv2_png(img):
    return cv2.imencode(".png", img)[1].tobytes()


def _libpng_version():
    m = re.search(r"PNG:.*?\(ver ([^)]+)\)", cv2.getBuildInformation())
    return m.group(1) if m else "?"


def _env():
    return "cv2 %s, libpng %s, zlib %s" % (cv2.__version__, _libpng_version(), zlib.ZLIB_RUNTIME_VERSION)


def idat(png):
    """The concatenated IDAT payloads of a PNG file, and the chunk kinds in order."""
    at, body, kinds = 8, b"", []
    while at < len(png):
        n = int.from_bytes(png[at:at + 4], "big")
        kind = png[at + 4:at + 8]
        kinds.append(kind)
        if kind == b"IDAT":
            body += png[at + 8:at + 8 + n]
        at += 12 + n
    return body, kinds


def test_cv2_png_is_zlib_rle_level_1():
    """The environment this encoder restates: cv2's IDAT stream after its 2-byte header is zlib level 1, memLevel 8, Z_RLE
    over the Sub-filtered rows, and the file has IHDR, IDAT and IEND only."""
    rs = np.random.RandomState(1)
    for kind in CONTENTS:
        for c in (1, 3):
            a = content(kind, 77, 301, c, rs)
            body, kinds = idat(cv2_png(a))
            z = zlib.compressobj(1, zlib.DEFLATED, 15, 8, zlib.Z_RLE)
            want = z.compress(P.filtered(a).tobytes()) + z.flush()
            assert body[2:] == want[2:], "cv2's PNG stream is not zlib Z_RLE level 1 (%s; %s, %d channels)" % (_env(), kind, c)
            assert set(kinds) == {b"IHDR", b"IDAT", b"IEND"}, (_env(), kinds)


@pytest.mark.parametrize("channels", [1, 3])
def test_restatement_is_cv2(channels):
    rs = np.random.RandomState(channels)
    for h, w in SIZES:
        for kind in CONTENTS:
            a = content(kind, h, w, channels, rs)
            assert P.png(a) == cv2_png(a), (h, w, kind, channels, _env())


def test_window_steps_and_chunking():
    rs = np.random.RandomState(5)
    for h, w, c in window_steps():
        for kind in ("noise", "gradient", "face_602_256x256.npz"):
            a = content(kind, h, w, c, rs)
            got = P.png(a)
            assert got == cv2_png(a), (h, w, c, kind, _env())
            n = h * (1 + w * c)
            assert got[41] == (0x78 if n > 16384 else 0x08 | (max(0, (n - 1).bit_length() - 8) << 4)), (h, w, c)


def test_large_photo_and_imwrite(tmp_path):
    """A 2667x4000 photo, and the file cv2.imwrite writes for a case of each block form."""
    rs = np.random.RandomState(8)
    a = content("places_11_512x408.npz", 2667, 4000, 3, rs)
    assert P.png(a) == cv2_png(a)
    for kind, c in (("noise", 3), ("flat", 1), ("face_602_256x256.npz", 3)):
        a = content(kind, 100, 93, c, rs)
        path = str(tmp_path / ("x_%s_%d.PNG" % (kind[:4], c)))
        assert cv2.imwrite(path, a)
        with open(path, "rb") as f:
            assert f.read() == P.png(a), (kind, c)


def _from_filtered_row(stream):
    """The 1-row grey image whose filtered bytes are ``stream`` (filter byte 1, then Sub differences)."""
    assert stream[0] == 1
    return (np.cumsum(np.asarray(stream[1:], np.int64)) % 256).astype(np.uint8)[None, :]


def _no_repeats(counts, rs):
    """A byte sequence with counts[v] copies of byte v, no two neighbours equal (so every byte is a literal)."""
    left = dict(counts)
    out, prev = [], -1
    while left:
        cands = sorted((n, v) for v, n in left.items() if v != prev)
        n, v = cands[-1]
        out.append(v)
        left[v] -= 1
        if not left[v]:
            del left[v]
        prev = v
    return out


def test_constructed_blocks():
    rs = np.random.RandomState(12)
    # 16383 symbols exactly: every byte a literal, so the final block is empty
    stream = [1]
    while len(stream) < P.BLOCK_SYMS:
        v = int(rs.randint(0, 256))
        if v != stream[-1]:
            stream.append(v)
    a = _from_filtered_row(stream)
    assert (P.filtered(a) == stream).all()
    blks = list(P.blocks(P.filtered(a)))
    assert [hi - lo for _, lo, hi, *_ in blks] == [P.BLOCK_SYMS, 0]
    assert P.png(a) == cv2_png(a)

    # Fibonacci literal counts next to the filter byte's and END_BLOCK's 1: the unrestricted tree is 17 deep, so gen_bitlen
    # repairs it to 15 bits
    fib = [2, 3]
    while len(fib) < 16:
        fib.append(fib[-1] + fib[-2])
    stream = [1] + _no_repeats({v + 2: n for v, n in enumerate(fib)}, rs)
    a = _from_filtered_row(stream)
    data = P.filtered(a)
    (blk, lo, hi, _, _, sym, _, _), = list(P.blocks(data))
    lfreq = np.bincount(sym, minlength=P.L_CODES)
    lfreq[P.END_BLOCK] += 1
    assert max(P.build_tree(lfreq, P.STATIC_LLEN, P.EXTRA_LBITS, 257, 99).lens) > 15
    assert blk.kind == P.DYNAMIC and max(blk.llen) == 15
    assert P.png(a) == cv2_png(a)

    # short inputs take static trees; noise is stored
    kinds = lambda img: [b[0].kind for b in P.blocks(P.filtered(img))]
    a = content("gradient", 4, 20, 1, rs)
    assert kinds(a) == [P.STATIC] and P.png(a) == cv2_png(a)
    a = content("noise", 64, 300, 3, rs)
    assert set(kinds(a)) == {P.STORED} and P.png(a) == cv2_png(a)
    a = content("flat", 64, 300, 1, rs)                        # one literal plus 258-matches per row, forced distance code
    assert P.png(a) == cv2_png(a)


def test_max_bytes_bounds_the_files():
    rs = np.random.RandomState(4)
    for h, w in SIZES + [(1, 5461), (3, 4000)]:
        for c in (1, 3):
            a = content("noise", h, w, c, rs)
            assert len(cv2_png(a)) <= P.max_bytes(h, w, c), (h, w, c)


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _call(lib, hw, pitch, n=1, channels=3, swap_rb=0, out_off=0, scratch=None, need=None, src=None, out=None, out_bytes=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    hw_a = (ctypes.c_int * (2 * k))(*(list(hw) * k))
    p_a = (ctypes.c_longlong * k)(*([pitch] * k))
    o_a = (ctypes.c_longlong * k)(*([out_off] * k))
    rc = lib.se_png_encode_u8(src, p_a, hw_a, n, channels, swap_rb, out, o_a, out_bytes, scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    rc, need, _ = _call(lib, (10, 10), 30)
    assert rc == 0 and need > 0
    rc, need1, _ = _call(lib, (10, 10), 10, channels=1)
    assert rc == 0 and need1 < need
    rc, need2, _ = _call(lib, (10, 10), 30, n=2)
    assert rc == 0 and need2 > need
    assert _call(lib, (10, 10), 30, n=0)[:2] == (0, 512)          # the per-image state and the scan sums, one slot each
    for kw, msg in [(dict(channels=2), "channels must be 1 or 3"), (dict(channels=4), "channels must be 1 or 3"),
                    (dict(swap_rb=2), "swap_rb must be 0 or 1"), (dict(n=33), "n must be in"), (dict(n=-1), "n must be in"),
                    (dict(out_off=-1), "negative offset")]:
        rc, _, err = _call(lib, (10, 10), 30, **kw)
        assert rc != 0 and msg in err, (kw, err)
    for hw, pitch, channels, msg in [((0, 10), 30, 3, "image 0: sizes must be in [1, 65535]"),
                                     ((10, 65536), 3 * 65536, 3, "image 0: sizes must be in [1, 65535]"),
                                     ((10, 10), 29, 3, "image 0: the source pitch of 29 bytes is narrower than its row of 30 bytes"),
                                     ((10, 10), 9, 1, "image 0: the source pitch of 9 bytes is narrower than its row of 10 bytes")]:
        rc, _, err = _call(lib, hw, pitch, channels=channels)
        assert rc != 0 and msg in err, (hw, pitch, channels, err)
    assert lib.se_png_encode_u8(None, None, None, 1, 3, 0, None, None, None, None, ctypes.byref(ctypes.c_longlong(0)), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()
    # past the query: scratch too small, then null pointers, all refused before anything is enqueued
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes, needs %d" % need in err
    rc, _, err = _call(lib, (10, 10), 30, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(need))
    assert rc != 0 and "null src / out / out_bytes" in err
    assert _call(lib, (10, 10), 30, n=0, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(512))[0] == 0
    assert lib.se_png_max_bytes(0, 5, 3) == -1 and lib.se_png_max_bytes(5, 65536, 1) == -1 and lib.se_png_max_bytes(5, 5, 2) == -1
    assert lib.se_png_max_bytes(65535, 65535, 3) == P.max_bytes(65535, 65535, 3)

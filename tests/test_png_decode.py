"""PNG decoding on the host: the numpy restatement (tests/util_png_decode.py) against Pillow, the container parser's routing,
the inflate core of se_png_decode.cu built for the host (one lane) against zlib on malformed and mutated streams, and the
argument checks se_png_decode_u8 makes before anything runs."""
import ctypes
import io
import os
import random
import shutil
import struct
import subprocess
import zlib

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build, pngfile
from tests import util_png_decode as U

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "sketchedit_b200", "csrc")


def pillow(f, mode):
    return np.asarray(Image.open(io.BytesIO(f)).convert(mode))


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_restatement_is_pillow(mode):
    for name, f in U.corpus():
        pngfile.parse(f)   # every corpus file goes to the device
        ref, got = pillow(f, mode), U.decode(f, mode)
        assert ref.shape == got.shape and np.array_equal(ref, got), name


def test_parser_fields():
    for name, f in U.corpus():
        hd = pngfile.parse(f)
        w, h, depth, ctype = struct.unpack(">IIBB", f[16:26])
        assert (hd.h, hd.w, hd.depth, hd.ctype) == (h, w, depth, ctype), name
        assert hd.stream == b"".join(b for c, b in U.chunks(f) if c == b"IDAT"), name
        assert pngfile.size(f) == (h, w)


def test_parser_routes_to_pillow():
    for name, f, why in U.fallbacks():
        with pytest.raises(pngfile.Host, match=why):
            pngfile.parse(f)
    good = U.make_png(U.photo(5, 6), 8, 2)
    bad_crc = bytearray(good)
    bad_crc[30] ^= 1   # inside IHDR's CRC
    cases = {
        "truncated chunk": good[:-6],
        "bad CRC": bytes(bad_crc),
        "APNG": U.make_png(U.photo(5, 6), 8, 2, extra=[(b"acTL", bytes(8))]),
        "chunk b'iCCP'": U.make_png(U.photo(5, 6), 8, 2, extra=[(b"iCCP", b"x\0\0" + zlib.compress(b"p"))]),
        "chunk b'gAMA'": U.make_png(U.photo(5, 6), 8, 2, extra=[(b"gAMA", b"\0\0")]),
        "no PLTE": U.make_png(np.zeros((3, 3, 1), np.uint8), 8, 3),
        "IDAT chunks apart": good.replace(U.chunk(b"IEND", b""), U.chunk(b"tIME", bytes(7)) + U.chunk(b"IDAT", b"") +
                                          U.chunk(b"IEND", b"")),
        "not a PNG": b"",
    }
    for why, f in cases.items():
        with pytest.raises(pngfile.Host, match=why.replace("(", r"\(")):
            pngfile.parse(f)
    pngfile.parse(good)


def test_malformed_files_parse():
    # the container of each is sound, so they reach the device, whose status must refuse them (tests/test_gpu_png_decode.py)
    for name, f in U.malformed():
        pngfile.parse(f)


# ------------------------------------------------------------------------------------------------ the inflate core on the host
DRIVER = r"""
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "se_inflate.cuh"
// cases on stdin: int64 raw_n, int64 n, n stream bytes; on stdout per case: int32 status, then raw_n bytes when it is 0.
// Each buffer is allocated at its exact size, so the address sanitizer reports any access outside it.
int main() {
  long long hdr[2];
  static se::InflateTabs tabs;
  while (fread(hdr, 8, 2, stdin) == 2) {
    unsigned char* src = (unsigned char*)malloc(hdr[1] ? hdr[1] : 1);
    unsigned char* raw = (unsigned char*)malloc(hdr[0] ? hdr[0] : 1);
    if (hdr[1] && fread(src, 1, hdr[1], stdin) != (size_t)hdr[1]) return 3;
    int st = se::inflate_zlib(hdr[1] ? src : nullptr, hdr[1], raw, hdr[0], tabs, 0, 1);
    fwrite(&st, 4, 1, stdout);
    if (st == 0) fwrite(raw, 1, hdr[0], stdout);
    free(src);
    free(raw);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def inflate_host(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("inflate_host")
    src, exe = d / "driver.cpp", d / "inflate_host"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(cases):
        blob = b"".join(struct.pack("<qq", n, len(z)) + z for z, n in cases)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
        p = subprocess.run([str(exe)], input=blob, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode()[-3000:]
        res, at = [], 0
        for z, n in cases:
            (st,) = struct.unpack("<i", p.stdout[at:at + 4])
            at += 4
            res.append((st, p.stdout[at:at + n] if st == 0 else None))
            at += n if st == 0 else 0
        assert at == len(p.stdout)
        return res
    return run


def zlib_says(z, n):
    """zlib's bytes when z is a complete stream of exactly n bytes, else None."""
    d = zlib.decompressobj()
    try:
        out = d.decompress(z, n + 1)
    except zlib.error:
        return None
    return out if d.eof and len(out) == n else None


def check(run, cases):
    for (z, n), (st, raw) in zip(cases, run(cases)):
        want = zlib_says(z, n)
        if st == 0:   # accepted: zlib accepts it too, with the same bytes
            assert want is not None and raw == want, (z[:40], n)
        else:
            assert want is None or 1 <= st <= 9, (z[:40], n, st)


def streams():
    rng = np.random.default_rng(3)
    photo = U.photo(30, 40).tobytes()
    noise = rng.integers(0, 256, 5000, dtype=np.uint8).tobytes()
    out = []
    for data in (photo, noise, b"\0" * 3000, b"ab" * 700):
        for lvl in (0, 1, 6, 9):
            for strat in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE):
                c = zlib.compressobj(lvl, strategy=strat)
                out.append((c.compress(data) + c.flush(), len(data)))
    return out


def test_inflate_host_valid(inflate_host):
    cases = streams()
    res = inflate_host(cases)
    for (z, n), (st, raw) in zip(cases, res):
        assert st == 0 and raw == zlib.decompress(z)


def test_inflate_host_malformed(inflate_host):
    z = zlib.compress(U.photo(9, 8).tobytes())
    n = 9 * 8 * 3
    far, _ = U.fixed_deflate([1, (5, 2)])
    cases = [(b"", n), (z[:1], n), (b"\x78\x02" + z[2:], n), (bytes([0x78, 0xBB]) + z[2:], n), (z[:-1], n),
             (z[:-1] + bytes([z[-1] ^ 1]), n), (b"\x78\x01\x07" + z[3:], n), (far, 6), (z, n - 1), (z, n + 1),
             (b"\x78\x01\x01\x05\x00\xfb\xff", 5),   # stored LEN 5 with no data
             (b"\x78\x01\x01\x05\x00\xfa\xff" + b"abcde", 5),   # LEN != ~NLEN
             (b"\x78\x01\x05\xe0\xff" + b"\xff" * 8, 4)]   # dynamic block with too many codes
    res = inflate_host(cases)
    assert all(st != 0 for st, _ in res), [st for st, _ in res]
    check(inflate_host, cases)


def test_inflate_host_mutated(inflate_host):
    rnd = random.Random(11)
    base = streams()
    cases = []
    for _ in range(3000):
        z, n = base[rnd.randrange(len(base))]
        z = bytearray(z)
        kind = rnd.randrange(4)
        if kind == 0:
            for _ in range(rnd.randint(1, 4)):
                k = rnd.randrange(len(z))
                z[k] ^= 1 << rnd.randrange(8)
        elif kind == 1:
            z = z[:rnd.randrange(len(z))]
        elif kind == 2:
            k = rnd.randrange(len(z))
            z[k:k + rnd.randint(1, 8)] = b""
        else:
            k = rnd.randrange(len(z))
            z[k:k] = bytes(rnd.randrange(256) for _ in range(rnd.randint(1, 8)))
        cases.append((bytes(z), n + rnd.choice((0, 0, 0, -1, 1))))
    check(inflate_host, cases)


# ------------------------------------------------------------------------------------------------ se_png_decode_u8's host checks
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _call(lib, info, n=1, src_off=0, src_len=100, plte_off=0, scratch=None, need=None, src=None, out=None, status=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    L = ctypes.c_longlong
    info_a = (ctypes.c_int * (6 * k))(*(list(info) * k))
    rc = lib.se_png_decode_u8(src, (L * k)(*([src_off] * k)), (L * k)(*([src_len] * k)), info_a, (L * k)(*([plte_off] * k)), n,
                              out, status, scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    rgb = (10, 10, 8, 2, 0, 3)                                     # h, w, depth, colour type, palette entries, output channels
    assert _call(lib, rgb)[:2] == (0, 320)                         # 10 filtered rows of 1 + 30 bytes, rounded up to 16
    assert _call(lib, rgb, n=3)[:2] == (0, 960)
    assert _call(lib, (5, 7, 1, 3, 2, 1))[:2] == (0, 5 * (1 + 1) + 6)   # 1-bit palette: 1 byte per row
    assert _call(lib, rgb, n=0)[:2] == (0, 0)
    for info, kw, msg in [(rgb, dict(n=257), "n must be in"), (rgb, dict(n=-1), "n must be in"),
                          ((0, 10, 8, 2, 0, 3), {}, "file 0: sizes must be in [1, 65535]"),
                          ((10, 65536, 8, 2, 0, 3), {}, "file 0: sizes must be in [1, 65535]"),
                          ((10, 10, 16, 2, 0, 3), {}, "colour type 2 at depth 16 is not decoded here"),
                          ((10, 10, 8, 5, 0, 3), {}, "colour type 5 at depth 8 is not decoded here"),
                          ((10, 10, 8, 3, 0, 3), {}, "a palette of 1 to 256 entries"),
                          ((10, 10, 8, 3, 257, 3), {}, "a palette of 1 to 256 entries"),
                          ((10, 10, 8, 3, 4, 3), dict(plte_off=-1), "a palette of 1 to 256 entries"),
                          ((10, 10, 8, 2, 4, 3), {}, "a palette of 1 to 256 entries"),
                          ((10, 10, 8, 2, 0, 2), {}, "mode must be 1 (L) or 3 (RGB)"),
                          (rgb, dict(src_off=-1), "negative offset or length"), (rgb, dict(src_len=-1), "negative offset or length")]:
        rc, _, err = _call(lib, info, **kw)
        assert rc != 0 and msg in err, (info, kw, err)
    assert lib.se_png_decode_u8(None, None, None, None, None, 1, None, None, None, ctypes.byref(ctypes.c_longlong(0)), None) != 0
    assert "null length / offset / info array" in lib.se_last_error().decode()
    # past the query: scratch too small, then null pointers, all refused before anything is enqueued
    rc, _, err = _call(lib, rgb, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes, needs 320" in err
    rc, _, err = _call(lib, rgb, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(320))
    assert rc != 0 and "null src / out / status" in err
    rc, _, err = _call(lib, rgb, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(320), src=ctypes.c_void_p(256),
                       out=(ctypes.c_void_p * 1)(None), status=ctypes.c_void_p(256))
    assert rc != 0 and "null out" in err
    assert _call(lib, rgb, n=0, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(0))[0] == 0

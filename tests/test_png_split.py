"""The split inflate of se_png_split.cu on the host: its stages (se_inflate_split.cuh: find, count, link, emit, resolve and the
Adler-32 check) built with the host compiler and run in order with one lane against zlib, over every encoder setting, flush
points, chunk spacings from 1 byte to 64 KB, far matches whose markers cross chunks, malformed and mutated streams and a
crafted false block start; se_png_split_u8's argument checks and scratch query; and edit sessions opened from upload bytes
with the Pillow flow."""
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

from sketchedit_b200 import _lib, build
from tests import util_png_decode as U
from tests.test_png_decode import CSRC, zlib_says

INF_LINK = 12

DRIVER = r"""
#include <stdio.h>
#include <stdlib.h>
#include "se_inflate_split.cuh"
using namespace se;
// The stages in launch order, one lane. Chunks are counted in order (each one's end is only compared in link), emitted and
// resolved from the last to the first: no chunk reads another's entries, and resolve_byte reads entries only.
static int split(const unsigned char* src, long long n, unsigned char* raw, long long raw_n, long long S, InflateTabs& t,
                 long long* used) {
  const long long nc = n / S + 1;
  SplitChunk* c = (SplitChunk*)malloc(sizeof(SplitChunk) * nc);
  for (long long k = 0; k < nc; ++k) {
    long long lo, hi, start = 16;
    if (k > 0) {
      chunk_bits(k, S, n, &lo, &hi);
      start = find_block(src, n, lo, hi, 0, 1);
    }
    c[k] = SplitChunk{start, -1, 0, 0, 0, 0, 0};
  }
  *used = 0;
  for (long long k = 0; k < nc; ++k) {
    if (c[k].start < 0) continue;
    ++*used;
    for (long long j = k + 1; j < nc; ++j)
      if (c[j].start >= 0) {
        c[k].next = c[j].start;
        break;
      }
    c[k].status = chunk_count(src, n, raw_n, c[k], k == 0, t, 0, 1);
  }
  long long tail = 0;
  int st = chunks_link(c, nc, raw_n, &tail);
  unsigned* e = (unsigned*)malloc(4 * (raw_n ? raw_n : 1));
  for (long long k = nc - 1; k >= 0 && st == 0; --k)
    if (c[k].start >= 0) st = chunk_emit(src, n, c[k], e, t, 0, 1);
  for (long long i = raw_n - 1; i >= 0 && st == 0; --i) {
    const int v = resolve_byte(e, i);
    if (v < 0) st = INF_LINK;
    raw[i] = (unsigned char)v;
  }
  if (st == 0) {
    const long long want = stored_adler(src, n, tail);
    st = want < 0 ? INF_SHORT_INPUT : adler32_lanes(raw, raw_n, 0, 1) == (unsigned)want ? INF_OK : INF_ADLER;
  }
  free(e);
  free(c);
  return st;
}
// cases on stdin: int64 raw_n, int64 S, int64 n, n stream bytes; on stdout per case: int32 status, int64 non-empty chunks,
// then raw_n bytes when the status is 0. Each buffer is allocated at its exact size for the address sanitizer.
int main() {
  long long hdr[3];
  static InflateTabs tabs;
  while (fread(hdr, 8, 3, stdin) == 3) {
    unsigned char* src = (unsigned char*)malloc(hdr[2] ? hdr[2] : 1);
    unsigned char* raw = (unsigned char*)malloc(hdr[0] ? hdr[0] : 1);
    if (hdr[2] && fread(src, 1, hdr[2], stdin) != (size_t)hdr[2]) return 3;
    long long used = 0;
    int st = split(hdr[2] ? src : nullptr, hdr[2], raw, hdr[0], hdr[1], tabs, &used);
    fwrite(&st, 4, 1, stdout);
    fwrite(&used, 8, 1, stdout);
    if (st == 0) fwrite(raw, 1, hdr[0], stdout);
    free(src);
    free(raw);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def split_host(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("split_host")
    src, exe = d / "driver.cpp", d / "split_host"
    src.write_text(DRIVER)
    subprocess.run([cxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-I", CSRC, str(src), "-o", str(exe)], check=True)

    def run(cases):
        """cases: (stream, raw_n, S) -> [(status, non-empty chunks, bytes or None)]"""
        blob = b"".join(struct.pack("<qqq", n, S, len(z)) + z for z, n, S in cases)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
        p = subprocess.run([str(exe)], input=blob, capture_output=True, env=env)
        assert p.returncode == 0, p.stderr.decode()[-3000:]
        res, at = [], 0
        for z, n, S in cases:
            st, used = struct.unpack("<iq", p.stdout[at:at + 12])
            at += 12
            res.append((st, used, p.stdout[at:at + n] if st == 0 else None))
            at += n if st == 0 else 0
        assert at == len(p.stdout)
        return res
    return run


def check(run, cases):
    """Status 0 only with zlib's bytes; nonzero wherever zlib refuses. Returns the results."""
    res = run(cases)
    for (z, n, S), (st, _, raw) in zip(cases, res):
        want = zlib_says(z, n)
        if st == 0:
            assert want is not None and raw == want, (z[:40], n, S)
        else:
            assert want is None or 1 <= st <= 12, (z[:40], n, S, st)
    return res


def deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem=8, flushes=()):
    """zlib's stream of data; memLevel `mem` sets how many symbols a block holds (2^(mem + 6)), `flushes` are (offset, mode)
    points where the compressor flushes (Z_SYNC_FLUSH, Z_FULL_FLUSH: an empty stored block)."""
    c = zlib.compressobj(level, zlib.DEFLATED, 15, mem, strategy)
    out, at = b"", 0
    for o, mode in flushes:
        out += c.compress(data[at:o]) + c.flush(mode)
        at = o
    return out + c.compress(data[at:]) + c.flush()


def datas():
    rng = np.random.default_rng(3)
    text = (b"the quick brown fox jumps over the lazy dog %d; " * 400) % tuple(range(400))
    return {"filtered": U.filt(U.photo(60, 80).reshape(60, 240), 3, (1, 2, 4)), "text": text,
            "noise": rng.integers(0, 256, 6000, dtype=np.uint8).tobytes(), "zeros": b"\0" * 5000, "ab": b"ab" * 1500}


SPACINGS = (1, 2, 3, 7, 64, 1000)


def test_encoder_settings_and_spacings(split_host):
    """Levels 0, 1, 6, 9 and Z_RLE, Z_HUFFMAN_ONLY, Z_FIXED, with small blocks (memLevel 1: 128 symbols) and zlib's default:
    every chunk spacing decodes each stream to zlib's bytes, and small spacings use many chunks."""
    cases, dynamic = [], []
    for name, data in datas().items():
        for lvl in (0, 1, 6, 9):
            for strat in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_RLE, zlib.Z_HUFFMAN_ONLY, zlib.Z_FIXED):
                for mem in (1, 8):
                    z = deflate(data, lvl, strat, mem)
                    if name == "filtered" and lvl and strat != zlib.Z_FIXED and mem == 1:
                        dynamic.append(len(cases))   # dynamic blocks of 128 symbols: cut at every byte, many chunks
                    cases += [(z, len(data), S) for S in SPACINGS]
    res = check(split_host, cases)
    assert all(st == 0 for st, _, _ in res), [(len(z), S, st) for (z, _, S), (st, _, _) in zip(cases, res) if st]
    assert min(res[k][1] for k in dynamic) > 20


def test_flush_points(split_host):
    """Empty stored blocks from Z_SYNC_FLUSH and Z_FULL_FLUSH between dynamic blocks, at several offsets."""
    data = datas()["filtered"]
    cases = []
    for flushes in ([(10, zlib.Z_SYNC_FLUSH)], [(3000, zlib.Z_FULL_FLUSH), (3001, zlib.Z_SYNC_FLUSH)],
                    [(o, zlib.Z_SYNC_FLUSH if o % 2 else zlib.Z_FULL_FLUSH) for o in range(500, len(data), 1777)]):
        for mem in (1, 8):
            z = deflate(data, 6, mem=mem, flushes=flushes)
            cases += [(z, len(data), S) for S in SPACINGS]
    res = check(split_host, cases)
    assert all(st == 0 for st, _, _ in res)


def test_large_spacings(split_host):
    """A 400 KB photo at zlib's defaults cut every 4 KB to 64 KB: chunks start inside every kind of block."""
    data = U.filt(U.photo(400, 340, 5).reshape(400, 1020), 3, (1, 2, 4))
    cases = [(deflate(data, lvl), len(data), S) for lvl in (1, 6) for S in (4096, 16384, 65536)]
    res = check(split_host, cases)
    assert all(st == 0 for st, _, _ in res)
    assert max(used for _, used, _ in res) >= 8


def test_far_matches_cross_chunks(split_host):
    """32 KB of filtered scanlines written four times, a byte changed every 97: matches of distance 32768 between the changes,
    in 128-symbol blocks, so each marker chain walks back through several chunks to the first copy."""
    base = np.frombuffer(U.filt(U.photo(64, 171, 9).reshape(64, 513), 3, (1, 4)), np.uint8)[:32768]
    copies = [base]
    for k in range(3):
        c = copies[-1].copy()
        c[k::97] ^= 0x5A
        copies.append(c)
    data = np.concatenate(copies).tobytes()
    cases = [(deflate(data, lvl, mem=mem), len(data), S) for lvl in (6, 9) for mem in (1, 8) for S in (64, 1000, 4096)]
    res = check(split_host, cases)
    assert all(st == 0 for st, _, _ in res)
    assert max(used for _, used, _ in res) > 10


def test_malformed_and_mutated(split_host):
    """The one-warp decoder's malformed streams and 2000 mutations (bit flips, cuts, deletions, insertions) of the streams
    above at small spacings: nonzero wherever zlib refuses, zlib's bytes wherever the status is 0."""
    z = zlib.compress(U.photo(9, 8).tobytes())
    n = 9 * 8 * 3
    far, _ = U.fixed_deflate([1, (5, 2)])
    bad = [(b"", n), (z[:1], n), (b"\x78\x02" + z[2:], n), (bytes([0x78, 0xBB]) + z[2:], n), (z[:-1], n),
           (z[:-1] + bytes([z[-1] ^ 1]), n), (b"\x78\x01\x07" + z[3:], n), (far, 6), (z, n - 1), (z, n + 1),
           (b"\x78\x01\x01\x05\x00\xfb\xff", 5), (b"\x78\x01\x01\x05\x00\xfa\xff" + b"abcde", 5),
           (b"\x78\x01\x05\xe0\xff" + b"\xff" * 8, 4)]
    res = check(split_host, [(z_, n_, S) for z_, n_ in bad for S in (1, 5, 64)])
    assert all(st != 0 for st, _, _ in res)
    rnd = random.Random(13)
    base = [(deflate(d, lvl, mem=mem), len(d)) for d in datas().values() for lvl in (1, 6, 9) for mem in (1, 8)]
    cases = []
    for _ in range(2000):
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
        cases.append((bytes(z), n + rnd.choice((0, 0, 0, -1, 1)), rnd.choice((1, 3, 16, 100))))
    check(split_host, cases)


def test_false_block_start_is_refused(split_host):
    """A stored block whose payload is a valid dynamic block (BFINAL 0) from its first bit, placed so that payload starts at
    a chunk's nominal offset: the finder takes it as chunk 1's start, chunk 0 ends after the stored block instead, and the
    stream is refused (never decoded to other bytes), though zlib accepts it."""
    inner = zlib.compressobj(6, zlib.DEFLATED, -15, 1)   # raw deflate, 128-symbol blocks: the first is dynamic, not final
    payload = inner.compress(datas()["filtered"]) + inner.flush()
    payload = payload[:200]
    assert payload[0] & 7 == 4   # BFINAL 0, BTYPE 2
    stored = bytes([0]) + struct.pack("<HH", len(payload), 0xFFFF ^ len(payload)) + payload
    last = b"\x01\x00\x00\xff\xff"   # an empty final stored block
    z = b"\x78\x01" + stored + last + struct.pack(">I", zlib.adler32(payload))
    assert zlib.decompress(z) == payload
    S = 7   # the payload starts at byte 7: zlib header 2, stored header 1, LEN and NLEN 4
    (st, used, raw), = check(split_host, [(z, len(payload), S)])
    assert st == INF_LINK and used >= 2
    (st, _, raw), = check(split_host, [(z, len(payload), 1000)])   # one chunk: decoded
    assert st == 0 and raw == payload


# ------------------------------------------------------------------------------------------------ se_png_split_u8's host checks
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _call(lib, info, n=1, src_off=0, src_len=100, plte_off=0, chunk=16, scratch=None, need=None, src=None, out=None,
          status=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    L = ctypes.c_longlong
    info_a = (ctypes.c_int * (6 * k))(*(list(info) * k))
    rc = lib.se_png_split_u8(src, (L * k)(*([src_off] * k)), (L * k)(*([src_len] * k)), info_a, (L * k)(*([plte_off] * k)), n,
                             out, status, chunk, scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_split_entry_checks_and_scratch_query(lib):
    rgb = (10, 10, 8, 2, 0, 3)   # h, w, depth, colour type, palette entries, output channels: 310 raw bytes
    # 256 bytes of file state, 48 bytes per chunk (100 / 16 + 1 = 7 chunks) rounded to 256, 320 raw bytes and 4 x 320 entries
    assert _call(lib, rgb)[:2] == (0, 256 + 512 + 5 * 320)
    assert _call(lib, rgb, chunk=1000)[:2] == (0, 256 + 256 + 5 * 320)
    assert _call(lib, rgb, n=3)[:2] == (0, 256 + 1024 + 5 * 960)
    assert _call(lib, rgb, n=0)[:2] == (0, 0)
    for info, kw, msg in [(rgb, dict(n=257), "n must be in"), (rgb, dict(chunk=0), "chunk_bytes must be at least 1"),
                          ((0, 10, 8, 2, 0, 3), {}, "file 0: sizes must be in [1, 65535]"),
                          ((10, 10, 16, 2, 0, 3), {}, "colour type 2 at depth 16 is not decoded here"),
                          ((10, 10, 8, 3, 0, 3), {}, "a palette of 1 to 256 entries"),
                          ((10, 10, 8, 2, 0, 2), {}, "mode must be 1 (L) or 3 (RGB)"),
                          ((40000, 20000, 8, 6, 0, 3), {}, "more than the split decoder's 2^31 - 1"),
                          (rgb, dict(src_len=-1), "negative offset or length")]:
        rc, _, err = _call(lib, info, **kw)
        assert rc != 0 and msg in err, (info, kw, err)
    rc, _, err = _call(lib, rgb, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes, needs" in err
    rc, _, err = _call(lib, rgb, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(1 << 20))
    assert rc != 0 and "null src / out / status" in err
    assert _call(lib, rgb, n=0, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(0))[0] == 0


def test_chunk_spacing_follows_the_stream():
    from sketchedit_b200 import engine as E
    assert E.png_split_chunk_bytes(100) == E.PNG_SPLIT_MIN_CHUNK
    big = E.png_split_chunk_bytes(1 << 30)
    assert big >= E.PNG_SPLIT_MIN_CHUNK and (1 << 30) // big <= E.PNG_SPLIT_MAX_CHUNKS


# ------------------------------------------------------------------------------------------------ sessions from upload bytes
def _uploads():
    ph = U.photo(45, 61, 2)
    buf = io.BytesIO()
    Image.fromarray(ph).save(buf, "JPEG", quality=90, subsampling=1)
    jpeg = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray(ph).save(buf, "PNG", icc_profile=b"\0" * 300)
    icc_png = buf.getvalue()
    return {"png": U.pil_png(ph), "png_grey": U.pil_png(ph[..., 0]), "png_palette": U.make_png(
        np.arange(45 * 61).reshape(45, 61, 1) % 7, 4, 3, palette=np.arange(21).reshape(7, 3) * 9),
        "png_interlaced": U.adam7(ph), "png_icc": icc_png, "jpeg": jpeg}


def test_session_from_bytes_is_session_from_pillow():
    """resize='host': a session opened from the upload's bytes (bytes, bytearray, memoryview) is the session opened from
    Image.open of them: photo, size, exif, icc_profile, keep, and the same files after an edit and an undo; garbage bytes
    raise Pillow's exception."""
    from tests.test_edit_session import _FakeProcessor, _mask, _NoForward
    proc = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    try:
        for name, data in _uploads().items():
            for given in (data, bytearray(data), memoryview(data)):
                a, b = proc.open_session(given), proc.open_session(Image.open(io.BytesIO(data)))
                assert a.size == b.size and a.exif == b.exif and a.icc_profile == b.icc_profile, name
                assert a.image().tobytes() == b.image().tobytes(), name
                for s in (a, b):
                    s.edit(_mask(*s.size, [(5, 6, 30, 25)]), None, region="auto")
                assert a.png() == b.png() and a.jpeg(80) == b.jpeg(80), name
                if name == "jpeg":
                    assert a.jpeg(quality="keep") == b.jpeg(quality="keep")
                else:
                    with pytest.raises(ValueError, match="not a JPEG"):
                        a.jpeg(quality="keep")
                a.undo()
                b.undo()
                assert a.image().tobytes() == b.image().tobytes(), name
                a.close()
                b.close()
        for bad in (b"", b"\x89PNG\r\n\x1a\n" + b"\0" * 40, b"garbage bytes"):
            with pytest.raises(Exception) as want:
                Image.open(io.BytesIO(bad)).convert("RGB")
            with pytest.raises(type(want.value)):
                proc.open_session(bad)
    finally:
        proc.close()

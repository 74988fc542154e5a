"""PNG decoding restated in numpy (zlib does the inflate), and the corpus the decoder is tested on.

``decode(data, mode)`` restates what se_png_decode_u8 computes for the files ``sketchedit_b200.pngfile`` sends to the
device: container parse, unfilter, bit unpack, palette and conversion. tests/test_png_decode.py pins it to
``np.asarray(Image.open(f).convert(mode))``; tests/test_gpu_png_decode.py pins the kernels to Pillow over the same corpus."""
import io
import struct
import zlib

import numpy as np
from PIL import Image

SIG = b"\x89PNG\r\n\x1a\n"


# ---------------------------------------------------------------------------------------------------------------- restatement
def chunks(data):
    at = 8
    while at + 8 <= len(data):
        n, cid = struct.unpack(">I4s", data[at:at + 8])
        yield cid, data[at + 8:at + 8 + n]
        at += 12 + n


def unfilter(raw, h, rowb, bpp):
    """Rows of the filtered scanlines ``raw`` (h rows of 1 + rowb bytes) after undoing each row's filter."""
    rows = np.frombuffer(raw, np.uint8).reshape(h, rowb + 1)
    out = np.zeros((h, rowb), np.uint8)
    prev = np.zeros(rowb, np.int32)
    for r in range(h):
        ft, x = rows[r, 0], rows[r, 1:].astype(np.int32)
        cur = np.zeros(rowb, np.int32)
        if ft == 0:
            cur = x
        elif ft == 2:
            cur = (x + prev) & 255
        else:
            for i in range(rowb):
                a = cur[i - bpp] if i >= bpp else 0
                b, c = prev[i], (prev[i - bpp] if i >= bpp else 0)
                if ft == 1:
                    pred = a
                elif ft == 3:
                    pred = (a + b) >> 1
                elif ft == 4:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = a if pa <= pb and pa <= pc else b if pb <= pc else c
                else:
                    raise ValueError("filter type %d" % ft)
                cur[i] = (x[i] + pred) & 255
        out[r] = cur
        prev = cur
    return out


def luma(rgb):
    rgb = rgb.astype(np.uint32)
    return ((rgb[..., 0] * 19595 + rgb[..., 1] * 38470 + rgb[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def decode(data, mode):
    """np.asarray(Image.open(f).convert(mode)) for a non-interlaced PNG of 8 bits or less, restated."""
    cs = list(chunks(data))
    w, h, depth, ctype, _, _, lace = struct.unpack(">IIBBBBB", cs[0][1])
    assert lace == 0 and depth <= 8
    pal = next((np.frombuffer(b, np.uint8).reshape(-1, 3) for c, b in cs if c == b"PLTE"), None)
    raw = zlib.decompress(b"".join(b for c, b in cs if c == b"IDAT"))
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    rowb = (w * ch * depth + 7) // 8
    rows = unfilter(raw[:h * (rowb + 1)], h, rowb, max(1, ch * depth // 8))
    if depth < 8:
        bits = np.unpackbits(rows, axis=1).reshape(h, -1, depth)[:, :w]
        v = (bits * (1 << np.arange(depth - 1, -1, -1))).sum(-1).astype(np.uint8)
    else:
        v = rows.reshape(h, w, ch)
    if ctype == 3:
        idx = v if depth < 8 else v[..., 0]
        if idx.max() >= len(pal):
            raise IndexError("palette index past the palette")
        rgb = pal[idx]
    elif ctype in (0, 4):
        g = (v * (255 // ((1 << depth) - 1))).astype(np.uint8) if depth < 8 else v[..., 0]
        rgb = np.repeat(g[..., None], 3, -1)
    else:
        rgb = v[..., :3]
    return rgb if mode == "RGB" else luma(rgb)


# ---------------------------------------------------------------------------------------------------------------- writing
def chunk(cid, body):
    return struct.pack(">I", len(body)) + cid + body + struct.pack(">I", zlib.crc32(body, zlib.crc32(cid)))


def filt(rows, bpp, ftypes):
    """Filtered scanlines of the uint8 rows [h, rowb]; row r uses filter ftypes[r % len(ftypes)]."""
    h, rowb = rows.shape
    out, prev = bytearray(), np.zeros(rowb, np.int32)
    for r in range(h):
        x, ft = rows[r].astype(np.int32), ftypes[r % len(ftypes)]
        if ft in (0, 2):
            y = x - (prev if ft == 2 else 0)
        else:
            y = np.zeros(rowb, np.int32)
            for i in range(rowb):
                a = x[i - bpp] if i >= bpp else 0
                b, c = prev[i], (prev[i - bpp] if i >= bpp else 0)
                if ft == 1:
                    pred = a
                elif ft == 3:
                    pred = (a + b) >> 1
                else:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = a if pa <= pb and pa <= pc else b if pb <= pc else c
                y[i] = x[i] - pred
        out += bytes([ft]) + (y & 255).astype(np.uint8).tobytes()
        prev = x
    return bytes(out)


def pack_rows(v, depth):
    """Sample rows [h, w * channels] of values below 2^depth packed at `depth` bits, MSB first."""
    if depth == 8:
        return v.astype(np.uint8)
    bits = ((v[..., None] >> np.arange(depth - 1, -1, -1)) & 1).astype(np.uint8).reshape(v.shape[0], -1)
    return np.packbits(bits, axis=1)


def make_png(v, depth, ctype, ftypes=(0, 1, 2, 3, 4), palette=None, trns=None, stream=None, idat=8192, lace=0, extra=(),
             **z):
    """A PNG of the samples v [h, w, channels] built by hand: filters ftypes per row, zlib with the compressobj keywords z
    (or the given stream, a function of the filtered bytes), IDAT chunks of `idat` bytes, extra (cid, body) chunks before
    IDAT."""
    h, w = v.shape[:2]
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    rows = pack_rows(v.reshape(h, w * ch), depth)
    raw = filt(rows, max(1, ch * depth // 8), ftypes)
    if stream is None:
        c = zlib.compressobj(**z)
        data = c.compress(raw) + c.flush()
    else:
        data = stream(raw)
    out = SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, lace))
    for cid, body in extra:
        out += chunk(cid, body)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    if trns is not None:
        out += chunk(b"tRNS", trns)
    for k in range(0, max(len(data), 1), idat):
        out += chunk(b"IDAT", data[k:k + idat])
    return out + chunk(b"IEND", b"")


class BitWriter:
    def __init__(self):
        self.bits, self.n = 0, 0

    def put(self, v, k):
        self.bits |= v << self.n
        self.n += k

    def code(self, c, k):   # Huffman codes go MSB first
        self.put(int(format(c, "0%db" % k)[::-1], 2), k)

    def bytes(self):
        return self.bits.to_bytes((self.n + 7) // 8, "little")


def fixed_deflate(symbols):
    """One final fixed-Huffman block of symbols: ints (literals) and (length, distance) pairs; zlib-wrapped."""
    lbase = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
    lext = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    dbase = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
    dext = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
    bw = BitWriter()
    bw.put(1, 1)
    bw.put(1, 2)

    def lit(s):
        if s < 144:
            bw.code(0x30 + s, 8)
        elif s < 256:
            bw.code(0x190 + s - 144, 9)
        elif s < 280:
            bw.code(s - 256, 7)
        else:
            bw.code(0xC0 + s - 280, 8)

    out = bytearray()
    for s in symbols:
        if isinstance(s, int):
            lit(s)
            out.append(s)
            continue
        ln, d = s
        lc = max(i for i in range(29) if lbase[i] <= ln)
        lit(257 + lc)
        bw.put(ln - lbase[lc], lext[lc])
        dc = max(i for i in range(30) if dbase[i] <= d)
        bw.code(dc, 5)
        bw.put(d - dbase[dc], dext[dc])
        for _ in range(ln):
            out.append(out[-d] if d <= len(out) else 0)   # (a distance too far back: malformed())
    lit(256)
    return b"\x78\x01" + bw.bytes() + struct.pack(">I", zlib.adler32(bytes(out))), bytes(out)


# ---------------------------------------------------------------------------------------------------------------- corpus
def photo(h, w, seed=0):
    """A photo-like RGB image: smooth gradients plus a little noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * 255 / max(w - 1, 1), y * 255 / max(h - 1, 1), (x + y) * 127 / max(h + w - 2, 1)], -1)
    return np.clip(base + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)


def sketch(h, w, seed=0):
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w), np.uint8)
    for _ in range(max(1, h // 16)):
        img[rng.integers(0, h), :] = 255
        img[:, rng.integers(0, w)] = 255
    return img


def pil_png(arr, **kw):
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, "PNG", **kw)
    return buf.getvalue()


def corpus(big=False):
    """(name, bytes) of files the device decodes; every one's pixels are Pillow's."""
    import cv2
    rng = np.random.default_rng(7)
    out = []
    ph = photo(37, 53, 1)
    for lvl in range(10):
        out.append(("pil_level%d" % lvl, pil_png(ph, compress_level=lvl)))
    out.append(("pil_optimize", pil_png(ph, optimize=True)))
    out.append(("pil_grey", pil_png(sketch(40, 31, 2))))
    strategies = [v for k, v in vars(cv2).items() if k.startswith("IMWRITE_PNG_STRATEGY_")]
    for lvl in range(10):
        for s in sorted(set(strategies)):
            img = ph[..., ::-1] if (lvl + s) % 2 else sketch(29, 41, lvl)
            out.append(("cv2_l%d_s%d" % (lvl, s), cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, lvl,
                                                                              cv2.IMWRITE_PNG_STRATEGY, s])[1].tobytes()))
    small = photo(19, 23, 3)
    out.append(("filters_rgb", make_png(small, 8, 2)))
    out.append(("filters_rgba", make_png(np.dstack([small, small[..., :1]]), 8, 6, ftypes=(4, 3, 2, 1, 0))))
    for name, z in (("z_fixed", dict(strategy=zlib.Z_FIXED)), ("z_huffman", dict(strategy=zlib.Z_HUFFMAN_ONLY)),
                    ("z_rle", dict(strategy=zlib.Z_RLE))):
        out.append((name, make_png(small, 8, 2, **z)))
    for wb in range(9, 16):
        out.append(("wbits%d" % wb, make_png(photo(40, 60, wb), 8, 2, ftypes=(1, 4), wbits=wb)))

    def window256(raw):   # windowBits 8: zlib's deflate writes 8 as 9, so CINFO 0 goes in by hand over a distance-1 stream
        c = zlib.compressobj(9, zlib.DEFLATED, -15, strategy=zlib.Z_RLE)
        return bytes([0x08, 0x1D]) + c.compress(raw) + c.flush() + struct.pack(">I", zlib.adler32(raw))
    out.append(("wbits8", make_png(photo(40, 60, 8), 8, 2, ftypes=(1,), stream=window256)))

    def stored_flushes(raw):   # an empty stored block from each sync flush, then level 0: stored blocks of 65535
        c = zlib.compressobj(0)
        return c.compress(raw[:10]) + c.flush(zlib.Z_SYNC_FLUSH) + c.flush(zlib.Z_FULL_FLUSH) + c.compress(raw[10:]) + c.flush()
    out.append(("stored", make_png(photo(120, 250, 4), 8, 2, ftypes=(0,), stream=stored_flushes)))
    flat = np.full((3, 300, 3), 9, np.uint8)
    out.append(("match258_d1", make_png(flat, 8, 2, ftypes=(0,), level=9)))
    # matches of 258 at distance 32768: two equal rows of 32767 grey pixels (a row and its filter byte are 32768 bytes)
    first = bytes([0]) + rng.integers(0, 256, 32767, dtype=np.uint8).tobytes()
    z, _ = fixed_deflate(list(first) + [(258, 32768)] * 126 + [(257, 32768), (3, 32768)])
    out.append(("match258_d32768", make_png(np.zeros((2, 32767, 1), np.uint8), 8, 0, stream=lambda _r: z)))
    out.append(("idat_1byte", make_png(photo(9, 11, 5), 8, 2, idat=1)))
    # every colour type and depth, short palettes, tRNS
    for depth in (1, 2, 4, 8):
        v = rng.integers(0, 1 << depth, (13, 17, 1))
        out.append(("grey%d" % depth, make_png(v, depth, 0)))
        out.append(("grey%d_trns" % depth, make_png(v, depth, 0, trns=struct.pack(">H", 1))))
        npal = min(3, 1 << depth)
        pv = rng.integers(0, npal, (11, 21, 1))
        pal = rng.integers(0, 256, (npal, 3))
        out.append(("pal%d_short" % depth, make_png(pv, depth, 3, palette=pal)))
        out.append(("pal%d_trns" % depth, make_png(pv, depth, 3, palette=pal, trns=b"\x00\x80")))
    out.append(("rgb_trns", make_png(photo(7, 9, 6), 8, 2, trns=struct.pack(">HHH", 1, 2, 3))))
    out.append(("la", make_png(rng.integers(0, 256, (10, 13, 2)), 8, 4)))
    out.append(("rgba", make_png(rng.integers(0, 256, (10, 13, 4)), 8, 6)))
    out.append(("pal8_full", make_png(rng.integers(0, 256, (16, 16, 1)), 8, 3, palette=rng.integers(0, 256, (256, 3)))))
    out.append(("ancillary", make_png(photo(6, 7, 8), 8, 2, extra=[(b"gAMA", b"\0\0\xb1\x8f"), (b"pHYs", bytes(9)),
                                                                   (b"sRGB", b"\0")])))
    for h, w in ((1, 1), (1, 37), (41, 1), (5, 333), (17, 2)):
        out.append(("size%dx%d" % (h, w), pil_png(photo(h, w, h + w))))
        out.append(("size%dx%d_1bit" % (h, w), make_png(rng.integers(0, 2, (h, w, 1)), 1, 0)))
    if big:
        out.append(("big_4000x2667", pil_png(photo(2667, 4000, 9))))
    return out


def fallbacks():
    """(name, bytes, reason) of files pngfile routes to Pillow."""
    ph = photo(12, 10, 11)
    buf = io.BytesIO()
    Image.fromarray(ph).save(buf, "PNG", save_all=True, append_images=[Image.fromarray(ph[::-1])])
    apng = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray((np.arange(120).reshape(12, 10) * 500).astype(np.uint16)).save(buf, "PNG")
    deep = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray(ph).save(buf, "JPEG")
    return [("interlaced", adam7(ph), "interlaced"), ("16bit", deep, "16-bit"), ("apng", apng, "APNG"),
            ("jpeg_named_png", buf.getvalue(), "not a PNG"),
            ("text", make_png(ph, 8, 2, extra=[(b"tEXt", b"k\0v")]), "chunk b'tEXt'")]


def adam7(rgb):
    """An interlaced RGB PNG of rgb (filter None)."""
    h, w = rgb.shape[:2]
    raw = b""
    for y0, x0, dy, dx in ((0, 0, 8, 8), (0, 4, 8, 8), (4, 0, 8, 4), (0, 2, 4, 4), (2, 0, 4, 2), (0, 1, 2, 2), (1, 0, 2, 1)):
        sub = rgb[y0::dy, x0::dx]
        if sub.size:
            raw += b"".join(b"\0" + r.tobytes() for r in sub)
    return (SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 1)) + chunk(b"IDAT", zlib.compress(raw)) +
            chunk(b"IEND", b""))


def malformed():
    """(name, bytes) of files the parser accepts and the decoder must refuse (nonzero status)."""
    ph = photo(9, 8, 12)
    rows = (b"\x01" + ph[0].tobytes()) * 9

    def with_stream(z):
        return make_png(ph, 8, 2, ftypes=(1,), stream=lambda _r: z)
    zs = zlib.compress(rows)
    bad = [("bad_header", with_stream(b"\x78\x02" + zs[2:])),
           ("fdict", with_stream(bytes([0x78, 0xBB]) + b"\0\0\0\0" + zs[2:])),
           ("truncated", with_stream(zs[:len(zs) // 2])),
           ("bad_adler", with_stream(zs[:-1] + bytes([zs[-1] ^ 1]))),
           ("block_type3", with_stream(b"\x78\x01\x07" + zs[3:])),
           ("too_far", with_stream(fixed_deflate([1, (5, 2)])[0])),
           ("too_many", make_png(ph, 8, 2, stream=lambda r: zlib.compress(r + b"\0" * 5))),
           ("too_few", make_png(ph, 8, 2, stream=lambda r: zlib.compress(r[:-5]))),
           ("bad_filter", make_png(ph, 8, 2, stream=lambda r: zlib.compress(b"\x05" + r[1:]))),
           ("palette_index", make_png(np.full((4, 4, 1), 5), 8, 3, palette=[[1, 2, 3]] * 3))]
    return bad

"""What ``cv2.imencode(".png", img)`` writes with no parameters (OpenCV 4.13, libpng 1.6, zlib 1.3), restated in numpy and
plain Python. It is the spec se_png.cu follows, and its stages (``filtered``, ``parse``, ``deflate``, ``zlib_stream``) split a
failing GPU case by stage. Tests pin it to cv2.

  * Filter: every row is Sub (type 1), or None (type 0) when the image is 1 pixel wide. A colour image is written as RGB
    (cv2 takes BGR), one channel as greyscale.
  * Parse: zlib level 1, memLevel 8, strategy Z_RLE. deflate_rle only looks back one byte and matches greedily, so every
    maximal run of L equal bytes is one literal, (L - 1) // 258 matches of 258, then for r = (L - 1) % 258 one match of r
    when r >= 3, else r literals. All matches are at distance 1.
  * Blocks: a block ends after every 16383 symbols ((lit_bufsize - 1), lit_bufsize = 1 << 14); the last block holds the rest
    and is empty when the count is a multiple of 16383. Each block's trees and its choice of stored / static / dynamic are
    zlib's trees.c (build_tree, gen_bitlen, gen_codes, scan_tree, send_tree, build_bl_tree, _tr_flush_block).
  * zlib stream: CMF / FLG with libpng's window rewrite (the smallest window covering the filtered data), the LSB-first bit
    stream, Adler-32 big-endian.
  * File: signature, IHDR, the stream in IDAT chunks of 8192 bytes (the last shorter), IEND.
"""
import struct
import zlib

import numpy as np

BLOCK_SYMS = 16383          # symbols per deflate block (sym_end / 3 at memLevel 8)
MAX_MATCH = 258
IDAT_CHUNK = 8192           # libpng's zbuffer: bytes of zlib stream per IDAT chunk
STORED_MAX = 32506          # a stored block's bytes lie in zlib's window (buf != NULL) up to wsize - MIN_LOOKAHEAD bytes
L_CODES, D_CODES, BL_CODES, HEAP_SIZE = 286, 30, 19, 2 * 286 + 1
MAX_BITS, MAX_BL_BITS, END_BLOCK = 15, 7, 256
EXTRA_LBITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
STORED, STATIC, DYNAMIC = 0, 1, 2


def _length_tables():
    """(length_code[lc], base_length[code]) of trees.c for lc = match length - 3; lc 255 (258) is code 28, not 27 + 31."""
    code_of, base = [0] * 256, [0] * 29
    lc = 0
    for code in range(28):
        base[code] = lc
        for _ in range(1 << EXTRA_LBITS[code]):
            code_of[lc] = code
            lc += 1
    code_of[255] = 28
    base[28] = 255
    return np.array(code_of, np.int64), np.array(base, np.int64)


LENGTH_CODE, BASE_LENGTH = _length_tables()
STATIC_LLEN = np.array([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, np.int64)   # 288 codes
STATIC_DLEN = np.full(D_CODES, 5, np.int64)


def bi_reverse(code, n):
    return int("{:0{}b}".format(code, n)[::-1], 2) if n else 0


def canonical_codes(lens):
    """gen_codes: bit-reversed canonical codes of the code lengths ``lens``."""
    count = [0] * (MAX_BITS + 1)
    for l in lens:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * (MAX_BITS + 1), 0
    for bits in range(1, MAX_BITS + 1):
        code = (code + count[bits - 1]) << 1
        nxt[bits] = code
    out = []
    for l in lens:
        out.append(bi_reverse(nxt[l], l) if l else 0)
        if l:
            nxt[l] += 1
    return out


STATIC_LCODE = np.array(canonical_codes(list(STATIC_LLEN)), np.int64)
STATIC_DCODE = np.array([bi_reverse(n, 5) for n in range(D_CODES)], np.int64)


# ------------------------------------------------------------------------------------------------ filter and parse
def filtered(img):
    """The filtered rows libpng deflates: per row the filter type byte, then the row in PNG channel order (RGB from BGR)."""
    img = np.asarray(img, np.uint8)
    if img.ndim == 3:
        img = img[:, :, ::-1]
    h, w = img.shape[:2]
    rows = img.reshape(h, -1).astype(np.int64)
    c = rows.shape[1] // w
    if w > 1:
        rows = rows.copy()
        rows[:, c:] = (rows[:, c:] - rows[:, :-c]) & 0xFF
    out = np.empty((h, rows.shape[1] + 1), np.uint8)
    out[:, 0] = 1 if w > 1 else 0
    out[:, 1:] = rows
    return out.reshape(-1)


def parse(data):
    """deflate_rle's symbols of ``data``: (pos, length, value) per symbol, in order. A literal has length 1 and its byte as
    value; a match (distance 1) has its length (3..258) and the value of the byte it repeats."""
    data = np.asarray(data, np.uint8)
    n = data.size
    starts = np.flatnonzero(np.r_[True, data[1:] != data[:-1]])
    L = np.r_[starts[1:], n] - starts
    nfull, r = (L - 1) // MAX_MATCH, (L - 1) % MAX_MATCH
    ntail = np.where(r >= 3, 1, r)
    nsym = 1 + nfull + ntail
    run = np.repeat(np.arange(starts.size), nsym)
    q = np.arange(run.size) - np.repeat(np.cumsum(nsym) - nsym, nsym)        # symbol index within its run
    s, nf, rr = starts[run], nfull[run], r[run]
    tail = q - nf - 1
    pos = np.where(q == 0, s, np.where(q <= nf, s + 1 + MAX_MATCH * (q - 1), s + 1 + MAX_MATCH * nf + np.maximum(tail, 0)))
    length = np.where(q == 0, 1, np.where(q <= nf, MAX_MATCH, np.where(rr >= 3, rr, 1)))
    return pos.astype(np.int64), length.astype(np.int64), data[pos].astype(np.int64)


# ------------------------------------------------------------------------------------------------ trees.c
class Tree:
    """One build_tree result: code lengths and codes of the leaves 0..elems-1, max_code, and what build_tree added to
    opt_len and static_len."""

    def __init__(self, lens, codes, max_code, opt_len, static_len):
        self.lens, self.codes, self.max_code, self.opt_len, self.static_len = lens, codes, max_code, opt_len, static_len


def build_tree(freq_in, stree_len, extra, base, max_length):
    elems = len(freq_in)
    freq = [int(f) for f in freq_in] + [0] * (HEAP_SIZE - elems)
    length, dad, depth = [0] * HEAP_SIZE, [0] * HEAP_SIZE, [0] * HEAP_SIZE
    heap = [0] * (HEAP_SIZE + 1)
    heap_len, heap_max, max_code = 0, HEAP_SIZE, -1
    opt_len = static_len = 0
    for n in range(elems):
        if freq[n]:
            heap_len += 1
            heap[heap_len] = max_code = n
            depth[n] = 0
        else:
            length[n] = 0
    while heap_len < 2:                          # at least two codes: force 0 / 1 / 2 in
        node = 0
        if max_code < 2:
            max_code += 1
            node = max_code
        heap_len += 1
        heap[heap_len] = node
        freq[node] = 1
        depth[node] = 0
        opt_len -= 1
        if stree_len is not None:
            static_len -= int(stree_len[node])

    def smaller(a, b):
        return freq[a] < freq[b] or (freq[a] == freq[b] and depth[a] <= depth[b])

    def downheap(k):
        v, j = heap[k], k << 1
        while j <= heap_len:
            if j < heap_len and smaller(heap[j + 1], heap[j]):
                j += 1
            if smaller(v, heap[j]):
                break
            heap[k] = heap[j]
            k, j = j, j << 1
        heap[k] = v

    for k in range(heap_len // 2, 0, -1):
        downheap(k)
    node = elems
    while True:
        n = heap[1]                              # pqremove
        heap[1] = heap[heap_len]
        heap_len -= 1
        downheap(1)
        m = heap[1]
        heap_max -= 1
        heap[heap_max] = n
        heap_max -= 1
        heap[heap_max] = m
        freq[node] = freq[n] + freq[m]
        depth[node] = max(depth[n], depth[m]) + 1
        dad[n] = dad[m] = node
        heap[1] = node
        node += 1
        downheap(1)
        if heap_len < 2:
            break
    heap_max -= 1
    heap[heap_max] = heap[1]

    # gen_bitlen
    bl_count = [0] * (max(MAX_BITS, max_length) + 1)
    length[heap[heap_max]] = 0
    overflow = 0
    for h in range(heap_max + 1, HEAP_SIZE):
        n = heap[h]
        bits = length[dad[n]] + 1
        if bits > max_length:
            bits, overflow = max_length, overflow + 1
        length[n] = bits
        if n > max_code:
            continue
        bl_count[bits] += 1
        xbits = extra[n - base] if n >= base else 0
        opt_len += freq[n] * (bits + xbits)
        if stree_len is not None:
            static_len += freq[n] * (int(stree_len[n]) + xbits)
    if overflow:
        while True:
            bits = max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[max_length] -= 1
            overflow -= 2
            if overflow <= 0:
                break
        h = HEAP_SIZE
        for bits in range(max_length, 0, -1):
            n = bl_count[bits]
            while n:
                h -= 1
                m = heap[h]
                if m > max_code:
                    continue
                if length[m] != bits:
                    opt_len += (bits - length[m]) * freq[m]
                    length[m] = bits
                n -= 1
    lens = length[:elems]
    # gen_codes, from bl_count as gen_bitlen left it
    nxt, code = [0] * len(bl_count), 0
    for bits in range(1, len(bl_count)):
        code = (code + bl_count[bits - 1]) << 1
        nxt[bits] = code
    codes = [0] * elems
    for n in range(max_code + 1):
        if lens[n]:
            codes[n] = bi_reverse(nxt[lens[n]], lens[n])
            nxt[lens[n]] += 1
    return Tree(lens, codes, max_code, opt_len, static_len)


def tree_runs(lens, max_code):
    """scan_tree / send_tree: the bit-length symbols (sym, extra value, extra bits) that describe lens[0..max_code]."""
    out = []
    prevlen, nextlen, count = -1, lens[0], 0
    max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
    for n in range(max_code + 1):
        curlen = nextlen
        nextlen = lens[n + 1] if n + 1 <= max_code else 0xFFFF     # the guard
        count += 1
        if count < max_count and curlen == nextlen:
            continue
        if count < min_count:
            out += [(curlen, 0, 0)] * count
        elif curlen != 0:
            if curlen != prevlen:
                out.append((curlen, 0, 0))
                count -= 1
            out.append((16, count - 3, 2))
        elif count <= 10:
            out.append((17, count - 3, 3))
        else:
            out.append((18, count - 11, 7))
        count, prevlen = 0, curlen
        if nextlen == 0:
            max_count, min_count = 138, 3
        elif curlen == nextlen:
            max_count, min_count = 6, 3
        else:
            max_count, min_count = 7, 4
    return out


class Block:
    """One deflate block: its type, its literal/length and distance codes, and for a dynamic block the header's bit
    fields (value, bits) after the 3 type bits."""

    def __init__(self, kind, lcode, llen, dcode, dlen, header):
        self.kind, self.lcode, self.llen, self.dcode, self.dlen, self.header = kind, lcode, llen, dcode, dlen, header


def block_trees(lfreq, nmatch, stored_len):
    """_tr_flush_block's trees and choice for a block with literal/length counts ``lfreq`` (END_BLOCK included), ``nmatch``
    matches (all distance code 0) and ``stored_len`` input bytes."""
    dfreq = [nmatch] + [0] * (D_CODES - 1)
    lt = build_tree(lfreq, STATIC_LLEN, EXTRA_LBITS, 257, MAX_BITS)
    dt = build_tree(dfreq, STATIC_DLEN, EXTRA_DBITS, 0, MAX_BITS)
    lruns, druns = tree_runs(lt.lens, lt.max_code), tree_runs(dt.lens, dt.max_code)
    blfreq = [0] * BL_CODES
    for sym, _, _ in lruns + druns:
        blfreq[sym] += 1
    bt = build_tree(blfreq, None, EXTRA_BLBITS, 0, MAX_BL_BITS)
    max_blindex = BL_CODES - 1
    while max_blindex >= 3 and bt.lens[BL_ORDER[max_blindex]] == 0:
        max_blindex -= 1
    opt_len = lt.opt_len + dt.opt_len + bt.opt_len + 3 * (max_blindex + 1) + 5 + 5 + 4
    static_len = lt.static_len + dt.static_len
    opt_lenb, static_lenb = (opt_len + 3 + 7) >> 3, (static_len + 3 + 7) >> 3
    if static_lenb <= opt_lenb:
        opt_lenb = static_lenb
    if stored_len + 4 <= opt_lenb:
        assert stored_len <= STORED_MAX, "a stored block past zlib's window (buf == NULL) is not restated"
        return Block(STORED, None, None, None, None, None)
    if static_lenb == opt_lenb:
        return Block(STATIC, STATIC_LCODE, STATIC_LLEN, STATIC_DCODE, STATIC_DLEN, None)
    header = [(lt.max_code + 1 - 257, 5), (dt.max_code + 1 - 1, 5), (max_blindex + 1 - 4, 4)]
    header += [(bt.lens[BL_ORDER[r]], 3) for r in range(max_blindex + 1)]
    for sym, val, nb in lruns + druns:
        header.append((bt.codes[sym], bt.lens[sym]))
        if nb:
            header.append((val, nb))
    return Block(DYNAMIC, np.array(lt.codes, np.int64), np.array(lt.lens, np.int64), np.array(dt.codes, np.int64),
                 np.array(dt.lens, np.int64), header)


# ------------------------------------------------------------------------------------------------ bit stream
class BitWriter:
    """An LSB-first bit stream (send_bits), kept as a list of (value, bits) runs and byte-aligned raw byte strings."""

    def __init__(self):
        self.parts, self.vals, self.nbits, self.bits = [], [], [], 0

    def put(self, vals, nbits):
        vals, nbits = np.atleast_1d(np.asarray(vals, np.int64)), np.atleast_1d(np.asarray(nbits, np.int64))
        self.vals.append(vals)
        self.nbits.append(nbits)
        self.bits += int(nbits.sum())

    def _flush_bits(self, pad):
        if not self.vals:
            return
        vals, nbits = np.concatenate(self.vals), np.concatenate(self.nbits)
        self.vals, self.nbits = [], []
        keep = nbits > 0
        vals, nbits = vals[keep], nbits[keep]
        idx = np.repeat(np.arange(vals.size), nbits)
        shift = np.arange(idx.size) - np.repeat(np.cumsum(nbits) - nbits, nbits)
        bitarr = ((vals[idx] >> shift) & 1).astype(np.uint8)
        bitarr = np.r_[bitarr, np.zeros(pad, np.uint8)]
        self.parts.append(np.packbits(bitarr, bitorder="little"))

    def align(self):
        """bi_windup: pad with zero bits to a byte boundary."""
        pad = -self.bits % 8
        self.bits += pad
        pending = sum(int(n.sum()) for n in self.nbits)
        self._flush_bits(-pending % 8)

    def raw(self, data):
        assert self.bits % 8 == 0
        self.parts.append(np.asarray(data, np.uint8))
        self.bits += 8 * len(data)

    def getvalue(self):
        self.align()
        return b"".join(p.tobytes() for p in self.parts)


def block_ranges(nsym):
    """[first, last) symbol index of each block: every BLOCK_SYMS symbols, then the rest (empty on an exact multiple)."""
    nfull = nsym // BLOCK_SYMS
    return [(b * BLOCK_SYMS, (b + 1) * BLOCK_SYMS) for b in range(nfull)] + [(nfull * BLOCK_SYMS, nsym)]


def block_input(data, pos, length, lo, hi):
    """Histograms and stored length of symbols lo..hi: (lfreq with END_BLOCK, matches, stored_len, lit/len codes, lc)."""
    ln = length[lo:hi]
    match = ln >= 3
    sym = np.where(match, 257 + LENGTH_CODE[np.clip(ln - 3, 0, 255)], np.asarray(data, np.int64)[pos[lo:hi]])
    lfreq = np.bincount(sym, minlength=L_CODES)
    lfreq[END_BLOCK] += 1
    return lfreq, int(match.sum()), int(ln.sum()), sym, match, ln


def blocks(data):
    """Per deflate block of ``data``: (Block, lo, hi, stored_len, sym, match, ln) with the symbol range [lo, hi), the
    block's input bytes and its symbols' literal/length codes, match flags and lengths."""
    data = np.asarray(data, np.uint8)
    pos, length, _ = parse(data)
    for lo, hi in block_ranges(pos.size):
        lfreq, nmatch, stored_len, sym, match, ln = block_input(data, pos, length, lo, hi)
        yield block_trees(lfreq, nmatch, stored_len), lo, hi, int(pos[lo]) if hi > lo else data.size, stored_len, sym, match, ln


def deflate(data):
    """The raw deflate stream zlib's deflate_rle writes for ``data`` (no zlib header or trailer)."""
    data = np.asarray(data, np.uint8)
    bw = BitWriter()
    allb = list(blocks(data))
    for k, (blk, lo, hi, start, stored_len, sym, match, ln) in enumerate(allb):
        last = int(k == len(allb) - 1)
        bw.put((blk.kind << 1) + last, 3)
        if blk.kind == STORED:
            bw.align()
            bw.raw(np.frombuffer(struct.pack("<HH", stored_len, stored_len ^ 0xFFFF), np.uint8))
            bw.raw(data[start:start + stored_len])
            continue
        if blk.kind == DYNAMIC:
            bw.put([v for v, _ in blk.header], [n for _, n in blk.header])
        code = blk.lcode[sym]
        nb = blk.llen[sym]
        lcode = np.clip(sym - 257, 0, 28)
        xb = np.where(match, np.array(EXTRA_LBITS, np.int64)[lcode], 0)
        xv = np.where(match, (ln - 3) - BASE_LENGTH[lcode], 0)
        dc, dl = np.where(match, blk.dcode[0], 0), np.where(match, blk.dlen[0], 0)
        vals = np.stack([code, xv, dc], 1).reshape(-1)
        bits = np.stack([nb, xb, dl], 1).reshape(-1)
        bw.put(vals, bits)
        bw.put(blk.lcode[END_BLOCK], blk.llen[END_BLOCK])
    return bw.getvalue()


def zlib_header(data_size):
    """CMF, FLG as libpng leaves them: zlib writes 0x78 0x01 (level 1 with Z_RLE: FLEVEL 0), then libpng lowers CINFO to the
    smallest window that covers data_size bytes when that is at most 16384, and recomputes FCHECK."""
    cinfo, half = 7, 1 << 14
    if data_size <= half:
        while True:
            half >>= 1
            cinfo -= 1
            if not (cinfo > 0 and data_size <= half):
                break
    cmf = (cinfo << 4) | 8
    flg = 0x1F - ((cmf << 8) % 0x1F)
    return bytes([cmf, flg])


def zlib_stream(data):
    data = np.asarray(data, np.uint8)
    return zlib_header(data.size) + deflate(data) + struct.pack(">I", zlib.adler32(data.tobytes()))


def chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def png(img):
    """The bytes of ``cv2.imencode(".png", img)[1]`` for a uint8 [h, w, 3] BGR or [h, w] image."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[:2]
    z = zlib_stream(filtered(img))
    out = [b"\x89PNG\r\n\x1a\n", chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2 if img.ndim == 3 else 0, 0, 0, 0))]
    out += [chunk(b"IDAT", z[o:o + IDAT_CHUNK]) for o in range(0, len(z), IDAT_CHUNK)]
    out.append(chunk(b"IEND", b""))
    return b"".join(out)


def max_bytes(h, w, channels):
    """se_png_max_bytes: a true upper bound of the file of an h x w image."""
    n = h * (1 + w * channels)
    deflate_max = n + 8 * (n // BLOCK_SYMS + 2) + 8
    z = 2 + deflate_max + 4
    return 8 + 25 + z + 12 * ((z + IDAT_CHUNK - 1) // IDAT_CHUNK) + 12

"""libjpeg-turbo's two-pass JPEG encode with optimal Huffman tables, restated in integer numpy: what ``PIL.Image.save(buf,
"JPEG", quality=q, subsampling=s, optimize=True)`` writes for an RGB image without ``info``, s = 0 or 2. It is the spec of
se_jpeg_encode_opt_u8 with optimize = 1; tests pin it to Pillow. The coefficients are tests/util_jpeg.py's, unchanged.

  * Statistics: one histogram per table (DC luma, AC luma, DC chroma, AC chroma; Cb and Cr share the chroma tables) of the
    symbols the baseline coder emits for the image: DC difference categories, AC run/size symbols, ZRL (0xF0) and EOB (0x00).
    A dummy luma block of a 4:2:0 MCU counts as DC difference 0 and EOB, as it is coded.
  * Table (ITU T.81 Annex K.2, with the tie rule libjpeg uses): a reserved symbol 256 of count 1 joins the symbols of nonzero
    count; each step merges the least frequent entry c1 and the next least frequent c2, where among equal counts the higher
    symbol number is taken first, and a count above 10^9 is never chosen; every symbol of the two merged trees gets one bit
    longer. Code lengths over 16 are limited by Annex K.3's procedure, then one code of the longest length, the reserved
    one, is dropped. The symbols are listed by their unlimited code length, then by value, and take the limited lengths in
    that order; codes are canonical (Annex C).
  * The header is the baseline one with these four tables in its DHT segments, so its length depends on the image.
"""
import numpy as np

from tests import util_jpeg as J

MAX_CANDIDATE = 1000000000   # a count above this is never picked for a merge (libjpeg's starting minimum)


def symbols(coef, per_mcu):
    """Every Huffman symbol of the scan in coding order: arrays (table, symbol, value bits, value length), table 0 DC luma,
    1 DC chroma, 2 AC luma, 3 AC chroma; the value bits are the low ``length`` bits of the coefficient (negative: minus 1)."""
    nb = coef.shape[0]
    comp = np.arange(nb) % per_mcu
    chroma = (comp >= per_mcu - 2).astype(np.int64)
    cid = np.where(chroma == 1, 1 + (comp - (per_mcu - 2)), 0)
    dc = coef[:, 0].astype(np.int64)
    prev = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(cid == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    diff = dc - prev
    parts = []

    def add(block, key, table, sym, val, nval):
        parts.append((block, key, table, sym, np.where(val < 0, val - 1, val) & ((1 << nval) - 1), nval))

    n = J._nbits(diff)
    add(np.arange(nb), np.zeros(nb, np.int64), chroma, n, diff, n)
    b, k = np.nonzero(coef[:, 1:])
    k = k + 1
    v = coef[b, k].astype(np.int64)
    first = np.r_[True, b[1:] != b[:-1]]
    run = k - np.where(first, 1, np.r_[0, k[:-1]] + 1)
    zrl = run // 16
    n = J._nbits(v)
    add(b, k * 8 + 7, 2 + chroma[b], (run % 16) * 16 + n, v, n)
    zb = np.repeat(b, zrl)
    zk = np.repeat(k * 8, zrl) + (np.arange(zb.size) - np.repeat(np.cumsum(zrl) - zrl, zrl))
    z = np.zeros(zb.size, np.int64)
    add(zb, zk, 2 + chroma[zb], z + 0xF0, z, z)
    last = np.zeros(nb, np.int64)
    np.maximum.at(last, b, k)
    eb = np.nonzero(last < 63)[0]
    z = np.zeros(eb.size, np.int64)
    add(eb, z + 64 * 8, 2 + chroma[eb], z, z, z)
    blk, key, table, sym, val, nval = (np.concatenate([p[i] for p in parts]) for i in range(6))
    order = np.lexsort((key, blk))
    return table[order], sym[order], val[order], nval[order]


def histograms(coef, per_mcu):
    """[4, 256] int64 symbol counts per table (0 DC luma, 1 DC chroma, 2 AC luma, 3 AC chroma)."""
    table, sym, _, _ = symbols(coef, per_mcu)
    return np.bincount(table * 256 + sym, minlength=4 * 256).reshape(4, 256)


def code_lengths(freq):
    """The unlimited code length of each of the 257 symbols (0: unused), symbol 256 the reserved one: Annex K.2's merges."""
    freq = [int(f) for f in freq[:256]] + [1]
    size = [0] * 257
    root = list(range(257))                       # the tree each symbol is in, named by the entry holding its count
    while True:
        cand = [i for i in range(257) if freq[i] and freq[i] <= MAX_CANDIDATE]
        if len(cand) < 2:
            break
        c1 = min(cand, key=lambda i: (freq[i], -i))
        c2 = min((i for i in cand if i != c1), key=lambda i: (freq[i], -i))
        freq[c1] += freq[c2]
        freq[c2] = 0
        for j in range(257):
            if root[j] in (c1, c2):
                size[j] += 1
                root[j] = c1
    return size


def limit_lengths(size):
    """Annex K.3: the count of codes per length 1..16 after limiting, with the reserved code removed."""
    bits = [0] * (max(max(size), 16) + 1)
    for s in size:
        if s:
            bits[s] += 1
    for i in range(len(bits) - 1, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    return bits[1:17]


def optimal_table(freq):
    """(counts per length 1..16, symbols) of the optimal table of one histogram of 256 counts."""
    size = code_lengths(freq)
    order = sorted((s, j) for j, s in enumerate(size[:256]) if s)
    return limit_lengths(size), bytes(j for _, j in order)


def tables(coef, per_mcu):
    """The four optimal tables, in histogram order (DC luma, DC chroma, AC luma, AC chroma)."""
    return [optimal_table(h) for h in histograms(coef, per_mcu)]


def header(h, w, quality, subsampling, tabs):
    """The baseline header with the DHT segments of ``tabs`` (DC luma, DC chroma, AC luma, AC chroma)."""
    base = J.header(h, w, quality, subsampling)
    sof_end, sos_at = 177, J.HEADER_BYTES - 14
    dht = b""
    for cls_id, t in ((0x00, 0), (0x10, 2), (0x01, 1), (0x11, 3)):
        counts, syms = tabs[t]
        dht += bytes([0xFF, 0xC4]) + (3 + 16 + len(syms)).to_bytes(2, "big") + bytes([cls_id]) + bytes(counts) + syms
    return base[:sof_end] + dht + base[sos_at:]


def entropy(coef, per_mcu, tabs):
    """The entropy-coded segment (stuffed and padded) of the coefficients coded with ``tabs``."""
    table, sym, val, nval = symbols(coef, per_mcu)
    code, size = np.zeros((4, 256), np.int64), np.zeros((4, 256), np.int64)
    for t, tab in enumerate(tabs):
        for s, (c, n) in J.huff_codes(tab).items():
            code[t, s], size[t, s] = c, n
    assert (size[table, sym] > 0).all()
    length = size[table, sym] + nval
    word = (code[table, sym] << nval) | val
    start = np.cumsum(length) - length
    total = int(length.sum())
    pos = np.arange(total) - np.repeat(start, length)
    bits = (np.repeat(word, length) >> (np.repeat(length, length) - 1 - pos)) & 1
    bits = np.concatenate([bits, np.ones(-total % 8, np.int64)]).astype(np.uint8)
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def encode(rgb, quality=75, subsampling=2):
    """The bytes Pillow writes for Image.fromarray(rgb).save(buf, "JPEG", quality=quality, subsampling=subsampling,
    optimize=True)."""
    rgb = np.asarray(rgb, np.uint8)
    h, w = rgb.shape[:2]
    coef, per_mcu = J.coefficients(rgb, quality, subsampling)
    tabs = tables(coef, per_mcu)
    return header(h, w, quality, subsampling, tabs) + entropy(coef, per_mcu, tabs) + b"\xff\xd9"

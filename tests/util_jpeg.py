"""libjpeg-turbo's baseline JPEG encoder, restated in integer numpy: what ``PIL.Image.save(buf, "JPEG", quality=q,
subsampling=s)`` writes for an RGB image without ``info``, with s = 0 (4:4:4) or 2 (4:2:0). It is the spec se_jpeg.cu follows,
and its stages (``planes``, ``coefficients``, ``entropy``) split a failing GPU case by stage. Tests pin it to Pillow.

Stages, as libjpeg-turbo runs them with Pillow's defaults (islow DCT, no smoothing, standard Huffman tables):
  * RGB -> YCbCr in 16-bit fixed point (jccolor.c);
  * 4:2:0: columns repeated to the MCU width (16) and rows to an even count, 2x2 averaged with the bias 1, 2, 1, 2, ... along
    each output row (jcsample.c h2v2_downsample), then the chroma rows repeated to a multiple of 8; luma and 4:4:4 planes repeat
    their last column and row up to the block grid (jcprepct.c);
  * a luma block of a 4:2:0 MCU that lies wholly outside the image is a dummy block: no AC, the DC of the block before it in the
    MCU (jccoefct.c), so its DC difference is 0;
  * level shift, islow FDCT (jfdctint.c, output scaled by 8), quantisation by 8 q with libjpeg-turbo's reciprocal, correction
    and shift (jcdctmgr.c compute_reciprocal / quantize);
  * Huffman coding with the Annex K tables in zigzag order, 0x00 after every 0xFF, the last byte padded with 1-bits.
"""
import numpy as np

# Annex K.1 quantisation bases (natural order)
LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100,
    103, 99], np.int64)
CHROMA_Q = np.full(64, 99, np.int64)
CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# Annex K.3 Huffman tables: code counts per length 1..16, then the symbols
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a434445464748"
    "494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3"
    "c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"))
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a43444546"
    "4748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8"
    "b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"))


def _zigzag():
    order = sorted(((y, x) for y in range(8) for x in range(8)), key=lambda p: (p[0] + p[1], p[0] if (p[0] + p[1]) % 2 else p[1]))
    return np.array([y * 8 + x for y, x in order])


ZIGZAG = _zigzag()                    # ZIGZAG[k] = natural index of zigzag position k
MAX_BLOCK_BITS = 64 * 26              # DC: <= 11-bit code + 11 bits; AC: <= 16-bit code + 10 bits each
HEADER_BYTES = 623


def quant_table(quality, base):
    """jpeg_quality_scaling + jpeg_add_quant_table with force_baseline (natural order)."""
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * scale + 50) // 100, 1, 255)


def huff_codes(table):
    """symbol -> (code, length) of a canonical table (Annex C)."""
    counts, symbols = table
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            codes[symbols[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def _lut(table):
    codes = huff_codes(table)
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    for s, (c, n) in codes.items():
        code[s], size[s] = c, n
    return code, size


def max_bytes(h, w, subsampling):
    """A true worst case of the file size: the header, MAX_BLOCK_BITS per block doubled for stuffing, and EOI."""
    m = 16 if subsampling == 2 else 8
    blocks = -(-h // m) * -(-w // m) * (6 if subsampling == 2 else 3)
    return HEADER_BYTES + 2 * (blocks * MAX_BLOCK_BITS // 8) + 2


def header(h, w, quality, subsampling):
    """SOI, JFIF APP0 1.01 (density 1:1, units 0), DQT 0 and 1, SOF0, DHT DC0 AC0 DC1 AC1, SOS: HEADER_BYTES bytes."""
    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body

    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t, base in enumerate((LUMA_Q, CHROMA_Q)):
        out += seg(0xDB, bytes([t]) + bytes(quant_table(quality, base)[ZIGZAG].astype(np.uint8)))
    y = 0x22 if subsampling == 2 else 0x11
    out += seg(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3, 1, y, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls_id, table in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        out += seg(0xC4, bytes([cls_id]) + bytes(table[0]) + bytes(table[1]))
    out += seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    assert len(out) == HEADER_BYTES
    return out


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc(rgb):
    """jccolor.c rgb_ycc_convert: three int64 planes."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def _pad(p, rows, cols):
    return np.pad(p, ((0, rows - p.shape[0]), (0, cols - p.shape[1])), mode="edge")


def planes(rgb, subsampling):
    """The sample planes the DCT reads, each a multiple of 8 in both directions, and the MCU grid (rows, cols)."""
    h, w = rgb.shape[:2]
    y, cb, cr = ycc(rgb)
    if subsampling == 0:
        my, mx = -(-h // 8), -(-w // 8)
        return [_pad(p, 8 * my, 8 * mx) for p in (y, cb, cr)], (my, mx)
    my, mx = -(-h // 16), -(-w // 16)
    out = [_pad(y, 16 * my, 16 * mx)]         # luma blocks past the image are dummies; their samples are never used
    bias = np.tile([1, 2], 4 * mx)
    for p in (cb, cr):
        p = _pad(p, 2 * -(-h // 2), 16 * mx)
        d = (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias) >> 2
        out.append(_pad(d, 8 * my, 8 * mx))
    return out, (my, mx)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, axis, first):
    """One pass of jfdctint.c over axis 1 (rows) or 2 (columns) of [N, 8, 8] int64."""
    d = np.moveaxis(d, axis, -1)
    c, p = 13, 2
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o = np.empty_like(d)
    sh = c - p if first else c + p
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << p, (t10 - t11) << p
    else:
        o[..., 0], o[..., 4] = _descale(t10 + t11, p), _descale(t10 - t11, p)
    z1 = (t12 + t13) * 4433
    o[..., 2] = _descale(z1 + t13 * 6270, sh)
    o[..., 6] = _descale(z1 - t12 * 15137, sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * 9633
    t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    o[..., 7] = _descale(t4 + z1 + z3, sh)
    o[..., 5] = _descale(t5 + z2 + z4, sh)
    o[..., 3] = _descale(t6 + z2 + z3, sh)
    o[..., 1] = _descale(t7 + z1 + z4, sh)
    return np.moveaxis(o, -1, axis)


def fdct(blocks):
    """islow FDCT of level-shifted [N, 8, 8] samples: rows, then columns."""
    return _fdct_1d(_fdct_1d(blocks, 2, True), 1, False)


def reciprocal(divisor):
    """jcdctmgr.c compute_reciprocal for 16-bit DCTELEM: (recip, corr, shift) with q = ((|x| + corr) * recip) >> shift."""
    b = int(divisor).bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, int(divisor))
    c = divisor // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= divisor // 2:
        c += 1
    else:
        fq += 1
    return fq, c, r


def quantize(coef, qtable):
    recip, corr, shift = (np.array(v, np.int64).reshape(8, 8) for v in zip(*[reciprocal(8 * int(q)) for q in qtable.ravel()]))
    a = np.abs(coef)
    return np.sign(coef) * (((a + corr) * recip) >> shift)


def _blocks(p):
    """[rows/8 * cols/8, 8, 8] blocks of a plane, row-major."""
    r, c = p.shape[0] // 8, p.shape[1] // 8
    return p.reshape(r, 8, c, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


def coefficients(rgb, quality=75, subsampling=2):
    """Quantised coefficients in zigzag order, [blocks, 64] in scan order (MCU by MCU: the luma blocks row-major, Cb, Cr), and
    the number of blocks per MCU."""
    h, w = rgb.shape[:2]
    pl, (my, mx) = planes(rgb, subsampling)
    qs = [quant_table(quality, LUMA_Q), quant_table(quality, CHROMA_Q), quant_table(quality, CHROMA_Q)]
    q = [quantize(fdct(_blocks(p) - 128), t.reshape(8, 8)).reshape(-1, 64)[:, ZIGZAG] for p, t in zip(pl, qs)]
    if subsampling == 0:
        return np.stack(q, 1).reshape(-1, 64), 3
    y = q[0].reshape(my, 2, mx, 2, 64).transpose(0, 2, 1, 3, 4).reshape(my * mx, 4, 64)
    ys, xs = np.meshgrid(np.arange(my * 2), np.arange(mx * 2), indexing="ij")
    dummy = ((ys >= -(-h // 8)) | (xs >= -(-w // 8))).reshape(my, 2, mx, 2).transpose(0, 2, 1, 3).reshape(my * mx, 4)
    y[dummy] = 0
    for k in range(1, 4):                      # a dummy takes the DC of the block before it (block 0 is never a dummy)
        y[:, k, 0] = np.where(dummy[:, k], y[:, k - 1, 0], y[:, k, 0])
    return np.concatenate([y, q[1][:, None], q[2][:, None]], 1).reshape(-1, 64), 6


def _nbits(v):
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while (a >> n).any():
        n += (a >> n) > 0
    return n


def entropy(coef, per_mcu):
    """The entropy-coded segment (stuffed and padded) of [blocks, 64] zigzag coefficients in scan order."""
    nb = coef.shape[0]
    comp = np.arange(nb) % per_mcu
    chroma = comp >= per_mcu - 2
    cid = np.where(chroma, 1 + (comp - (per_mcu - 2)), 0)
    dc = coef[:, 0]
    prev = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(cid == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    diff = dc - prev
    luts = {(False, False): _lut(DC_LUMA), (True, False): _lut(DC_CHROMA), (False, True): _lut(AC_LUMA),
            (True, True): _lut(AC_CHROMA)}

    def items(block, key, sym, val, nval, is_chroma, ac):
        lc, ls = (np.where(is_chroma, luts[(True, ac)][i][sym], luts[(False, ac)][i][sym]) for i in (0, 1))
        v = val & ((1 << nval) - 1)
        return block, key, (lc << nval) | v, ls + nval

    parts = []
    n = _nbits(diff)
    parts.append(items(np.arange(nb), np.zeros(nb, np.int64), n, np.where(diff < 0, diff - 1, diff), n, chroma, False))
    b, k = np.nonzero(coef[:, 1:])
    k = k + 1
    v = coef[b, k]
    first = np.r_[True, b[1:] != b[:-1]]
    run = k - np.where(first, 1, np.r_[0, k[:-1]] + 1)
    zrl = run // 16
    n = _nbits(v)
    parts.append(items(b, k * 8 + 7, (run % 16) * 16 + n, np.where(v < 0, v - 1, v), n, chroma[b], True))
    zb = np.repeat(b, zrl)
    zk = np.repeat(k * 8, zrl) + (np.arange(zb.size) - np.repeat(np.cumsum(zrl) - zrl, zrl))
    parts.append(items(zb, zk, np.full(zb.size, 0xF0), np.zeros(zb.size, np.int64), np.zeros(zb.size, np.int64), chroma[zb], True))
    last = np.zeros(nb, np.int64)
    np.maximum.at(last, b, k)
    eb = np.nonzero(last < 63)[0]
    parts.append(items(eb, np.full(eb.size, 64 * 8), np.zeros(eb.size, np.int64), np.zeros(eb.size, np.int64),
                       np.zeros(eb.size, np.int64), chroma[eb], True))
    blk, key, code, length = (np.concatenate([p[i] for p in parts]) for i in range(4))
    order = np.lexsort((key, blk))
    code, length = code[order], length[order]
    start = np.cumsum(length) - length
    total = int(length.sum())
    pos = np.arange(total) - np.repeat(start, length)
    bits = (np.repeat(code, length) >> (np.repeat(length, length) - 1 - pos)) & 1
    bits = np.concatenate([bits, np.ones(-total % 8, np.int64)]).astype(np.uint8)
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def encode(rgb, quality=75, subsampling=2):
    """The bytes Pillow writes for Image.fromarray(rgb).save(buf, "JPEG", quality=quality, subsampling=subsampling)."""
    rgb = np.asarray(rgb, np.uint8)
    h, w = rgb.shape[:2]
    coef, per_mcu = coefficients(rgb, quality, subsampling)
    return header(h, w, quality, subsampling) + entropy(coef, per_mcu) + b"\xff\xd9"

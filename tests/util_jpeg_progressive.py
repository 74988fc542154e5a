"""libjpeg-turbo's progressive JPEG encode (jcphuff.c), restated in integer numpy: what ``PIL.Image.save(buf, "JPEG",
quality=q, subsampling=s, progressive=True)`` writes for an RGB image without ``info``, s = 0 or 2. It is the spec of
se_jpeg_encode_progressive_u8; tests pin it to Pillow. The coefficients are tests/util_jpeg.py's and the tables are built as
tests/util_jpeg_optimize.py builds them (libjpeg-turbo forces optimal tables in progressive mode), one set per scan.

  * The scan script is jpeg_simple_progression's for YCbCr (SCANS). The interleaved DC scans cover every block of every MCU,
    dummy luma blocks of 4:2:0 included (their DC is the block before them in the MCU, as in the baseline coder); every other
    scan covers one component's blocks, ceil(w_c / 8) x ceil(h_c / 8) in raster order, without dummies.
  * Point transform: DC first codes the difference of DC >> Al; DC refinement emits bit Al of the DC; AC first codes
    |v| >> Al (the value bits of a negative coefficient are those of ~(|v| >> Al)); AC refinement codes the coefficients whose
    |v| >> Al is 1 (newly nonzero: run/1 symbol and a sign bit, 1 for positive) and emits bit 0 of |v| >> Al for those
    already nonzero (correction bits).
  * EOB runs: a block of an AC scan ends in a run ("T") when anything follows its last coded symbol. The run counter is
    emitted as symbol (n << 4) with n = bitlength - 1 extra bits before the next coded symbol of a later block, when it
    reaches 0x7FFF, and at the end of the scan. In refinement scans the correction bits that follow a block's last coded
    symbol wait in a buffer and go out after the emitted run; a run is also emitted once the buffer holds more than
    MAX_CORR_BITS - 64 + 1 bits. Inside a block, pending correction bits go out after each ZRL or run/1 symbol, and ZRLs are
    only emitted up to the last newly nonzero coefficient (later zero runs fold into the EOB run).
  * Each scan's data is padded with 1-bits to a byte and stuffed; before it come DHT segments for the tables it uses, built
    from that scan's own counts, and its SOS. The frame is SOF2.
"""
import numpy as np

from tests import util_jpeg as J
from tests import util_jpeg_optimize as O

# (component: None for Y, Cb, Cr interleaved, else 0 Y, 1 Cb, 2 Cr), Ss, Se, Ah, Al
SCANS = [(None, 0, 0, 0, 1), (0, 1, 5, 0, 2), (2, 1, 63, 0, 1), (1, 1, 63, 0, 1), (0, 6, 63, 0, 2),
         (0, 1, 63, 2, 1), (None, 0, 0, 1, 0), (2, 1, 63, 1, 0), (1, 1, 63, 1, 0), (0, 1, 63, 1, 0)]
MAX_RUN = 0x7FFF
CORR_LIMIT = 1000 - 64 + 1   # MAX_CORR_BITS - DCTSIZE2 + 1: a run is emitted once more bits than this wait
SOF_END = 177


def component_blocks(coef, per_mcu, h, w, c):
    """[n, 64] zigzag coefficients of component c's own blocks in raster order."""
    if per_mcu == 3:
        return coef[c::3]
    if c:
        return coef[3 + c::6]
    my, mx = -(-h // 16), -(-w // 16)
    y = coef.reshape(my * mx, 6, 64)[:, :4].reshape(my, mx, 2, 2, 64).transpose(0, 2, 1, 3, 4).reshape(2 * my, 2 * mx, 64)
    return y[:-(-h // 8), :-(-w // 8)].reshape(-1, 64)


class Items:
    """Everything a scan emits: per item its block, sort keys within the block, table (-1: raw bits), symbol, bits, length."""

    def __init__(self):
        self.parts = []

    def add(self, blk, key, sub, table, sym, val, nval):
        n = np.broadcast_shapes(np.shape(blk))[0]
        f = lambda x: np.broadcast_to(np.asarray(x, np.int64), (n,))
        nval = f(nval)
        self.parts.append((f(blk), f(key), f(sub), f(table), f(sym), f(val) & ((np.int64(1) << nval) - 1), nval))

    def ordered(self):
        cols = [np.concatenate([p[i] for p in self.parts]) if self.parts else np.zeros(0, np.int64) for i in range(7)]
        order = np.lexsort((cols[2], cols[1], cols[0]))
        return [c[order] for c in cols[3:]]


def _dc_first(coef, per_mcu, al, items):
    nb = coef.shape[0]
    comp = np.arange(nb) % per_mcu
    cid = np.where(comp >= per_mcu - 2, comp - (per_mcu - 3), 0)
    dc = coef[:, 0].astype(np.int64) >> al
    prev = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(cid == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    diff = dc - prev
    n = J._nbits(diff)
    items.add(np.arange(nb), 0, 0, (cid > 0).astype(np.int64), n, np.where(diff < 0, diff - 1, diff), n)


def _ac_first(x, ss, se, al, t, items):
    """The block-local symbols of an AC first scan; returns (N, T, trailing correction bits: none)."""
    nb = x.shape[0]
    v = x[:, ss:se + 1].astype(np.int64)
    a = np.abs(v) >> al
    b, kk = np.nonzero(a)
    k = kk + ss
    first = np.r_[True, b[1:] != b[:-1]]
    run = k - np.where(first, ss, np.r_[0, k[:-1]] + 1)
    zrl = run // 16
    n = J._nbits(a[b, kk])
    items.add(b, k * 16 + 8, 0, t, (run % 16) * 16 + n, np.where(v[b, kk] < 0, ~a[b, kk], a[b, kk]), n)
    zb = np.repeat(b, zrl)
    zj = np.arange(zb.size) - np.repeat(np.cumsum(zrl) - zrl, zrl)
    items.add(zb, np.repeat(k * 16, zrl) + 2 * zj, 0, t, 0xF0, 0, 0)
    has = np.zeros(nb, bool)
    has[b] = True
    last = np.full(nb, ss - 1)
    np.maximum.at(last, b, k)
    empty = np.zeros(0, np.int64)
    return has, last < se, (empty, empty, empty)


def _ac_refine(x, ss, se, al, t, items):
    """The block-local symbols of an AC refinement scan; returns (N, T, trailing correction bits as (block, k, bit))."""
    nb, L = x.shape[0], se - ss + 1
    v = x[:, ss:se + 1].astype(np.int64)
    a = np.abs(v) >> al
    newly = a == 1
    idx = np.arange(L)
    eob = np.where(newly, idx, -1).max(1)                          # band index of the last newly nonzero, -1: none
    zero = (a == 0).astype(np.int64)
    czero = np.cumsum(zero, 1)                                     # zeros up to and including each position
    lastnew = np.maximum.accumulate(np.where(newly, idx, -1), 1)
    lastnew = np.c_[np.full(nb, -1), lastnew[:, :-1]]              # the last newly nonzero strictly before
    base = np.where(lastnew >= 0, np.take_along_axis(czero, np.maximum(lastnew, 0), 1), 0)
    z = czero - zero - base                                        # zeros since the last run/1 symbol
    b, kk = np.nonzero(a)
    zk = z[b, kk]
    same = np.r_[False, b[1:] == b[:-1]]
    prev_corr = same & np.r_[False, ~newly[b, kk][:-1]]
    zprev = np.where(prev_corr, np.r_[0, zk[:-1]], 0)
    coded = kk <= eob[b]
    nzrl = np.where(coded, zk // 16 - zprev // 16, 0)
    isnew = newly[b, kk]
    k = kk + ss
    zb = np.repeat(b, nzrl)
    zj = np.arange(zb.size) - np.repeat(np.cumsum(nzrl) - nzrl, nzrl)
    items.add(zb, np.repeat(k * 16, nzrl) + 2 * zj, 0, t, 0xF0, 0, 0)
    nb_i = np.nonzero(isnew)[0]
    items.add(b[nb_i], k[nb_i] * 16 + 8, 0, t, (zk[nb_i] % 16) * 16 + 1, (v[b, kk][nb_i] > 0).astype(np.int64), 1)
    # a correction bit goes out after the first ZRL or run/1 symbol of a later coefficient of its block, else it trails
    flush = (nzrl > 0) | isnew
    m = b.size
    nxt = np.where(flush, np.arange(m), m)
    nxt = np.r_[np.minimum.accumulate(nxt[::-1])[::-1][1:], m] if m else nxt
    ci = np.nonzero(~isnew)[0]
    f = nxt[ci]
    held = (f < m)
    held[held] = b[f[held]] == b[ci[held]]
    fh, ch = f[held], ci[held]
    items.add(b[ch], k[fh] * 16 + np.where(nzrl[fh] > 0, 1, 9), k[ch], -1, -1, a[b[ch], kk[ch]] & 1, 1)
    tr = ci[~held]
    has = eob >= 0
    return has, eob < L - 1, (b[tr], k[tr], a[b[tr], kk[tr]] & 1)


def _runs(has, ends, corr, refine, t, items, stats):
    """Walks the EOB runs of a scan in block order and adds each emitted run (symbol, extra bits, waiting correction bits)
    to the block that emits it: before a block's first coded symbol (key -4) or after its last (key 2000)."""
    cb, ck, cbit = corr
    ncorr = np.bincount(cb, minlength=has.size) if cb.size else np.zeros(has.size, np.int64)

    def emit(j, key, count, start, end):
        n = int(count).bit_length() - 1
        items.add([j], key, 0, t, n << 4, count, n)
        lo, hi = np.searchsorted(cb, start), np.searchsorted(cb, end + 1)
        if hi > lo:
            items.add(np.full(hi - lo, j), key + 1, cb[lo:hi] * 64 + ck[lo:hi], -1, -1, cbit[lo:hi], 1)

    count = bits = 0
    start = 0
    for j in range(has.size):
        if has[j]:
            if count:
                emit(j, -4, count, start, j - 1)
            count = bits = 0
        if ends[j]:
            if count == 0:
                start = j
            count += 1
            bits += int(ncorr[j])
            if count == MAX_RUN or (refine and bits > CORR_LIMIT):
                stats["max_run" if count == MAX_RUN else "corr_limit"] += 1
                emit(j, 2000, count, start, j)
                count = bits = 0
    if count:
        emit(has.size - 1, 2000, count, start, has.size - 1)


def scan_items(coef, per_mcu, h, w, s, stats=None):
    """(table, symbol, bits, length) of everything scan s emits, in order; table -1 marks raw bits."""
    comp, ss, se, ah, al = SCANS[s]
    items = Items()
    stats = stats if stats is not None else {"max_run": 0, "corr_limit": 0}
    if comp is None:
        if ah == 0:
            _dc_first(coef, per_mcu, al, items)
        else:
            items.add(np.arange(coef.shape[0]), 0, 0, -1, -1, coef[:, 0].astype(np.int64) >> al, 1)
        return items.ordered()
    x = component_blocks(coef, per_mcu, h, w, comp)
    t = int(comp > 0)
    has, ends, corr = (_ac_refine if ah else _ac_first)(x, ss, se, al, t, items)
    _runs(has, ends, corr, ah > 0, t, items, stats)
    return items.ordered()


def scan_tables(table, sym):
    """The optimal tables of one scan, [table 0, table 1] (None where the scan codes nothing with that table)."""
    out = []
    for t in (0, 1):
        sel = table == t
        out.append(O.optimal_table(np.bincount(sym[sel], minlength=256)) if sel.any() else None)
    return out


def pack(table, sym, val, nval, tabs):
    """The stuffed, 1-padded bytes of one scan's items coded with ``tabs``."""
    code, size = np.zeros((3, 256), np.int64), np.zeros((3, 256), np.int64)
    for t, tab in enumerate(tabs):
        if tab is not None:
            for s, (c, n) in J.huff_codes(tab).items():
                code[t, s], size[t, s] = c, n
    t = np.where(table < 0, 2, table)
    sy = np.where(table < 0, 0, sym)
    assert (size[t, sy][table >= 0] > 0).all()
    length = size[t, sy] + nval
    word = (code[t, sy] << nval) | val
    start = np.cumsum(length) - length
    total = int(length.sum())
    pos = np.arange(total) - np.repeat(start, length)
    bits = (np.repeat(word, length) >> (np.repeat(length, length) - 1 - pos)) & 1
    bits = np.concatenate([bits, np.ones(-total % 8, np.int64)]).astype(np.uint8)
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def scan_header(s, tabs):
    """The DHT segments of scan s's tables and its SOS."""
    comp, ss, se, ah, al = SCANS[s]
    out = b""
    for t, tab in enumerate(tabs):
        if tab is not None:
            counts, syms = tab
            cls_id = (0x10 if se else 0x00) | t
            out += bytes([0xFF, 0xC4]) + (3 + 16 + len(syms)).to_bytes(2, "big") + bytes([cls_id]) + bytes(counts) + syms
    if comp is None:
        sel = [(1, 0x00), (2, 0x10), (3, 0x10)] if ah == 0 else [(1, 0), (2, 0), (3, 0)]
    else:
        sel = [(comp + 1, int(comp > 0))]
    body = bytes([len(sel)]) + b"".join(bytes(p) for p in sel) + bytes([ss, se, ah << 4 | al])
    return out + bytes([0xFF, 0xDA]) + (len(body) + 2).to_bytes(2, "big") + body


def encode(rgb, quality=75, subsampling=2, stats=None):
    """The bytes Pillow writes for Image.fromarray(rgb).save(buf, "JPEG", quality=quality, subsampling=subsampling,
    progressive=True). ``stats`` (a dict) counts the runs emitted early at MAX_RUN ("max_run") and at CORR_LIMIT
    ("corr_limit")."""
    rgb = np.asarray(rgb, np.uint8)
    h, w = rgb.shape[:2]
    coef, per_mcu = J.coefficients(rgb, quality, subsampling)
    head = bytearray(J.header(h, w, quality, subsampling)[:SOF_END])
    head[SOF_END - 18] = 0xC2                                     # SOF2
    out = bytes(head)
    if stats is not None:
        stats.setdefault("max_run", 0)
        stats.setdefault("corr_limit", 0)
    for s in range(len(SCANS)):
        table, sym, val, nval = scan_items(coef, per_mcu, h, w, s, stats)
        tabs = scan_tables(table, sym)
        out += scan_header(s, tabs) + pack(table, sym, val, nval, tabs)
    return out + b"\xff\xd9"

"""libjpeg-turbo's encoder with the caller's quantisation tables, 4:2:2 and APP1 / APP2 segments, restated in integer numpy:
what ``PIL.Image.save(buf, "JPEG", qtables=T, subsampling=s, optimize=o, progressive=p, exif=E, icc_profile=I)`` writes for
an RGB image, and so ``src.save(buf, "JPEG", quality="keep", ...)``'s file. It is the spec se_jpeg_encode_tables_u8 follows.
The colour conversion, FDCT, quantisation, Huffman coding and scans are tests/util_jpeg.py's, util_jpeg_optimize.py's and
util_jpeg_progressive.py's, unchanged; what is new here:
  * 4:2:2 (subsampling 1): 16x8 MCUs of Y0, Y1, Cb, Cr; chroma columns repeated to the MCU width and averaged in pairs with
    the bias 0, 1, 0, 1, ... along each row (jcsample.c h2v1_downsample), rows repeated to the block grid; a luma block wholly
    right of the image is a dummy (DC of the block before it, EOB);
  * Pillow's table assignment (JpegEncode.c): one table serves all components, two split luma / chroma, three or four give
    component c table c; DQT segments 0 .. min(n, 3) - 1 are written, entries <= 0 taken as 1 (jpeg_add_quant_table);
  * the APP1 / APP2 segments (``engine.jpeg_app_segments``) right after APP0.
"""
import numpy as np

from tests import util_jpeg as J
from tests import util_jpeg_optimize as O
from tests import util_jpeg_progressive as P

SAMPLING = {0: 0x11, 1: 0x21, 2: 0x22}   # Y's sampling byte in SOF
LUMA_BLOCKS = {0: (1, 1), 1: (1, 2), 2: (2, 2)}   # luma blocks per MCU, (rows, columns)


def sampling(subsampling):
    """Pillow's subsampling (-1: libjpeg's default) as 0, 1 or 2."""
    return 2 if subsampling == -1 else subsampling


def comp_tables(qtables):
    """(each component's table as int64 [64] natural order with entries >= 1, the number of DQT segments)."""
    qtables = list(qtables.values()) if isinstance(qtables, dict) else list(qtables)
    nq = min(len(qtables), 3)
    tabs = [np.maximum(np.asarray(qtables[t], np.int64), 1) for t in range(nq)]
    return [tabs[min(c, nq - 1)] for c in range(3)], tabs


def planes(rgb, subsampling):
    """The sample planes the DCT reads and the MCU grid (rows, cols); 4:4:4 and 4:2:0 are util_jpeg.planes."""
    if subsampling != 1:
        return J.planes(rgb, subsampling)
    h, w = rgb.shape[:2]
    y, cb, cr = J.ycc(rgb)
    my, mx = -(-h // 8), -(-w // 16)
    out = [J._pad(y, 8 * my, 16 * mx)]        # luma blocks past the image are dummies
    bias = np.tile([0, 1], 4 * mx)
    for p in (cb, cr):
        p = J._pad(p, h, 16 * mx)
        out.append(J._pad((p[:, 0::2] + p[:, 1::2] + bias) >> 1, 8 * my, 8 * mx))
    return out, (my, mx)


def coefficients(rgb, qtables, subsampling):
    """Quantised zigzag coefficients [blocks, 64] in scan order and the blocks per MCU (util_jpeg.coefficients with the
    component tables of ``qtables`` and 4:2:2)."""
    h, w = rgb.shape[:2]
    pl, (my, mx) = planes(rgb, subsampling)
    qs, _ = comp_tables(qtables)
    q = [J.quantize(J.fdct(J._blocks(p) - 128), t.reshape(8, 8)).reshape(-1, 64)[:, J.ZIGZAG] for p, t in zip(pl, qs)]
    v, u = LUMA_BLOCKS[subsampling]
    nl = v * u
    y = q[0].reshape(my, v, mx, u, 64).transpose(0, 2, 1, 3, 4).reshape(my * mx, nl, 64)
    ys, xs = np.meshgrid(np.arange(my * v), np.arange(mx * u), indexing="ij")
    dummy = ((ys >= -(-h // 8)) | (xs >= -(-w // 8))).reshape(my, v, mx, u).transpose(0, 2, 1, 3).reshape(my * mx, nl)
    y[dummy] = 0
    for k in range(1, nl):                     # a dummy takes the DC of the block before it (block 0 is never a dummy)
        y[:, k, 0] = np.where(dummy[:, k], y[:, k - 1, 0], y[:, k, 0])
    return np.concatenate([y, q[1][:, None], q[2][:, None]], 1).reshape(-1, 64), nl + 2


def header(h, w, qtables, subsampling, segments=b"", tabs=None):
    """SOI, JFIF APP0, the segments, the DQTs, SOF0, DHT DC0 AC0 DC1 AC1 (Annex K, or ``tabs`` in util_jpeg_optimize's
    order), SOS."""
    def seg(marker, body):
        return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body

    _, dqt = comp_tables(qtables)
    nq = len(dqt)
    out = b"\xff\xd8" + seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00") + segments
    for t, q in enumerate(dqt):
        out += seg(0xDB, bytes([t]) + bytes(q[J.ZIGZAG].astype(np.uint8)))
    comps = b"".join(bytes([c + 1, SAMPLING[subsampling] if c == 0 else 0x11, min(c, nq - 1)]) for c in range(3))
    out += seg(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([3]) + comps)
    huff = (J.DC_LUMA, J.DC_CHROMA, J.AC_LUMA, J.AC_CHROMA) if tabs is None else tabs
    for cls_id, t in ((0x00, 0), (0x10, 2), (0x01, 1), (0x11, 3)):
        counts, syms = huff[t]
        out += seg(0xC4, bytes([cls_id]) + bytes(counts) + bytes(syms))
    return out + seg(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))


def sof_end(ntables, segments_len):
    """Header bytes through SOF0."""
    return 20 + segments_len + 69 * min(ntables, 3) + 19


def component_blocks(coef, per_mcu, h, w, c):
    """[n, 64] zigzag coefficients of component c's own blocks in raster order (util_jpeg_progressive's, with 4:2:2)."""
    if per_mcu != 4:
        return P.component_blocks(coef, per_mcu, h, w, c)
    if c:
        return coef[1 + c::4]
    my, mx = -(-h // 8), -(-w // 16)
    return coef.reshape(my * mx, 4, 64)[:, :2].reshape(my, 2 * mx, 64)[:, :-(-w // 8)].reshape(-1, 64)


def scan_items(coef, per_mcu, h, w, s):
    """util_jpeg_progressive.scan_items with component_blocks above."""
    comp, ss, se, ah, al = P.SCANS[s]
    if comp is None or per_mcu != 4:
        return P.scan_items(coef, per_mcu, h, w, s)
    items = P.Items()
    x = component_blocks(coef, per_mcu, h, w, comp)
    t = int(comp > 0)
    has, ends, corr = (P._ac_refine if ah else P._ac_first)(x, ss, se, al, t, items)
    P._runs(has, ends, corr, ah > 0, t, items, {"max_run": 0, "corr_limit": 0})
    return items.ordered()


def encode(rgb, qtables, subsampling, optimize=False, progressive=False, segments=b""):
    """The bytes Pillow writes for Image.fromarray(rgb).save(buf, "JPEG", qtables=qtables, subsampling=subsampling,
    optimize=optimize, progressive=progressive, ...) with the APP1 / APP2 ``segments`` those metadata arguments make."""
    rgb = np.asarray(rgb, np.uint8)
    h, w = rgb.shape[:2]
    sub = sampling(subsampling)
    coef, per_mcu = coefficients(rgb, qtables, sub)
    if progressive:
        end = sof_end(len(comp_tables(qtables)[1]), len(segments))
        head = bytearray(header(h, w, qtables, sub, segments)[:end])
        head[end - 18] = 0xC2                                     # SOF2
        out = bytes(head)
        for s in range(len(P.SCANS)):
            table, sym, val, nval = scan_items(coef, per_mcu, h, w, s)
            tabs = P.scan_tables(table, sym)
            out += P.scan_header(s, tabs) + P.pack(table, sym, val, nval, tabs)
        return out + b"\xff\xd9"
    if optimize:
        tabs = O.tables(coef, per_mcu)
        return header(h, w, qtables, sub, segments, tabs) + O.entropy(coef, per_mcu, tabs) + b"\xff\xd9"
    return header(h, w, qtables, sub, segments) + J.entropy(coef, per_mcu) + b"\xff\xd9"


def max_bytes(h, w, subsampling, ntables, progressive=False, segments_len=0):
    """The bound se_jpeg_tables_max_bytes states (DESIGN §7b): the header with min(ntables, 3) DQTs and the segments; per
    block 208 bytes (baseline) or each scan's most bits per slot; every byte possibly stuffed; EOI."""
    sub = sampling(subsampling)
    v, u = LUMA_BLOCKS[sub]
    mcus = -(-h // (8 * v)) * -(-w // (8 * u))
    per = v * u + 2
    end = sof_end(ntables, segments_len)
    if not progressive:
        return end + 432 + 14 + 2 * (mcus * per * J.MAX_BLOCK_BITS // 8) + 2
    total = 0
    for comp, ss, se, ah, al in P.SCANS:
        slots = mcus * per if comp is None else (-(-h // 8) * -(-w // 8) if comp == 0 else mcus)
        bits = (1 if ah else 27) if comp is None else (se - ss + 1) * (18 if ah else 26) + 30
        total += -(-slots * bits // 8)
    return end + 2 * (21 + 12) + 14 + 14 + 8 * (21 + 176 + 10) + 2 + 2 * total

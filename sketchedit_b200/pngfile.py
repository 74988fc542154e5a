"""PNG container parsing for the device decoder (``se_png_decode_u8``): signature, chunks and their CRCs, without decompressing.

``parse(data)`` says whether the device decodes a file to what ``np.asarray(Image.open(f).convert(mode))`` gives, and if so
returns what the decoder needs: the IHDR fields, the palette and the IDAT payloads joined into one zlib stream. Everything
else goes to Pillow (``host`` below), so results are always Pillow's, pixels or exception: a file that is not a PNG; 16-bit
or interlaced; an APNG (``acTL``); a chunk outside the few known not to change what Pillow returns; a bad CRC, length or
order; more pixels than Pillow opens without a warning."""
import io
import struct
import zlib
from collections import namedtuple

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
MAX_DIM = 65535
# (colour type) -> bit depths decoded on the device
DEPTHS = {0: (1, 2, 4, 8), 2: (8,), 3: (1, 2, 4, 8), 4: (8,), 6: (8,)}
# ancillary chunks Pillow reads without effect on pixels (or not at all), with the lengths Pillow reads them at
SAFE = {b"gAMA": 4, b"cHRM": 32, b"sRGB": 1, b"pHYs": 9, b"tIME": 7}
MODES = {"RGB": 3, "L": 1}

PngHead = namedtuple("PngHead", "h w depth ctype palette stream")
PngHead.__doc__ = """A file the device decodes: IHDR height, width, bit depth and colour type; the PLTE bytes (b"" unless colour
type 3); the IDAT payloads joined into one zlib stream."""


class Host(Exception):
    """The file goes to Pillow; the message says why."""


def parse(data):
    """``PngHead`` of the PNG bytes ``data``, or raises ``Host`` naming why Pillow must decode them."""
    data = memoryview(data).cast("B") if not isinstance(data, bytes) else data
    if len(data) < 8 or bytes(data[:8]) != SIGNATURE:
        raise Host("not a PNG")
    at, n = 8, len(data)
    ihdr = palette = trns = None
    idat, state = [], "head"   # head -> idat -> tail (after the IDAT run) -> end (IEND)
    while state != "end":
        if at + 8 > n:
            raise Host("truncated chunk")
        length, cid = struct.unpack(">I4s", data[at:at + 8])
        if length > 0x7FFFFFFF or at + 12 + length > n:
            raise Host("truncated chunk")
        body = data[at + 8:at + 8 + length]
        (crc,) = struct.unpack(">I", data[at + 8 + length:at + 12 + length])
        if zlib.crc32(body, zlib.crc32(cid)) != crc:
            raise Host("bad CRC in %r" % cid)
        at += 12 + length
        if ihdr is None:
            if cid != b"IHDR" or length != 13:
                raise Host("no IHDR first")
            w, h, depth, ctype, comp, filt, lace = struct.unpack(">IIBBBBB", body)
            if depth == 16:
                raise Host("16-bit")
            if lace != 0:
                raise Host("interlaced")
            if depth not in DEPTHS.get(ctype, ()) or comp or filt:
                raise Host("colour type %d at depth %d" % (ctype, depth))
            if not (1 <= w <= MAX_DIM and 1 <= h <= MAX_DIM):
                raise Host("size %dx%d" % (w, h))
            from PIL import Image
            if Image.MAX_IMAGE_PIXELS is not None and w * h > Image.MAX_IMAGE_PIXELS:
                raise Host("more pixels than Pillow opens without a warning")
            ihdr = (h, w, depth, ctype)
            continue
        if cid in (b"acTL", b"fcTL", b"fdAT"):
            raise Host("APNG")
        if cid == b"IDAT":
            if state == "tail":
                raise Host("IDAT chunks apart")
            if state == "head" and ihdr[3] == 3 and palette is None:
                raise Host("no PLTE")
            state = "idat"
            idat.append(body)
        elif cid == b"IEND":
            if length or state != "idat" and state != "tail":
                raise Host("IEND before IDAT, or not empty")
            state = "end"
        else:
            if state == "idat":
                state = "tail"
            if cid == b"PLTE" and state == "head" and palette is None and trns is None and ihdr[3] in (2, 3, 6):
                if length % 3 or not 3 <= length <= 768:
                    raise Host("PLTE of %d bytes" % length)
                palette = bytes(body)
            elif cid == b"tRNS" and state == "head" and trns is None and (
                    (ihdr[3] == 3 and palette is not None and length <= 256) or (ihdr[3] == 0 and length == 2) or
                    (ihdr[3] == 2 and length == 6)):
                trns = bytes(body)
            elif SAFE.get(cid) != length:
                raise Host("chunk %r" % cid)
    h, w, depth, ctype = ihdr
    return PngHead(h, w, depth, ctype, palette if ctype == 3 else b"", b"".join(idat))


def size(data):
    """(h, w) of a PNG's IHDR without checking the rest of the file, None when it has none."""
    if len(data) < 24 or bytes(data[:8]) != SIGNATURE or bytes(data[12:16]) != b"IHDR":
        return None
    w, h = struct.unpack(">II", data[16:24])
    return h, w


def stage(heads, alloc):
    """The device decoder's input for the ``PngHead`` list ``heads``: each file's stream followed by its palette, packed in
    order, one copy of each into the buffer ``alloc(total)`` returns (total >= 1 bytes; a uint8 numpy array or CPU tensor).
    Returns ``(buffer, offsets, lengths)`` of the streams."""
    offsets, at = [], 0
    for hd in heads:
        offsets.append(at)
        at += len(hd.stream) + len(hd.palette)
    buf = alloc(max(at, 1))
    view = np.asarray(buf)
    for hd, o in zip(heads, offsets):
        n = len(hd.stream)
        view[o:o + n] = np.frombuffer(hd.stream, np.uint8)
        view[o + n:o + n + len(hd.palette)] = np.frombuffer(hd.palette, np.uint8)
    return buf, offsets, [len(hd.stream) for hd in heads]


def pillow_decode(data, mode):
    """What the device decoder stands for: np.asarray(Image.open(f).convert(mode)), Pillow's exception included."""
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert(mode))

"""Serving side of the reference's second entry point (reference demo.py:39-73, SURVEY.md 8f-3), without the Flask UI.

The reference's demo handles one request per Flask thread (``app.run(threaded=True)``) and every request runs its own
batch-1 forward. Here concurrent requests are BATCHED: ``RequestBatcher`` collects the requests that arrive within a short
window, groups them by input size and runs each group as one forward (``Engine.inference_u8``: the codecs of
demo.py:52-53,64-66 run on the device); ``DemoProcessor.process_image`` is the reference's ``process_image`` around it
(floor the size to a multiple of 8, PIL resize in, forward, PIL resize back). By default the two resizes run on the device
too (``engine.resize_u8_packed``, bit-identical to Pillow), so a batch is one upload and one download of raw bytes.

    proc = DemoProcessor(models.create_model(opt), max_batch=16, max_wait_ms=2.0)
    result_pil = proc.process_image(image_pil, mask_pil)       # callable from any number of threads
    result_pil, mask = proc.process_image(image_pil, mask_pil, return_mask=True)       # ... and the predicted edit mask
    result_pil = proc.process_image(image_pil, mask_pil, edit_mask=corrected_mask)      # run on a revised edit mask
    result_pil = proc.process_image(image_pil, mask_pil, region="auto")                 # edit a crop around the strokes only
    result_pil = proc.process_image(image_pil, mask_pil, region="strokes")              # one crop per group of strokes
    result_pil = proc.process_image(image_pil, mask_pil, region="auto", feather=16)     # paste fading over 16 px at inner edges
    result_pil = proc.process_image(image_pil, mask_pil, region="auto", detail=True)    # restore the photo's fine detail in the hole
    s = proc.open_session(image_pil)                  # the photo stays on the device across edits
    r = s.edit(mask_pil, region="strokes")            # r.boxes, r.patches: what changed; s.undo() restores it
    p = s.propose(mask_pil, region="strokes")         # p.boxes, p.masks: the edit's region, from netM alone
    r = s.accept(p)                                   # that edit, byte for byte (or accept(p, edit_masks=corrections))
    preview = s.jpeg(size=(640, 640))                 # Pillow's thumbnail of the photo, made and encoded on the device
    mask = proc.predict_mask(image_pil, mask_pil)     # process_image's returned mask, without the image
    proc.close()

A region edit (``region=``) crops a box of the photo, runs the forward on it at ``DemoProcessor(region_size=...)`` and pastes
the result back with the edit mask: its cost follows the box, not the photo, and region requests on photos of any size
batch together. A request may carry several boxes (``region="strokes"`` or a list), pasted in order. ``feather=F`` fades each
box's paste mask to 0 along the box edges that lie inside the photo (``feather_widths``, ``feather_ramp``), so the paste shows no
seam there. ``detail=True`` adds back, inside the hole, the photo's high frequencies that the box's resize round trip lost,
gathered with netG's own attention weights (``process_image``). An ``EditSession`` keeps one photo on the device for a chain of edits, each drawn on the previous result, with undo.

Everything except the forward itself (``run_batch``) is plain host logic and is unit-tested on the CPU with a fake forward.
"""
import threading
import time
from collections import OrderedDict, deque, namedtuple

import numpy as np


class _Request:
    __slots__ = ("key", "payload", "event", "result", "error", "t_submit")

    def __init__(self, key, payload):
        self.key, self.payload = key, payload
        self.event = threading.Event()
        self.result = self.error = None
        self.t_submit = time.monotonic()


class RequestBatcher:
    """Thread-safe request batching.

    ``run_batch(key, payloads) -> list of results`` (same length and order) is called from ONE worker thread with all the
    pending requests that share ``key`` (at most ``max_batch``). A request is dispatched as soon as ``max_batch`` requests of
    its key are pending or ``max_wait_ms`` after it was submitted, whichever comes first; keys are served oldest request first.
    ``submit`` blocks the calling thread until its result is ready and re-raises the worker's exception for that batch.
    """

    def __init__(self, run_batch, max_batch=16, max_wait_ms=2.0):
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self.run_batch, self.max_batch, self.max_wait = run_batch, int(max_batch), max_wait_ms / 1e3
        self._cv = threading.Condition()
        self._pending = OrderedDict()          # key -> deque of requests, keys in order of their oldest pending request
        self._closed = False
        self.batches = []                      # (key, size) of every dispatched batch (observability / tests)
        self._worker = threading.Thread(target=self._loop, name="sketchedit-batcher", daemon=True)
        self._worker.start()

    def submit(self, key, payload):
        req = _Request(key, payload)
        with self._cv:
            if self._closed:
                raise RuntimeError("RequestBatcher is closed")
            self._pending.setdefault(key, deque()).append(req)
            self._cv.notify_all()
        req.event.wait()
        if req.error is not None:
            raise req.error
        return req.result

    def close(self):
        with self._cv:
            self._closed = True
            self._cv.notify_all()
        self._worker.join()

    # -- worker
    def _take(self):
        """Under the lock: the next batch to run, or (None, seconds to sleep) / (None, None) when closed and drained."""
        now = time.monotonic()
        best_wait = None
        for key, q in self._pending.items():
            age = now - q[0].t_submit
            if len(q) >= self.max_batch or age >= self.max_wait or self._closed:
                reqs = [q.popleft() for _ in range(min(self.max_batch, len(q)))]
                if not q:
                    del self._pending[key]
                else:
                    self._pending.move_to_end(key)          # the rest of this key queues behind the other keys
                return reqs, None
            w = self.max_wait - age
            best_wait = w if best_wait is None else min(best_wait, w)
        if self._closed and not self._pending:
            return None, None
        return None, (best_wait if best_wait is not None else 3600.0)

    def _loop(self):
        while True:
            with self._cv:
                reqs, wait = self._take()
                while reqs is None:
                    if wait is None:
                        return
                    self._cv.wait(timeout=wait)
                    reqs, wait = self._take()
            self._dispatch(reqs)
            reqs = None                     # the results belong to their requesters: device memory in them is not kept here

    def _dispatch(self, reqs):
        key = reqs[0].key
        try:
            results = self.run_batch(key, [r.payload for r in reqs])
            if len(results) != len(reqs):
                raise RuntimeError("run_batch returned %d results for %d requests" % (len(results), len(reqs)))
            for r, res in zip(reqs, results):
                r.result = res
        except BaseException as e:      # noqa: BLE001 - delivered to every requester of this batch
            for r in reqs:
                r.error = e
        self.batches.append((key, len(reqs)))
        for r in reqs:
            r.event.set()


def floor8(n):
    return n // 8 * 8


def region_box(bbox, photo_size, region_size):
    """The PIL box ``(left, upper, right, lower)`` of an automatic region edit: the crop of the photo that is resized to the
    working size ``region_size = (Hn, Wn)``. ``bbox`` is the strokes' PIL bounding box, ``photo_size`` the photo's PIL size
    ``(w, h)``.

    The scale ``s = max(1, 2*bw/Wn, 2*bh/Hn)``, rounded up to a multiple of 1/8: the strokes span at most half of each side, the
    crop is never upsampled unless the photo is smaller than the working size, and box sizes repeat (the resize's coefficient
    tables are cached per size). The box is ``min(w, s*Wn)`` x ``min(h, s*Hn)``, centred on the bbox (floored) and shifted to
    lie inside the photo, so it always contains the bbox."""
    left, upper, right, lower = (int(v) for v in bbox)
    w, h = (int(v) for v in photo_size)
    Hn, Wn = (int(v) for v in region_size)
    if not (0 <= left < right <= w and 0 <= upper < lower <= h):
        raise ValueError("bbox %r is not a non-empty box inside the %dx%d photo" % (tuple(bbox), w, h))
    e8 = max(8, -(-16 * (right - left) // Wn), -(-16 * (lower - upper) // Hn))    # 8*s = ceil(8 * 2*b/n), at least 8
    bw, bh = min(w, e8 * Wn // 8), min(h, e8 * Hn // 8)

    def place(lo, hi, size, extent):
        return min(max((lo + hi - size) // 2, 0), extent - size)

    x, y = place(left, right, bw, w), place(upper, lower, bh, h)
    return x, y, x + bw, y + bh


GROUP_CELL = 8     # region_groups connects strokes on a grid of 8x8-pixel cells


def _intersects(a, b):
    return a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]


def region_groups(mask, edit_mask=None, region_size=(256, 256), photo_size=None, offset=(0, 0)):
    """The stroke groups of a region edit with ``region="strokes"``: a list of ``(bbox, box)`` PIL boxes, one per group,
    ordered by the (upper, left) corner of ``bbox``. ``mask`` and ``edit_mask`` are PIL images of the photo's size, or of one
    smaller size placed at ``offset = (x, y)`` in a photo of PIL size ``photo_size`` (zero elsewhere); the boxes are then those
    of the zero-padded photo-sized masks, in photo coordinates.

    1. The non-zero pixels of ``mask`` and ``edit_mask`` are connected (8-neighbourhood) on a grid of 8x8-pixel cells; a cell is
       set when any of its pixels is. ``bbox`` is the exact pixel bounding box of a group's non-zero pixels.
    2. Two groups merge while one's ``bbox`` intersects the other's ``region_box``; the merged ``bbox`` is the union.
    3. ``box = region_box(bbox, mask.size, region_size)``.
    So every box holds its own group's strokes and no other group's: ``mask.crop(box)`` is that group's sketch alone. Boxes
    may still overlap, in stroke-free margins. One group gives the box of ``region="auto"``. No stroke is a ValueError."""
    w, h = photo_size or mask.size
    dx, dy = (int(v) for v in offset)
    if edit_mask is not None and edit_mask.size != mask.size:
        raise ValueError("edit_mask is %dx%d, mask %dx%d: they must have one size" % (edit_mask.size + mask.size))
    c = GROUP_CELL
    ims = [m if m.mode == "L" else m.convert("L") for m in (mask, edit_mask) if m is not None]
    bbs = [(b[0] + dx, b[1] + dy, b[2] + dx, b[3] + dy) for b in (m.getbbox() for m in ims) if b]
    if not bbs:
        raise ValueError("region='strokes' needs a sketch stroke or a non-zero edit mask")
    # only the cells of the union bbox are examined, from a cell corner of the photo's grid
    ox, oy = min(b[0] for b in bbs) // c * c, min(b[1] for b in bbs) // c * c
    crop = (ox, oy, max(b[2] for b in bbs), max(b[3] for b in bbs))
    ch, cw = crop[3] - oy, crop[2] - ox
    H8, W8 = -(-ch // c), -(-cw // c)
    pad = np.zeros((H8 * c, W8 * c), np.uint8)
    for m in ims:                                               # PIL pads a crop reaching past the mask with zeros
        np.maximum(pad[:ch, :cw], np.asarray(m.crop((crop[0] - dx, crop[1] - dy, crop[2] - dx, crop[3] - dy))), out=pad[:ch, :cw])
    blocks = pad.reshape(H8, c, W8, c)
    cells = (pad.view(np.uint64).reshape(H8, c, W8) != 0).any(axis=1)     # a cell row's 8 pixels as one word: exact
    # runs of set cells per cell row, joined by union-find with the overlapping (8-neighbour) runs of the row above
    d = np.diff(np.pad(cells.astype(np.int8), ((0, 0), (1, 1))), axis=1)
    starts, ends = np.nonzero(d == 1), np.nonzero(d == -1)[1]   # both in row-major order: run k is [s, e) of row r
    run_r, run_s, run_e = starts[0], starts[1], ends
    parent = list(range(len(run_r)))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    row_first = np.searchsorted(run_r, np.arange(H8 + 1))
    for r in range(1, H8):
        i, i1 = row_first[r - 1], row_first[r]
        for k in range(row_first[r], row_first[r + 1]):
            while i < i1 and run_e[i] < run_s[k]:                  # runs above that end before this one's diagonal neighbour
                i += 1
            j = i
            while j < i1 and run_s[j] <= run_e[k]:
                a, b = find(j), find(k)
                if a != b:
                    parent[b] = a
                j += 1
    roots = np.array([find(k) for k in range(len(run_r))])
    label = np.full((H8, W8), -1, np.int64)
    for k in range(len(run_r)):
        label[run_r[k], run_s[k]:run_e[k]] = roots[k]
    cy, cx = np.nonzero(cells)
    lab = label[cy, cx]
    # exact pixel bounds of each set cell, then their extremes per group
    px = blocks[cy, :, cx, :] != 0                                # [cells, c, c]
    rows, cols = px.any(axis=2), px.any(axis=1)
    y0 = oy + cy * c + rows.argmax(axis=1)
    y1 = oy + cy * c + c - rows[:, ::-1].argmax(axis=1)
    x0 = ox + cx * c + cols.argmax(axis=1)
    x1 = ox + cx * c + c - cols[:, ::-1].argmax(axis=1)
    ids, inv = np.unique(lab, return_inverse=True)
    bb = np.empty((len(ids), 4), np.int64)
    bb[:, :2] = np.iinfo(np.int64).max
    bb[:, 2:] = -1
    np.minimum.at(bb[:, 0], inv, x0)
    np.minimum.at(bb[:, 1], inv, y0)
    np.maximum.at(bb[:, 2], inv, x1)
    np.maximum.at(bb[:, 3], inv, y1)
    groups = [tuple(int(v) for v in b) for b in bb]
    boxes = [region_box(g, (w, h), region_size) for g in groups]
    merged = True
    while merged:
        merged = False
        for i in range(len(groups)):
            for j in range(i + 1, len(groups)):
                if _intersects(groups[j], boxes[i]) or _intersects(groups[i], boxes[j]):
                    a, b = groups[i], groups.pop(j)
                    groups[i] = (min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3]))
                    boxes.pop(j)
                    boxes[i] = region_box(groups[i], (w, h), region_size)
                    merged = True
                    break
            if merged:
                break
    return sorted(zip(groups, boxes), key=lambda gb: (gb[0][1], gb[0][0]))


def detail_box_ok(size, region_size):
    """Whether a box of PIL size ``(w, h)`` can take detail at the working size ``(Hn, Wn)``: every patch position of the
    working grid must have a box-pixel anchor, ``u(w - 1) >= Wn - 16`` with ``u(x) = ((2x + 1) Wn) // (2 w)`` (and likewise
    rows), which holds from ``w >= Wn / 32``. A narrower box has patches no box column maps into (DESIGN.md section 7b)."""
    w, h = (int(v) for v in size)
    Hn, Wn = (int(v) for v in region_size)
    return (2 * w - 1) * Wn // (2 * w) >= Wn - 16 and (2 * h - 1) * Hn // (2 * h) >= Hn - 16


def _check_detail(detail, region_none, host, has_attention=True):
    """``detail`` checked against the request: a bool, and only for a region edit of the device flow on a model with the
    contextual attention (whose weights it uses). Checked before the request is queued, so a detail request never makes a
    batch it shares with other requests fail."""
    if not isinstance(detail, bool):
        raise ValueError("detail must be True or False, got %r" % (detail,))
    if detail and not has_attention:
        raise ValueError("detail=True needs the model's contextual attention (use_cam): it aggregates with its weights")
    if detail and region_none:
        raise ValueError("detail=True needs a region edit: the whole-photo flow only floors the photo to a multiple of 8, so no "
                         "detail is lost to restore")
    if detail and host:
        raise ValueError("detail=True needs resize='device': the host flow has no GPU forward export to take it from")
    return detail


def _check_detail_boxes(boxes, region_size):
    for b in boxes:
        if not detail_box_ok((b[2] - b[0], b[3] - b[1]), region_size):
            raise ValueError("detail=True needs boxes of at least 1/32 of the working size %dx%d per side, got box %r"
                             % (region_size[1], region_size[0], tuple(b)))


def _check_feather(feather):
    if isinstance(feather, bool) or not isinstance(feather, (int, np.integer)) or feather < 0:
        raise ValueError("feather must be an int >= 0 (photo pixels), got %r" % (feather,))
    return int(feather)


def feather_widths(box, photo_size, feather):
    """The feather widths ``(left, top, right, bottom)`` of a region edit's PIL box ``(left, upper, right, lower)`` in a photo
    of PIL size ``(w, h)``: a side on the photo's border gets 0 (it stays hard), any other ``min(feather, bw // 4)`` (left,
    right) or ``min(feather, bh // 4)`` (top, bottom) for a ``bw x bh`` box. The quarter cap keeps the band off the strokes of
    an 'auto' or 'strokes' box: ``region_box`` centres strokes that span at most half of each side, and it only shifts a box
    towards a photo border, whose side is not feathered."""
    left, upper, right, lower = (int(v) for v in box)
    w, h = (int(v) for v in photo_size)
    fx, fy = min(int(feather), (right - left) // 4), min(int(feather), (lower - upper) // 4)
    return (0 if left == 0 else fx, 0 if upper == 0 else fy, 0 if right == w else fx, 0 if lower == h else fy)


def feather_ramp(size, widths):
    """The feather ramp [h, w] uint8 of a box of PIL size ``(w, h)`` with ``widths = (left, top, right, bottom)``: a side of
    width f gives the pixel at distance d from its edge pixel (d = 0 on it) ``255 if d >= f else (255 * (d + 1)) // (f + 1)``,
    and a pixel takes the least over the four sides. The pasted mask is ``feather_mask(m, widths) = DIV255(m * ramp)``, with
    Pillow's blend rounding ``DIV255(a) = (((a + 128) >> 8) + a + 128) >> 8``; widths of 0 leave m unchanged."""
    w, h = (int(v) for v in size)
    fl, ft, fr, fb = (int(v) for v in widths)

    def side(d, f):
        return np.where(d >= f, 255, (255 * (d + 1)) // (f + 1))

    x, y = np.arange(w), np.arange(h)
    rx = np.minimum(side(x, fl), side(w - 1 - x, fr))
    ry = np.minimum(side(y, ft), side(h - 1 - y, fb))
    return np.minimum(ry[:, None], rx[None, :]).astype(np.uint8)


def feather_mask(m, widths):
    """``DIV255(m * feather_ramp)`` of an [h, w] uint8 mask (see ``feather_ramp``)."""
    m = np.asarray(m)
    a = m.astype(np.int32) * feather_ramp(m.shape[::-1], widths) + 128
    return (((a >> 8) + a) >> 8).astype(np.uint8)


def _check_box(box, w, h):
    if not (isinstance(box, (tuple, list)) and len(box) == 4 and all(isinstance(v, (int, np.integer)) for v in box)):
        raise ValueError("region must be None, 'auto', 'strokes', a PIL box (left, upper, right, lower) of integers or a list of "
                         "such boxes, got %r" % (box,))
    left, upper, right, lower = (int(v) for v in box)
    if not (0 <= left < right <= w and 0 <= upper < lower <= h):
        raise ValueError("region %r must satisfy 0 <= left < right <= %d and 0 <= upper < lower <= %d" % (tuple(box), w, h))
    return left, upper, right, lower


def _overlap_sets(boxes):
    """Indices of the boxes, split into connected sets of boxes that overlap (each set in box order)."""
    parent = list(range(len(boxes)))

    def find(a):
        while parent[a] != a:
            a = parent[a]
        return a

    for i in range(len(boxes)):
        for j in range(i):
            if _intersects(boxes[i], boxes[j]):
                parent[find(i)] = find(j)
    sets = {}
    for i in range(len(boxes)):
        sets.setdefault(find(i), []).append(i)
    return list(sets.values())


class DemoProcessor:
    """``process_image`` of the reference demo (demo.py:39-73) on the batched uint8 forward.

    Differences from the reference function, none of them numerical: it returns the PIL result instead of writing
    ``static/results/<name>``, and concurrent calls share forwards. ``precision``: 'bf16' | 'fp32' | 'fp32_direct'.

    ``resize``: where the three Pillow resizes of the demo run (photo and sketch mask down to the floored size, result back).
    'device' (default): on the GPU with ``engine.resize_u8_packed``, bit-identical to Pillow; a batch is one upload of the raw
    photos and masks from pinned memory and one download of the results. 'host': with Pillow on the requesting thread.
    The device flow's two pinned staging buffers are reused and grow to the largest batch seen (raw photos plus masks in, raw
    photos out: about 680 MB at 16 requests of 12 MP); ``close()`` releases them.

    ``region_size = (Hn, Wn)``: the working size of region edits (``process_image(..., region=...)``), multiples of 8, at
    least 16.
    """

    def __init__(self, model, precision=None, max_batch=16, max_wait_ms=2.0, resize="device", region_size=(256, 256)):
        import torch
        if resize not in ("device", "host"):
            raise ValueError("resize must be 'device' or 'host'")
        region_size = tuple(int(v) for v in region_size)
        if len(region_size) != 2 or any(v < 16 or v % 8 for v in region_size):
            raise ValueError("region_size must be (Hn, Wn), multiples of 8 and at least 16, got %r" % (region_size,))
        self._torch = torch
        self.model = model
        self.precision = precision or getattr(model, "precision", "bf16")
        self.resize = resize
        self.region_size = region_size
        self.engine = model.engine()
        self._pinned = {}              # name -> reused pinned host staging buffer (grown on demand)
        self._sessions = set()         # open EditSessions, closed by close()
        self._sessions_mu = threading.Lock()
        self._closed = False
        self.batcher = RequestBatcher(self._run_batch if resize == "host" else self._run_batch_device, max_batch=max_batch,
                                      max_wait_ms=max_wait_ms)

    def close(self):
        with self._sessions_mu:
            self._closed = True
            sessions = list(self._sessions)
        for sess in sessions:
            sess.close()
        self.batcher.close()
        self._pinned.clear()

    def open_session(self, img, history_bytes=256 << 20):
        """An ``EditSession`` on ``img`` (converted to RGB): with ``resize='device'`` the photo is uploaded once to the engine's
        device and stays there until ``close()``. ``history_bytes`` bounds the bytes its undo snapshots hold.

        ``img`` is a PIL image or the upload's bytes (``bytes``, ``bytearray`` or ``memoryview``); the session on bytes is
        the session on ``Image.open(io.BytesIO(img))``, Pillow's exception included for a file it cannot open. With
        ``resize='device'`` a PNG that ``pngfile.parse`` accepts and that has at least ``engine.PNG_SPLIT_MIN_RAW`` bytes of
        scanlines (about 1200x1200 RGB and up) is decoded across the whole GPU straight into the session's photo
        (``engine.png_decode_into``: only the compressed stream is uploaded, no full-size host array); JPEG, smaller PNG
        files (where Pillow is faster) and every other file go through Pillow."""
        sess = EditSession(self, img, history_bytes)
        with self._sessions_mu:
            closed = self._closed
            if not closed:
                self._sessions.add(sess)
        if closed:
            sess.close()
            raise RuntimeError("DemoProcessor is closed")
        return sess

    def _staging(self, name, nbytes):
        buf = self._pinned.get(name)
        if buf is None or buf.numel() < nbytes:
            buf = self._pinned[name] = self._torch.empty(max(nbytes, 1), dtype=self._torch.uint8, pin_memory=True)
        return buf

    def _run_batch_device(self, key, payloads):
        """payloads: (raw RGB photo [h,w,3] or None, raw 'L' mask [hm,wm], raw 'L' edit mask [he,we] or None, return_mask,
        session photo or None) at their own sizes; key: the floored network size, plus True when the batch runs on edit masks.
        With SOFT in place of True (``EditSession.accept``) each payload ends with a proposal's fp32 soft masks [1,1,H,W] on
        the device, which the batch runs on, and none returns a mask. A PREDICT key is ``_run_predict_device``'s.
        A session's photo ([h,w,3] on the device, with the raw photo None) is resized from where it lies, and the result is
        resized back into it after a snapshot of its previous bytes; its result is then (photo, mask, [snapshot])."""
        if key[-1] == PREDICT:
            return self._run_predict_device(key, payloads)
        if key[0] == "region":
            return self._run_region_device(key, payloads)
        torch = self._torch
        from .engine import _aligned_offsets, resize_u8_packed, resize_window_u8_packed
        H, W = key[:2]
        edit, soft = key[-1] is True, key[-1] == SOFT
        B = len(payloads)
        dev = self.engine.device
        sess = [p[4] for p in payloads]
        sizes = [tuple(p[4].shape[:2]) if p[4] is not None else p[0].shape[:2] for p in payloads]
        photos, masks = [p[0] for p in payloads if p[4] is None], [p[1] for p in payloads]
        edits = [p[2] for p in payloads] if edit else []
        back = [i for i, p in enumerate(payloads) if p[3] and not edit]   # predicted masks to resize back and download
        offs, total = _aligned_offsets([a.nbytes for a in photos + masks + edits])
        photo_at = iter(offs)                       # upload offset of each raw photo, in order
        srcs = [sess[i].view(-1) if sess[i] is not None else None for i in range(B)]
        src_offs = [0 if sess[i] is not None else next(photo_at) for i in range(B)]
        np_ = len(photos)
        out_offs, out_total = _aligned_offsets([h * w * 3 for h, w in sizes] + [sizes[i][0] * sizes[i][1] for i in back])
        stage = self._staging("in", total)          # free: every batch, failed ones included, ends with a stream synchronise
        host = stage.numpy()
        for a, o in zip(photos + masks + edits, offs):
            host[o:o + a.nbytes] = a.reshape(-1)
        down = self._staging("out", out_total)
        snaps = {}
        with torch.cuda.device(dev):
            try:
                src = stage[:total].to(dev, non_blocking=True)
                srcs = [t if t is not None else src for t in srcs]
                img = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
                msk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                resize_window_u8_packed(srcs, src_offs, [w * 3 for _, w in sizes], sizes, [(H, W)] * B, 3, out=img,
                                        dst_offsets=[i * H * W * 3 for i in range(B)])
                # the resized mask goes to the forward as it is: its input codec applies > 0 (demo.py:52)
                resize_u8_packed(src, offs[np_:np_ + B], [a.shape[:2] for a in masks], [(H, W)] * B, 1, out=msk,
                                 dst_offsets=[i * H * W for i in range(B)])
                with torch.no_grad():
                    if edit:
                        edt = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                        resize_u8_packed(src, offs[np_ + B:], [a.shape[:2] for a in edits], [(H, W)] * B, 1, out=edt,
                                         dst_offsets=[i * H * W for i in range(B)])
                        bgr = self.engine.inference_with_mask_u8(img, msk, edt, precision=self.precision)
                    elif soft:
                        slab = self._soft_slab([p[5] for p in payloads], H, W)
                        bgr = self.engine.inference_u8_with_soft_mask(img, msk, slab, precision=self.precision)
                    else:
                        bgr, mk = self.engine.inference_u8(img, msk, precision=self.precision)
                # back to each photo's own size; the forward writes BGR, the demo keeps RGB
                res = torch.empty(max(out_total, 1), device=dev, dtype=torch.uint8)
                resize_u8_packed(bgr, [i * H * W * 3 for i in range(B)], [(H, W)] * B, sizes, 3,
                                 swap_rb=True, out=res, dst_offsets=out_offs[:B])
                for i, t in enumerate(sess):
                    if t is not None:
                        snaps[i] = t.clone()
                        t.view(-1).copy_(res[out_offs[i]:out_offs[i] + t.numel()])
                if back:
                    resize_u8_packed(mk, [i * H * W for i in back], [(H, W)] * len(back), [sizes[i] for i in back], 1,
                                     out=res, dst_offsets=out_offs[B:])
                down[:out_total].copy_(res[:out_total], non_blocking=True)
            finally:
                torch.cuda.current_stream().synchronize()
        host = down.numpy()
        results = [host[o:o + h * w * 3].reshape(h, w, 3).copy() for (h, w), o in zip(sizes, out_offs)]
        masks_back = dict(zip(back, [host[o:o + sizes[i][0] * sizes[i][1]].reshape(sizes[i]).copy()
                                     for i, o in zip(back, out_offs[B:])]))
        return [(r, masks_back.get(i), [snaps[i]]) if i in snaps else (r, masks_back.get(i)) for i, r in enumerate(results)]

    def _run_region_device(self, key, payloads):
        """payloads: (photo crops [bh,bw,3] or None, sketch crops [bh,bw], edit-mask crops [bh,bw] or None, return_mask, boxes,
        session photo or None, feather, photo PIL size, detail): one crop per PIL box of the request, at its box size; key: ("region",
        Hn, Wn), plus True when the batch runs on edit masks. Returns per request one (patch, mask) per box: patch [bh,bw,3] is
        the box's bytes once all of the request's boxes are pasted in order, mask the box's paste mask resized back to [bh,bw]
        (feathered as pasted) when asked for and predicted, else None. A box's feather widths follow from its place in the
        photo (``feather_widths``), wherever it is pasted. A session's request has no photo crops: its boxes are resized from
        its photo ([h,w,3] on the device), snapshotted and pasted into it, and its result is (that list, [previous bytes of
        each box]). With SOFT in place of True (``EditSession.accept``) the edit-mask crops are a proposal's paste masks at
        the working size [H,W], and the payload ends with its fp32 soft masks [k,1,H,W] on the device, which the forward runs
        on; no mask is returned. When a request asks for detail the batch's forward also exports netG's attention and hole
        (``Engine.inference_u8_export``; the same bytes), and that request's boxes are pasted with their detail planes
        (``detail_u8_packed``), computed from the photo before any box of the batch is pasted."""
        torch = self._torch
        from .engine import (_aligned_offsets, detail_u8_packed, feather_u8_packed, resize_composite_u8_packed, resize_u8_packed,
                             resize_window_u8_packed)
        H, W = key[1:3]
        edit, soft = key[-1] is True, key[-1] == SOFT
        dev = self.engine.device
        items = [(r, j) for r, p in enumerate(payloads) for j in range(len(p[4]))]   # (request, box) per box
        B = len(items)
        boxes = [payloads[r][4][j] for r, j in items]
        sizes = [(b[3] - b[1], b[2] - b[0]) for b in boxes]
        sess = [payloads[r][5] for r, _ in items]
        plain = [i for i in range(B) if sess[i] is None]
        photos = {i: payloads[r][0][j] for i, (r, j) in enumerate(items) if sess[i] is None}
        masks = [payloads[r][1][j] for r, j in items]
        edits = [payloads[r][2][j] for r, j in items] if edit or soft else []
        back = [i for i, (r, _) in enumerate(items) if payloads[r][3] and not edit and not soft]   # predicted masks to return
        fw = [feather_widths(boxes[i], payloads[r][7], payloads[r][6]) for i, (r, _) in enumerate(items)]
        det = [i for i, (r, _) in enumerate(items) if payloads[r][8]]   # boxes pasted with detail
        # The work buffer: the plain requests' photo crops (uploaded; a box that overlaps no other box of its request is pasted
        # in place over its crop), the session boxes' patches, the predicted masks resized back (these three are the one
        # download), then the sketch and edit-mask crops (uploaded), then the canvases. A set of overlapping boxes of a plain
        # request is pasted into a canvas, their bounding rectangle, assembled from the crops after the upload; its boxes are
        # then copied back into their crop slots. A session's boxes are pasted into its photo and copied out to their slots.
        slots = plain + [i for i in range(B) if sess[i] is not None] + back
        so, n_down = _aligned_offsets([sizes[i][0] * sizes[i][1] * (3 if k < B else 1) for k, i in enumerate(slots)])
        rgb_at, mask_at = dict(zip(slots[:B], so[:B])), dict(zip(back, so[B:]))
        n_plain = so[len(plain)] if len(plain) < len(slots) else n_down   # the end of the plain crops: the first upload
        mo, m_total = _aligned_offsets([a.nbytes for a in masks + edits])
        sk_at, total = [n_down + o for o in mo], n_down + m_total
        canvas = {}                                   # item -> (canvas offset, pitch, y, x) for boxes in a set of several
        canvas_end, first = total, 0
        for p in payloads:
            rb = p[4]
            for s in (_overlap_sets(rb) if p[5] is None else []):
                if len(s) < 2:
                    continue
                L, U = min(rb[i][0] for i in s), min(rb[i][1] for i in s)
                R, D = max(rb[i][2] for i in s), max(rb[i][3] for i in s)
                for i in s:
                    canvas[first + i] = (canvas_end, (R - L) * 3, rb[i][1] - U, rb[i][0] - L)
                canvas_end += ((D - U) * (R - L) * 3 + 15) // 16 * 16
            first += len(rb)
        stage = self._staging("in", total)          # free: every batch, failed ones included, ends with a stream synchronise
        host = stage.numpy()
        for i, a in photos.items():
            host[rgb_at[i]:rgb_at[i] + a.nbytes] = a.reshape(-1)
        for a, o in zip(masks + edits, sk_at):
            host[o:o + a.nbytes] = a.reshape(-1)
        down = self._staging("out", n_down)
        net3, net1 = [i * H * W * 3 for i in range(B)], [i * H * W for i in range(B)]

        def crop_slot(work, i):
            return work[rgb_at[i]:rgb_at[i] + sizes[i][0] * sizes[i][1] * 3].view(*sizes[i], 3)

        def in_canvas(work, i):                       # item i's box in its canvas, and its crop slot, as [bh,bw,3] views
            co, pitch, y, x = canvas[i]
            bh, bw = sizes[i]
            rows = work[co:co + (y + bh) * pitch].view(y + bh, pitch)
            return rows[y:, x * 3:(x + bw) * 3].view(bh, bw, 3), crop_slot(work, i)

        def in_photo(i):                              # a session item's box in its photo, as a [bh,bw,3] view
            left, upper, right, lower = boxes[i]
            return sess[i][upper:lower, left:right]

        snaps = {}
        with torch.cuda.device(dev):
            try:
                work = torch.empty(canvas_end, device=dev, dtype=torch.uint8)
                if n_plain:
                    work[:n_plain].copy_(stage[:n_plain], non_blocking=True)
                work[n_down:total].copy_(stage[n_down:total], non_blocking=True)
                for i in canvas:                      # 2-D copies; overlapping crops hold the same photo bytes
                    dst, crop = in_canvas(work, i)
                    dst.copy_(crop)
                img = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
                msk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                # the photo crops: plain ones from their upload slots, a session's as windows of its photo
                srcs = [work if sess[i] is None else sess[i].view(-1) for i in range(B)]
                src_offs = [rgb_at[i] if sess[i] is None else (boxes[i][1] * sess[i].shape[1] + boxes[i][0]) * 3 for i in range(B)]
                pitches = [sizes[i][1] * 3 if sess[i] is None else sess[i].shape[1] * 3 for i in range(B)]
                resize_window_u8_packed(srcs, src_offs, pitches, sizes, [(H, W)] * B, 3, out=img, dst_offsets=net3)
                resize_u8_packed(work, sk_at[:B], sizes, [(H, W)] * B, 1, out=msk, dst_offsets=net1)
                pm_at = net1                          # the paste masks: pm at pm_at[i]
                with torch.no_grad():
                    if edit:
                        pm = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                        resize_u8_packed(work, sk_at[B:], sizes, [(H, W)] * B, 1, out=pm, dst_offsets=net1)
                        if det:
                            bgr, _, attn, hole = self.engine.inference_u8_export(img, msk, edit_mask_u8=pm, precision=self.precision)
                        else:
                            bgr = self.engine.inference_with_mask_u8(img, msk, pm, precision=self.precision)
                    elif soft:                        # the proposal's mask bytes were uploaded at the working size
                        pm, pm_at = work, sk_at[B:]
                        slab = self._soft_slab([p[9] for p in payloads], H, W)
                        if det:
                            bgr, _, attn, hole = self.engine.inference_u8_export(img, msk, edit_mask=slab, precision=self.precision)
                        else:
                            bgr = self.engine.inference_u8_with_soft_mask(img, msk, slab, precision=self.precision)
                    elif det:
                        bgr, pm, attn, hole = self.engine.inference_u8_export(img, msk, precision=self.precision)
                    else:
                        bgr, pm = self.engine.inference_u8(img, msk, precision=self.precision)
                D = d_at = None
                if det:                               # from the photo's bytes, before any box is pasted
                    low, low_at = resize_u8_packed(img, [net3[i] for i in det], [(H, W)] * len(det), [sizes[i] for i in det], 3)
                    L = attn.shape[1]
                    D, d_offs, _ = detail_u8_packed([srcs[i] for i in det], [src_offs[i] for i in det], [pitches[i] for i in det],
                                                    [sizes[i] for i in det], (H, W), low, low_at, hole, [net1[i] for i in det],
                                                    attn, [i * L * L for i in det])
                    d_at = dict(zip(det, d_offs))
                for i in range(B):
                    if sess[i] is not None:
                        snaps[i] = in_photo(i).clone()
                groups = [plain] if plain else []     # one composite for the plain boxes, one per session
                groups += [[i for i in range(B) if items[i][0] == r] for r, p in enumerate(payloads) if p[5] is not None]
                for g in groups:
                    if sess[g[0]] is None:
                        place = [canvas.get(i, (rgb_at[i], sizes[i][1] * 3, 0, 0)) for i in g]
                        target = work
                    else:
                        place = [(0, sess[i].shape[1] * 3, boxes[i][1], boxes[i][0]) for i in g]
                        target = sess[g[0]].view(-1)
                    gd = D is not None and any(i in d_at for i in g)
                    resize_composite_u8_packed(bgr, [net3[i] for i in g], pm, [pm_at[i] for i in g], [(H, W)] * len(g), target,
                                               [c[0] for c in place], [c[1] for c in place], [c[2:] for c in place],
                                               [sizes[i] for i in g], swap_rb=True,
                                               feather=[fw[i] for i in g] if any(any(fw[i]) for i in g) else None,
                                               detail=D if gd else None, detail_offsets=[d_at.get(i, -1) for i in g] if gd else None)
                for i in canvas:
                    src, crop = in_canvas(work, i)
                    crop.copy_(src)
                for i in snaps:
                    crop_slot(work, i).copy_(in_photo(i))
                if back:
                    resize_u8_packed(pm, [net1[i] for i in back], [(H, W)] * len(back), [sizes[i] for i in back], 1, out=work,
                                     dst_offsets=[mask_at[i] for i in back])
                    fb = [i for i in back if any(fw[i])]
                    if fb:                            # the masks as pasted
                        feather_u8_packed(work, [mask_at[i] for i in fb], [sizes[i] for i in fb], [fw[i] for i in fb])
                down[:n_down].copy_(work[:n_down], non_blocking=True)
            finally:
                torch.cuda.current_stream().synchronize()
        host = down.numpy()
        out = [[] for _ in payloads]
        for i, (r, _) in enumerate(items):
            (h, w), o = sizes[i], rgb_at[i]
            m = host[mask_at[i]:mask_at[i] + h * w].reshape(h, w).copy() if i in mask_at else None
            out[r].append((host[o:o + h * w * 3].reshape(h, w, 3).copy(), m))
        return [(o, [snaps[i] for i in range(B) if items[i][0] == r]) if p[5] is not None else o
                for r, (o, p) in enumerate(zip(out, payloads))]

    def _run_predict_device(self, key, payloads):
        """The mask-only forward of ``predict_mask`` and ``EditSession.propose``. payloads: (photo crops [bh,bw,3] or None,
        sketch crops, boxes, session photo or None, feather, photo PIL size); key: the working size (the floored photo size, or
        ("region", Hn, Wn)) and PREDICT. A whole-photo request is the one box (0, 0, w, h) with its sketch at its own size.
        Each crop is resized to the working size like the edit's (a session's from its photo), and each box's predicted mask
        is resized back to the box and feathered as the edit pastes it. Returns per request (fp32 soft masks [k,1,H,W] on the
        device, mask bytes [k,H,W], [the box's paste mask [bh,bw] per box])."""
        torch = self._torch
        from .engine import _aligned_offsets, feather_u8_packed, resize_u8_packed, resize_window_u8_packed
        H, W = key[-3:-1]
        dev = self.engine.device
        items = [(r, j) for r, p in enumerate(payloads) for j in range(len(p[2]))]
        B = len(items)
        boxes = [payloads[r][2][j] for r, j in items]
        sizes = [(b[3] - b[1], b[2] - b[0]) for b in boxes]
        sess = [payloads[r][3] for r, _ in items]
        photos = [payloads[r][0][j] for r, j in items if payloads[r][3] is None]
        sketches = [payloads[r][1][j] for r, j in items]
        fw = [feather_widths(boxes[i], payloads[r][5], payloads[r][4]) for i, (r, _) in enumerate(items)]
        offs, total = _aligned_offsets([a.nbytes for a in photos + sketches])
        photo_at = iter(offs)
        net3, net1 = [i * H * W * 3 for i in range(B)], [i * H * W for i in range(B)]
        back, n_down = _aligned_offsets([B * H * W] + [h * w for h, w in sizes])   # the working-size bytes, then the masks
        back = back[1:]
        stage = self._staging("in", total)          # free: every batch, failed ones included, ends with a stream synchronise
        host = stage.numpy()
        for a, o in zip(photos + sketches, offs):
            host[o:o + a.nbytes] = a.reshape(-1)
        down = self._staging("out", n_down)
        with torch.cuda.device(dev):
            try:
                src = stage[:total].to(dev, non_blocking=True)
                img = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
                msk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                srcs = [src if t is None else t.view(-1) for t in sess]
                src_offs = [next(photo_at) if t is None else (b[1] * t.shape[1] + b[0]) * 3 for t, b in zip(sess, boxes)]
                pitches = [w * 3 if t is None else t.shape[1] * 3 for t, (_, w) in zip(sess, sizes)]
                resize_window_u8_packed(srcs, src_offs, pitches, sizes, [(H, W)] * B, 3, out=img, dst_offsets=net3)
                resize_u8_packed(src, offs[len(photos):], [a.shape[:2] for a in sketches], [(H, W)] * B, 1, out=msk,
                                 dst_offsets=net1)
                with torch.no_grad():
                    soft, mk = self.engine.predict_mask_u8(img, msk, precision=self.precision)
                res = torch.empty(n_down, device=dev, dtype=torch.uint8)
                res[:B * H * W].copy_(mk.view(-1))
                resize_u8_packed(mk, net1, [(H, W)] * B, sizes, 1, out=res, dst_offsets=back)
                fb = [i for i in range(B) if any(fw[i])]
                if fb:                                # the masks as pasted
                    feather_u8_packed(res, [back[i] for i in fb], [sizes[i] for i in fb], [fw[i] for i in fb])
                down[:n_down].copy_(res, non_blocking=True)
                ends = np.cumsum([len(p[2]) for p in payloads]).tolist()
                kept = [soft[e - len(p[2]):e].clone() for e, p in zip(ends, payloads)]   # each proposal holds its own
            finally:
                torch.cuda.current_stream().synchronize()
        host = down.numpy()
        work = host[:B * H * W].reshape(B, H, W)
        masks = [host[o:o + h * w].reshape(h, w).copy() for o, (h, w) in zip(back, sizes)]
        return [(k, work[e - len(p[2]):e].copy(), masks[e - len(p[2]):e]) for k, e, p in zip(kept, ends, payloads)]

    def _soft_slab(self, softs, H, W):
        """The requests' fp32 soft masks [k,1,H,W], in order, gathered into one [B,1,H,W] tensor by device copies."""
        torch = self._torch
        slab = torch.empty(sum(len(t) for t in softs), 1, H, W, device=self.engine.device, dtype=torch.float32)
        at = 0
        for t in softs:
            slab[at:at + len(t)].copy_(t)
            at += len(t)
        return slab

    def _run_masks_host(self, key, payloads):
        """The host flow's PREDICT and SOFT batches. payloads: (photos [k,H,W,3], masks [k,H,W]), plus for SOFT the fp32 soft
        masks [k,1,H,W] on the device. Results: PREDICT (soft masks [k,1,H,W] on the device, mask bytes [k,H,W]), SOFT
        rgb [k,H,W,3]."""
        torch = self._torch
        dev = self.engine.device
        ends = np.cumsum([len(p[0]) for p in payloads]).tolist()
        with torch.cuda.device(dev):
            img = torch.from_numpy(np.concatenate([p[0] for p in payloads])).to(dev, non_blocking=True)
            msk = torch.from_numpy(np.concatenate([p[1] for p in payloads])).to(dev, non_blocking=True)
            with torch.no_grad():
                if key[-1] == PREDICT:
                    soft, mk = self.engine.predict_mask_u8(img, msk, precision=self.precision)
                    mk = mk.cpu().numpy()
                    return [(soft[e - len(p[0]):e].clone(), mk[e - len(p[0]):e]) for e, p in zip(ends, payloads)]
                bgr = self.engine.inference_u8_with_soft_mask(img, msk, self._soft_slab([p[2] for p in payloads], *msk.shape[1:]),
                                                              precision=self.precision)
            rgb = bgr.cpu().numpy()[..., ::-1]
        return [np.ascontiguousarray(rgb[e - len(p[0]):e]) for e, p in zip(ends, payloads)]

    def _run_batch(self, key, payloads):
        """payloads: (photo [H,W,3], mask [H,W], edit mask [H,W] or None, return_mask) at the network size of ``key`` (the
        floored size), or for a region key (photos [k,H,W,3], masks [k,H,W], edit masks [k,H,W] or None, return_mask) with one
        item per box at the working size, and then each result is (rgb [k,H,W,3], mask [k,H,W] or None); True as the key's
        last element: the batch runs on edit masks. PREDICT or SOFT there: ``_run_masks_host``."""
        if key[-1] in (PREDICT, SOFT):
            return self._run_masks_host(key, payloads)
        torch = self._torch
        join = np.concatenate if key[0] == "region" else np.stack
        img = torch.from_numpy(join([p[0] for p in payloads])).cuda(non_blocking=True)         # [B,H,W,3] RGB uint8
        msk = torch.from_numpy(join([p[1] for p in payloads])).cuda(non_blocking=True)         # [B,H,W] uint8 (> 0 = stroke)
        mk = None
        with torch.no_grad():
            if key[-1] is True:
                edt = torch.from_numpy(join([p[2] for p in payloads])).cuda(non_blocking=True)
                bgr = self.engine.inference_with_mask_u8(img, msk, edt, precision=self.precision)
            else:
                bgr, mk = self.engine.inference_u8(img, msk, precision=self.precision)
        rgb = bgr.cpu().numpy()[..., ::-1]                                                     # demo.py keeps RGB (test.py swaps to BGR)
        mk = mk.cpu().numpy() if mk is not None else None
        if key[0] == "region":
            ends = np.cumsum([len(p[0]) for p in payloads])
            return [(np.ascontiguousarray(rgb[e - len(p[0]):e]), mk[e - len(p[0]):e] if mk is not None and p[3] else None)
                    for e, p in zip(ends, payloads)]
        return [(np.ascontiguousarray(rgb[i]), mk[i] if mk is not None and p[3] else None) for i, p in enumerate(payloads)]

    def process_image(self, img, mask, edit_mask=None, return_mask=False, region=None, feather=0, detail=False):
        """img: PIL image; mask: PIL 'L' image, usually of the same size (non-zero = sketch stroke). Returns the edited PIL
        image at the input's size. Sizes are floored to a multiple of 8 for the network exactly like demo.py:43.

        edit_mask: PIL 'L' image of any size that replaces the predicted edit mask (mask revising): resized to the floored
        size like the sketch mask, v/255 blends the result and v >= 128 is inpainted. return_mask=True returns
        ``(result, mask)``: the predicted mask as an 'L' image at the photo's size (resized back like the result), or
        ``edit_mask`` itself when one was given.

        region: None edits the whole photo as above. A PIL box ``(left, upper, right, lower)`` of integers, or 'auto' for
        ``region_box`` around the strokes (and the edit mask's non-zero pixels), runs a region edit: the box is cropped, resized
        to ``region_size``, edited, resized back and pasted with the edit mask (predicted or given) resized back to the box,
        exactly as Pillow's ``out = img.copy(); out.paste(res, box, m)``. Pixels outside the box are the photo's own; strokes
        outside it are ignored. mask and edit_mask must then have the photo's size. Region requests on photos of any size
        share forwards. With return_mask=True a predicted mask comes back at the photo's size, zero outside the box.

        A list of PIL boxes, or 'strokes' for one box per stroke group (``region_groups``), edits several regions in one
        forward. Every crop is taken from the photo itself and the results are pasted in the list's order, exactly as
        ``out = img.copy()`` followed by the single-box paste of each box into ``out``; a later box blends over an earlier one
        where they overlap. The returned predicted mask is then the largest of the boxes' paste masks at each pixel.

        feather: an int >= 0 (photo pixels, default 0). A region edit pastes each box with ``feather_mask(m, widths)`` in place
        of its paste mask m, ``widths = feather_widths(box, img.size, feather)``: the mask fades to 0 over a band along the box
        edges inside the photo, while edges on the photo's border stay hard. A predicted mask is returned as pasted (feathered);
        a given edit_mask is returned as given. 0 pastes exactly as without it. It does not change the forward, so requests
        with different values share forwards. region=None has no inner edges: feather is checked and has no effect.

        detail: False (default) or True, for region edits with resize='device'. The network sees each box resampled to the
        working size, so the pasted result is an upsample without the photo's fine detail. True adds it back inside the hole
        (contextual residual aggregation): the detail the resize round trip removes from the photo, zero in the hole, is
        gathered into each hole patch with the softmax weights netG's contextual attention computed, and added to the
        resized result before the paste (DESIGN.md section 7b). False pastes exactly as without it. It needs a model with the
        contextual attention (use_cam) and boxes of at least 1/32 of the working size per side (``detail_box_ok``); requests
        that do not meet this raise ValueError before they are queued. It changes no forward
        output, so requests with and without it share forwards; a batch with any detail request runs the forward that also
        returns the attention weights, 4 L^2 bytes per box (L = (Hn/8 - 1)(Wn/8 - 1): 3.7 MB at 256 x 256, 63 MB at
        512 x 512), held until the batch ends, and runs the attention in one band, so its L x L workspace is not held to
        ``engine.set_attention_workspace_limit``; each detail box takes transient scratch (``engine.detail_u8_packed``).
        Whether it looks better needs trained weights to judge. With region=None or resize='host' it is a ValueError."""
        from PIL import Image
        feather = _check_feather(feather)
        detail = self._check_detail(detail, region is None)
        img = img.convert("RGB")
        if region is not None:
            return self._process_region(img, mask, edit_mask, return_mask, region, feather, detail)
        w_raw, h_raw = img.size
        h_t, w_t = floor8(h_raw), floor8(w_raw)
        if h_t < 16 or w_t < 16:
            raise ValueError("image smaller than 16x16 (two stride-2 convolutions, 4x4 mask pool, stride-2 patch grid)")
        # requests on edit masks run their own forward: a batch never mixes them with predicted-mask requests
        key = (h_t, w_t) if edit_mask is None else (h_t, w_t, True)
        if self.resize == "device":
            for m, nm in ((mask, "mask"), (edit_mask, "edit_mask")):
                if m is not None and m.mode != "L":
                    raise ValueError("resize='device' takes an 'L' %s (got mode %r); resize='host' resizes it with Pillow" % (nm, m.mode))
            edit_raw = np.asarray(edit_mask) if edit_mask is not None else None
            out, mk = self.batcher.submit(key, (np.asarray(img), np.asarray(mask), edit_raw, return_mask, None))
            res = Image.fromarray(out)
            mk = Image.fromarray(mk) if mk is not None else None
        else:
            img_t = np.ascontiguousarray(np.array(img.resize((w_t, h_t))), dtype=np.uint8)
            mask_t = np.array(mask.resize((w_t, h_t)))
            mask_t = np.ascontiguousarray((mask_t > 0).astype(np.uint8) * 255)
            edit_t = np.ascontiguousarray(np.array(edit_mask.convert("L").resize((w_t, h_t))), dtype=np.uint8) if edit_mask is not None else None
            out, mk = self.batcher.submit(key, (img_t, mask_t, edit_t, return_mask))
            res = Image.fromarray(out).resize((w_raw, h_raw))
            mk = Image.fromarray(mk).resize((w_raw, h_raw)) if mk is not None else None
        if not return_mask:
            return res
        return res, (edit_mask if edit_mask is not None else mk)

    def _region_boxes(self, size, mask, edit_mask, region, offset=(0, 0)):
        """The PIL boxes of a region edit of a photo of PIL size ``size``; the masks lie at ``offset`` in it."""
        w, h = size
        dx, dy = offset
        if isinstance(region, str):
            if region == "strokes":
                return [box for _, box in region_groups(mask, edit_mask, self.region_size, size, offset)]
            if region != "auto":
                raise ValueError("region must be None, 'auto', 'strokes', a PIL box or a list of PIL boxes, got %r" % region)
            bbs = [b for b in (mask.getbbox(), edit_mask.getbbox() if edit_mask is not None else None) if b]
            if not bbs:
                raise ValueError("region='auto' needs a sketch stroke or a non-zero edit mask")
            return [region_box((min(b[0] for b in bbs) + dx, min(b[1] for b in bbs) + dy, max(b[2] for b in bbs) + dx,
                                max(b[3] for b in bbs) + dy), size, self.region_size)]
        if isinstance(region, list) and not region:
            raise ValueError("region=[] is empty: give at least one PIL box")
        if isinstance(region, (list, tuple)) and all(isinstance(b, (list, tuple)) for b in region):   # a list of boxes
            return [_check_box(b, w, h) for b in region]
        return [_check_box(region, w, h)]

    def predict_mask(self, img, mask, region=None, feather=0):
        """The edit mask ``process_image(img, mask, region=region, return_mask=True, feather=feather)[1]`` returns, bit for
        bit, from netM alone (``Engine.predict_mask_u8``): netG does not run and no image is made, for about a quarter of the
        forward's arithmetic. Takes the arguments, and raises the errors, of ``process_image`` without an edit mask. Requests
        share mask-only forwards with each other and with ``EditSession.propose``, never with edits."""
        from PIL import Image
        feather = _check_feather(feather)
        img = img.convert("RGB")
        w, h = img.size
        if region is None:
            if floor8(h) < 16 or floor8(w) < 16:
                raise ValueError("image smaller than 16x16 (two stride-2 convolutions, 4x4 mask pool, stride-2 patch grid)")
            if self.resize == "device" and mask.mode != "L":
                raise ValueError("resize='device' takes an 'L' mask (got mode %r); resize='host' resizes it with Pillow" % mask.mode)
            return self._predict(img, None, mask, [(0, 0, w, h)], True, 0, img.size, (0, 0))[2][0]
        self._check_region_masks(img.size, mask, None)
        boxes = self._region_boxes(img.size, mask, None, region)
        return Image.fromarray(_union_mask(img.size, boxes, self._predict(img, None, mask, boxes, False, feather, img.size, (0, 0))[2]))

    def _predict(self, img, photo, mask, boxes, whole, feather, size, offset):
        """The mask-only forward of a request: ``(soft, work, masks, inputs)``. ``soft``: the fp32 soft masks [k,1,H,W] on the
        engine's device, one per box at the working size; ``work``: their bytes [k,H,W] (the device flow's paste masks at
        the working size); ``masks``: the 'L' paste mask per box at the box's size (feathered) or, ``whole``, at the photo's;
        ``inputs``: what ``EditSession.accept`` submits again (the device flow: the sketch crops; the host flow: the resized
        photo and sketch). The photo is the PIL ``img`` or, with the device flow of a session, ``photo`` on the device; the
        mask lies at ``offset`` in a photo of PIL size ``size``."""
        from PIL import Image
        w, h = size
        key = (floor8(h), floor8(w), PREDICT) if whole else ("region",) + self.region_size + (PREDICT,)
        if self.resize == "device":
            at = [(b[0] - offset[0], b[1] - offset[1], b[2] - offset[0], b[3] - offset[1]) for b in boxes]   # mask coordinates
            sketches = [np.asarray(mask)] if whole else [np.asarray(mask.crop(b)) for b in at]
            crops = None if photo is not None else [np.asarray(img)] if whole else [np.asarray(img.crop(b)) for b in boxes]
            soft, work, mks = self.batcher.submit(key, (crops, sketches, boxes, photo, feather, size))
            return soft, work, [Image.fromarray(m) for m in mks], sketches
        if whole:
            h_t, w_t = key[:2]
            img_t = np.ascontiguousarray(np.array(img.resize((w_t, h_t))), dtype=np.uint8)[None]
            mask_t = np.ascontiguousarray((np.array(mask.resize((w_t, h_t))) > 0).astype(np.uint8) * 255)[None]
            soft, mk = self.batcher.submit(key, (img_t, mask_t))
            return soft, mk, [Image.fromarray(mk[0]).resize(size)], (img_t, mask_t)
        Hn, Wn = self.region_size
        fm = _placed(mask, size, offset)
        img_t = np.stack([np.array(img.crop(b).resize((Wn, Hn))) for b in boxes]).astype(np.uint8)
        mask_t = np.stack([(np.array(fm.crop(b).resize((Wn, Hn))) > 0).astype(np.uint8) * 255 for b in boxes])
        soft, mk = self.batcher.submit(key, (img_t, mask_t))
        mks = [Image.fromarray(mk[i]).resize((b[2] - b[0], b[3] - b[1])) for i, b in enumerate(boxes)]
        if feather:
            mks = [Image.fromarray(feather_mask(m, feather_widths(b, size, feather))) for m, b in zip(mks, boxes)]
        return soft, mk, mks, (img_t, mask_t)

    def _check_region_masks(self, size, mask, edit_mask):
        w, h = size
        for m, nm in ((mask, "mask"), (edit_mask, "edit_mask")):
            if m is not None and m.size != size:
                raise ValueError("a region edit needs the %s at the photo's size %dx%d (got %dx%d)" % ((nm, w, h) + m.size))
            if self.resize == "device" and m is not None and m.mode != "L":
                raise ValueError("resize='device' takes an 'L' %s (got mode %r); resize='host' resizes it with Pillow" % (nm, m.mode))

    def _process_region(self, img, mask, edit_mask, return_mask, region, feather=0, detail=False):
        from PIL import Image
        self._check_region_masks(img.size, mask, edit_mask)
        boxes = self._region_boxes(img.size, mask, edit_mask, region)
        if detail:
            _check_detail_boxes(boxes, self.region_size)
        if self.resize == "device":
            out = img.copy()
            crops = [np.asarray(img.crop(b)) for b in boxes]
            sketches = [np.asarray(mask.crop(b)) for b in boxes]
            edits = [np.asarray(edit_mask.crop(b)) for b in boxes] if edit_mask is not None else None
            got = self.batcher.submit(self._region_key(edit_mask),
                                      (crops, sketches, edits, return_mask, boxes, None, feather, img.size, detail))
            for b, (patch, _) in zip(boxes, got):        # in order: a later patch holds the final bytes where boxes overlap
                out.paste(Image.fromarray(patch), b[:2])
            mks = [Image.fromarray(mk) if mk is not None else None for _, mk in got]
        else:
            out, mks = self._region_host(img, mask, edit_mask, boxes, feather)
        if not return_mask:
            return out
        if edit_mask is not None:
            return out, edit_mask
        return out, Image.fromarray(_union_mask(img.size, boxes, mks))

    def _check_detail(self, detail, region_none):
        return _check_detail(detail, region_none, self.resize == "host", getattr(self.engine, "use_cam", True))

    def _region_key(self, edit_mask):
        # region requests on edit masks run their own forward, and region requests never share one with whole-photo requests
        Hn, Wn = self.region_size
        return ("region", Hn, Wn) if edit_mask is None else ("region", Hn, Wn, True)

    def _region_host(self, img, mask, edit_mask, boxes, feather=0):
        """The Pillow flow of a region edit: ``(out, paste masks)``, one 'L' paste mask per box at the box's size (feathered
        with ``feather_widths(box, img.size, feather)``). ``edit_mask`` may also be a list of each box's edit mask."""
        from PIL import Image
        Hn, Wn = self.region_size
        sizes = [(b[2] - b[0], b[3] - b[1]) for b in boxes]
        out = img.copy()
        img_t = np.stack([np.array(img.crop(b).resize((Wn, Hn))) for b in boxes]).astype(np.uint8)
        mask_t = np.stack([(np.array(mask.crop(b).resize((Wn, Hn))) > 0).astype(np.uint8) * 255 for b in boxes])
        if edit_mask is not None:
            ems = edit_mask if isinstance(edit_mask, list) else [edit_mask.convert("L").crop(b) for b in boxes]
        edit_t = np.stack([np.array(e.convert("L").resize((Wn, Hn))) for e in ems]).astype(np.uint8) \
            if edit_mask is not None else None
        res, mk = self.batcher.submit(self._region_key(edit_mask), (img_t, mask_t, edit_t, True))
        mks = [Image.fromarray(edit_t[i] if edit_t is not None else mk[i]).resize(s) for i, s in enumerate(sizes)]
        if feather:
            mks = [Image.fromarray(feather_mask(m, feather_widths(b, img.size, feather))) for m, b in zip(mks, boxes)]
        for i, (b, s) in enumerate(zip(boxes, sizes)):   # every crop above came from the photo, not from `out`
            out.paste(Image.fromarray(res[i]).resize(s), b, mks[i])
        return out, mks


EditResult = namedtuple("EditResult", ["boxes", "patches", "masks"])

# last element of the batch keys of mask-only forwards (``predict_mask``, ``EditSession.propose``) and of forwards on a
# proposal's fp32 soft masks (``EditSession.accept``): neither shares a forward with an edit
PREDICT, SOFT = "predict", "soft"


def _union_mask(size, boxes, mks):
    """The largest of the boxes' paste masks at each pixel of a photo of PIL size ``size``, 0 outside every box, [h,w]."""
    w, h = size
    full = np.zeros((h, w), np.uint8)
    for b, mk in zip(boxes, mks):
        sub = full[b[1]:b[3], b[0]:b[2]]
        np.maximum(sub, np.asarray(mk), out=sub)
    return full


def _placed(m, size, offset):
    """m as a PIL 'L' image of PIL size ``size``: placed at ``offset`` and zero elsewhere."""
    if m is None or (m.size == tuple(size) and tuple(offset) == (0, 0)):
        return m
    from PIL import Image
    full = Image.new("L", tuple(size), 0)
    full.paste(m, tuple(offset))
    return full


class EditSession:
    """A photo kept across a chain of edits, each drawn on the result of the one before, with undo
    (``DemoProcessor.open_session``). ``edit(...)`` is

        cur = proc.process_image(cur, mask, edit_mask, region=region, feather=feather)

    with ``cur`` starting as the photo in RGB, and returns ``EditResult(boxes, patches, masks)``: the edit's PIL boxes in
    paste order (``region=None``: the whole photo), ``patches[i] = cur.crop(boxes[i])`` after the edit, and ``masks[i]`` the
    box's paste mask (feathered as pasted) as an 'L' image when ``return_mask`` is set and the mask was predicted, else None. Outside the union of
    the boxes ``cur`` keeps the previous photo's bytes.

    ``mask`` and ``edit_mask`` are 'L' images of one size, placed at ``offset = (x, y)`` in the photo and zero elsewhere: the
    boxes and bytes are those of the zero-padded photo-sized masks, without building them (``region=None`` takes photo-sized
    masks at (0, 0)). ``undo()`` restores the photo from before the last edit not yet undone, exactly; its snapshots hold the
    previous bytes of each edit's boxes and are dropped oldest first to keep within ``history_bytes``. Edits of one session run
    one at a time; edits of several sessions share forwards with each other and with ``process_image`` requests of their
    batch key.

    With ``resize='device'`` the photo lives on the engine's device: an edit uploads only the masks' box crops, resizes the
    photo's boxes where they lie (``engine.resize_window_u8_packed``), pastes the results into the photo and downloads only the
    patches; undo snapshots stay on the device. With ``resize='host'`` the session holds a PIL image and runs the Pillow flow.

    ``propose(mask, ...)`` previews an edit: the boxes and paste masks ``edit`` would use, from netM alone. ``accept(p)`` then
    runs that edit on netM's exact fp32 masks (the same bytes as ``edit``), or ``accept(p, edit_masks=...)`` on the user's
    corrections. Any ``edit``, ``undo``, ``accept`` or ``close`` of the session invalidates its open proposals."""

    def __init__(self, proc, img, history_bytes):
        if int(history_bytes) < 0:
            raise ValueError("history_bytes must be >= 0")
        self._proc = proc
        self._mu = threading.Lock()
        self._history = deque()         # (boxes, previous bytes of each box, bytes held), oldest first
        self._held = 0
        self.history_bytes = int(history_bytes)
        # what jpeg(quality="keep", exif=s.exif, icc_profile=s.icc_profile) keeps of the upload, read before the conversion
        self._keep = None               # a JPEG upload's (quantisation tables, JpegImagePlugin.get_sampling)
        self._exif, self._icc_profile = b"", None
        self._img = self._photo = None
        self._proposals = set()         # open proposals, computed on the current photo
        head = None
        if isinstance(img, (bytes, bytearray, memoryview)):   # the upload's bytes: Image.open(io.BytesIO(img)) below
            img = bytes(img)
            if proc.resize == "device":
                from . import engine, pngfile
                try:
                    head = pngfile.parse(img)
                except pngfile.Host:
                    pass
                if head is not None and engine.png_raw_bytes(head) < engine.PNG_SPLIT_MIN_RAW:
                    head = None   # below the split decoder's size Pillow is faster (DESIGN.md 7b)
            if head is None:
                import io

                from PIL import Image
                img = Image.open(io.BytesIO(img))
        if head is not None:   # a PNG the device decodes; it has no EXIF or ICC chunk (pngfile sends those to Pillow)
            self.size = (head.w, head.h)
            self._photo = self._decode_png(img, head)
        else:
            if getattr(img, "format", None) == "JPEG" and getattr(img, "quantization", None):
                from PIL import JpegImagePlugin
                self._keep = (dict(img.quantization), JpegImagePlugin.get_sampling(img))
            self._exif = img.info.get("exif", b"")
            self._icc_profile = img.info.get("icc_profile")
            img = img.convert("RGB")
            self.size = img.size
            if proc.resize == "host":
                self._img = img
            else:
                torch = proc._torch
                w, h = img.size
                self._photo = torch.empty(h, w, 3, device=proc.engine.device, dtype=torch.uint8)
                self._photo.copy_(torch.from_numpy(np.array(img)))
        self._closed = False

    def _check_open(self):
        if self._closed:
            raise RuntimeError("EditSession is closed")

    def _decode_png(self, data, head):
        """The photo of the PNG upload ``data`` (``pngfile.parse`` gave ``head``) in a new tensor on the engine's device:
        its stream staged in pinned memory and decoded there (``engine.png_decode_into``), no full-size host array; the host
        reads the status once, and a file the device refuses is decoded by Pillow (its exception included) into the tensor."""
        from . import engine
        torch = self._proc._torch
        dev = self._proc.engine.device
        with torch.cuda.device(dev):
            photo = torch.empty(head.h, head.w, 3, device=dev, dtype=torch.uint8)
            engine.png_decode_into(engine.png_stage([head]), [head], ["RGB"], [data], [(photo.view(-1), 0, (head.h, head.w))],
                                   ["the upload"], dev)
        return photo

    @property
    def exif(self):
        """The upload's EXIF block (its ``info["exif"]``), or ``b""``: ``jpeg(exif=s.exif)`` carries it into the file. Its
        contents are not rewritten, so an IFD1 thumbnail in it still shows the unedited photo."""
        return self._exif

    @property
    def icc_profile(self):
        """The upload's ICC profile (its ``info["icc_profile"]``), or None: ``jpeg(icc_profile=s.icc_profile)`` carries it."""
        return self._icc_profile

    def close(self):
        """Releases the photo and the snapshots (idempotent); also run by ``DemoProcessor.close()``."""
        with self._mu:
            self._closed = True
            self._drop_proposals()
            self._img = self._photo = None
            self._history.clear()
            self._held = 0
        with self._proc._sessions_mu:
            self._proc._sessions.discard(self)

    def image(self, size=None):
        """The current photo as a PIL RGB image. ``size = (width, height)`` gives a preview instead: the photo as
        ``Image.thumbnail(size)`` leaves a copy of it (Pillow 12.2: BICUBIC, reducing_gap=2.0), at most ``size`` and with its
        aspect ratio kept; a photo that already fits comes back whole. With ``resize='device'`` the preview is made on the
        device (``engine.thumbnail_u8``) and only it is downloaded."""
        from PIL import Image
        size = self._size(size)
        with self._mu:
            self._check_open()
            if self._img is not None:
                img = self._host_image(None, size)
                return img.copy() if img is self._img else img
            with self._proc._torch.cuda.device(self._photo.device):
                return Image.fromarray(self._pixels(None, size).cpu().numpy())

    def jpeg(self, quality=75, subsampling=2, box=None, optimize=False, progressive=False, size=None, exif=b"",
             icc_profile=None):
        """The current photo, or its PIL box ``(left, upper, right, lower)``, as a JPEG file: the bytes of

            img = s.image().crop(box);  img.thumbnail(size)
        buf = io.BytesIO();  img.save(buf, "JPEG", quality=quality, subsampling=subsampling, optimize=optimize,
                                      progressive=progressive)

        (no crop when ``box`` is None, no thumbnail when ``size`` is None). ``size = (width, height)`` makes a preview:
        the photo or box scaled down to fit ``size`` as ``Image.thumbnail`` does (Pillow 12.2: BICUBIC, reducing_gap=2.0);
        one that already fits is encoded whole. On the device the preview is made from the photo where it lies into a
        small buffer (``engine.thumbnail_u8``, about 6 MB of transient memory for a 4000x2667 photo to 640x427) and
        encoded there, so the encode's memory follows the preview's size (about 5 MB at 640x427, 4:2:0). ``quality`` in [1, 100]; ``subsampling`` 0 (4:4:4) or 2 (4:2:0, Pillow's default);
        ``optimize`` a bool: True builds Huffman tables for the image, a smaller file of the same pixels. Pillow fails
        (OSError) to write an optimized file larger than its buffer of max(64 KiB, w h) bytes (2 w h from quality 95 on),
        as a noisy photo at quality 90, 4:4:4 can be; the device encode still writes the file, the one Pillow writes
        with a larger buffer. ``progressive`` a bool: True writes a progressive file (ten scans, each with its own optimal
        tables, whatever ``optimize`` is), which a page shows coarse at once and sharpens as the rest arrives; Pillow
        refuses the same large files there.
        With ``resize='device'`` the photo is encoded on its device where it lies (``engine.jpeg_encode_u8``) and only the
        file is downloaded; with ``resize='host'`` Pillow encodes it. quality, subsampling and the box's entries are Python or
        numpy integers, not bools. The device encode holds transient device memory sized for the worst-case file (about
        200 MB for a 4000x2667 photo at 4:2:0, 400 MB at 4:4:4, with or without optimize, and about 450 MB at 4:2:0 for a
        progressive file; ``engine.jpeg_encode_u8``).

        ``quality="keep"`` keeps the format of a JPEG upload (the image given to ``open_session``): its quantisation tables
        and subsampling, 4:2:2 included, as Pillow's ``upload.save(buf, "JPEG", quality="keep")`` does, so the blocks an edit
        did not touch come out nearly as they went in; ``subsampling`` is then ignored, as Pillow ignores it. The file is

            img.save(buf, "JPEG", qtables=upload.quantization, subsampling=JpegImagePlugin.get_sampling(upload), ...)

        with the other arguments as above, and ValueError("Cannot use 'keep' when original image is not a JPEG") when the
        upload is not a JPEG. ``exif`` (bytes or a ``PIL.Image.Exif``, at most 65533 bytes) and ``icc_profile`` (bytes or
        None) are written as Pillow's ``save(exif=..., icc_profile=...)`` writes them, after APP0; ``s.exif`` and
        ``s.icc_profile`` are the upload's, so ``s.jpeg(quality="keep", exif=s.exif, icc_profile=s.icc_profile)`` gives back
        the photo as it was uploaded, edits included. An upload table with an entry above 255 (a 16-bit table; no 8-bit
        baseline file has one) is refused with ValueError. On the device these calls run ``engine.jpeg_encode_tables_u8``,
        a numeric quality with the tables of ``engine.jpeg_quality_tables``."""
        import io

        from . import engine
        keep = isinstance(quality, str) and quality == "keep"
        if keep:
            engine._check_jpeg_args(75, 2, optimize, progressive)
        else:
            quality, subsampling = engine._check_jpeg_args(quality, subsampling, optimize, progressive)
        segments = engine.jpeg_app_segments(exif, icc_profile)
        size = self._size(size)
        with self._mu:
            self._check_open()
            if keep and self._keep is None:
                raise ValueError("Cannot use 'keep' when original image is not a JPEG")
            qtables, sampling = self._keep if keep else (None, None)
            if keep:
                engine._check_qtables(qtables)
            box = self._box(box)
            kw = dict(optimize=bool(optimize), progressive=bool(progressive))
            if self._img is not None:
                img = self._host_image(box, size)
                buf = io.BytesIO()
                fmt = dict(qtables=qtables, subsampling=sampling) if keep else dict(quality=quality, subsampling=subsampling)
                img.save(buf, "JPEG", exif=exif, icc_profile=icc_profile, **fmt, **kw)
                return buf.getvalue()
            pixels = self._pixels(box, size)
            if keep:
                return engine.jpeg_encode_tables_u8([pixels], qtables, sampling, exif=exif, icc_profile=icc_profile, **kw)[0]
            if segments:
                return engine.jpeg_encode_tables_u8([pixels], engine.jpeg_quality_tables(quality), subsampling, exif=exif,
                                                    icc_profile=icc_profile, **kw)[0]
            return engine.jpeg_encode_u8([pixels], quality, subsampling, optimize, progressive)[0]

    def png(self, box=None, size=None):
        """The current photo, or its PIL box ``(left, upper, right, lower)``, as a PNG file: the bytes of

            img = s.image().crop(box);  img.thumbnail(size)
            cv2.imencode(".png", np.array(img)[:, :, ::-1])[1]

        (no crop when ``box`` is None, no thumbnail when ``size`` is None), the file ``cv2.imwrite`` writes for the photo;
        ``size`` makes a preview as in ``jpeg``. With ``resize='device'`` the photo is
        encoded on its device where it lies (``engine.png_encode_u8``) and only the file is downloaded; with ``resize='host'``
        cv2 encodes it. The box's entries are Python or numpy integers, not bools. The device encode holds transient device
        memory of about 2.2 bytes per photo byte (``engine.png_encode_u8``)."""
        from . import engine
        size = self._size(size)
        with self._mu:
            self._check_open()
            box = self._box(box)
            if self._img is not None:
                import cv2
                import numpy as np
                img = self._host_image(box, size)
                return cv2.imencode(".png", np.ascontiguousarray(np.asarray(img)[:, :, ::-1]))[1].tobytes()
            return engine.png_encode_u8([self._pixels(box, size)])[0]

    @staticmethod
    def _size(size):
        """A preview bound checked: None, or ``(width, height)`` as Python ints."""
        from . import engine
        return None if size is None else engine.check_thumbnail_size(size)

    def _host_image(self, box, size):
        """The host flow's PIL image of ``box`` (the whole photo for None), thumbnailed to ``size`` unless it is None. The
        thumbnail is made on a copy (``thumbnail`` works in place), so the session's photo is never touched."""
        img = self._img if box is None else self._img.crop(box)
        if size is not None:
            img = img.copy() if img is self._img else img
            img.thumbnail(size)
        return img

    def _pixels(self, box, size):
        """The device flow's pixels of ``box``: the resident photo's window, or when ``size`` is given and the window does
        not fit it, the window's thumbnail in a new device buffer."""
        from . import engine
        win = self._window(box)
        if size is not None and engine.thumbnail_size(win.shape[1], win.shape[0], size) is not None:
            win = engine.thumbnail_u8([win], size)[0]
        return win

    def _box(self, box):
        """``box`` checked against the photo, as a tuple of ints (None stays None)."""
        from . import engine
        if box is None:
            return None
        w, h = self.size
        if not (isinstance(box, (tuple, list)) and len(box) == 4 and all(engine._is_int(v) for v in box)):
            raise ValueError("box must be None or a PIL box (left, upper, right, lower) of integers, got %r" % (box,))
        box = tuple(int(v) for v in box)
        if not (0 <= box[0] < box[2] <= w and 0 <= box[1] < box[3] <= h):
            raise ValueError("box %r must satisfy 0 <= left < right <= %d and 0 <= upper < lower <= %d" % (box, w, h))
        return box

    def _window(self, box):
        """The resident photo's view of ``box`` (the whole photo for None)."""
        w, h = self.size
        left, upper, right, lower = box if box is not None else (0, 0, w, h)
        return self._photo[upper:lower, left:right]

    def _boxes(self, mask, edit_mask, region, offset):
        w, h = self.size
        for m, nm in ((mask, "mask"), (edit_mask, "edit_mask")):
            if m is not None and m.mode != "L":
                raise ValueError("an EditSession takes an 'L' %s (got mode %r)" % (nm, m.mode))
        if edit_mask is not None and edit_mask.size != mask.size:
            raise ValueError("edit_mask is %dx%d, mask %dx%d: they must have one size" % (edit_mask.size + mask.size))
        if not (isinstance(offset, (tuple, list)) and len(offset) == 2 and all(isinstance(v, (int, np.integer)) for v in offset)):
            raise ValueError("offset must be (x, y) of integers, got %r" % (offset,))
        ox, oy = (int(v) for v in offset)
        if region is None:
            if (ox, oy) != (0, 0) or mask.size != (w, h):
                raise ValueError("region=None needs the mask at the photo's size %dx%d and offset (0, 0)" % (w, h))
            if floor8(h) < 16 or floor8(w) < 16:
                raise ValueError("image smaller than 16x16 (two stride-2 convolutions, 4x4 mask pool, stride-2 patch grid)")
            return [(0, 0, w, h)]
        mw, mh = mask.size
        if not (0 <= ox and 0 <= oy and ox + mw <= w and oy + mh <= h):
            raise ValueError("a %dx%d mask at offset (%d, %d) does not fit the %dx%d photo" % (mw, mh, ox, oy, w, h))
        return self._proc._region_boxes(self.size, mask, edit_mask, region, (ox, oy))

    def _drop_proposals(self):
        for p in self._proposals:
            p._drop()
        self._proposals.clear()

    def propose(self, mask, region="auto", offset=(0, 0), feather=0):
        """The edit ``edit(mask, region=region, offset=offset, feather=feather)`` would make, before it is made: returns a
        ``Proposal`` whose ``boxes`` are that edit's boxes and whose ``masks`` are its paste masks (feathered as pasted),
        bit for bit ``edit(..., return_mask=True).masks``, from netM alone (``Engine.predict_mask_u8``; netG does not run,
        about a quarter of an edit's arithmetic). The photo does not change. The proposal holds each box's fp32 soft mask at
        the working size on the engine's device (4 bytes per working pixel) until it is accepted, closed or invalidated.
        Proposals share mask-only forwards with each other and with ``DemoProcessor.predict_mask``."""
        feather = _check_feather(feather)
        with self._mu:
            self._check_open()
            boxes = self._boxes(mask, None, region, offset)
            off = tuple(int(v) for v in offset)
            soft, work, masks, inputs = self._proc._predict(self._img, self._photo, mask, boxes, region is None, feather,
                                                            self.size, off)
            p = Proposal(self, boxes, masks, region is None, mask, off, feather, soft, work, inputs)
            self._proposals.add(p)
            return p

    def accept(self, p, edit_masks=None, return_mask=False, detail=False):
        """Makes the edit of the open proposal ``p`` of this session and returns its ``EditResult``, like ``edit``.

        ``edit_masks=None`` runs the forward on the proposal's fp32 soft masks (``Engine.inference_u8_with_soft_mask``; netM
        does not run again): the photo, the result, ``undo`` and ``jpeg`` afterwards are bit for bit those of
        ``edit(mask, region=p.boxes, offset=offset, feather=feather)``, which is the ``edit`` of the ``region`` given to
        ``propose``; ``return_mask`` returns ``p.masks``. A list of one 'L' image per box, of the box's size, runs the edit
        on those corrected masks: it is ``edit(mask, edit_mask=M, region=p.boxes, ...)`` whenever ``edit_masks[i]`` is
        ``M``'s crop of box i. ``p.masks`` given back unchanged is not "no change": those bytes are feathered and truncated
        (up to 1/255 off netM's mask, and pixels of soft mask in (0.5, 128/255) are no longer inpainted). No change is
        ``edit_masks=None``.

        The photo is not uploaded again: the device flow resizes the boxes again from the photo on the device, as ``edit``
        does, which keeps a proposal at its soft masks alone; the host flow keeps the Pillow-resized inputs it uploaded.
        The proposal is then closed, and so are the session's other proposals. ``detail`` is ``edit``'s: ``accept(p,
        detail=True)`` is ``edit(..., detail=True)`` byte for byte."""
        from PIL import Image
        if not isinstance(p, Proposal):
            raise TypeError("accept takes a Proposal of this session, got %r" % (type(p).__name__,))
        detail = self._proc._check_detail(detail, p._whole)
        if detail:
            _check_detail_boxes(p.boxes, self._proc.region_size)
        with self._mu:
            self._check_open()
            if p._session is not self:
                raise ValueError("the proposal belongs to another session")
            if p._soft is None:
                raise RuntimeError("the proposal is closed: it was accepted or closed, or the photo changed since it was made")
            if edit_masks is not None:
                if not isinstance(edit_masks, (list, tuple)) or len(edit_masks) != len(p.boxes):
                    raise ValueError("edit_masks must be None or a list of %d 'L' images, one per box" % len(p.boxes))
                for i, (m, b) in enumerate(zip(edit_masks, p.boxes)):
                    if getattr(m, "mode", None) != "L" or m.size != (b[2] - b[0], b[3] - b[1]):
                        raise ValueError("edit_masks[%d] must be an 'L' image of its box's size %dx%d" % ((i, b[2] - b[0], b[3] - b[1])))
            soft, work, inputs = p._soft, p._work, p._inputs
            self._drop_proposals()
            if edit_masks is not None:
                return self._edit(p._mask, list(edit_masks), p.boxes, p._whole, return_mask, p._offset, p._feather, detail)
            proc, boxes = self._proc, p.boxes
            if self._img is not None:
                prev = [self._img.crop(b) for b in boxes]
                key = inputs[0].shape[1:3] + (SOFT,) if p._whole else ("region",) + proc.region_size + (SOFT,)
                res = proc.batcher.submit(key, inputs + (soft,))
                if p._whole:
                    out = Image.fromarray(res[0]).resize(self.size)
                else:
                    out = self._img.copy()
                    for i, b in enumerate(boxes):    # the edit's paste, with its paste masks
                        out.paste(Image.fromarray(res[i]).resize((b[2] - b[0], b[3] - b[1])), b, p.masks[i])
                self._img = out
                patches = [out.crop(b) for b in boxes]
            else:
                if p._whole:
                    w, h = self.size
                    patch, _, prev = proc.batcher.submit((floor8(h), floor8(w), SOFT),
                                                         (None, inputs[0], None, False, self._photo, soft))
                    got = [(patch, None)]
                else:
                    got, prev = proc.batcher.submit(("region",) + proc.region_size + (SOFT,),
                                                    (None, inputs, list(work), False, boxes, self._photo, p._feather, self.size,
                                                     detail, soft))
                patches = [Image.fromarray(q) for q, _ in got]
            return self._record(boxes, prev, patches, list(p.masks) if return_mask else [None] * len(boxes))

    def _record(self, boxes, prev, patches, masks):
        nbytes = sum((b[2] - b[0]) * (b[3] - b[1]) * 3 for b in boxes)
        self._history.append((boxes, prev, nbytes))
        self._held += nbytes
        while self._history and self._held > self.history_bytes:
            self._held -= self._history.popleft()[2]
        return EditResult(boxes, patches, masks)

    def edit(self, mask, edit_mask=None, region="auto", return_mask=False, offset=(0, 0), feather=0, detail=False):
        """One edit of the current photo; see the class. Returns ``EditResult(boxes, patches, masks)``. ``detail`` is
        ``DemoProcessor.process_image``'s (region edits of the device flow); undo restores the photo exactly either way."""
        feather = _check_feather(feather)
        detail = self._proc._check_detail(detail, region is None)
        with self._mu:
            self._check_open()
            boxes = self._boxes(mask, edit_mask, region, offset)
            if detail:
                _check_detail_boxes(boxes, self._proc.region_size)
            self._drop_proposals()
            return self._edit(mask, edit_mask, boxes, region is None, return_mask, tuple(int(v) for v in offset), feather, detail)

    def _edit(self, mask, edit_mask, boxes, whole, return_mask, off, feather, detail=False):
        """``edit`` under the lock, on checked arguments; ``edit_mask`` may also be a list of each box's edit mask."""
        from PIL import Image
        if whole and isinstance(edit_mask, list):
            edit_mask = edit_mask[0]
        proc = self._proc
        if self._img is not None:
            fm = _placed(mask, self.size, off)
            fe = edit_mask if isinstance(edit_mask, list) else _placed(edit_mask, self.size, off)
            prev = [self._img.crop(b) for b in boxes]
            if whole:
                out, mk = proc.process_image(self._img, fm, fe, return_mask=True)
                mks = [mk]
            else:
                out, mks = proc._region_host(self._img, fm, fe, boxes, feather)
            self._img = out
            patches = [out.crop(b) for b in boxes]
        else:
            if whole:
                w, h = self.size
                key = (floor8(h), floor8(w)) if edit_mask is None else (floor8(h), floor8(w), True)
                edit_raw = np.asarray(edit_mask) if edit_mask is not None else None
                patch, mk, prev = proc.batcher.submit(key, (None, np.asarray(mask), edit_raw, return_mask, self._photo))
                got = [(patch, mk)]
            else:
                at = [(b[0] - off[0], b[1] - off[1], b[2] - off[0], b[3] - off[1]) for b in boxes]   # mask coordinates
                sketches = [np.asarray(mask.crop(b)) for b in at]
                edits = None if edit_mask is None else [np.asarray(e) for e in edit_mask] if isinstance(edit_mask, list) \
                    else [np.asarray(edit_mask.crop(b)) for b in at]
                got, prev = proc.batcher.submit(proc._region_key(edit_mask),
                                                (None, sketches, edits, return_mask, boxes, self._photo, feather, self.size, detail))
            patches = [Image.fromarray(p) for p, _ in got]
            mks = [Image.fromarray(m) if m is not None else None for _, m in got]
        return self._record(boxes, prev, patches, [m if return_mask and edit_mask is None else None for m in mks])

    def undo(self):
        """Restores the photo from before the last edit not yet undone. Returns ``(boxes, patches)``: that edit's boxes and the
        restored photo's bytes in them. Raises RuntimeError when no snapshot is left."""
        from PIL import Image
        with self._mu:
            self._check_open()
            if not self._history:
                raise RuntimeError("nothing to undo: no snapshot is left")
            self._drop_proposals()
            boxes, prev, nbytes = self._history.pop()
            self._held -= nbytes
            if self._img is not None:
                for b, crop in reversed(list(zip(boxes, prev))):
                    self._img.paste(crop, b[:2])
                return boxes, [self._img.crop(b) for b in boxes]
            torch, photo = self._proc._torch, self._photo
            with torch.cuda.device(photo.device):
                for (left, upper, right, lower), t in reversed(list(zip(boxes, prev))):
                    photo[upper:lower, left:right].copy_(t.view(lower - upper, right - left, 3))
                down = torch.cat([photo[b[1]:b[3], b[0]:b[2]].reshape(-1) for b in boxes]).cpu().numpy()
            patches, pos = [], 0
            for left, upper, right, lower in boxes:
                n = (lower - upper) * (right - left) * 3
                patches.append(Image.fromarray(down[pos:pos + n].reshape(lower - upper, right - left, 3)))
                pos += n
            return boxes, patches


class Proposal:
    """A previewed edit of an ``EditSession`` (``EditSession.propose``): ``boxes``, the PIL boxes the edit would use, and
    ``masks``, each box's 'L' paste mask as the edit would paste it. It holds each box's fp32 soft mask on the engine's
    device until ``EditSession.accept`` takes it, ``close()`` releases it, or an ``edit``, ``undo``, ``accept`` or ``close``
    of its session invalidates it (the photo it was computed on has changed). It is accepted at most once."""

    def __init__(self, session, boxes, masks, whole, mask, offset, feather, soft, work, inputs):
        self.boxes, self.masks = boxes, masks
        self._session, self._whole, self._mask, self._offset, self._feather = session, whole, mask, offset, feather
        self._soft, self._work, self._inputs = soft, work, inputs

    @property
    def open(self):
        """True until the proposal is accepted, closed or invalidated."""
        return self._soft is not None

    def _drop(self):
        self._soft = self._work = self._inputs = None

    def close(self):
        """Releases the proposal's device memory (idempotent); ``accept`` then raises."""
        with self._session._mu:
            self._drop()
            self._session._proposals.discard(self)

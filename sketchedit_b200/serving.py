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
    proc.close()

A region edit (``region=``) crops a box of the photo, runs the forward on it at ``DemoProcessor(region_size=...)`` and pastes
the result back with the edit mask: its cost follows the box, not the photo, and region requests on photos of any size
batch together.

Everything except the forward itself (``run_batch``) is plain host logic and is unit-tested on the CPU with a fake forward.
"""
import threading
import time
from collections import OrderedDict, deque

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


def _check_box(box, w, h):
    if not (isinstance(box, (tuple, list)) and len(box) == 4 and all(isinstance(v, (int, np.integer)) for v in box)):
        raise ValueError("region must be None, 'auto' or a PIL box (left, upper, right, lower) of integers, got %r" % (box,))
    left, upper, right, lower = (int(v) for v in box)
    if not (0 <= left < right <= w and 0 <= upper < lower <= h):
        raise ValueError("region %r must satisfy 0 <= left < right <= %d and 0 <= upper < lower <= %d" % (tuple(box), w, h))
    return left, upper, right, lower


def _aligned_offsets(nbytes, align=16):
    offs, total = [], 0
    for n in nbytes:
        offs.append(total)
        total += (n + align - 1) // align * align
    return offs, total


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
        self.batcher = RequestBatcher(self._run_batch if resize == "host" else self._run_batch_device, max_batch=max_batch,
                                      max_wait_ms=max_wait_ms)

    def close(self):
        self.batcher.close()
        self._pinned.clear()

    def _staging(self, name, nbytes):
        buf = self._pinned.get(name)
        if buf is None or buf.numel() < nbytes:
            buf = self._pinned[name] = self._torch.empty(max(nbytes, 1), dtype=self._torch.uint8, pin_memory=True)
        return buf

    def _run_batch_device(self, key, payloads):
        """payloads: (raw RGB photo [h,w,3], raw 'L' mask [hm,wm], raw 'L' edit mask [he,we] or None, return_mask) at their own
        sizes; key: the floored network size, plus True when the batch runs on edit masks."""
        if key[0] == "region":
            return self._run_region_device(key, payloads)
        torch = self._torch
        from .engine import resize_u8_packed
        H, W = key[:2]
        edit = len(key) > 2
        B = len(payloads)
        dev = self.engine.device
        photos, masks = [p[0] for p in payloads], [p[1] for p in payloads]
        edits = [p[2] for p in payloads] if edit else []
        back = [i for i, p in enumerate(payloads) if p[3] and not edit]   # predicted masks to resize back and download
        offs, total = _aligned_offsets([a.nbytes for a in photos + masks + edits])
        out_offs, out_total = _aligned_offsets([a.nbytes for a in photos] + [photos[i].shape[0] * photos[i].shape[1] for i in back])
        stage = self._staging("in", total)          # free: every batch, failed ones included, ends with a stream synchronise
        host = stage.numpy()
        for a, o in zip(photos + masks + edits, offs):
            host[o:o + a.nbytes] = a.reshape(-1)
        down = self._staging("out", out_total)
        with torch.cuda.device(dev):
            try:
                src = stage[:total].to(dev, non_blocking=True)
                img = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
                msk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                resize_u8_packed(src, offs[:B], [a.shape[:2] for a in photos], [(H, W)] * B, 3, out=img,
                                 dst_offsets=[i * H * W * 3 for i in range(B)])
                # the resized mask goes to the forward as it is: its input codec applies > 0 (demo.py:52)
                resize_u8_packed(src, offs[B:2 * B], [a.shape[:2] for a in masks], [(H, W)] * B, 1, out=msk,
                                 dst_offsets=[i * H * W for i in range(B)])
                with torch.no_grad():
                    if edit:
                        edt = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                        resize_u8_packed(src, offs[2 * B:], [a.shape[:2] for a in edits], [(H, W)] * B, 1, out=edt,
                                         dst_offsets=[i * H * W for i in range(B)])
                        bgr = self.engine.inference_with_mask_u8(img, msk, edt, precision=self.precision)
                    else:
                        bgr, mk = self.engine.inference_u8(img, msk, precision=self.precision)
                # back to each photo's own size; the forward writes BGR, the demo keeps RGB
                res = torch.empty(max(out_total, 1), device=dev, dtype=torch.uint8)
                resize_u8_packed(bgr, [i * H * W * 3 for i in range(B)], [(H, W)] * B, [a.shape[:2] for a in photos], 3,
                                 swap_rb=True, out=res, dst_offsets=out_offs[:B])
                if back:
                    resize_u8_packed(mk, [i * H * W for i in back], [(H, W)] * len(back), [photos[i].shape[:2] for i in back], 1,
                                     out=res, dst_offsets=out_offs[B:])
                down[:out_total].copy_(res[:out_total], non_blocking=True)
            finally:
                torch.cuda.current_stream().synchronize()
        host = down.numpy()
        results = [host[o:o + a.nbytes].reshape(a.shape).copy() for a, o in zip(photos, out_offs)]
        masks_back = dict(zip(back, [host[o:o + photos[i].shape[0] * photos[i].shape[1]].reshape(photos[i].shape[:2]).copy()
                                     for i, o in zip(back, out_offs[B:])]))
        return [(r, masks_back.get(i)) for i, r in enumerate(results)]

    def _run_region_device(self, key, payloads):
        """payloads: (photo crop [bh,bw,3], sketch crop [bh,bw], edit-mask crop [bh,bw] or None, return_mask) at their box sizes;
        key: ("region", Hn, Wn), plus True when the batch runs on edit masks. Returns (patch [bh,bw,3]: the crop with the result
        pasted in, the paste mask resized back to the box [bh,bw] when asked for and predicted, else None)."""
        torch = self._torch
        from .engine import resize_paste_u8_packed, resize_u8_packed
        H, W = key[1:3]
        edit = key[-1] is True
        B = len(payloads)
        dev = self.engine.device
        photos, masks = [p[0] for p in payloads], [p[1] for p in payloads]
        edits = [p[2] for p in payloads] if edit else []
        sizes = [a.shape[:2] for a in photos]
        back = [i for i, p in enumerate(payloads) if p[3] and not edit]   # predicted masks to resize back and download
        offs, total = _aligned_offsets([a.nbytes for a in photos + masks + edits])
        # the patches are pasted in place over the uploaded photo crops, which come first; a predicted mask is resized back into
        # the slot of its sketch crop. One download covers both.
        n_down = offs[B + back[-1]] + masks[back[-1]].nbytes if back else offs[B - 1] + photos[-1].nbytes
        stage = self._staging("in", total)          # free: every batch, failed ones included, ends with a stream synchronise
        host = stage.numpy()
        for a, o in zip(photos + masks + edits, offs):
            host[o:o + a.nbytes] = a.reshape(-1)
        down = self._staging("out", n_down)
        net3, net1 = [i * H * W * 3 for i in range(B)], [i * H * W for i in range(B)]
        with torch.cuda.device(dev):
            try:
                src = stage[:total].to(dev, non_blocking=True)
                img = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
                msk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                resize_u8_packed(src, offs[:B], sizes, [(H, W)] * B, 3, out=img, dst_offsets=net3)
                resize_u8_packed(src, offs[B:2 * B], sizes, [(H, W)] * B, 1, out=msk, dst_offsets=net1)
                with torch.no_grad():
                    if edit:
                        pm = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
                        resize_u8_packed(src, offs[2 * B:], sizes, [(H, W)] * B, 1, out=pm, dst_offsets=net1)
                        bgr = self.engine.inference_with_mask_u8(img, msk, pm, precision=self.precision)
                    else:
                        bgr, pm = self.engine.inference_u8(img, msk, precision=self.precision)
                resize_paste_u8_packed(bgr, net3, pm, net1, [(H, W)] * B, src, offs[:B], sizes, swap_rb=True, out=src,
                                       dst_offsets=offs[:B])
                if back:
                    resize_u8_packed(pm, [net1[i] for i in back], [(H, W)] * len(back), [sizes[i] for i in back], 1, out=src,
                                     dst_offsets=[offs[B + i] for i in back])
                down[:n_down].copy_(src[:n_down], non_blocking=True)
            finally:
                torch.cuda.current_stream().synchronize()
        host = down.numpy()
        out = []
        for i, (a, o) in enumerate(zip(photos, offs)):
            m = host[offs[B + i]:offs[B + i] + masks[i].nbytes].reshape(sizes[i]).copy() if i in back else None
            out.append((host[o:o + a.nbytes].reshape(a.shape).copy(), m))
        return out

    def _run_batch(self, key, payloads):
        """payloads: (photo [H,W,3], mask [H,W], edit mask [H,W] or None, return_mask) at the network size of ``key`` (the
        floored size, or a region's working size); True as the key's last element: the batch runs on edit masks."""
        torch = self._torch
        img = torch.from_numpy(np.stack([p[0] for p in payloads])).cuda(non_blocking=True)     # [B,H,W,3] RGB uint8
        msk = torch.from_numpy(np.stack([p[1] for p in payloads])).cuda(non_blocking=True)     # [B,H,W] uint8 (> 0 = stroke)
        mk = None
        with torch.no_grad():
            if key[-1] is True:
                edt = torch.from_numpy(np.stack([p[2] for p in payloads])).cuda(non_blocking=True)
                bgr = self.engine.inference_with_mask_u8(img, msk, edt, precision=self.precision)
            else:
                bgr, mk = self.engine.inference_u8(img, msk, precision=self.precision)
        rgb = bgr.cpu().numpy()[..., ::-1]                                                     # demo.py keeps RGB (test.py swaps to BGR)
        mk = mk.cpu().numpy() if mk is not None else None
        return [(np.ascontiguousarray(rgb[i]), mk[i] if mk is not None and p[3] else None) for i, p in enumerate(payloads)]

    def process_image(self, img, mask, edit_mask=None, return_mask=False, region=None):
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
        share forwards. With return_mask=True a predicted mask comes back at the photo's size, zero outside the box."""
        from PIL import Image
        img = img.convert("RGB")
        if region is not None:
            return self._process_region(img, mask, edit_mask, return_mask, region)
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
            out, mk = self.batcher.submit(key, (np.asarray(img), np.asarray(mask), edit_raw, return_mask))
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

    def _process_region(self, img, mask, edit_mask, return_mask, region):
        from PIL import Image
        w, h = img.size
        for m, nm in ((mask, "mask"), (edit_mask, "edit_mask")):
            if m is not None and m.size != img.size:
                raise ValueError("a region edit needs the %s at the photo's size %dx%d (got %dx%d)" % ((nm, w, h) + m.size))
            if self.resize == "device" and m is not None and m.mode != "L":
                raise ValueError("resize='device' takes an 'L' %s (got mode %r); resize='host' resizes it with Pillow" % (nm, m.mode))
        if isinstance(region, str):
            if region != "auto":
                raise ValueError("region must be None, 'auto' or a PIL box, got %r" % region)
            bbs = [b for b in (mask.getbbox(), edit_mask.getbbox() if edit_mask is not None else None) if b]
            if not bbs:
                raise ValueError("region='auto' needs a sketch stroke or a non-zero edit mask")
            box = region_box((min(b[0] for b in bbs), min(b[1] for b in bbs), max(b[2] for b in bbs), max(b[3] for b in bbs)),
                             img.size, self.region_size)
        else:
            box = _check_box(region, w, h)
        Hn, Wn = self.region_size
        box_size = (box[2] - box[0], box[3] - box[1])
        # region requests on edit masks run their own forward, and region requests never share one with whole-photo requests
        key = ("region", Hn, Wn) if edit_mask is None else ("region", Hn, Wn, True)
        out = img.copy()
        if self.resize == "device":
            edit_raw = np.asarray(edit_mask.crop(box)) if edit_mask is not None else None
            patch, mk = self.batcher.submit(key, (np.asarray(img.crop(box)), np.asarray(mask.crop(box)), edit_raw, return_mask))
            out.paste(Image.fromarray(patch), box[:2])
            mk = Image.fromarray(mk) if mk is not None else None
        else:
            img_t = np.ascontiguousarray(np.array(img.crop(box).resize((Wn, Hn))), dtype=np.uint8)
            mask_t = np.ascontiguousarray((np.array(mask.crop(box).resize((Wn, Hn))) > 0).astype(np.uint8) * 255)
            edit_t = np.ascontiguousarray(np.array(edit_mask.convert("L").crop(box).resize((Wn, Hn))), dtype=np.uint8) \
                if edit_mask is not None else None
            res, mk = self.batcher.submit(key, (img_t, mask_t, edit_t, True))
            mk = Image.fromarray(edit_t if edit_t is not None else mk).resize(box_size)
            out.paste(Image.fromarray(res).resize(box_size), box, mk)
        if not return_mask:
            return out
        if edit_mask is not None:
            return out, edit_mask
        full = Image.new("L", img.size, 0)
        full.paste(mk, box[:2])
        return out, full

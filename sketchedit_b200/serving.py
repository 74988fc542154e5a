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
    proc.close()

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
    """

    def __init__(self, model, precision=None, max_batch=16, max_wait_ms=2.0, resize="device"):
        import torch
        if resize not in ("device", "host"):
            raise ValueError("resize must be 'device' or 'host'")
        self._torch = torch
        self.model = model
        self.precision = precision or getattr(model, "precision", "bf16")
        self.resize = resize
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

    def _run_batch(self, key, payloads):
        """payloads: (photo [H,W,3], mask [H,W], edit mask [H,W] or None, return_mask) at the floored size ``key[:2]``."""
        torch = self._torch
        img = torch.from_numpy(np.stack([p[0] for p in payloads])).cuda(non_blocking=True)     # [B,H,W,3] RGB uint8
        msk = torch.from_numpy(np.stack([p[1] for p in payloads])).cuda(non_blocking=True)     # [B,H,W] uint8 (> 0 = stroke)
        mk = None
        with torch.no_grad():
            if len(key) > 2:
                edt = torch.from_numpy(np.stack([p[2] for p in payloads])).cuda(non_blocking=True)
                bgr = self.engine.inference_with_mask_u8(img, msk, edt, precision=self.precision)
            else:
                bgr, mk = self.engine.inference_u8(img, msk, precision=self.precision)
        rgb = bgr.cpu().numpy()[..., ::-1]                                                     # demo.py keeps RGB (test.py swaps to BGR)
        mk = mk.cpu().numpy() if mk is not None else None
        return [(np.ascontiguousarray(rgb[i]), mk[i] if mk is not None and p[3] else None) for i, p in enumerate(payloads)]

    def process_image(self, img, mask, edit_mask=None, return_mask=False):
        """img: PIL image; mask: PIL 'L' image, usually of the same size (non-zero = sketch stroke). Returns the edited PIL
        image at the input's size. Sizes are floored to a multiple of 8 for the network exactly like demo.py:43.

        edit_mask: PIL 'L' image of any size that replaces the predicted edit mask (mask revising): resized to the floored
        size like the sketch mask, v/255 blends the result and v >= 128 is inpainted. return_mask=True returns
        ``(result, mask)``: the predicted mask as an 'L' image at the photo's size (resized back like the result), or
        ``edit_mask`` itself when one was given."""
        from PIL import Image
        img = img.convert("RGB")
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

"""A chain of edits on one photo: an EditSession against process_image fed its own result.

    python tools/session_bench.py [--reps 5] [--out FILE]

For 1000x667 and 4000x2667 photos (bf16, synthetic weights, device resize, 256x256 working size) it runs a chain of 10 edits,
each a face-sized stroke group with region="auto" at a new place, in two modes alternated in one process:
  - session: DemoProcessor.open_session(photo), then session.edit(mask, region="auto", offset=...) with the stroke's own
    small mask placed at its offset;
  - process_image: cur = process_image(cur, mask, region="auto") with the photo-sized mask.
It reports the median wall time per edit of a chain from one thread, and edits/s of 16 threads each running its own chain
(medians of --reps). The host-to-device and device-to-host bytes per edit are computed from the box sizes. The window resize
of the session flow (resize_window_u8_packed of 16 boxes out of their photo to 256x256) is timed alone in a separate
torch.profiler run. Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is
written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from serving_bench import card, model  # noqa: E402

WORK = (256, 256)
EDITS = 10


def chain(w, h, seed):
    """The photo and the chain's strokes: (small 'L' mask, its offset, the photo-sized mask) per edit."""
    from PIL import Image
    rs = np.random.RandomState(seed)
    img = Image.fromarray(rs.randint(0, 256, (h, w, 3), dtype=np.uint8))
    fw, fh = max(16, w // 25), max(16, h // 13)                  # a face-sized group: 160x200 at 4000x2667
    steps = []
    for k in range(EDITS):
        x, y = int(rs.randint(0, w - fw)), int(rs.randint(0, h - fh))
        small = np.zeros((fh, fw), np.uint8)
        small[:, ::3] = 255                                      # vertical strokes 3 pixels apart
        full = np.zeros((h, w), np.uint8)
        full[y:y + fh, x:x + fw] = small
        steps.append((Image.fromarray(small), (x, y), Image.fromarray(full)))
    return img, steps


def traffic(w, h, steps, proc):
    """Bytes per edit over the PCIe bus, from the box sizes: (session H2D, session D2H, process_image H2D, D2H)."""
    from sketchedit_b200.serving import region_box
    s_in = s_out = p_in = p_out = 0
    for small, (x, y), _ in steps:
        bb = small.getbbox()
        box = region_box((bb[0] + x, bb[1] + y, bb[2] + x, bb[3] + y), (w, h), WORK)
        px = (box[2] - box[0]) * (box[3] - box[1])
        s_in, s_out = s_in + px, s_out + 3 * px                  # the mask crop in, the patch out
        p_in, p_out = p_in + 4 * px, p_out + 3 * px              # the photo and mask crops in, the patch out
    return [v / len(steps) for v in (s_in, s_out, p_in, p_out)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200.engine import resize_window_u8_packed
    from sketchedit_b200.serving import DemoProcessor
    assert torch.cuda.is_available(), "session_bench.py needs a GPU"
    name, power = card()
    mdl = model(args.precision)
    results = []
    for w, h in ((1000, 667), (4000, 2667)):
        img, steps = chain(w, h, seed=w)
        proc = DemoProcessor(mdl, max_batch=16, max_wait_ms=2.0, region_size=WORK)

        def run(mode):
            """One chain; returns the wall time per edit in ms."""
            t0 = time.perf_counter()
            if mode == "session":
                s = proc.open_session(img)
                for small, off, _ in steps:
                    s.edit(small, region="auto", offset=off)
                s.close()
            else:
                cur = img
                for _, _, full in steps:
                    cur = proc.process_image(cur, full, region="auto")
            return (time.perf_counter() - t0) * 1e3 / EDITS

        modes = ("session", "process_image")
        for m in modes:                                          # warm-up: graphs, coefficient tables, staging buffers
            run(m)
        lat = {m: [] for m in modes}
        for _ in range(args.reps):
            for m in modes:
                lat[m].append(run(m))

        def burst(mode):
            ts = [threading.Thread(target=run, args=(mode,)) for _ in range(args.threads)]
            t0 = time.perf_counter()
            [t.start() for t in ts]
            [t.join() for t in ts]
            return args.threads * EDITS / (time.perf_counter() - t0)

        for m in modes:
            burst(m)
        thr = {m: [] for m in modes}
        for _ in range(args.reps):
            for m in modes:
                thr[m].append(burst(m))
        proc.close()

        # the window resize alone: 16 boxes of the chain out of the resident photo, to the working size
        photo = torch.from_numpy(np.array(img)).cuda().view(-1)
        from sketchedit_b200.serving import region_box
        boxes = []
        for small, (x, y), _ in (steps * 2)[:16]:
            bb = small.getbbox()
            boxes.append(region_box((bb[0] + x, bb[1] + y, bb[2] + x, bb[3] + y), (w, h), WORK))
        out = torch.empty(16 * WORK[0] * WORK[1] * 3, dtype=torch.uint8, device="cuda")

        def windows():
            resize_window_u8_packed(photo, [(b[1] * w + b[0]) * 3 for b in boxes], [3 * w] * 16,
                                    [(b[3] - b[1], b[2] - b[0]) for b in boxes], [WORK] * 16, 3, out=out,
                                    dst_offsets=[i * WORK[0] * WORK[1] * 3 for i in range(16)])

        iters = 50
        windows()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                windows()
            torch.cuda.synchronize()
        k_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                   for e in prof.key_averages() if "resize_" in e.key and "kernel" in e.key)
        del photo, out
        torch.cuda.empty_cache()

        s_in, s_out, p_in, p_out = traffic(w, h, steps, proc)
        rec = {"size": "%dx%d" % (w, h), "edits": EDITS,
               "ms_per_edit": {m: round(statistics.median(v), 2) for m, v in lat.items()},
               "ms_per_edit_all": {m: [round(x, 2) for x in v] for m, v in lat.items()},
               "threads": args.threads, "edits_per_s": {m: round(statistics.median(v), 1) for m, v in thr.items()},
               "edits_per_s_all": {m: [round(x, 1) for x in v] for m, v in thr.items()},
               "bytes_per_edit": {"session": {"h2d": int(s_in), "d2h": int(s_out)},
                                  "process_image": {"h2d": int(p_in), "d2h": int(p_out)}},
               "window_resize_16_boxes_ms": round(k_us / 1e3 / iters, 4)}
        results.append(rec)
        print("%s (%s, %s, %s): ms/edit session %.2f / process_image %.2f; %d threads: %.1f / %.1f edits/s; "
              "bytes/edit in %d / %d, out %d / %d; window resize of 16 boxes %.4f ms"
              % (rec["size"], name, power, args.precision, rec["ms_per_edit"]["session"], rec["ms_per_edit"]["process_image"],
                 args.threads, rec["edits_per_s"]["session"], rec["edits_per_s"]["process_image"], s_in, p_in, s_out, p_out,
                 rec["window_resize_16_boxes_ms"]), flush=True)
    line = {"gpu": name, "power_limit": power, "precision": args.precision, "host_cpus": os.cpu_count(), "results": results}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

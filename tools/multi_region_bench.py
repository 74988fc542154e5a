"""One box per stroke group against one box around all strokes (DemoProcessor.process_image(..., region=...)).

    python tools/multi_region_bench.py [--reps 5] [--out FILE]

For 1000x667 and 4000x2667 photos (bf16, synthetic weights, device resize, 256x256 working size) and two stroke layouts,
two distant groups and three groups of which two have overlapping boxes, it compares region='auto' (the union box) with
region='strokes' (region_groups), alternated in one process:
  - latency: median wall time of process_image from one thread (includes the batcher's max_wait_ms window);
  - throughput: requests/s of 16 threads submitting 16 requests each;
  - the composite kernel alone (paste_v_kernel of se_resize_composite_feather_detail_u8) for 16 requests' boxes pasted into their canvases
    as the device flow does it (a canvas per set of overlapping boxes): its device time from a separate torch.profiler run,
    the bytes it moves (the result and mask rows it reads once, each canvas pixel a box covers read and written once) and
    that rate over the H100 SXM data-sheet 3.35 TB/s.
It also reports the host time of region_groups. Prints the card's name and power limit with the numbers and one JSON line.
Needs an H100; nothing is written to the tree.
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

from serving_bench import HBM_BYTES_PER_S, card, model  # noqa: E402

WORK = (256, 256)
# (width, height) -> layout -> face-sized stroke groups (left, upper, right, lower)
LAYOUTS = {
    (1000, 667): {"two": [(100, 100, 140, 160), (800, 500, 860, 560)],
                  "three": [(100, 100, 140, 160), (330, 120, 370, 170), (800, 500, 860, 560)]},
    (4000, 2667): {"two": [(600, 500, 760, 700), (3200, 1900, 3360, 2100)],
                   "three": [(600, 500, 760, 700), (960, 500, 1120, 700), (3200, 1900, 3360, 2100)]},
}


def request(w, h, rects, seed):
    from PIL import Image
    rs = np.random.RandomState(seed)
    img = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1:3] = 255                                 # vertical strokes 3 pixels apart
    return Image.fromarray(img), Image.fromarray(m)


def canvases(boxes):
    """The device flow's canvases: (bounding rectangle, [(y, x, h, w) of each box in it]) per set of overlapping boxes."""
    from sketchedit_b200.serving import _overlap_sets
    out = []
    for s in _overlap_sets(boxes):
        L, U = min(boxes[i][0] for i in s), min(boxes[i][1] for i in s)
        R, D = max(boxes[i][2] for i in s), max(boxes[i][3] for i in s)
        out.append(((U, L, D - U, R - L), [(boxes[i][1] - U, boxes[i][0] - L, boxes[i][3] - boxes[i][1], boxes[i][2] - boxes[i][0])
                                           for i in s]))
    return out


def composite_bytes(src, rect, boxes):
    """Bytes paste_v_kernel moves for one canvas: each box's result (3 bytes) and mask (1 byte) rows at the working height
    and the box width, read once, and every canvas pixel some box covers, read once and written once."""
    cover = np.zeros(rect[2:], bool)
    for y, x, h, w in boxes:
        cover[y:y + h, x:x + w] = True
    return sum(src[0] * w * 4 for _, _, _, w in boxes) + 2 * 3 * int(cover.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    from sketchedit_b200.serving import DemoProcessor, region_box, region_groups
    assert torch.cuda.is_available(), "multi_region_bench.py needs a GPU"
    name, power = card()
    mdl = model(args.precision)
    results = []
    for (w, h), layouts in LAYOUTS.items():
        for layout, rects in layouts.items():
            img, msk = request(w, h, rects, seed=w + len(rects))
            t_groups = []
            for _ in range(7):
                t0 = time.perf_counter()
                groups = region_groups(msk, region_size=WORK)
                t_groups.append((time.perf_counter() - t0) * 1e3)
            boxes = {"auto": [region_box(msk.getbbox(), img.size, WORK)], "strokes": [b for _, b in groups]}
            proc = DemoProcessor(mdl, max_batch=16, max_wait_ms=2.0, region_size=WORK)

            def call(c):
                return proc.process_image(img, msk, region=c)

            for c in boxes:                                         # warm-up: graph capture, coefficient tables
                call(c)
                call(c)
            lat = {c: [] for c in boxes}
            for _ in range(args.reps):
                for c in boxes:
                    t0 = time.perf_counter()
                    call(c)
                    lat[c].append((time.perf_counter() - t0) * 1e3)

            def burst(c):
                def worker():
                    for _ in range(16):
                        call(c)
                ts = [threading.Thread(target=worker) for _ in range(args.threads)]
                t0 = time.perf_counter()
                [t.start() for t in ts]
                [t.join() for t in ts]
                return args.threads * 16 / (time.perf_counter() - t0)

            for c in boxes:
                burst(c)                                           # warm-up of the batched shapes
            thr = {c: [] for c in boxes}
            for _ in range(max(2, args.reps // 2)):
                for c in boxes:
                    thr[c].append(burst(c))
            proc.close()

            # the composite kernel alone: 16 requests' boxes into their canvases
            B, (Hn, Wn) = 16, WORK
            canv = canvases(boxes["strokes"]) * B
            items = [b for _, bs in canv for b in bs]
            k = len(items)
            res = torch.randint(0, 256, (k * Hn * Wn * 4,), dtype=torch.uint8, device="cuda")
            offs, pos = [], 0
            for (_, _, ch, cw), _ in canv:
                offs.append(pos)
                pos += (ch * cw * 3 + 15) // 16 * 16
            base = torch.randint(0, 256, (pos,), dtype=torch.uint8, device="cuda")
            c_off = [o for o, (_, bs) in zip(offs, canv) for _ in bs]
            pitch = [r[3] * 3 for r, bs in canv for _ in bs]

            def composite():
                resize_composite_u8_packed(res, [i * Hn * Wn * 3 for i in range(k)], res,
                                           [k * Hn * Wn * 3 + i * Hn * Wn for i in range(k)], [(Hn, Wn)] * k, base, c_off, pitch,
                                           [b[:2] for b in items], [b[2:] for b in items], swap_rb=True)

            iters = 50
            composite()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    composite()
                torch.cuda.synchronize()
            k_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                       for e in prof.key_averages() if "paste_v_kernel" in e.key)
            k_ms = k_us / 1e3 / iters
            nbytes = sum(composite_bytes((Hn, Wn), r, bs) for r, bs in canv)
            kern = {"requests": B, "boxes": k, "canvases": len(canv), "bytes": nbytes, "kernel_ms": round(k_ms, 4),
                    "kernel_gb_per_s": round(nbytes / k_ms / 1e6, 1),
                    "kernel_share_of_3_35_tb_s": round(nbytes / (k_ms / 1e3) / HBM_BYTES_PER_S, 3)}
            del res, base
            torch.cuda.empty_cache()

            rec = {"size": "%dx%d" % (w, h), "layout": layout, "boxes": {c: [list(b) for b in bx] for c, bx in boxes.items()},
                   "region_groups_ms": round(statistics.median(t_groups), 2),
                   "latency_ms": {c: round(statistics.median(v), 2) for c, v in lat.items()},
                   "latency_ms_all": {c: [round(x, 2) for x in v] for c, v in lat.items()},
                   "threads": args.threads, "throughput_rps": {c: round(statistics.median(v), 2) for c, v in thr.items()},
                   "throughput_rps_all": {c: [round(x, 2) for x in v] for c, v in thr.items()}, "composite_kernel": kern}
            results.append(rec)
            print("%s %s groups %s (%s, %s): latency auto %.2f / strokes %.2f ms; %d threads: auto %.1f / strokes %.1f req/s; "
                  "region_groups %.2f ms; boxes %s" % (rec["size"], layout, name, power, args.precision, rec["latency_ms"]["auto"],
                                                       rec["latency_ms"]["strokes"], args.threads, rec["throughput_rps"]["auto"],
                                                       rec["throughput_rps"]["strokes"], rec["region_groups_ms"], rec["boxes"]),
                  flush=True)
            print("  paste_v_kernel: %d boxes of %d requests into %d canvases, %.1f MB in %.4f ms (%.0f GB/s, %.1f%% of 3.35 TB/s)"
                  % (k, B, len(canv), nbytes / 1e6, k_ms, kern["kernel_gb_per_s"], 100 * kern["kernel_share_of_3_35_tb_s"]),
                  flush=True)
    line = {"gpu": name, "power_limit": power, "precision": args.precision, "host_cpus": os.cpu_count(), "results": results}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

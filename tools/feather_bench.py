"""The cost of feathered region pastes (process_image(..., feather=F), EditSession.edit(..., feather=F)).

    python tools/feather_bench.py [--reps 5] [--out FILE]

On 1000x667 and 4000x2667 photos (bf16, synthetic weights, device resize, 256x256 working size), alternated in one process:
  - paste_v_kernel alone, as tools/multi_region_bench.py times it (16 requests' 'strokes' boxes of its two- and three-group
    layouts pasted into their canvases), with every box's widths from feather_widths for F = 0 and F = 32: its device time
    from separate torch.profiler runs, and the bytes it moves over that time;
  - process_image(region='strokes') latency (two-group layout), median of --reps, F = 0 and 32;
  - session-edit latency: a session edit of the same strokes, median of --reps, F = 0 and 32.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from multi_region_bench import LAYOUTS, WORK, canvases, composite_bytes, request  # noqa: E402
from serving_bench import card, model  # noqa: E402

FS = (0, 32)


def kernel_ms(torch, fn, iters=50):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
             for e in prof.key_averages() if "paste_v_kernel" in e.key)
    return us / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    from sketchedit_b200.serving import DemoProcessor, _overlap_sets, feather_widths, region_groups
    assert torch.cuda.is_available(), "feather_bench.py needs a GPU"
    name, power = card()
    mdl = model(args.precision)
    results = []
    for (w, h), layouts in LAYOUTS.items():
        # the composite kernel alone, F = 0 and 32 in alternated profiler runs
        kern = {}
        for layout, rects in layouts.items():
            img, msk = request(w, h, rects, seed=w + len(rects))
            boxes = [b for _, b in region_groups(msk, region_size=WORK)]
            B, (Hn, Wn) = 16, WORK
            canv = canvases(boxes) * B
            items = [b for _, bs in canv for b in bs]
            order = [i for s in _overlap_sets(boxes) for i in s] * B        # the boxes of `items`, as canvases() lists them
            k = len(items)
            res = torch.randint(0, 256, (k * Hn * Wn * 4,), dtype=torch.uint8, device="cuda")
            offs, pos = [], 0
            for (_, _, ch, cw), _ in canv:
                offs.append(pos)
                pos += (ch * cw * 3 + 15) // 16 * 16
            base = torch.randint(0, 256, (pos,), dtype=torch.uint8, device="cuda")
            c_off = [o for o, (_, bs) in zip(offs, canv) for _ in bs]
            pitch = [r[3] * 3 for r, bs in canv for _ in bs]

            def composite(F):
                fw = [feather_widths(boxes[i], (w, h), F) for i in order] if F else None
                return lambda: resize_composite_u8_packed(res, [i * Hn * Wn * 3 for i in range(k)], res,
                                                          [k * Hn * Wn * 3 + i * Hn * Wn for i in range(k)], [(Hn, Wn)] * k,
                                                          base, c_off, pitch, [b[:2] for b in items], [b[2:] for b in items],
                                                          swap_rb=True, feather=fw)

            fns = {F: composite(F) for F in FS}
            for F in FS:
                fns[F]()
            torch.cuda.synchronize()
            ms = {F: [] for F in FS}
            for _ in range(3):
                for F in FS:
                    ms[F].append(kernel_ms(torch, fns[F]))
            nbytes = sum(composite_bytes((Hn, Wn), r, bs) for r, bs in canv)
            kern[layout] = {"boxes": k, "bytes": nbytes, "widths_f32": [list(feather_widths(b, (w, h), 32)) for b in boxes],
                            "kernel_ms": {F: round(statistics.median(v), 4) for F, v in ms.items()},
                            "kernel_ms_all": {F: [round(x, 4) for x in v] for F, v in ms.items()},
                            "gb_per_s": {F: round(nbytes / statistics.median(v) / 1e6, 1) for F, v in ms.items()}}
            del res, base
            torch.cuda.empty_cache()

        # end to end: process_image and a session edit of the two-group strokes, F alternated
        img, msk = request(w, h, layouts["two"], seed=w + 2)
        proc = DemoProcessor(mdl, max_batch=16, max_wait_ms=2.0, region_size=WORK)
        sess = proc.open_session(img, history_bytes=0)
        calls = {("process_image", F): (lambda F=F: proc.process_image(img, msk, region="strokes", feather=F)) for F in FS}
        calls.update({("session", F): (lambda F=F: sess.edit(msk, region="strokes", feather=F)) for F in FS})
        for c in calls.values():                                   # warm-up: graphs, tables, staging buffers
            c()
            c()
        lat = {c: [] for c in calls}
        for _ in range(args.reps):
            for c, fn in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                lat[c].append((time.perf_counter() - t0) * 1e3)
        proc.close()
        e2e = {"%s_f%d" % c: round(statistics.median(v), 2) for c, v in lat.items()}
        rec = {"size": "%dx%d" % (w, h), "composite_kernel": kern, "latency_ms": e2e,
               "latency_ms_all": {"%s_f%d" % c: [round(x, 2) for x in v] for c, v in lat.items()}}
        results.append(rec)
        for layout, kr in kern.items():
            print("%dx%d %s (%s, %s): paste_v_kernel %d boxes, %.1f MB: F=0 %.4f ms, F=32 %.4f ms (runs %s / %s)"
                  % (w, h, layout, name, power, kr["boxes"], kr["bytes"] / 1e6, kr["kernel_ms"][0], kr["kernel_ms"][32],
                     kr["kernel_ms_all"][0], kr["kernel_ms_all"][32]), flush=True)
        print("%dx%d (%s, %s, %s): process_image F=0 %.2f / F=32 %.2f ms; session edit F=0 %.2f / F=32 %.2f ms (medians of %d)"
              % (w, h, name, power, args.precision, e2e["process_image_f0"], e2e["process_image_f32"], e2e["session_f0"],
                 e2e["session_f32"], args.reps), flush=True)
    line = {"gpu": name, "power_limit": power, "precision": args.precision, "results": results}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

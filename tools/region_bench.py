"""Region edits against whole-photo edits in the demo serving path (DemoProcessor.process_image(..., region=...)).

    python tools/region_bench.py [--reps 5] [--out FILE]

For 1000x667 and 4000x2667 photos with the local sketch of tools/serving_bench.py (bf16, synthetic weights, device resize) it
reports three cases, alternated in one process: the whole photo, region='auto' at 256x256 and region='auto' at 512x512:
  - latency: median wall time of process_image from one thread (includes the batcher's max_wait_ms window);
  - throughput: requests/s of 16 threads submitting together (16 requests per thread, or 1 for whole 4000x2667 photos);
  - the paste kernel alone (paste_v_kernel of se_resize_composite_feather_detail_u8, one box per canvas) for a batch of 16 region
    results pasted into their boxes:
    its device time from a separate torch.profiler run, the bytes it moves (the result and mask rows it reads once, the base
    it reads and the patch it writes) and that rate over the H100 SXM data-sheet 3.35 TB/s.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from serving_bench import HBM_BYTES_PER_S, card, model, request  # noqa: E402

SIZES = [(1000, 667), (4000, 2667)]       # (width, height) as the requests arrive
CASES = [("whole", None), ("region256", (256, 256)), ("region512", (512, 512))]


def paste_bytes(src, dst):
    """Bytes paste_v_kernel moves for one image: the result (3 bytes) and mask (1 byte) rows at the working height and the
    box width, read once, and the box's base bytes read and patch bytes written."""
    (ih, _), (oh, ow) = src, dst
    return ih * ow * 4 + 2 * oh * ow * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    from sketchedit_b200.serving import DemoProcessor, region_box
    assert torch.cuda.is_available(), "region_bench.py needs a GPU"
    name, power = card()
    mdl = model(args.precision)
    results = []
    for w, h in SIZES:
        big = w * h > 4e6
        img, msk = request(w, h, seed=w)
        procs = {c: DemoProcessor(mdl, max_batch=2 if big and rs is None else 16, max_wait_ms=2.0,
                                  **({"region_size": rs} if rs else {})) for c, rs in CASES}
        region = {c: ("auto" if rs else None) for c, rs in CASES}
        boxes = {c: region_box(msk.getbbox(), img.size, rs) for c, rs in CASES if rs}

        def call(c):
            return procs[c].process_image(img, msk, region=region[c])

        for c in procs:                                             # warm-up: graph capture, coefficient tables
            call(c)
            call(c)
        lat = {c: [] for c in procs}
        for _ in range(args.reps):
            for c in procs:
                t0 = time.perf_counter()
                call(c)
                lat[c].append((time.perf_counter() - t0) * 1e3)

        def burst(c):
            per_thread = 1 if big and region[c] is None else 16

            def worker():
                for _ in range(per_thread):
                    call(c)
            ts = [threading.Thread(target=worker) for _ in range(args.threads)]
            t0 = time.perf_counter()
            [t.start() for t in ts]
            [t.join() for t in ts]
            return args.threads * per_thread / (time.perf_counter() - t0)

        for c in procs:
            burst(c)                                               # warm-up of the batched shapes
        thr = {c: [] for c in procs}
        for _ in range(max(2, args.reps // 2)):
            for c in procs:
                thr[c].append(burst(c))
        batches = {c: len(p.batcher.batches) for c, p in procs.items()}
        for p in procs.values():
            p.close()

        kernels = {}
        for c, rs in CASES:                                         # the paste kernel alone, 16 results into their boxes
            if not rs:
                continue
            B, (Hn, Wn) = 16, rs
            l, u, r, b = boxes[c]
            bh, bw = b - u, r - l
            res = torch.randint(0, 256, (B * Hn * Wn * 4,), dtype=torch.uint8, device="cuda")
            base = torch.randint(0, 256, (B * bh * bw * 3,), dtype=torch.uint8, device="cuda")
            ro, mo, bo = [i * Hn * Wn * 3 for i in range(B)], [B * Hn * Wn * 3 + i * Hn * Wn for i in range(B)], \
                [i * bh * bw * 3 for i in range(B)]

            def paste():
                resize_composite_u8_packed(res, ro, res, mo, [(Hn, Wn)] * B, base, bo, [bw * 3] * B, [(0, 0)] * B, [(bh, bw)] * B,
                                           swap_rb=True)

            iters = 50
            paste()
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    paste()
                torch.cuda.synchronize()
            k_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                       for e in prof.key_averages() if "paste_v_kernel" in e.key)
            k_ms = k_us / 1e3 / iters
            nbytes = B * paste_bytes((Hn, Wn), (bh, bw))
            kernels[c] = {"batch": B, "box": [bw, bh], "bytes": nbytes, "kernel_ms": round(k_ms, 4),
                          "kernel_gb_per_s": round(nbytes / k_ms / 1e6, 1),
                          "kernel_share_of_3_35_tb_s": round(nbytes / (k_ms / 1e3) / HBM_BYTES_PER_S, 3)}
            del res, base
        torch.cuda.empty_cache()

        rec = {"size": "%dx%d" % (w, h), "boxes": {c: list(bx) for c, bx in boxes.items()},
               "latency_ms": {c: round(statistics.median(v), 2) for c, v in lat.items()},
               "latency_ms_all": {c: [round(x, 2) for x in v] for c, v in lat.items()},
               "threads": args.threads, "throughput_rps": {c: round(statistics.median(v), 2) for c, v in thr.items()},
               "throughput_rps_all": {c: [round(x, 2) for x in v] for c, v in thr.items()},
               "forwards": batches, "paste_kernel": kernels}
        results.append(rec)
        print("%s %s (%s, %s): latency whole %.2f / region256 %.2f / region512 %.2f ms; %d threads: whole %.1f / region256 %.1f "
              "/ region512 %.1f req/s; boxes %s" % (rec["size"], name, power, args.precision, rec["latency_ms"]["whole"],
                                                   rec["latency_ms"]["region256"], rec["latency_ms"]["region512"], args.threads,
                                                   rec["throughput_rps"]["whole"], rec["throughput_rps"]["region256"],
                                                   rec["throughput_rps"]["region512"], rec["boxes"]), flush=True)
        for c, k in kernels.items():
            print("  paste_v_kernel %s: %d results into %dx%d boxes, %.1f MB in %.4f ms (%.0f GB/s, %.1f%% of 3.35 TB/s)"
                  % (c, k["batch"], k["box"][0], k["box"][1], k["bytes"] / 1e6, k["kernel_ms"], k["kernel_gb_per_s"],
                     100 * k["kernel_share_of_3_35_tb_s"]), flush=True)
    line = {"gpu": name, "power_limit": power, "precision": args.precision, "host_cpus": os.cpu_count(), "results": results}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

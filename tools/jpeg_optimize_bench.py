"""JPEG with optimal Huffman tables (optimize=True) on the GPU against the Annex K tables and against Pillow on the host.

    python tools/jpeg_optimize_bench.py [--reps 21] [--out FILE]

On jpeg_bench.py's photo-like images (a golden image upscaled, plus noise) at 1000x667 and 4000x2667, quality 75, 4:2:0:
1. The file size with and without optimize.
2. Kernel time: the sum of the library's kernels of one se_jpeg_encode_opt_u8 call (engine.jpeg_encode_u8_packed, one
   image), from torch.profiler over 50 calls of each mode in a run of their own.
3. session.jpeg() and session.jpeg(optimize=True) on a session holding the image (resize='device'; the file is downloaded),
   alternated call by call, --reps times each: median and min-max ms.
4. Pillow's save(buf, "JPEG", quality=75, optimize=True) of the same image on one host thread, median of 5.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from jpeg_bench import photo_like  # noqa: E402
from serving_bench import card, model  # noqa: E402


def kernel_ms(t, h, w, optimize, iters=50):
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed, jpeg_max_bytes
    buf = torch.empty(jpeg_max_bytes(h, w, 2), dtype=torch.uint8, device="cuda")

    def call():
        jpeg_encode_u8_packed(t.view(-1), [0], [3 * w], [(h, w)], out=buf, out_offsets=[0], optimize=optimize)

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
             for e in prof.key_averages() if "jpeg_" in e.key or "scan_" in e.key)
    return us / 1e3 / iters


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    from PIL import Image
    assert torch.cuda.is_available(), "jpeg_optimize_bench.py needs a GPU"
    from sketchedit_b200.serving import DemoProcessor
    name, power = card()
    proc = DemoProcessor(model("bf16"), region_size=(256, 256))
    rows = []
    for w, h in ((1000, 667), (4000, 2667)):
        a = photo_like(w, h, seed=w)
        img = Image.fromarray(a)
        t = torch.from_numpy(a).cuda()
        kern = {opt: kernel_ms(t, h, w, opt) for opt in (False, True)}
        s = proc.open_session(img)
        files = {opt: s.jpeg(optimize=opt) for opt in (False, True)}
        buf = io.BytesIO()
        img.save(buf, "JPEG", quality=75, optimize=True)
        assert files[True] == buf.getvalue()
        for _ in range(3):
            s.jpeg(), s.jpeg(optimize=True)
        ms = {False: [], True: []}
        for _ in range(args.reps):
            for opt in (False, True):
                t0 = time.perf_counter()
                s.jpeg(optimize=opt)
                ms[opt].append((time.perf_counter() - t0) * 1e3)
        s.close()
        pil = []
        for _ in range(5):
            t0 = time.perf_counter()
            img.save(io.BytesIO(), "JPEG", quality=75, optimize=True)
            pil.append((time.perf_counter() - t0) * 1e3)
        r = {"size": "%dx%d" % (w, h), "quality": 75, "subsampling": "4:2:0",
             "bytes": len(files[False]), "bytes_optimize": len(files[True]),
             "saved_percent": round(100 * (1 - len(files[True]) / len(files[False])), 2),
             "kernels_ms": round(kern[False], 4), "kernels_ms_optimize": round(kern[True], 4),
             "session_jpeg_ms": stats(ms[False]), "session_jpeg_ms_optimize": stats(ms[True]),
             "pillow_optimize_ms": round(statistics.median(pil), 2)}
        rows.append(r)
        print("%s (%s, %s): %d -> %d bytes (%.2f%% smaller); kernels %.4f -> %.4f ms; session.jpeg() %.3f [%.3f-%.3f] -> "
              "%.3f [%.3f-%.3f] ms; Pillow optimize=True %.2f ms" %
              (r["size"], name, power, r["bytes"], r["bytes_optimize"], r["saved_percent"], r["kernels_ms"],
               r["kernels_ms_optimize"], *ms_triplet(r["session_jpeg_ms"]), *ms_triplet(r["session_jpeg_ms_optimize"]),
               r["pillow_optimize_ms"]), flush=True)
    proc.close()
    line = {"gpu": name, "power_limit": power, "reps": args.reps, "rows": rows}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


def ms_triplet(d):
    return d["median"], d["min"], d["max"]


if __name__ == "__main__":
    main()

"""Previews of an edit session's photo: s.jpeg(size=...) on the GPU against the full-size download and Pillow's thumbnail.

    python tools/thumbnail_bench.py [--reps 21] [--out FILE]

On jpeg_bench.py's photo-like images (a golden image upscaled, plus noise) at 4000x2667 and 1000x667, with the bounds
(640, 640) and (1280, 1280), quality 75, 4:2:0, on a session holding the image (resize='device'):
1. Call time, the three alternated call by call, --reps times each (median and min-max ms):
   (a) s.jpeg(size=bound): the thumbnail made and encoded on the device, the file downloaded;
   (b) s.image() then Pillow's thumbnail(bound) and save on one host thread (what a server does without size=);
   (c) s.jpeg(): the full-size file.
   The file bytes of each ((a) and (b) are the same file).
2. Kernel time, from torch.profiler in a run of its own over 50 calls of engine.thumbnail_u8 on the resident photo: each
   kernel's mean device time per call, and the reduce's read rate (the window's bytes over its time).
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

SIZES = ((4000, 2667), (1000, 667))
BOUNDS = ((640, 640), (1280, 1280))


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def kernel_us(t, bound, iters=50):
    """Mean device time per engine.thumbnail_u8 call of each kernel it launches, in microseconds."""
    import torch

    from sketchedit_b200.engine import thumbnail_u8
    for _ in range(3):
        thumbnail_u8([t], bound)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            thumbnail_u8([t], bound)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("reduce_kernel", "resize_h_kernel", "resize_v_kernel"):
            if k in e.key:
                us = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                out[k] = out.get(k, 0.0) + us / iters
    return {k: round(v, 2) for k, v in out.items()}


def pillow_preview(s, bound):
    img = s.image()
    img.thumbnail(bound)
    buf = io.BytesIO()
    img.save(buf, "JPEG", quality=75, subsampling=2)
    return buf.getvalue()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    from PIL import Image
    assert torch.cuda.is_available(), "thumbnail_bench.py needs a GPU"
    from sketchedit_b200.engine import thumbnail_size
    from sketchedit_b200.serving import DemoProcessor
    name, power = card()
    proc = DemoProcessor(model("bf16"), region_size=(256, 256))
    rows = []
    for w, h in SIZES:
        a = photo_like(w, h, seed=w)
        s = proc.open_session(Image.fromarray(a))
        for bound in BOUNDS:
            calls = {"device_preview": lambda: s.jpeg(size=bound), "host_preview": lambda: pillow_preview(s, bound),
                     "full_jpeg": lambda: s.jpeg()}
            files = {k: f() for k, f in calls.items()}
            assert files["device_preview"] == files["host_preview"], (w, h, bound)
            for _ in range(2):
                for f in calls.values():
                    f()
            ms = {k: [] for k in calls}
            for _ in range(args.reps):
                for k, f in calls.items():
                    t0 = time.perf_counter()
                    f()
                    ms[k].append((time.perf_counter() - t0) * 1e3)
            r = {"size": "%dx%d" % (w, h), "bound": list(bound), "preview": list(thumbnail_size(w, h, bound) or (w, h)),
                 "quality": 75, "subsampling": "4:2:0", "bytes": {k: len(v) for k, v in files.items()},
                 "call_ms": {k: stats(v) for k, v in ms.items()}}
            rows.append(r)
            print("%s -> %s (%s, %s): bytes %s; call ms %s" % (r["size"], r["preview"], name, power, r["bytes"],
                                                                 {k: v["median"] for k, v in r["call_ms"].items()}), flush=True)
        s.close()
    kern = []
    for w, h in SIZES:
        t = torch.from_numpy(photo_like(w, h, seed=w)).cuda()
        for bound in BOUNDS:
            us = kernel_us(t, bound)
            k = {"size": "%dx%d" % (w, h), "bound": list(bound), "kernels_us": us}
            if "reduce_kernel" in us:
                k["reduce_read_GBps"] = round(w * h * 3 / us["reduce_kernel"] / 1e3, 1)
            kern.append(k)
            print("kernels %s -> bound %s (%s, %s): %s" % (k["size"], bound, name, power, k), flush=True)
    proc.close()
    line = {"gpu": name, "power_limit": power, "reps": args.reps, "rows": rows, "kernels": kern}
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()

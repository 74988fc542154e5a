"""Progressive JPEG (progressive=True) on the GPU against baseline and optimize=True files, and against Pillow on the host.

    python tools/jpeg_progressive_bench.py [--reps 21] [--out FILE]

On jpeg_bench.py's photo-like images (a golden image upscaled, plus noise) at 1000x667 and 4000x2667, quality 75, 4:2:0:
1. The file size: baseline, optimize=True and progressive=True.
2. Kernel time: the sum of the library's kernels of one encode call (engine.jpeg_encode_u8_packed, one image) in each mode,
   from torch.profiler over 50 calls of each mode in a run of their own.
3. session.jpeg(), session.jpeg(optimize=True) and session.jpeg(progressive=True) on a session holding the image
   (resize='device'; the file is downloaded), alternated call by call, --reps times each: median and min-max ms.
4. Pillow's save(buf, "JPEG", quality=75, progressive=True) of the same image on one host thread, median of 5.
5. Kernel time of progressive=True on the worst content for the EOB-run walk, 4000x2667: grey blocks whose eight lowest
   luma AC coefficients are about +-3 after quantisation and all others 0, so the last luma refinement scan codes few
   coefficients for the first time and its runs are long, each carrying 8 correction bits per block and cut every 118
   blocks by the correction-bit limit, and every chroma AC scan is one run of all its blocks; and a flat image, where
   every AC scan of every component is one run.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import io
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from jpeg_bench import photo_like  # noqa: E402
from serving_bench import card, model  # noqa: E402

MODES = {"baseline": {}, "optimize": {"optimize": True}, "progressive": {"progressive": True}}
LUMA_Q75 = [8, 6, 5, 8, 12, 20, 26, 31, 6, 6, 7, 10, 13, 29, 30, 28, 7, 7, 8, 12, 20, 29, 35, 28, 7, 9, 11, 15, 26, 44, 40, 31,
            9, 11, 19, 28, 34, 55, 52, 39, 12, 18, 28, 32, 41, 52, 57, 46, 25, 32, 39, 44, 52, 61, 60, 51, 36, 46, 48, 49, 56,
            50, 52, 50]   # Annex K luma table at quality 75, natural order
ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24]


def refine_run_image(w, h, seed=0):
    """Grey 8x8 blocks built from eight quantised AC values of +-3 at zigzag positions 1..8 (quality 75)."""
    rs = np.random.RandomState(seed)
    n = np.arange(8)
    c = np.where(n == 0, np.sqrt(0.5), 1.0)
    basis = c[:, None] * np.cos((2 * n[None, :] + 1) * n[:, None] * np.pi / 16) / 2
    tiles = []
    for _ in range(64):
        f = np.zeros(64)
        for z in ZIGZAG[1:9]:
            f[z] = rs.choice([-3, 3]) * LUMA_Q75[z]
        tiles.append(np.clip(np.rint(128 + np.einsum("uv,ux,vy->xy", f.reshape(8, 8), basis, basis)), 0, 255))
    bh, bw = -(-h // 8), -(-w // 8)
    pick = rs.randint(0, 64, (bh, bw))
    g = np.array(tiles)[pick].transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)[:h, :w].astype(np.uint8)
    return np.repeat(g[..., None], 3, -1)


def kernel_ms(t, h, w, mode, iters=50):
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed, jpeg_max_bytes
    buf = torch.empty(jpeg_max_bytes(h, w, 2, progressive=True), dtype=torch.uint8, device="cuda")

    def call():
        jpeg_encode_u8_packed(t.view(-1), [0], [3 * w], [(h, w)], out=buf, out_offsets=[0], **MODES[mode])

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


def pillow_prog(a):
    from PIL import Image, ImageFile
    buf = io.BytesIO()
    old, ImageFile.MAXBLOCK = ImageFile.MAXBLOCK, max(ImageFile.MAXBLOCK, 8 * a.shape[0] * a.shape[1])
    try:
        Image.fromarray(a).save(buf, "JPEG", quality=75, progressive=True)
    finally:
        ImageFile.MAXBLOCK = old
    return buf.getvalue()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    from PIL import Image
    assert torch.cuda.is_available(), "jpeg_progressive_bench.py needs a GPU"
    from sketchedit_b200.engine import jpeg_encode_u8
    from sketchedit_b200.serving import DemoProcessor
    name, power = card()
    proc = DemoProcessor(model("bf16"), region_size=(256, 256))
    rows = []
    for w, h in ((1000, 667), (4000, 2667)):
        a = photo_like(w, h, seed=w)
        img = Image.fromarray(a)
        t = torch.from_numpy(a).cuda()
        kern = {m: kernel_ms(t, h, w, m) for m in MODES}
        s = proc.open_session(img)
        files = {m: s.jpeg(**kw) for m, kw in MODES.items()}
        assert files["progressive"] == pillow_prog(a)
        for _ in range(3):
            for kw in MODES.values():
                s.jpeg(**kw)
        ms = {m: [] for m in MODES}
        for _ in range(args.reps):
            for m, kw in MODES.items():
                t0 = time.perf_counter()
                s.jpeg(**kw)
                ms[m].append((time.perf_counter() - t0) * 1e3)
        s.close()
        pil = []
        for _ in range(5):
            t0 = time.perf_counter()
            img.save(io.BytesIO(), "JPEG", quality=75, progressive=True)
            pil.append((time.perf_counter() - t0) * 1e3)
        r = {"size": "%dx%d" % (w, h), "quality": 75, "subsampling": "4:2:0",
             "bytes": {m: len(f) for m, f in files.items()},
             "kernels_ms": {m: round(v, 4) for m, v in kern.items()},
             "session_jpeg_ms": {m: stats(v) for m, v in ms.items()},
             "pillow_progressive_ms": round(statistics.median(pil), 2)}
        rows.append(r)
        print("%s (%s, %s): bytes %s; kernels ms %s; session.jpeg() ms %s; Pillow progressive=True %.2f ms" %
              (r["size"], name, power, r["bytes"], r["kernels_ms"],
               {m: v["median"] for m, v in r["session_jpeg_ms"].items()}, r["pillow_progressive_ms"]), flush=True)
    worst = {}
    w, h = 4000, 2667
    for label, a in (("refine_run", refine_run_image(w, h)), ("flat", np.full((h, w, 3), 128, np.uint8))):
        t = torch.from_numpy(a).cuda()
        assert jpeg_encode_u8([t], 75, 2, progressive=True)[0] == pillow_prog(a)
        worst[label] = {m: round(kernel_ms(t, h, w, m), 4) for m in ("optimize", "progressive")}
        print("worst case %s %dx%d (%s, %s): kernels ms %s" % (label, w, h, name, power, worst[label]), flush=True)
    proc.close()
    line = {"gpu": name, "power_limit": power, "reps": args.reps, "rows": rows, "worst_case_kernels_ms": worst}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

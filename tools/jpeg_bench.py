"""JPEG encoding on the GPU against Pillow on the host.

    python tools/jpeg_bench.py [--reps 5] [--threads 16] [--out FILE]

1. Kernel time: se_jpeg_encode_u8 (engine.jpeg_encode_u8_packed, one image per call) on 1000x667 and 4000x2667 photo-like
   images (a golden image upscaled, plus noise) at quality 75 and 90, 4:2:0 and 4:4:4: CUDA events around 50 calls (the word
   memset, the header and every kernel of the call; no copies), and the sum of the library's kernels in a torch.profiler run
   of its own. The file sizes and Pillow's single-thread encode time of the same image are printed beside them.
2. A session edit followed by the file the page loads: session.edit(...) then session.jpeg() against session.edit(...) then
   session.image() and Pillow's save(buf, "JPEG") (quality 75, 4:2:0), and the edit alone, for a chain of 10 edits (the
   strokes of session_bench.py) on the same photo-like image as in 1 (bf16, synthetic weights), from one thread (median ms
   per edit + file) and from --threads threads each with its own session (files/s). The file's size is printed with them.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import io
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
from session_bench import EDITS, WORK, chain  # noqa: E402


def photo_like(w, h, seed):
    from PIL import Image
    rs = np.random.RandomState(seed)
    g = np.load(os.path.join(ROOT, "tests", "golden", "places_11_512x408.npz"))["image_u8"]
    a = np.asarray(Image.fromarray(g).resize((w, h))).astype(np.int16) + rs.randint(-8, 9, (h, w, 3))
    return np.clip(a, 0, 255).astype(np.uint8)


def pillow_save(img, quality=75, subsampling=2):
    buf = io.BytesIO()
    img.save(buf, "JPEG", quality=quality, subsampling=subsampling)
    return buf.getvalue()


def kernel_times(w, h, iters=50):
    import torch
    from PIL import Image

    from sketchedit_b200.engine import jpeg_encode_u8, jpeg_encode_u8_packed, jpeg_max_bytes
    a = photo_like(w, h, seed=w)
    t = torch.from_numpy(a).cuda()
    flat = t.view(-1)
    out = []
    for q in (75, 90):
        for sub in (2, 0):
            buf = torch.empty(jpeg_max_bytes(h, w, sub), dtype=torch.uint8, device="cuda")

            def call():
                jpeg_encode_u8_packed(flat, [0], [3 * w], [(h, w)], quality=q, subsampling=sub, out=buf, out_offsets=[0])

            call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            call_ms = e0.elapsed_time(e1) / iters
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    call()
                torch.cuda.synchronize()
            k_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                       for e in prof.key_averages() if "jpeg_" in e.key or "scan_" in e.key)
            data = jpeg_encode_u8([t], q, sub)[0]
            img = Image.fromarray(a)
            want = pillow_save(img, q, sub)
            assert data == want, (w, h, q, sub)
            t0 = time.perf_counter()
            for _ in range(5):
                pillow_save(img, q, sub)
            pil_ms = (time.perf_counter() - t0) * 1e3 / 5
            out.append({"size": "%dx%d" % (w, h), "quality": q, "subsampling": "4:2:0" if sub == 2 else "4:4:4",
                        "call_ms": round(call_ms, 4), "kernels_ms": round(k_us / 1e3 / iters, 4), "bytes": len(data),
                        "pillow_ms": round(pil_ms, 2)})
            del buf
    return out


def session_times(mdl, w, h, reps, threads):
    from sketchedit_b200.serving import DemoProcessor
    from PIL import Image
    _, steps = chain(w, h, seed=w)                               # the strokes of session_bench.py's chains
    img = Image.fromarray(photo_like(w, h, seed=w + 1))          # on a photo-like image, not session_bench.py's noise
    proc = DemoProcessor(mdl, max_batch=16, max_wait_ms=2.0, region_size=WORK)
    sizes = []

    def run(mode):
        """One chain of edits, each followed by its file ("edit": no file); returns ms per edit (+ file)."""
        s = proc.open_session(img)
        t0 = time.perf_counter()
        for small, off, _ in steps:
            s.edit(small, region="auto", offset=off)
            if mode == "jpeg":
                data = s.jpeg()
            elif mode == "image+pillow":
                data = pillow_save(s.image())
        ms = (time.perf_counter() - t0) * 1e3 / EDITS
        if mode == "jpeg" and not sizes:
            assert data == pillow_save(s.image())
            sizes.append(len(data))
        s.close()
        return ms

    modes = ("edit", "jpeg", "image+pillow")
    for m in modes:
        run(m)
    lat = {m: [] for m in modes}
    for _ in range(reps):
        for m in modes:
            lat[m].append(run(m))

    def burst(mode):
        ts = [threading.Thread(target=run, args=(mode,)) for _ in range(threads)]
        t0 = time.perf_counter()
        [t.start() for t in ts]
        [t.join() for t in ts]
        return threads * EDITS / (time.perf_counter() - t0)

    for m in modes:
        burst(m)
    thr = {m: [] for m in modes}
    for _ in range(reps):
        for m in modes:
            thr[m].append(burst(m))
    proc.close()
    return {"size": "%dx%d" % (w, h), "edits": EDITS, "file_bytes": sizes[0],
            "ms_per_edit_and_file": {m: round(statistics.median(v), 2) for m, v in lat.items()},
            "ms_all": {m: [round(x, 2) for x in v] for m, v in lat.items()},
            "threads": threads, "files_per_s": {m: round(statistics.median(v), 1) for m, v in thr.items()},
            "files_per_s_all": {m: [round(x, 1) for x in v] for m, v in thr.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "jpeg_bench.py needs a GPU"
    name, power = card()
    kernels = []
    for w, h in ((1000, 667), (4000, 2667)):
        for r in kernel_times(w, h):
            kernels.append(r)
            print("%s q%d %s (%s, %s): call %.4f ms, kernels %.4f ms, %d bytes; Pillow %.2f ms" %
                  (r["size"], r["quality"], r["subsampling"], name, power, r["call_ms"], r["kernels_ms"], r["bytes"],
                   r["pillow_ms"]), flush=True)
    mdl = model("bf16")
    sessions = []
    for w, h in ((1000, 667), (4000, 2667)):
        r = session_times(mdl, w, h, args.reps, args.threads)
        sessions.append(r)
        print("%s (%s, %s), %d-byte file: ms per edit: alone %.2f, + jpeg() %.2f, + image() + Pillow %.2f; %d threads, "
              "per s: %.1f / %.1f / %.1f" %
              (r["size"], name, power, r["file_bytes"], r["ms_per_edit_and_file"]["edit"], r["ms_per_edit_and_file"]["jpeg"],
               r["ms_per_edit_and_file"]["image+pillow"], args.threads, r["files_per_s"]["edit"], r["files_per_s"]["jpeg"],
               r["files_per_s"]["image+pillow"]), flush=True)
    line = {"gpu": name, "power_limit": power, "host_cpus": os.cpu_count(), "kernels": kernels, "sessions": sessions}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

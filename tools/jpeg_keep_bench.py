"""Edit-session JPEGs in the upload's own format (quality="keep" with its EXIF and ICC profile) against today's default file.

    python tools/jpeg_keep_bench.py [--reps 21] [--out FILE]

Uploads: jpeg_bench.py's photo-like image saved by Pillow at (quality 92, 4:2:2) and (95, 4:2:0), with an EXIF block
(orientation 6) and the 588-byte sRGB profile, at 4000x2667 and 1000x667; each opened in a resize='device' session.
1. session.jpeg(quality="keep", exif=s.exif, icc_profile=s.icc_profile) against session.jpeg() (quality 75, 4:2:0),
   alternated call by call, --reps times each: median and min-max ms (the file downloaded).
2. One encode of each from a device image (engine.jpeg_encode_tables_u8 with the upload's tables and metadata,
   engine.jpeg_encode_u8): CUDA events around 20 calls (allocation, segment copy and the file's download included), and
   the sum of the library's kernels from torch.profiler over 20 calls of its own.
3. Pillow's host save of the same keep statement, median of 5; the file sizes.
4. After one region edit: over the 8x8 blocks outside the edited boxes, the PSNR of each decoded file against the decoded
   upload, and the share of those blocks whose decoded pixels equal the upload's.
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

UPLOADS = ((92, 1), (95, 2))


def stats(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def kernel_ms(call, iters=20):
    """(CUDA-event ms per call, profiler ms of the library's kernels per call)."""
    import torch
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
             for e in prof.key_averages() if "jpeg_" in e.key or "scan_" in e.key)
    return e0.elapsed_time(e1) / iters, us / 1e3 / iters


def fidelity(file, ref, boxes):
    """Over the whole 8x8 blocks outside the edited boxes: (PSNR dB of the decoded file against ref, share of those blocks
    whose decoded pixels equal ref's)."""
    from PIL import Image
    a = np.asarray(Image.open(io.BytesIO(file)).convert("RGB")).astype(np.int64)
    h, w = ref.shape[:2]
    bh, bw = h // 8, w // 8
    d = (a[:bh * 8, :bw * 8] - ref[:bh * 8, :bw * 8]).reshape(bh, 8, bw, 8, 3)
    outside = np.ones((bh, bw), bool)
    for x0, y0, x1, y1 in boxes:
        outside[y0 // 8:-(-y1 // 8), x0 // 8:-(-x1 // 8)] = False
    d = d.transpose(0, 2, 1, 3, 4)[outside]
    mse = float((d ** 2).mean())
    psnr = 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)
    return round(float(psnr), 2), round(float((d == 0).all(axis=(1, 2, 3)).mean()), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch
    from PIL import Image, ImageCms, JpegImagePlugin
    assert torch.cuda.is_available(), "jpeg_keep_bench.py needs a GPU"
    from sketchedit_b200.engine import jpeg_encode_tables_u8, jpeg_encode_u8
    from sketchedit_b200.serving import DemoProcessor
    name, power = card()
    proc = DemoProcessor(model("bf16"), region_size=(256, 256))
    exif = Image.Exif()
    exif[0x0112] = 6
    icc = ImageCms.ImageCmsProfile(ImageCms.createProfile("sRGB")).tobytes()
    rows = []
    for w, h in ((4000, 2667), (1000, 667)):
        a = photo_like(w, h, seed=w)
        t = torch.from_numpy(a).cuda()
        for q, sub in UPLOADS:
            buf = io.BytesIO()
            Image.fromarray(a).save(buf, "JPEG", quality=q, subsampling=sub, exif=exif, icc_profile=icc)
            upload = buf.getvalue()
            src = Image.open(io.BytesIO(upload))
            ref = np.asarray(src.convert("RGB")).astype(np.int64)
            s = proc.open_session(src)
            keep = dict(quality="keep", exif=s.exif, icc_profile=s.icc_profile)
            files = {"keep": s.jpeg(**keep), "default": s.jpeg()}
            sampling = JpegImagePlugin.get_sampling(src)
            statement = io.BytesIO()
            s.image().save(statement, "JPEG", qtables=src.quantization, subsampling=sampling, exif=s.exif,
                           icc_profile=s.icc_profile)
            assert files["keep"] == statement.getvalue()
            for _ in range(3):
                s.jpeg(**keep)
                s.jpeg()
            ms = {"keep": [], "default": []}
            for _ in range(args.reps):
                for m, kw in (("keep", keep), ("default", {})):
                    t0 = time.perf_counter()
                    s.jpeg(**kw)
                    ms[m].append((time.perf_counter() - t0) * 1e3)
            kern = {"keep": kernel_ms(lambda: jpeg_encode_tables_u8([t], src.quantization, sampling, exif=s.exif,
                                                                     icc_profile=s.icc_profile)),
                    "default": kernel_ms(lambda: jpeg_encode_u8([t]))}
            img = s.image()
            pil = []
            for _ in range(5):
                t0 = time.perf_counter()
                img.save(io.BytesIO(), "JPEG", qtables=src.quantization, subsampling=sampling, exif=s.exif,
                         icc_profile=s.icc_profile)
                pil.append((time.perf_counter() - t0) * 1e3)
            m = np.zeros((h, w), np.uint8)
            m[h // 3:h // 3 + h // 10, w // 4:w // 4 + w // 8:3] = 255
            mask = Image.fromarray(m)
            r = s.edit(mask)
            after = {"keep": s.jpeg(**keep), "default": s.jpeg()}
            fid = {k: fidelity(f, ref, r.boxes) for k, f in after.items()}
            s.close()
            row = {"size": "%dx%d" % (w, h), "upload": "q%d %s" % (q, {1: "4:2:2", 2: "4:2:0"}[sub]),
                   "upload_bytes": len(upload), "bytes": {k: len(f) for k, f in files.items()},
                   "session_jpeg_ms": {k: stats(v) for k, v in ms.items()},
                   "events_ms": {k: round(v[0], 4) for k, v in kern.items()},
                   "kernels_ms": {k: round(v[1], 4) for k, v in kern.items()},
                   "pillow_keep_ms": round(statistics.median(pil), 2),
                   "after_edit": {k: {"psnr_db": v[0], "unchanged_blocks_outside": v[1]} for k, v in fid.items()}}
            rows.append(row)
            print("%s %s (%s, %s): bytes %s (upload %d); session.jpeg ms %s; events ms %s; kernels ms %s; Pillow keep %.2f ms; "
                  "after one edit %s" % (row["size"], row["upload"], name, power, row["bytes"], len(upload),
                                         {k: v["median"] for k, v in row["session_jpeg_ms"].items()}, row["events_ms"],
                                         row["kernels_ms"], row["pillow_keep_ms"], row["after_edit"]), flush=True)
    proc.close()
    line = {"gpu": name, "power_limit": power, "reps": args.reps, "rows": rows}
    out = json.dumps(line)
    print(out)
    if args.out:
        with open(args.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()

"""PNG decoding on the GPU against Pillow on the host.

    python tools/png_decode_bench.py [--reps 3] [--out-dir DIR] [--out FILE]

1. Kernel time of one se_png_decode_u8 call (engine.png_decode_u8_packed, streams already on the device, output
   preallocated), CUDA events around each of --reps decodes after a warm-up, median: 128 photo-like 256x256 photos ("RGB")
   plus their 128 sketches ("L"), 16 photos at 512x512, one 4000x2667 photo; all saved by Pillow at its default settings.
   This host's single-thread Pillow decode of the same files, np.asarray(Image.open(f).convert(mode)), is printed beside.
2. The test.py loop from PNG files on disk (written under --out-dir, a temporary directory by default), bf16 with synthetic
   weights, results encoded to PNG in memory (inference_stream(png=("image", "mask"))): the host loader (Pillow in
   DataLoader workers) against the device decoder (the workers only read the files), each at --nThreads 1 and 8: 256x256
   batch 128 and 512x512 batch 16 (6 batches per pass, --reps passes), then the crossover at batch 4 and 16 at 256x256,
   batch 4 at 512x512 and 1024x1024, and batch 1 with test_celeb.sh's flags (2 passes). The runs alternate in one process.
   Each pass reports images/s over the whole pass, DataLoader start-up included as test.py pays it, and the steady rate
   from the first batch's results to the last; the figures are medians over the passes.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import io
import json
import os
import shlex
import statistics
import sys
import tempfile
import time

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from png_bench import mask_like, photo_like  # noqa: E402
from serving_bench import card, model  # noqa: E402


def png(a):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "PNG")
    return buf.getvalue()


def decode_time(files, modes, reps):
    """Median ms of one device decode of the files, and this host's single-thread Pillow time for them."""
    import torch

    from sketchedit_b200 import engine as E
    from sketchedit_b200 import pngfile
    heads = [pngfile.parse(f) for f in files]
    staging, offs, lens = E.png_stage(heads)
    src = staging.cuda()
    out, out_offs, status = E.png_decode_u8_packed(src, offs, lens, heads, modes)
    assert status.cpu().tolist() == [0] * len(files)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        E.png_decode_u8_packed(src, offs, lens, heads, modes, out=out, out_offsets=out_offs)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    t0 = time.perf_counter()
    host = [pngfile.pillow_decode(f, m) for f, m in zip(files, modes)]
    host_ms = (time.perf_counter() - t0) * 1e3
    dev = out.cpu().numpy()
    for o, h in zip(out_offs, host):
        assert np.array_equal(dev[o:o + h.size], h.reshape(-1)), "device pixels differ from Pillow's"
    return statistics.median(ms), host_ms


def dataset(root, n, H, W):
    """n photo-like PNG photos and their sketches under root, and the list file."""
    for d in ("images", "edges"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for i in range(n):
        Image.fromarray(photo_like(W, H, i)).save(os.path.join(root, "images", "%04d.png" % i))
        Image.fromarray(mask_like(W, H, i)).save(os.path.join(root, "edges", "%04d.png" % i))
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("".join("%04d.png\n" % i for i in range(n)))


def loop_rate(m, root, B, threads, device):
    """(images/s of one pass of the test.py loop over the dataset under root, steady images/s): the first counts the
    DataLoader's start-up as test.py pays it; the second runs from the first batch's results to the last."""
    import torch

    import data
    from options.test_options import TestOptions
    txt = open(os.path.join(ROOT, "test_celeb.sh")).read().replace("\\\n", " ")
    argv = shlex.split(txt)[2:] + ["--image_dirs", os.path.join(root, "images"), "--mask_dirs", os.path.join(root, "edges"),
                                   "--image_lists", os.path.join(root, "list.txt"), "--output_dir", os.path.join(root, "out"),
                                   "--batchSize", str(B), "--nThreads", str(threads), "--output_mask_dir",
                                   os.path.join(root, "out_mask")]
    opt = TestOptions().parse(argv)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    loader = data.create_dataloader(opt)
    if device:
        loader = data.loader_of(loader.dataset, opt, files=True)
    n, n1, t1 = 0, 0, None
    with torch.no_grad():
        for files, mfiles in m.inference_stream(loader, uint8=True, png=("image", "mask")):
            n += len(files)
            if t1 is None:
                n1, t1 = n, time.perf_counter()
    t = time.perf_counter()
    return n / (t - t0), (n - n1) / max(t - t1, 1e-9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out-dir", default=None, help="where the PNG datasets are written (default: a temporary directory)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("png_decode_bench needs a CUDA device")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "decode": {}, "loop": {}}
    decode_time([png(photo_like(64, 64, 0))], ["RGB"], 2)   # warm-up: module load, allocator
    cases = {
        "256x256_b128_with_sketches": ([png(photo_like(256, 256, i)) for i in range(128)] +
                                       [png(mask_like(256, 256, i)) for i in range(128)], ["RGB"] * 128 + ["L"] * 128),
        "512x512_b16": ([png(photo_like(512, 512, i)) for i in range(16)], ["RGB"] * 16),
        "4000x2667_b1": ([png(photo_like(4000, 2667, 1))], ["RGB"]),
    }
    for key, (files, modes) in cases.items():
        dev_ms, host_ms = decode_time(files, modes, args.reps if len(files) > 1 else 1)
        res["decode"][key] = {"device_ms": round(dev_ms, 3), "host_pillow_ms": round(host_ms, 2),
                              "mean_file_bytes": round(sum(map(len, files)) / len(files))}
        print("decode %-28s device %8.3f ms   host Pillow (1 thread) %9.2f ms" % (key, dev_ms, host_ms), flush=True)
    m = model("bf16")
    tmp = tempfile.TemporaryDirectory() if args.out_dir is None else None
    base = args.out_dir or tmp.name
    # (batch, size, images, passes): the two workloads of the issue with 8 batches per pass, then the crossover in batch size
    # and image size, and batch 1 with test_celeb.sh's flags
    for (B, H, W, n, reps) in ((128, 256, 256, 768, args.reps), (16, 512, 512, 96, args.reps), (4, 256, 256, 64, 2),
                               (16, 256, 256, 96, 2), (4, 512, 512, 32, 2), (4, 1024, 1024, 16, 2), (1, 256, 256, 16, 2)):
        key = "%dx%d_b%d" % (H, W, B)
        root = os.path.join(base, "%dx%d" % (H, W))
        if not os.path.isdir(root) or len(os.listdir(os.path.join(root, "images"))) < n:
            dataset(root, n, H, W)
        with open(os.path.join(root, "list.txt"), "w") as f:
            f.write("".join("%04d.png\n" % i for i in range(n)))
        runs = [(threads, dev) for threads in (1, 8) for dev in (False, True)]
        for threads, dev in runs:   # warm-up pass of each
            loop_rate(m, root, B, threads, dev)
        rates = {r: [] for r in runs}
        for _ in range(reps):
            for r in runs:
                rates[r].append(loop_rate(m, root, B, *r))
        res["loop"][key] = {}
        for (threads, dev), v in rates.items():
            k = "%s_nThreads%d" % ("device" if dev else "host", threads)
            res["loop"][key][k] = round(statistics.median(a for a, _ in v), 1)
            res["loop"][key][k + "_steady"] = round(statistics.median(b for _, b in v), 1)
        print("loop %-16s " % key + "   ".join("%s %7.1f" % kv for kv in res["loop"][key].items()), flush=True)
    if tmp is not None:
        tmp.cleanup()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

"""PNG encoding on the GPU against cv2 on the host.

    python tools/png_bench.py [--reps 5] [--steps 8] [--out FILE]

1. Kernel time of one se_png_encode_u8 encode (engine.png_encode_u8_packed, all scratch and output preallocated, no copies),
   CUDA events around each of --reps encodes after a warm-up, median: batch 128 at 256x256 BGR plus its 128 masks, batch 16
   at 512x512, one 4000x2667 photo. The images are photo-like (a golden photo resized, plus noise) with binary masks, and
   the golden photos themselves; this host's single-thread cv2.imencode of the same images and the files' mean size are
   printed beside them.
2. test.py-style throughput, writing to memory: inference_stream(uint8=True) then cv2.imencode of every result and mask,
   against inference_stream(png=("image", "mask")), bf16 with synthetic weights (so the outputs are not photos), at 256x256
   batch 128 and 512x512 batch 16, --steps batches after one warm-up pass; images/s and the mean file size.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from serving_bench import card, model  # noqa: E402


def photo_like(w, h, seed):
    rs = np.random.RandomState(seed)
    g = np.load(os.path.join(ROOT, "tests", "golden", "places_11_512x408.npz"))["image_u8"]
    a = cv2.resize(g, (w, h), interpolation=cv2.INTER_CUBIC).astype(np.int16) + rs.randint(-8, 9, (h, w, 3))
    return np.clip(a, 0, 255).astype(np.uint8)


def mask_like(w, h, seed):
    rs = np.random.RandomState(seed)
    m = np.zeros((h, w), np.uint8)
    for _ in range(3):
        y, x = rs.randint(0, h), rs.randint(0, w)
        cv2.circle(m, (int(x), int(y)), int(rs.randint(h // 8, h // 3)), 255, -1)
    return m


def golden(name):
    return np.ascontiguousarray(np.load(os.path.join(ROOT, "tests", "golden", name))["image_u8"][:, :, ::-1])


def encode_time(images, masks, reps):
    """Median ms of one encode of the images (BGR) and masks on the device, and the host's single-thread cv2 time."""
    import torch

    from sketchedit_b200.engine import png_encode_u8_packed, png_max_bytes
    groups = [(np.stack(images), 3)] + ([(np.stack(masks), 1)] if masks else [])
    calls = []
    for arr, c in groups:
        n, h, w = arr.shape[:3]
        src = torch.from_numpy(arr).cuda().view(-1)
        step = h * w * c
        out, offs, _ = png_encode_u8_packed(src, [i * step for i in range(n)], [w * c] * n, [(h, w)] * n, c, swap_rb=True)
        calls.append(lambda src=src, n=n, h=h, w=w, c=c, step=step, out=out, offs=offs: png_encode_u8_packed(
            src, [i * step for i in range(n)], [w * c] * n, [(h, w)] * n, c, swap_rb=True, out=out, out_offsets=offs))
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = [f() for f in calls]
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    sizes = [int(v) for r in res for v in r[2].cpu().tolist()]
    t0 = time.perf_counter()
    host = [cv2.imencode(".png", x)[1].size for x in list(images) + list(masks)]
    host_ms = (time.perf_counter() - t0) * 1e3
    assert sizes == host, "device files differ in size from cv2's"
    return statistics.median(ms), host_ms, sum(sizes) / len(sizes)


def stream_rate(m, B, H, W, steps):
    """images/s of the test.py loop writing to memory: uint8 arrays + cv2.imencode against png=("image", "mask")."""
    import torch

    from sketchedit_b200 import synth
    rs = np.random.RandomState(B)
    batches = []
    for i in range(steps):
        _, sk = synth.synth_inputs(B, H, W, seed=200 + i)
        batches.append({"image_u8": torch.from_numpy(rs.randint(0, 256, (B, H, W, 3), dtype=np.uint8)).pin_memory(),
                        "mask_u8": (sk[:, 0] * 255).to(torch.uint8).pin_memory()})
    out = {}
    with torch.no_grad():
        for mode in ("cv2", "png", "cv2", "png"):   # a warm-up pass of each, then the timed ones
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            size = 0
            if mode == "cv2":
                for bgr, mk in m.inference_stream(iter(batches), uint8=True):
                    bgr, mk = bgr.numpy(), mk.numpy()
                    for b in range(B):
                        size += cv2.imencode(".png", bgr[b])[1].size + cv2.imencode(".png", mk[b])[1].size
            else:
                for files, mfiles in m.inference_stream(iter(batches), uint8=True, png=("image", "mask")):
                    size += sum(map(len, files)) + sum(map(len, mfiles))
            dt = time.perf_counter() - t0
            out[mode] = (B * steps / dt, size / (2 * B * steps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("png_bench needs a CUDA device")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "encode": {}, "stream": {}}
    encode_time([photo_like(64, 64, 0)], [mask_like(64, 64, 0)], 2)   # warm-up: module load, allocator
    cases = {
        "256x256_b128_with_masks": ([photo_like(256, 256, i) for i in range(128)], [mask_like(256, 256, i) for i in range(128)]),
        "512x512_b16": ([photo_like(512, 512, i) for i in range(16)], []),
        "4000x2667_b1": ([photo_like(4000, 2667, 1)], []),
        "golden_face_256x256": ([golden("face_602_256x256.npz")], []),
        "golden_places_512x408": ([golden("places_11_512x408.npz")], []),
    }
    for key, (imgs, masks) in cases.items():
        dev_ms, host_ms, size = encode_time(imgs, masks, args.reps)
        res["encode"][key] = {"device_ms": round(dev_ms, 3), "host_cv2_ms": round(host_ms, 2), "mean_file_bytes": round(size)}
        print("encode %-26s device %8.3f ms   host cv2 (1 thread) %9.2f ms   mean file %8d B" % (key, dev_ms, host_ms, size))
    m = model("bf16")
    for B, H, W in ((128, 256, 256), (16, 512, 512)):
        r = stream_rate(m, B, H, W, args.steps)
        key = "%dx%d_b%d" % (H, W, B)
        res["stream"][key] = {"cv2_images_per_s": round(r["cv2"][0], 1), "png_images_per_s": round(r["png"][0], 1),
                              "mean_file_bytes": round(r["png"][1])}
        print("stream %-12s uint8 + cv2.imencode %8.1f img/s   png= %8.1f img/s   mean file %7d B" % (key, r["cv2"][0], r["png"][0], r["png"][1]))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

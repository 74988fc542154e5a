"""Large PNG files decoded across the whole GPU (se_png_split_u8) against the one-warp decoder (se_png_decode_u8) and Pillow.

    python tools/png_split_bench.py [--reps 5] [--out FILE]

1. Per file, the decode time of the split decoder, the one-warp decoder (CUDA events around one png_decode_u8_packed call,
   streams already on the device, output preallocated; median of --reps runs alternated between the two; the one-warp
   decoder 1 run on files of more than 8 MB of scanlines) and Pillow on one host thread (np.asarray(Image.open(f).convert
   ("RGB")), median). Files: a 4000x2667 photo-like RGB image saved by Pillow and by cv2.imwrite, a flat 2048x2048
   screenshot-like image, and photo-like images from 512x512 to 2896x2896 for the crossover. Each stream's deflate blocks
   are counted by type with a host build of se_inflate.cuh (g++; "not measured" without it).
2. One torch.profiler breakdown per kernel of the split decode of the Pillow-saved 4000x2667 file.
3. The decode rows of tools/png_decode_bench.py (128 256x256 photos with their sketches, 16 photos at 512x512), each file
   through the split decoder and through the one-warp decoder, alternated.
4. DemoProcessor.open_session(bytes) against open_session(Image.open(io.BytesIO(bytes))) for Pillow-saved PNG photos at
   1000x667 and 4000x2667 (bf16, synthetic weights, device resize), each to the photo resident on the device; median of
   --reps alternated runs.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import io
import json
import os
import shutil
import statistics
import subprocess
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

COUNTER = r"""
#include <stdio.h>
#include <stdlib.h>
#include "se_inflate.cuh"
// a zlib stream on stdin -> its stored, fixed and dynamic block counts on stdout
struct Skip {
  int stored(const unsigned char*, unsigned) { return 0; }
  int lit(int) { return 0; }
  int match(long long, long long) { return 0; }
};
int main() {
  static unsigned char buf[1 << 28];
  const long long n = (long long)fread(buf, 1, sizeof(buf), stdin);
  static se::InflateTabs t;
  se::BitIn in{buf, 2, n, 0ull, 0};
  long long count[4] = {0};
  Skip out;
  for (unsigned last = 0; !last;) {
    se::BitIn peek = in;
    if (!peek.need(3)) return 1;
    count[(peek.buf >> 1) & 3]++;
    if (se::inflate_block(in, t, out, &last, 0, 1)) return 1;
  }
  printf("%lld %lld %lld\n", count[0], count[1], count[2]);
  return 0;
}
"""


def png(a):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, "PNG")
    return buf.getvalue()


def block_counter(tmp):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        return None
    src, exe = os.path.join(tmp, "count.cpp"), os.path.join(tmp, "count")
    with open(src, "w") as f:
        f.write(COUNTER)
    subprocess.run([cxx, "-O2", "-std=c++17", "-I", os.path.join(ROOT, "sketchedit_b200", "csrc"), src, "-o", exe], check=True)

    def count(stream):
        p = subprocess.run([exe], input=stream, capture_output=True, check=True)
        return dict(zip(("stored", "fixed", "dynamic"), map(int, p.stdout.split())))
    return count


def flat(h, w):
    a = np.full((h, w, 3), 240, np.uint8)
    a[: h // 12] = (40, 60, 90)
    a[h // 3: h // 2, w // 5: w // 2] = (255, 255, 255)
    a[::97] = 0
    rs = np.random.RandomState(4)
    for y in range(h // 10, h, h // 9):
        a[y:y + 12, 40:40 + w // 3] = rs.randint(0, 2, (12, w // 3, 1)) * 200
    return a


def device_ms(files, modes, split, reps):
    """ms of each of reps png_decode_u8_packed calls over the files with the split or one-warp decoder, and the status."""
    import torch

    from sketchedit_b200 import engine as E
    from sketchedit_b200 import pngfile
    E.PNG_SPLIT_MIN_RAW = 0 if split else 1 << 62
    heads = [pngfile.parse(f) for f in files]
    staging, offs, lens = E.png_stage(heads)
    src = staging.cuda()
    out, out_offs, status = E.png_decode_u8_packed(src, offs, lens, heads, modes)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        E.png_decode_u8_packed(src, offs, lens, heads, modes, out=out, out_offsets=out_offs)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    st = status.cpu().tolist()
    dev = out.cpu().numpy()
    for f, m, o, s in zip(files, modes, out_offs, st):
        if s == 0:
            want = pngfile.pillow_decode(f, m)
            assert np.array_equal(dev[o:o + want.size], want.reshape(-1)), "device pixels differ from Pillow's"
    return ms, st


def pillow_ms(files, modes, reps):
    from sketchedit_b200 import pngfile
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for f, m in zip(files, modes):
            pngfile.pillow_decode(f, m)
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def profile_split(f, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from sketchedit_b200 import engine as E
    from sketchedit_b200 import pngfile
    E.PNG_SPLIT_MIN_RAW = 0
    hd = pngfile.parse(f)
    staging, offs, lens = E.png_stage([hd])
    src = staging.cuda()
    out, out_offs, _ = E.png_decode_u8_packed(src, offs, lens, [hd], "RGB")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        E.png_decode_u8_packed(src, offs, lens, [hd], "RGB", out=out, out_offsets=out_offs)
        torch.cuda.synchronize()
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "png_split_4000x2667.pt.trace.json"))
    rows = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "device_time_total", 0):
            t = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
            if t:
                rows[e.key] = round(t / 1e3, 3)
    return rows


def session_ms(proc, data, reps):
    import torch
    ms = {"bytes": [], "pillow": []}
    for kind in ("bytes", "pillow"):   # warm-up
        proc.open_session(data if kind == "bytes" else Image.open(io.BytesIO(data))).close()
    for _ in range(reps):
        for kind in ("bytes", "pillow"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s = proc.open_session(data if kind == "bytes" else Image.open(io.BytesIO(data)))
            torch.cuda.synchronize()
            ms[kind].append((time.perf_counter() - t0) * 1e3)
            s.close()
    return {k: round(statistics.median(v), 2) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--trace-dir", default=None, help="where the profiler trace goes (default: none is written)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("png_split_bench needs a CUDA device")
    import cv2

    from sketchedit_b200 import engine as E
    from sketchedit_b200 import pngfile
    default_min = E.PNG_SPLIT_MIN_RAW
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = {"card": name, "power_limit": power, "files": {}, "rows": {}, "sessions": {}}
    tmp = tempfile.mkdtemp()
    count = block_counter(tmp)
    big = photo_like(4000, 2667, 1)
    files = {"pil_4000x2667": png(big), "cv2_4000x2667": cv2.imencode(".png", big[..., ::-1])[1].tobytes(),
             "flat_2048x2048": png(flat(2048, 2048))}
    for s in (512, 724, 1024, 1448, 2048, 2896):
        files["pil_%dx%d" % (s, s)] = png(photo_like(s, s, s))
    device_ms([png(photo_like(64, 64, 0))], ["RGB"], True, 2)   # warm-up: module load, allocator
    device_ms([png(photo_like(64, 64, 0))], ["RGB"], False, 2)
    for key, f in files.items():
        hd = pngfile.parse(f)
        raw = E.png_raw_bytes(hd)
        warp_reps = 1 if raw > 8 << 20 else args.reps
        split, warp = [], []
        st = None
        for r in range(args.reps):
            ms, st = device_ms([f], ["RGB"], True, 1)
            split += ms
            if r < warp_reps:
                warp += device_ms([f], ["RGB"], False, 1)[0]
        row = {"file_bytes": len(f), "raw_bytes": raw, "chunk_bytes": E.png_split_chunk_bytes(len(hd.stream)),
               "blocks": count(hd.stream) if count else "not measured", "split_status": st[0],
               "split_ms": round(statistics.median(split), 3), "one_warp_ms": round(statistics.median(warp), 3),
               "pillow_ms": round(pillow_ms([f], ["RGB"], 3), 2)}
        res["files"][key] = row
        print("%-16s %s" % (key, row), flush=True)
    res["profile_pil_4000x2667_ms"] = profile_split(files["pil_4000x2667"], args.trace_dir)
    print("profile", res["profile_pil_4000x2667_ms"], flush=True)
    rows = {
        "256x256_b128_with_sketches": ([png(photo_like(256, 256, i)) for i in range(128)] +
                                       [png(mask_like(256, 256, i)) for i in range(128)], ["RGB"] * 128 + ["L"] * 128),
        "512x512_b16": ([png(photo_like(512, 512, i)) for i in range(16)], ["RGB"] * 16),
    }
    for key, (fs, modes) in rows.items():
        split, warp = [], []
        for _ in range(args.reps):
            split += device_ms(fs, modes, True, 1)[0]
            warp += device_ms(fs, modes, False, 1)[0]
        res["rows"][key] = {"split_ms": round(statistics.median(split), 3), "one_warp_ms": round(statistics.median(warp), 3),
                            "pillow_ms": round(pillow_ms(fs, modes, 1), 2)}
        print("%-28s %s" % (key, res["rows"][key]), flush=True)
    E.PNG_SPLIT_MIN_RAW = default_min
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model("bf16"), region_size=(256, 256))
    try:
        for w, h in ((1000, 667), (4000, 2667)):
            res["sessions"]["%dx%d" % (w, h)] = session_ms(proc, png(photo_like(w, h, 3)), args.reps)
            print("open_session %dx%d (ms, bytes vs Image.open)" % (w, h), res["sessions"]["%dx%d" % (w, h)], flush=True)
    finally:
        proc.close()
    shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

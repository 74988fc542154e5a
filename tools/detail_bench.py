"""Cost of region-edit detail (process_image(..., detail=True) and EditSession.edit(..., detail=True)) on the GPU.

    python tools/detail_bench.py [--reps 5] [--out DIR]

Workloads: bf16, region="auto" at the 256 x 256 working size, on photos of 4000 x 2667 and 1000 x 667 (random weights: the
cost does not depend on them), each call with and without detail, alternated in one process; median and min-max of --reps
calls after a warm-up of each. Then the detail step on the forward's attn and hole, at 256 x 256 and once at 512 x 512, where
the aggregation GEMM grows as L^2: "call" is CUDA events around detail_u8_packed (the wrapper's host work and allocations
included, an upper bound), "kernels" the summed device time of its four launches (two packs, the GEMM, the fold) from
torch.profiler, in a run of its own. Prints one JSON line with the GPU's
name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:   # noqa: BLE001 - reported, not fatal
        return "unknown (%s)" % e, "unknown"


def photo(w, h, seed):
    from PIL import Image
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (127 + 60 * np.sin(xx / 37.0) * np.cos(yy / 53.0))[..., None] + rs.randint(-40, 40, (h, w, 3))
    img = Image.fromarray(np.clip(base, 0, 255).astype(np.uint8))
    m = np.zeros((h, w), np.uint8)
    cx, cy, s = w // 2, h // 2, max(16, w // 16)
    m[cy - s:cy + s, cx - s:cx + s:3] = 255
    return img, Image.fromarray(m)


def stats(ts):
    ts = sorted(ts)
    return {"median_ms": round(1e3 * ts[len(ts) // 2], 3), "min_ms": round(1e3 * ts[0], 3), "max_ms": round(1e3 * ts[-1], 3)}


def kernel_ms(eng, Hn, Wn, bw, bh, reps):
    import torch

    from sketchedit_b200.engine import detail_u8_packed, resize_u8_packed
    rs = np.random.RandomState(1)
    ph = torch.from_numpy(rs.randint(0, 256, (bh, bw, 3), dtype=np.uint8)).cuda()
    img = torch.from_numpy(rs.randint(0, 256, (1, Hn, Wn, 3), dtype=np.uint8)).cuda()
    sk = torch.zeros(1, Hn, Wn, dtype=torch.uint8, device="cuda")
    sk[0, Hn // 3:2 * Hn // 3, Wn // 3:2 * Wn // 3:3] = 255
    _, _, attn, hole = eng.inference_u8_export(img, sk, precision="bf16")
    low, low_at = resize_u8_packed(img, [0], [(Hn, Wn)], [(bh, bw)], 3)
    args = (ph, [0], [bw * 3], [(bh, bw)], (Hn, Wn), low, low_at, hole, [0], attn, [0])
    detail_u8_packed(*args)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record()
        for _ in range(10):
            detail_u8_packed(*args)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 10 / 1e3)
    from torch.profiler import ProfilerActivity, profile
    calls = 20
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            detail_u8_packed(*args)
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if "detail_" in e.key or "gemm_split_kernel" in e.key:
            us = getattr(e, "device_time_total", None)
            per[e.key.split("(")[0]] = round((us if us is not None else e.cuda_time_total) / calls / 1e3, 4)
    return {"call": stats(ts), "kernels_ms": round(sum(per.values()), 4), "per_kernel_ms": per}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "detail_bench needs a GPU: figures not taken on one are not measured"
    from sketchedit_b200 import build
    build.build(verbose=False)
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power, "precision": "bf16", "region_size": [256, 256], "reps": a.reps, "calls": {}}
    proc = DemoProcessor(_model("bf16"), max_batch=1, max_wait_ms=0.0, region_size=(256, 256))
    try:
        for w, h in ((4000, 2667), (1000, 667)):
            img, sk = photo(w, h, w)
            sess = proc.open_session(img, history_bytes=0)
            calls = {
                "process_image": lambda d: proc.process_image(img, sk, region="auto", detail=d),
                "session_edit": lambda d: sess.edit(sk, region="auto", detail=d),
            }
            for kind, f in calls.items():
                f(False), f(True), f(False), f(True)            # warm-up: graphs captured, tables uploaded
                t = {False: [], True: []}
                for _ in range(a.reps):
                    for d in (False, True):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        f(d)
                        t[d].append(time.perf_counter() - t0)
                res["calls"]["%s %dx%d" % (kind, w, h)] = {"plain": stats(t[False]), "detail": stats(t[True])}
            sess.close()
        eng = proc.engine
        res["detail_kernels"] = {"256x256, box 608x608 (scale 19/8)": kernel_ms(eng, 256, 256, 608, 608, a.reps),
                                 "256x256, box 256x256": kernel_ms(eng, 256, 256, 256, 256, a.reps),
                                 "512x512, box 1216x1216 (scale 19/8)": kernel_ms(eng, 512, 512, 1216, 1216, a.reps)}
    finally:
        proc.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "detail_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

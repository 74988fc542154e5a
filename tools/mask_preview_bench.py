"""Previewing the edit mask: what a preview costs against an edit.

    python tools/mask_preview_bench.py [--reps 5] [--out FILE]

Sessions: for 1000x667 and 4000x2667 photos (bf16, synthetic weights, device resize, 256x256 working size) and the strokes of
tools/session_bench.py (a face-sized stroke group per step, region="auto", small mask at an offset), three modes alternated in
one process, each over the whole chain of strokes on a fresh session:
  - propose: session.propose(mask, offset=...) then proposal.close() (the photo does not change);
  - edit: session.edit(mask, offset=...);
  - propose+accept: session.accept(session.propose(mask, offset=...)).
Reports the median wall time per step and its spread (min-max over --reps).

Engine: the mask-only forward (Engine.predict_mask_u8) against the whole forward (Engine.inference_u8) at 256x256, bf16, batch
128 and batch 1, alternated, CUDA events over 20 calls, medians and spread over --reps.

Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from serving_bench import card, model  # noqa: E402
from session_bench import WORK, chain  # noqa: E402


MODES = {
    "propose": lambda s, small, off: s.propose(small, offset=off).close(),
    "edit": lambda s, small, off: s.edit(small, offset=off),
    "propose+accept": lambda s, small, off: s.accept(s.propose(small, offset=off)),
}


def time_chain(proc, img, steps, fn):
    import torch
    s = proc.open_session(img)
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for small, off, _ in steps:
            fn(s, small, off)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / len(steps)
    finally:
        s.close()


def time_engine(eng, B, reps, iters=20):
    import torch
    rs = np.random.RandomState(B)
    img = torch.from_numpy(rs.randint(0, 256, (B, 256, 256, 3), dtype=np.uint8)).cuda()
    sk = torch.zeros(B, 256, 256, dtype=torch.uint8, device="cuda")
    sk[:, 100:160, 90:170:3] = 255
    calls = {"predict_mask_u8": lambda: eng.predict_mask_u8(img, sk, precision="bf16"),
             "inference_u8": lambda: eng.inference_u8(img, sk, precision="bf16")}
    for f in calls.values():                       # capture and warm both
        for _ in range(3):
            f()
    out = {k: [] for k in calls}
    for _ in range(reps):
        for k, f in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            out[k].append(a.elapsed_time(b) / iters)
    return out


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    from sketchedit_b200.serving import DemoProcessor
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = card()
    m = model("bf16")
    proc = DemoProcessor(m, max_batch=16, max_wait_ms=0.5, region_size=WORK)
    res = {"card": name, "power_limit": power, "sessions": {}, "engine": {}}
    try:
        for w, h in ((1000, 667), (4000, 2667)):
            img, steps = chain(w, h, seed=w)
            for fn in MODES.values():              # warm-up: graphs, tables, staging buffers
                time_chain(proc, img, steps[:3], fn)
            got = {k: [] for k in MODES}
            for _ in range(args.reps):
                for k, fn in MODES.items():
                    got[k].append(time_chain(proc, img, steps, fn) * 1e3)
            res["sessions"]["%dx%d" % (w, h)] = {k: summary(v) for k, v in got.items()}
        eng = m.engine()
        for B in (128, 1):
            res["engine"]["256x256_b%d" % B] = {k: summary(v) for k, v in time_engine(eng, B, args.reps).items()}
    finally:
        proc.close()
    print("card: %s, power limit %s" % (name, power))
    for size, d in res["sessions"].items():
        for k, s in d.items():
            print("session %-9s %-15s %8.2f ms/step  (%.2f-%.2f)" % (size, k, s["median"], s["min"], s["max"]))
    for cfg, d in res["engine"].items():
        p, f = d["predict_mask_u8"], d["inference_u8"]
        print("engine  %-11s predict_mask_u8 %8.3f ms (%.3f-%.3f)  inference_u8 %8.3f ms (%.3f-%.3f)  ratio %.2f"
              % (cfg, p["median"], p["min"], p["max"], f["median"], f["min"], f["max"], p["median"] / f["median"]))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

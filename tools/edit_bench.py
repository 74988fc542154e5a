"""Cost of the forward on a supplied edit mask against the plain forward, both in their uint8 serving form.

    python tools/edit_bench.py [--reps 5] [--out FILE]

For each workload, `Engine.inference_u8` (netM predicts the mask) and `Engine.inference_with_mask_u8` (the caller's mask; netM
does not run) are timed alternately in one process on the same seeded inputs. Each run of a form is a window of `iters` calls
between CUDA events, after a warm-up that also captures both CUDA graphs. The script reports the median per-call time over
`--reps` windows with its range, the launch count of each form, and the with-mask / plain ratio. The card's name and power limit
are read in the same run. It prints one line per workload and one JSON line. Needs an H100; it writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, precision, B, H, W, calls per timed window)
WORKLOADS = [("256x256 b128 bf16", "bf16", 128, 256, 256, 3),
             ("256x256 b32 fp32", "fp32", 32, 256, 256, 3),
             ("512x512 b16 bf16", "bf16", 16, 512, 512, 3),
             ("256x256 b1 bf16 latency", "bf16", 1, 256, 256, 30),
             ("512x512 b1 bf16 latency", "bf16", 1, 512, 512, 20)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], q[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import numpy as np
    import torch

    from sketchedit_b200 import synth
    from sketchedit_b200.engine import Engine
    assert torch.cuda.is_available(), "edit_bench.py needs a GPU"
    name, power = card()
    eng = Engine.from_state_dicts(synth.synth_state_dict("M"), synth.synth_state_dict("G"))
    results = []
    for label, prec, B, H, W, iters in WORKLOADS:
        rs = np.random.RandomState(B + H)
        dev = torch.device("cuda")
        img = torch.from_numpy(rs.randint(0, 256, (B, H, W, 3), dtype=np.uint8)).to(dev)
        _, sk = synth.synth_inputs(B, H, W, seed=B + W)
        sk = (sk[:, 0] * 255).to(torch.uint8).to(dev)
        bgr = torch.empty(B, H, W, 3, device=dev, dtype=torch.uint8)
        mk = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
        bgr2 = torch.empty_like(bgr)
        eng.inference_u8(img, sk, precision=prec, out=(bgr, mk))
        edit = mk.clone()                        # the mask the plain forward predicted, as a user would feed it back
        forms = {"plain": lambda: eng.inference_u8(img, sk, precision=prec, out=(bgr, mk)),
                 "with_mask": lambda: eng.inference_with_mask_u8(img, sk, edit, precision=prec, out=bgr2)}
        launches = {}
        for k, f in forms.items():
            for _ in range(3):                   # eager, capture, replay
                f()
            launches[k] = eng.launches()
        torch.cuda.synchronize()
        ms = {k: [] for k in forms}
        for _ in range(args.reps):
            for k, f in forms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    f()
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1) / iters)
        rec = {"workload": label, "precision": prec, "B": B, "H": H, "W": W, "launches": launches}
        for k in forms:
            rec[k + "_ms"] = {"median": statistics.median(ms[k]), "min": min(ms[k]), "max": max(ms[k])}
        rec["ratio"] = rec["with_mask_ms"]["median"] / rec["plain_ms"]["median"]
        results.append(rec)
        print("%-26s plain %9.3f ms [%.3f, %.3f] (%d launches)   with mask %9.3f ms [%.3f, %.3f] (%d launches)   ratio %.3f"
              % (label, rec["plain_ms"]["median"], rec["plain_ms"]["min"], rec["plain_ms"]["max"], launches["plain"],
                 rec["with_mask_ms"]["median"], rec["with_mask_ms"]["min"], rec["with_mask_ms"]["max"], launches["with_mask"],
                 rec["ratio"]), flush=True)
        del img, sk, bgr, mk, bgr2, edit
        torch.cuda.empty_cache()
    line = {"gpu": name, "power_limit": power, "reps": args.reps, "results": results}
    print("card: %s, power limit %s" % (name, power))
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

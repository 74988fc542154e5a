"""Batch-1 latency of the whole inference at photo sizes, with the attention run in bands under the workspace limit.

    python tools/highres_bench.py [--reps 5] [--out FILE]

Prints one JSON line: the card's name and power limit (read in the same run), then per (mode, size) the median latency of
`Engine.inference` (CUDA events, after a warm-up that also captures the CUDA graph), the workspace arena
(`se_workspace_bytes`) and the attention's band count; and the 2048 x 2048 bf16 forward with the limit forcing one band and
then four, alternated in the same process. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT_LIMIT = 16 << 30
SIZES = [(1024, 1024), (2048, 2048), (3000, 4000)]


def attention_bands(prec, B, H, W, limit):
    """Band count of the attention of an H x W input (the band planners of se_cam.cu / se_gemm_split.cu, restated)."""
    h, w = H // 4, W // 4
    hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
    if prec == "bf16":
        row = B * math.ceil(ws / 8) * math.ceil(hs / 32) * 32 * ws * 16
        if row * hs <= limit:
            return 1
        return math.ceil(hs / ((limit // row - 1) // 16 * 16))
    mp = math.ceil(hs * ws / 256) * 256
    row = B * mp * 8
    return 1 if row * mp <= limit else math.ceil(mp / (limit // row // 128 * 128))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], q[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200 import synth
    from sketchedit_b200.engine import Engine, set_attention_workspace_limit
    assert torch.cuda.is_available(), "highres_bench.py needs a GPU"
    name, power = card()
    eng = Engine.from_state_dicts(synth.synth_state_dict("M"), synth.synth_state_dict("G"))

    def timed(img, sk, prec):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.inference(img, sk, precision=prec)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    results = []
    set_attention_workspace_limit(0)
    for prec in ("bf16", "fp32"):
        for H, W in SIZES:
            img, sk = synth.synth_inputs(1, H, W, seed=H + W)
            img, sk = img.cuda(), sk.cuda()
            for _ in range(2):                       # eager run, then graph capture
                timed(img, sk, prec)
            ms = [timed(img, sk, prec) for _ in range(args.reps)]
            results.append({"mode": prec, "H": H, "W": W, "latency_ms": round(statistics.median(ms), 2),
                            "latency_ms_all": [round(v, 2) for v in ms], "arena_bytes": eng.workspace_bytes(),
                            "bands": attention_bands(prec, 1, H, W, DEFAULT_LIMIT), "launches": eng.launches()})
            del img, sk
            torch.cuda.empty_cache()

    # 2048 x 2048 bf16: one band (the default limit) against four (bands of 64 query rows), alternated
    H = W = 2048
    hs = ws = (H // 4 - 4) // 2 + 1
    row = math.ceil(ws / 8) * math.ceil(hs / 32) * 32 * ws * 16
    limits = {"1": DEFAULT_LIMIT, "4": row * 65}
    assert attention_bands("bf16", 1, H, W, limits["4"]) == 4 and attention_bands("bf16", 1, H, W, limits["1"]) == 1
    img, sk = synth.synth_inputs(1, H, W, seed=5)
    img, sk = img.cuda(), sk.cuda()
    alt = {"1": [], "4": []}
    for k, lim in limits.items():
        set_attention_workspace_limit(lim)
        for _ in range(2):
            timed(img, sk, "bf16")
    for _ in range(args.reps):
        for k, lim in limits.items():
            set_attention_workspace_limit(lim)
            alt[k].append(timed(img, sk, "bf16"))
    set_attention_workspace_limit(0)
    m1, m4 = statistics.median(alt["1"]), statistics.median(alt["4"])
    line = {"gpu": name, "power_limit": power, "batch": 1, "attention_limit_bytes": DEFAULT_LIMIT, "results": results,
            "bands_2048_bf16": {"one_band_ms": [round(v, 2) for v in alt["1"]], "four_band_ms": [round(v, 2) for v in alt["4"]],
                                "median_one_ms": round(m1, 2), "median_four_ms": round(m4, 2),
                                "four_over_one": round(m4 / m1, 4)}}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

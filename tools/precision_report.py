"""Error of every precision mode against the CPU oracle on the same inputs and weights (GPU side; test infrastructure):

    python tools/precision_report.py [B H W]   ->  markdown table on stdout

max / mean |difference| of the soft mask, the fine stage and the composed image, threshold flips of the binarised mask, and
the share of uint8 output values (test.py's PNG conversion) that differ from the oracle's.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from tests.util_parity import engine, weights

B, H, W = (int(a) for a in sys.argv[1:4]) if len(sys.argv) >= 4 else (4, 256, 256)
img, sk = synth.synth_inputs(B, H, W, seed=91)
WM, WG = weights()
ref = O.inference(WM, WG, img, sk)
rg, rm = O.to_uint8_outputs(ref["composed"], ref["mask"])
eng = engine()
print("# Precision modes vs the CPU oracle (%d images %dx%d, synthetic weights)\n" % (B, H, W))
print("| mode | mask flips | max abs mask | max abs fine | max abs composed | mean abs composed | uint8 values differing |")
print("|---|---:|---:|---:|---:|---:|---:|")
for prec in ("fp32_direct", "fp32", "bf16"):
    comp, mask, ex = eng.inference(img.cuda(), sk.cuda(), precision=prec, want=("mask_bin", "fine"))
    ours_bin = ex["mask_bin"].cpu()
    flips = int((ours_bin != ref["mask_bin"]).sum())
    r = ref if flips == 0 else O.inference(WM, WG, img, sk, mask_bin_override=ours_bin)
    g, m = O.to_uint8_outputs(comp.cpu(), mask.cpu())
    rg2, _ = O.to_uint8_outputs(r["composed"], r["mask"])
    d = lambda a, b: float((a.cpu().float() - b.float()).abs().max())
    print("| %s | %d / %d | %.2e | %.2e | %.2e | %.2e | %.4f%% |" % (
        prec, flips, ours_bin.numel(), d(mask, r["mask"]), d(ex["fine"], r["fine"]), d(comp, r["composed"]),
        float((comp.cpu() - r["composed"]).abs().mean()), 100.0 * float((np.asarray(g) != np.asarray(rg2)).mean())))

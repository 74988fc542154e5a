"""On-GPU diagnostic table: per-layer / per-stage max-abs error of each precision mode vs the CPU oracle.
Usage: python tools/gpu_diag.py <group> [...]   groups: fp32 tc_plain tc_s2 tc_dil tc_stem tc_deconv tc_small heads cam nets e2e
Each group should run in its own process (a device trap poisons the CUDA context)."""
import os
import sys
import time
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from sketchedit_b200.arch import layer_map
from tests.util_parity import bf16_round, engine, maxdiff, oracle_layer, rand_act, weights

GROUPS = {
    "tc_plain": [("M", "conv3", 16, 24), ("M", "conv5", 16, 16), ("G", "conv11", 16, 16), ("G", "pmconv6", 8, 16),
                 ("G", "xconv5", 8, 24), ("M", "conv5", 64, 64)],
    "tc_s2": [("M", "conv2_downsample", 32, 48), ("G", "xconv2_downsample", 16, 32), ("M", "conv4_downsample", 32, 32),
              ("G", "xconv4_downsample", 16, 48)],
    "tc_dil": [("M", "conv7_atrous", 16, 24), ("M", "conv8_atrous", 16, 16), ("M", "conv9_atrous", 24, 16),
               ("M", "conv10_atrous", 40, 24)],
    "tc_stem": [("M", "conv1", 24, 40), ("G", "conv1", 16, 16), ("G", "xconv1", 16, 32)],
    "tc_deconv": [("M", "conv13_upsample_conv", 8, 24), ("M", "conv15_upsample_conv", 16, 16)],
    "tc_small": [("M", "conv16", 16, 32), ("G", "xconv3", 16, 24)],
    "heads": [("M", "conv17", 16, 24), ("M", "conv_mask_17", 24, 16)],
}
GROUPS["fp32"] = sum((v for k, v in GROUPS.items()), [])


def layer_case(net, name, H, W, prec):
    spec = layer_map(net)[name]
    x = rand_act((2, spec.cin, H, W), seed=abs(hash((net, name))) % 1000)
    t0 = time.time()
    y = engine().gated_conv(net, name, x.cuda(), precision=prec)
    torch.cuda.synchronize()
    y = y.cpu()
    bfw = prec != "fp32" and spec.cin != 12
    ref = oracle_layer(net, name, x, bf16_weights=bfw)
    d = maxdiff(y, ref)
    print("%-10s net%s.%-28s %3dx%-3d max|ref| %7.3f  maxdiff %.3e  finite=%s  %.2fs" % (
        prec, net, name, H, W, float(ref.abs().max()), d, bool(torch.isfinite(y).all()), time.time() - t0), flush=True)
    return d


def run_group(g):
    print("=== group", g, flush=True)
    if g in GROUPS:
        precs = ["fp32"] if g == "fp32" else (["bf16"] if g != "heads" else ["fp32", "bf16"])
        for prec in precs:
            for case in GROUPS[g]:
                try:
                    layer_case(*case, prec)
                except Exception as e:
                    print("FAIL", prec, case, repr(e)[:300], flush=True)
    elif g == "cam":
        from sketchedit_b200.engine import contextual_attention
        for (h, w, B, scale) in [(16, 16, 2, 0.5), (12, 20, 1, 0.5), (32, 32, 1, 0.15), (64, 64, 1, 0.15)]:
            feat = F.relu(rand_act((B, 96, h, w), seed=h * w, scale=scale))
            mask = torch.zeros(B, 1, 4 * h, 4 * w)
            mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
            mask_s = F.avg_pool2d(mask, 4, 4)
            ref, A = O.contextual_attention(feat, mask_s)
            for prec in ("fp32", "bf16"):
                try:
                    out, attn = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec, want_attn=True)
                    torch.cuda.synchronize()
                    print("cam %-11s %dx%d B%d  max|ref| %.3f  out diff %.3e  attn diff %.3e  Amax-mean %.3f" % (
                        prec, h, w, B, float(ref.abs().max()), maxdiff(out.cpu(), ref), maxdiff(attn.cpu(), A),
                        float(A.max(1)[0].mean())), flush=True)
                except Exception as e:
                    print("FAIL cam", prec, h, w, repr(e)[:300], flush=True)
    elif g == "nets":
        WM, WG = weights()
        img, sk = synth.synth_inputs(2, 64, 96, seed=11)
        rm, rs = O.netM_forward(WM, img, sk)
        mask = torch.zeros(2, 1, 64, 96)
        mask[0, :, 16:40, 8:50] = 1
        mask[1, :, 30:60, 20:44] = 1
        r1, r2 = O.netG_forward(WG, img, img, mask, mask, sk)
        for prec in ("fp32", "bf16"):
            try:
                m, s = engine().netM(img.cuda(), sk.cuda(), precision=prec)
                print("netM %-11s mask diff %.3e  img diff %.3e  launches %d" % (prec, maxdiff(m.cpu(), rm), maxdiff(s.cpu(), rs), engine().launches()), flush=True)
                s1, s2 = engine().netG(img.cuda(), img.cuda(), mask.cuda(), mask.cuda(), sk.cuda(), precision=prec)
                print("netG %-11s coarse diff %.3e  fine diff %.3e  launches %d" % (prec, maxdiff(s1.cpu(), r1), maxdiff(s2.cpu(), r2), engine().launches()), flush=True)
            except Exception as e:
                print("FAIL nets", prec, repr(e)[:300], flush=True)
    elif g == "e2e":
        WM, WG = weights()
        for (B, H, W) in [(2, 64, 64), (1, 128, 104), (2, 256, 256)]:
            img, sk = synth.synth_inputs(B, H, W, seed=H + W)
            ref_free = O.inference(WM, WG, img, sk)
            for prec in ("fp32", "bf16"):
                try:
                    t0 = time.time()
                    comp, m, ex = engine().inference(img.cuda(), sk.cuda(), precision=prec, want=("coarse", "fine", "mask_bin"))
                    torch.cuda.synchronize()
                    dt = time.time() - t0
                    ob = ex["mask_bin"].cpu()
                    ref = O.inference(WM, WG, img, sk, mask_bin_override=ob)
                    print("e2e %-5s B%d %dx%d flips %d  mask %.3e coarse %.3e fine %.3e composed %.3e  launches %d  ws %.1f MB  %.2fs" % (
                        prec, B, H, W, int((ob != ref_free["mask_bin"]).sum()), maxdiff(m.cpu(), ref["mask"]),
                        maxdiff(ex["coarse"].cpu(), ref["coarse"]), maxdiff(ex["fine"].cpu(), ref["fine"]),
                        maxdiff(comp.cpu(), ref["composed"]), engine().launches(), engine().workspace_bytes() / 1e6, dt), flush=True)
                except Exception as e:
                    print("FAIL e2e", prec, B, H, W, repr(e)[:300], flush=True)
    else:
        print("unknown group", g)


if __name__ == "__main__":
    for g in sys.argv[1:]:
        try:
            run_group(g)
        except Exception:
            traceback.print_exc()

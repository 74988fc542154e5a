"""Demo serving path: Pillow resizes on the request threads against the device resize (DemoProcessor resize='host' / 'device').

    python tools/serving_bench.py [--reps 5] [--out FILE]

For each request size (641x481, 1000x667, 4000x2667; bf16, synthetic weights) it reports, host and device resize alternated in
one process:
  - latency: median wall time of process_image from one thread (includes the batcher's max_wait_ms window);
  - throughput: requests/s of 16 threads submitting together (16 requests per thread, or 1 at 4000x2667);
  - the device resizes alone for one batch (the two resizes in and the one back): the three calls' time from CUDA events
    (host enqueue included), the kernels' own device time from a separate torch.profiler run, the bytes they move (each pass
    reads its input and writes its output once) and that rate over the H100 SXM data-sheet 3.35 TB/s;
  - the three Pillow resizes of one request alone, on this host.
Prints the card's name and power limit with the numbers and one JSON line. Needs an H100; nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(641, 481), (1000, 667), (4000, 2667)]       # (width, height) as the requests arrive
HBM_BYTES_PER_S = 3.35e12                              # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return q[0], q[1]


def pass_bytes(src, dst, c):
    """Bytes the device resize moves for one image: each pass reads its input once and writes its output once."""
    (ih, iw), (oh, ow) = src, dst
    if (ih, iw) == (oh, ow):
        return 2 * ih * iw * c
    b = 0
    if iw != ow:
        b += ih * iw * c + ih * ow * c
    if ih != oh:
        b += ih * ow * c + oh * ow * c
    return b


def model(precision):
    from argparse import Namespace

    import models
    from sketchedit_b200 import synth
    opt = Namespace(gpu_ids=[0], isTrain=False, isSkip=True, netG="deepfillc2", init_type="xavier", init_variance=0.02,
                    use_cam=True, pool_type="max", no_mask_cc=False, no_mask_coarse=False, joint_train_inp=True,
                    model="editline2", precision=precision)
    m = models.create_model(opt)
    m.netM.load_state_dict(synth.synth_state_dict("M"))
    m.netG.load_state_dict(synth.synth_state_dict("G"))
    return m.eval()


def request(w, h, seed):
    from PIL import Image
    rs = np.random.RandomState(seed)
    img = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    m = np.zeros((h, w), np.uint8)
    m[h // 4:h // 2, w // 3:w // 3 + max(2, w // 100)] = 255
    return Image.fromarray(img), Image.fromarray(m)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line here")
    args = ap.parse_args()

    import torch

    from sketchedit_b200.engine import resize_u8_packed
    from sketchedit_b200.serving import DemoProcessor, floor8
    assert torch.cuda.is_available(), "serving_bench.py needs a GPU"
    name, power = card()
    mdl = model(args.precision)
    results = []
    for w, h in SIZES:
        big = w * h > 4e6
        max_batch = 2 if big else 16
        per_thread = 1 if big else 16
        procs = {r: DemoProcessor(mdl, max_batch=max_batch, max_wait_ms=2.0, resize=r) for r in ("host", "device")}
        img, msk = request(w, h, seed=w)
        for p in procs.values():                                   # warm-up: graph capture, coefficient tables
            p.process_image(img, msk)
            p.process_image(img, msk)
        lat = {"host": [], "device": []}
        for _ in range(args.reps):
            for r, p in procs.items():
                t0 = time.perf_counter()
                p.process_image(img, msk)
                lat[r].append((time.perf_counter() - t0) * 1e3)

        def burst(p, n_threads):
            def worker():
                for _ in range(per_thread):
                    p.process_image(img, msk)
            ts = [threading.Thread(target=worker) for _ in range(n_threads)]
            t0 = time.perf_counter()
            [t.start() for t in ts]
            [t.join() for t in ts]
            return n_threads * per_thread / (time.perf_counter() - t0)

        for p in procs.values():
            burst(p, args.threads)                                 # warm-up of the batched shapes
        thr = {"host": [], "device": []}
        for _ in range(max(2, args.reps // 2)):
            for r, p in procs.items():
                thr[r].append(burst(p, args.threads))
        for p in procs.values():
            p.close()

        # the device resize kernels alone, one batch of max_batch requests: photo and mask in, result back
        B, H, W = max_batch, floor8(h), floor8(w)
        raw = torch.randint(0, 256, (B * h * w * 4,), dtype=torch.uint8, device="cuda")
        net = torch.empty(B * H * W * 4, dtype=torch.uint8, device="cuda")
        back = torch.empty(B * h * w * 3, dtype=torch.uint8, device="cuda")
        img_offs, msk_offs = [i * h * w * 3 for i in range(B)], [B * h * w * 3 + i * h * w for i in range(B)]
        net_img, net_msk = [i * H * W * 3 for i in range(B)], [B * H * W * 3 + i * H * W for i in range(B)]

        def resizes():
            resize_u8_packed(raw, img_offs, [(h, w)] * B, [(H, W)] * B, 3, out=net, dst_offsets=net_img)
            resize_u8_packed(raw, msk_offs, [(h, w)] * B, [(H, W)] * B, 1, out=net, dst_offsets=net_msk)
            resize_u8_packed(net, net_img, [(H, W)] * B, [(h, w)] * B, 3, swap_rb=True, out=back, dst_offsets=img_offs)

        resizes()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 20
        call_ms = []
        for _ in range(args.reps):                                 # the three calls as issued, host enqueue included
            e0.record()
            for _ in range(iters):
                resizes()
            e1.record()
            torch.cuda.synchronize()
            call_ms.append(e0.elapsed_time(e1) / iters)
        # the kernels' own time: a separate profiled run, summing the device time of the resize kernels
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                resizes()
            torch.cuda.synchronize()
        k_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                   for e in prof.key_averages() if "resize_" in e.key and "kernel" in e.key)
        k_ms = k_us / 1e3 / iters
        ev_ms = statistics.median(call_ms)
        nbytes = B * (pass_bytes((h, w), (H, W), 3) + pass_bytes((h, w), (H, W), 1) + pass_bytes((H, W), (h, w), 3))
        del raw, net, back
        torch.cuda.empty_cache()

        t_pil = []
        for _ in range(args.reps):                                 # the three Pillow resizes of process_image, alone
            t0 = time.perf_counter()
            small = img.resize((W, H))
            msk.resize((W, H))
            small.resize((w, h))
            t_pil.append((time.perf_counter() - t0) * 1e3)

        rec = {"size": "%dx%d" % (w, h), "net_size": "%dx%d" % (W, H),
               "latency_ms": {r: round(statistics.median(v), 2) for r, v in lat.items()},
               "latency_ms_all": {r: [round(x, 2) for x in v] for r, v in lat.items()},
               "threads": args.threads, "max_batch": max_batch, "requests_per_burst": args.threads * per_thread,
               "throughput_rps": {r: round(statistics.median(v), 2) for r, v in thr.items()},
               "throughput_rps_all": {r: [round(x, 2) for x in v] for r, v in thr.items()},
               "resize_kernels": {"batch": B, "bytes": nbytes,
                                  # the same bytes over two times: the three calls bracketed by CUDA events (host enqueue
                                  # included) and the resize kernels' own device time summed by torch.profiler
                                  "events_ms": round(ev_ms, 4), "events_gb_per_s": round(nbytes / ev_ms / 1e6, 1),
                                  "events_share_of_3_35_tb_s": round(nbytes / (ev_ms / 1e3) / HBM_BYTES_PER_S, 3),
                                  "kernel_ms": round(k_ms, 4), "kernel_gb_per_s": round(nbytes / k_ms / 1e6, 1),
                                  "kernel_share_of_3_35_tb_s": round(nbytes / (k_ms / 1e3) / HBM_BYTES_PER_S, 3)},
               "pillow_resizes_ms_one_request": round(statistics.median(t_pil), 2)}
        results.append(rec)
        rk = rec["resize_kernels"]
        print("%s %s (%s): %s latency host %.2f ms / device %.2f ms; %d threads: host %.1f / device %.1f req/s; resizes of a "
              "batch of %d: %.1f MB in %.3f ms by CUDA events (%.0f GB/s, %.1f%% of 3.35 TB/s), %.3f ms of kernel time (%.0f GB/s, "
              "%.1f%%); Pillow resizes alone %.2f ms"
              % (rec["size"], name, power, args.precision, rec["latency_ms"]["host"], rec["latency_ms"]["device"], args.threads,
                 rec["throughput_rps"]["host"], rec["throughput_rps"]["device"], B, nbytes / 1e6, ev_ms, rk["events_gb_per_s"],
                 100 * rk["events_share_of_3_35_tb_s"], k_ms, rk["kernel_gb_per_s"], 100 * rk["kernel_share_of_3_35_tb_s"],
                 rec["pillow_resizes_ms_one_request"]), flush=True)
    line = {"gpu": name, "power_limit": power, "precision": args.precision, "host_cpus": os.cpu_count(), "results": results}
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

"""world_size-2 gloo test of the multi-GPU host logic: contiguous batch shards + the single all-gather of the
packed outputs reproduce the single-process result (per-sample independence of the path, SURVEY.md section 8e).
The per-shard compute is the CPU oracle (the CUDA kernels cannot run here); ordering / packing / gather are the
code bench.py uses on the GPU box."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from sketchedit_b200 import parallel, synth


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    from oracle import sketchedit_oracle as O
    WM, WG = synth.synth_state_dict("M"), synth.synth_state_dict("G")
    img, sk = synth.synth_inputs(4, 32, 32, seed=1)
    lo, hi = parallel.shard_bounds(4, world, rank)
    r = O.inference(WM, WG, img[lo:hi], sk[lo:hi])
    comp, mask = parallel.all_gather_outputs(r["composed"], r["mask"])
    if rank == 0:
        full = O.inference(WM, WG, img, sk)
        ret["comp"] = float((comp - full["composed"]).abs().max())
        ret["mask"] = float((mask - full["mask"]).abs().max())
        ret["shape"] = tuple(comp.shape)
    dist.destroy_process_group()


def test_two_rank_shard_and_gather():
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert ret["shape"] == (4, 3, 32, 32)
    assert ret["comp"] <= 2e-6 and ret["mask"] <= 2e-6, dict(ret)


def test_shard_bounds():
    assert [parallel.shard_bounds(1024, 8, r) for r in (0, 7)] == [(0, 128), (896, 1024)]
    with pytest.raises(ValueError):
        parallel.shard_bounds(10, 4, 0)

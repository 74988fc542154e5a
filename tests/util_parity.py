"""Helpers shared by the GPU parity tests."""
import numpy as np
import torch

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from sketchedit_b200.arch import layer_map

_W = {}


def golden(z, key, ours):
    """(ours, reference) for golden array `key`: large arrays are stored as a fixed sample of their flat positions
    (`<key>@idx`, oracle/make_golden.py shrink), and `ours` is then restricted to the same positions."""
    ref = torch.from_numpy(z[key])
    ours = torch.as_tensor(ours).detach().cpu()
    if key + "@idx" in z.files:
        return ours.reshape(-1)[torch.from_numpy(z[key + "@idx"].astype(np.int64))], ref
    return ours, ref


def weights():
    if not _W:
        _W["M"] = synth.synth_state_dict("M")
        _W["G"] = synth.synth_state_dict("G")
    return _W["M"], _W["G"]


_ENG = {}


def engine(**opts):
    from sketchedit_b200.engine import Engine
    key = tuple(sorted(opts.items()))
    if key not in _ENG:
        WM, WG = weights()
        _ENG[key] = Engine.from_state_dicts(WM, WG, **opts)
    return _ENG[key]


def bf16_round(t):
    return t.to(torch.bfloat16).to(torch.float32)


def rand_act(shape, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    return bf16_round(torch.randn(*shape, generator=g) * scale)


def oracle_layer(net, name, x, bf16_weights):
    WM, WG = weights()
    W = WM if net == "M" else WG
    spec = layer_map(net)[name]
    w, b = W[name + ".weight"], W[name + ".bias"]
    if bf16_weights:
        w = bf16_round(w)
    return O.gated_conv(x, w, b, spec)


def maxdiff(a, b):
    return float((a - b).abs().max())

"""conv_c8 layers with streamed weights, which run as 2-CTA clusters sharing each weight stage (TMA multicast).

A cluster runs pairs of neighbouring tiles; with an odd number of tiles the last pair has no second tile and its rank-1
CTA only helps load the weights (a phantom). Every streamed layer kind runs here at tile counts of 1, 2, 3, 2 * 132 - 1,
2 * 132 + 1 and one many-tile odd number, in bf16 and split-half fp32. Each case meets the per-element bound of
tests/util_bounds.py, and every image of the batch is bit-identical to its own batch-1 run (which has its own tile count,
so phantoms fall on other tiles).
"""
import pytest
import torch

from sketchedit_b200.arch import layer_map
from tests import util_bounds as UB
from tests.util_parity import engine, maxdiff

pytestmark = pytest.mark.gpu

STREAMED_LAYERS = [
    ("M", "conv5"),              # 96->192 3x3, halo
    ("M", "conv7_atrous"),       # rate 2, halo
    ("M", "conv8_atrous"),       # rate 4, one box per tap
    ("M", "conv10_atrous"),      # rate 16, one box per tap
    ("M", "conv4_downsample"),   # stride 2: space-to-depth input
    ("G", "xconv5"),             # 48->192
    ("G", "conv11"),             # 192->192 (split-half: one 64-channel chunk per stage)
]
# (batch, Ho, Wo) of the output; tiles = batch * ceil(Ho / 16) * ceil(Wo / 8)
TILE_SHAPES = [
    (1, 13, 7),      # 1 tile: a single cluster, rank 1 a phantom
    (2, 16, 8),      # 2
    (3, 11, 5),      # 3
    (1, 15, 2100),   # 263 = 2 * 132 - 1
    (5, 16, 424),    # 265 = 2 * 132 + 1
    (3, 136, 164),   # 567 = 3 * 9 * 21, partial tiles at both edges
]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("B,Ho,Wo", TILE_SHAPES)
@pytest.mark.parametrize("net,name", STREAMED_LAYERS)
def test_streamed_layer_pairs(net, name, B, Ho, Wo, prec):
    spec = layer_map(net)[name]
    H, W = UB.thin_input(spec, Ho, Wo)
    x = UB.conv_input(net, name, B, H, W, "unit", UB.stable_seed(net, name, B, Ho, Wo))
    y = engine().gated_conv(net, name, x.cuda(), precision=prec).cpu()
    r = UB.reference(net, name, x, prec)
    assert y.shape == r["Y"].shape, (y.shape, r["Y"].shape)
    q = UB.max_ratio(y, r["Y"], UB.gated_bound(r, prec))
    assert q <= 1.0, (net, name, B, Ho, Wo, prec, q)
    for i in range(B if B > 1 else 0):
        yi = engine().gated_conv(net, name, x[i:i + 1].cuda(), precision=prec).cpu()
        assert torch.equal(yi[0], y[i]), (name, prec, i, maxdiff(yi[0], y[i]))

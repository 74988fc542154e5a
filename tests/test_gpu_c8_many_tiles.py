"""conv_c8 layers at shapes where every CTA of the persistent grid runs several tiles.

The shapes of test_gpu_ops.py mostly give fewer tiles than the H100 has SMs, so each CTA runs one tile. Here a batch of 3
gives 231-405 tiles (or virtual tiles x sub-pixel classes) per launch: not a multiple of 132, with CTAs running an odd number
of tiles, and with partial tiles at the bottom edge. Each case is held to the tolerance of test_gpu_ops.py, and every image
of the batch must be bit-identical to its own batch-1 run.
"""
import pytest
import torch

from tests.util_parity import engine, maxdiff, oracle_layer, rand_act
from sketchedit_b200.arch import layer_map

pytestmark = pytest.mark.gpu

B = 3
# (net, layer, H, W) of the layer input; tiles per launch = B * ceil(Ho / 16) * ceil(Wo / 8) on the position grid
MANY_TILE_CASES = [
    ("M", "conv1", 120, 96),                    # 5x5 stem: 288 tiles
    ("M", "conv16", 136, 120),                  # 24->24: 405 tiles
    ("M", "conv3", 100, 88),                    # 48->96, resident weights: 231 tiles
    ("M", "conv5", 100, 88),                    # 96->192, streamed weights
    ("M", "conv9_atrous", 100, 88),             # rate 8, one box per tap
    ("G", "conv11", 100, 88),                   # 192->192
    ("M", "conv15_upsample_conv", 100, 88),     # deconv 48->48 (four classes fused in bf16)
    ("M", "conv13_upsample_conv", 100, 88),     # deconv 96->96 (two classes fused in bf16)
    ("G", "pmconv6", 100, 88),                  # ReLU gate
    ("M", "conv2_downsample", 200, 176),        # 24->96 stride 2: 231 tiles
]


def _per_image_identical(net, name, x, y, prec):
    for i in range(x.shape[0]):
        yi = engine().gated_conv(net, name, x[i:i + 1].cuda(), precision=prec).cpu()
        assert torch.equal(yi[0], y[i]), (name, prec, i, maxdiff(yi[0], y[i]))


@pytest.mark.parametrize("net,name,H,W", MANY_TILE_CASES)
def test_many_tiles_bf16(net, name, H, W):
    spec = layer_map(net)[name]
    x = rand_act((B, spec.cin, H, W), seed=(H * W + spec.cin) % 1000 + 11)
    y = engine().gated_conv(net, name, x.cuda(), precision="bf16").cpu()
    ref = oracle_layer(net, name, x, bf16_weights=True)
    assert y.shape == ref.shape
    tol = float(ref.abs().max()) * 2.0 ** -8 + 1e-3
    if spec.kind == "deconv":
        tol *= 2     # sub-pixel taps are summed in fp32 and THEN rounded to bf16 (oracle rounds each tap)
    assert maxdiff(y, ref) <= tol, (name, maxdiff(y, ref), tol)
    _per_image_identical(net, name, x, y, "bf16")


@pytest.mark.parametrize("net,name,H,W", MANY_TILE_CASES)
def test_many_tiles_fp32_split_half(net, name, H, W):
    spec = layer_map(net)[name]
    seed = (H * W + spec.cin) % 1000 + 13
    x = rand_act((B, spec.cin, H, W), seed=seed)
    x = x + 1e-3 * rand_act((B, spec.cin, H, W), seed=seed + 1)      # not bf16-representable: the lo halves matter
    y = engine().gated_conv(net, name, x.cuda(), precision="fp32").cpu()
    ref = oracle_layer(net, name, x, bf16_weights=False)
    assert y.shape == ref.shape
    assert maxdiff(y, ref) <= 1e-4, (name, maxdiff(y, ref))
    _per_image_identical(net, name, x, y, "fp32")

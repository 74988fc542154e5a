"""conv_c8 launches that run two teams of consumer warpgroups per CTA (resident weights, one k-step per tile).

A launch runs two teams when its CTAs run at least two tiles (more tiles than the H100's 132 SMs) and its halo ring is four
buffers deep; team t of a CTA runs the CTA's tiles t, t + 2, ... Each layer kind that takes this path through the
per-operator call runs here at tile counts that give a CTA 1-2, 2-3, 4-5 and 12-13 tiles, with image edges inside a tile,
in bf16 and split-half fp32, and every image of the batch must be bit-identical to its own batch-1 run: that run maps
tiles to CTAs and teams differently (the small shapes run one team, one tile per CTA), so an error that depends on the
team, the ring slot or the tile's place in a CTA's sequence shows. The stem pairs only run inside a forward: the whole
forward on a batch equals the batch-1 forwards. (The 96->96 deconv keeps one team, its ring is two deep: the control.)
"""
import pytest
import torch

from sketchedit_b200 import synth
from sketchedit_b200.arch import layer_map
from tests import util_bounds as UB
from tests.util_parity import engine, maxdiff

pytestmark = pytest.mark.gpu

TEAM_LAYERS = [
    ("M", "conv16"),                 # 24->24
    ("M", "conv1"),                  # 5x5 stem
    ("M", "conv3"),                  # 48->96
    ("G", "xconv3"),                 # 24->96 stride 1
    ("M", "conv2_downsample"),       # 24->96 stride 2: space-to-depth input
    ("G", "xconv2_downsample"),      # 24->48 stride 2
    ("M", "conv15_upsample_conv"),   # deconv 48->48: four classes fused in bf16, one launch per class in split-half
    ("M", "conv13_upsample_conv"),   # deconv 96->96: two classes fused, one team
]
# (batch, Ho, Wo) of the tile grid (the output; the input of a deconv); tiles = batch * ceil(Ho / 16) * ceil(Wo / 8)
TILE_SHAPES = [
    (2, 40, 180),    # 138: six CTAs run two tiles (their second team one), the others one
    (3, 72, 140),    # 270: two or three tiles per CTA, teams of 1 + 1 and 2 + 1
    (3, 136, 164),   # 567: four or five
    (5, 200, 196),   # 1625: twelve or thirteen; batch 1 (325 tiles) runs two teams too, on another mapping
]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("B,Ho,Wo", TILE_SHAPES)
@pytest.mark.parametrize("net,name", TEAM_LAYERS)
def test_batch_equals_its_images(net, name, B, Ho, Wo, prec):
    spec = layer_map(net)[name]
    H, W = (Ho, Wo) if spec.kind == "deconv" else UB.thin_input(spec, Ho, Wo)
    x = UB.conv_input(net, name, B, H, W, "unit", UB.stable_seed(net, name, B, Ho, Wo))
    y = engine().gated_conv(net, name, x.cuda(), precision=prec).cpu()
    assert torch.isfinite(y).all()
    for i in range(B):
        yi = engine().gated_conv(net, name, x[i:i + 1].cuda(), precision=prec).cpu()
        assert torch.equal(yi[0], y[i]), (name, prec, i, maxdiff(yi[0], y[i]))


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("B,H,W", [(5, 104, 136), (3, 88, 120)])
def test_forward_batch_equals_its_images(B, H, W, prec):
    # stem pairs: 595 / 165 tiles at full size for the batch (two teams), 119 / 55 for one image (one team)
    img, sk = synth.synth_inputs(B, H, W, seed=B * H + W)
    eng = engine()
    comp, mask, _ = eng.inference(img.cuda(), sk.cuda(), precision=prec)
    comp, mask = comp.cpu(), mask.cpu()
    for i in range(B):
        c1, m1, _ = eng.inference(img[i:i + 1].cuda(), sk[i:i + 1].cuda(), precision=prec)
        assert torch.equal(m1.cpu()[0], mask[i]), (prec, i)
        assert torch.equal(c1.cpu()[0], comp[i]), (prec, i, maxdiff(c1.cpu()[0], comp[i]))

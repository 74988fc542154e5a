"""The attention's softmax weights, as the callers receive them, against float64 with per-element bounds
(tests/util_bounds.py): contextual_attention(..., want_attn=True) in bf16 (cam_attn_export_kernel rewriting P from the S
kernel's key-tile order) and in fp32 / fp32_direct (the CUDA-core map), ReduceContextAttentionP1, and the maps the export
forward returns for region-edit detail in all three precisions, each on the forward's own tapped attention input.

Map shapes reach the key-tile index terms: one key (L = 1), exactly one 32 x 8 key tile, one key row and one key column past
it, several tile rows and columns, and the 256^2 and 512^2 forwards' 64 x 64 and 128 x 128 maps (hs = 63: two tile rows).
The float64 references run on the GPU (L = 3969 takes about 126 MB per [L, L] float64 map). Each check prints
max |attn - P| / bound."""
import pytest
import torch

from sketchedit_b200.engine import contextual_attention
from tests import util_bounds as UB
from tests.test_gpu_error_bounds import CAM_MASKS, _feat, _mask_s
from tests.test_gpu_mask_preview import _u8_inputs
from tests.test_gpu_region_detail import _softmax_bound
from tests.util_parity import engine
from tests.util_taps import decode_all

pytestmark = pytest.mark.gpu

# feature map (h, w) -> (hs, ws): 1 x 1; 32 x 8 (one key tile); 33 x 9; 65 x 17; 33 x 49; 31 x 31 (256^2); 63 x 63 (512^2)
MAPS = [(4, 4), (66, 18), (68, 20), (132, 36), (68, 100), (64, 64), (128, 128)]
MODES = ["bf16", "fp32", "fp32_direct"]


def _inputs(h, w, mkind):
    if mkind == "per_image":                    # B = 2, image 0 one rectangle, image 1 the 25/256 | 26/256 split
        feat = _feat("0.15", 2, h, w, seed=UB.stable_seed("map", h, w, mkind))
        return feat, torch.cat([_mask_s("rect", 1, h, w), _mask_s("frac25_26", 1, h, w)])
    return _feat("0.15", 1, h, w, seed=UB.stable_seed("map", h, w, mkind)), _mask_s(mkind, 1, h, w)


def map_reference(feat, mask_s, mode):
    """(P, bound) [B, keys, queries] of the map of `mode` on the GPU: bf16 Pb and Wp, the fp32 CUDA-core map's bound."""
    feat, mask_s = feat.cuda(), mask_s.cuda()
    return UB.attention_bf16_map(feat, mask_s) if mode == "bf16" else UB.attention_fp32_map(feat, mask_s)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("mkind", CAM_MASKS + ["per_image"])
@pytest.mark.parametrize("h,w", MAPS)
def test_attention_map_within_bound(h, w, mkind, mode, capsys):
    feat, mask_s = _inputs(h, w, mkind)
    _, attn = contextual_attention(feat.cuda(), mask_s.cuda(), precision=mode, want_attn=True)
    B, hs, ws = feat.shape[0], (h - 4) // 2 + 1, (w - 4) // 2 + 1
    assert attn.shape == (B, hs * ws, hs * ws)
    P, bound = map_reference(feat, mask_s, mode)
    q = UB.max_ratio(attn, P, bound)
    with capsys.disabled():
        print("\n[attention map %s %dx%d -> %dx%d B%d %s] max ratio %.3g" % (mode, h, w, hs, ws, B, mkind, q))
    assert q <= 1.0, q


def test_p1_returns_the_checked_map():
    from models.networks.splitcam import ReduceContextAttentionP1
    cam_1 = ReduceContextAttentionP1(nn_hard=False, ufstride=2, stride=2, bkg_patch_size=4, pd=0, is_th=True, th=0.1, norm_type=1)
    feat, mask_s = _inputs(68, 20, "per_image")
    f, m = feat.cuda(), mask_s.cuda()
    got = cam_1(f, f, m)
    _, attn = contextual_attention(f, m, precision="bf16", want_attn=True)
    assert got.shape == (2, 33 * 9, 33, 9) and torch.equal(got.reshape(attn.shape), attn)
    Pb, Wp = UB.attention_bf16_map(f, m)
    assert UB.max_ratio(attn, Pb, Wp) <= 1.0


# working sizes of the export forward: 512 x 512 (map 128 x 128, hs = 63) and 272 x 200 (map 68 x 50, hs = 33, ws = 24)
@pytest.mark.parametrize("prec", MODES)
@pytest.mark.parametrize("B,H,W", [(1, 512, 512), (2, 272, 200)])
def test_export_forward_map_within_bound(B, H, W, prec, capsys):
    eng = engine()
    img, sk = _u8_inputs(B, H, W, seed=H + W)
    eng.set_taps(True)
    try:
        _, _, attn, _ = eng.inference_u8_export(img, sk, precision=prec)
        taps = decode_all(eng.taps())
    finally:
        eng.set_taps(False)
    feat = taps["in:G.cam.f32" if prec == "fp32" else "in:G.cam"][0].cuda().double()
    mask_s = taps["in:G.cam.mask_s"][0].cuda().double()
    assert feat.shape[2:] == (H // 4, W // 4)
    if prec == "bf16":
        P, bound = UB.attention_bf16_map(feat, mask_s)
    elif prec == "fp32":
        # the split-half softmax's own fp32 write, bounded from its logit error model around the exact softmax
        P = UB.attention_fp32_map(feat, mask_s)[0]
        bound = _softmax_bound(feat, P, "fp32").double()
    else:
        P, bound = UB.attention_fp32_map(feat, mask_s)
    q = UB.max_ratio(attn, P, bound)
    with capsys.disabled():
        print("\n[export map %s %dx%d B%d] max ratio %.3g" % (prec, H, W, B, q))
    assert q <= 1.0, q

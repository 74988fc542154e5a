"""Contextual attention in bands of query rows under a workspace limit (se_set_attention_workspace_limit).

The L x L temporaries of the attention (probabilities; logits in the fp32 modes) are computed band by band through one
band-sized buffer, so the output must not depend on the band split (torch.equal against one band), and map sizes whose
L x L tensors exceed the device's memory run. Large sizes are checked at sampled pixels against the pointwise fp64
reference in tests/util_attention.py.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sketchedit_oracle as O
from tests.util_attention import contextual_attention_at, sample_pixels
from tests.util_parity import rand_act

GiB = 1 << 30


# ----------------------------------------------------------------------------- CPU: the pointwise reference
@pytest.mark.parametrize("h,w,B", [(64, 64, 2), (128, 102, 1)])
def test_pointwise_reference_matches_the_oracle(h, w, B):
    feat = F.relu(rand_act((B, 96, h, w), seed=h * w + 3))
    mask = torch.zeros(B, 1, 4 * h, 4 * w)
    mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
    mask[0, :, :24, :40] = 1.0                       # a masked corner
    mask_s = F.avg_pool2d(mask, 4, 4)
    ref, _ = O.contextual_attention(feat.double(), mask_s.double())
    px = sample_pixels(B, h, w, 24, seed=h + w, extra=[(0, 2, 3), (0, h // 2, w // 3), (B - 1, 3 * h // 4, w // 2)])
    got = contextual_attention_at(feat, mask_s, px, key_rows=7)    # several key-row chunks, one of them short
    want = torch.stack([ref[b, :, y, x] for b, y, x in px])
    assert float((got - want).abs().max()) <= 1e-6


# ----------------------------------------------------------------------------- band plans (bytes per query row, mirrored)
def _grid(h, w):
    return (h - 4) // 2 + 1, (w - 4) // 2 + 1


def bf16_row_bytes(B, h, w):
    """P of one query row (se_cam.cu cam_plan): B x key blocks x ws x 16 B; bands of 16-row multiples + one carried row."""
    hs, ws = _grid(h, w)
    kb = math.ceil(ws / 8) * math.ceil(hs / 32) * 32
    return B * kb * ws * 16


def split_row_bytes(B, h, w):
    """S (fp32) + P (fp16 hi + lo) of one query row (se_gemm_split.cu cam_split_plan); bands of 128-row multiples."""
    hs, ws = _grid(h, w)
    return B * math.ceil(hs * ws / 256) * 256 * 8


def direct_row_bytes(B, h, w):
    """S + P (both fp32) of one row of queries (se_engine.cu run_cam); bands of R class rows hold R + 1 query rows."""
    hs, ws = _grid(h, w)
    return B * ws * math.ceil(hs * ws / 128) * 128 * 8


def forced_limits(prec, B, h, w):
    """Limits that force several bands: the minimum band height, and a taller band that leaves an awkward remainder."""
    hs, ws = _grid(h, w)
    if prec == "bf16":
        r = bf16_row_bytes(B, h, w)
        return [r * 17, r * 49] if hs > 48 else [r * 17]
    if prec == "fp32":
        r = split_row_bytes(B, h, w)
        return [r * 128, r * 384]
    r = direct_row_bytes(B, h, w)
    return [r * 2, r * 6]                            # 1 and 5 class rows per band


def _launches():
    from sketchedit_b200 import _lib
    return int(_lib.load().se_last_launch_count())


@pytest.fixture
def attention_limit():
    """Sets the process-wide limit for one test and restores the default afterwards."""
    from sketchedit_b200.engine import set_attention_workspace_limit
    yield set_attention_workspace_limit
    set_attention_workspace_limit(0)


def _cam_inputs(B, h, w, seed, scale=0.5):
    feat = F.relu(rand_act((B, 96, h, w), seed=seed, scale=scale))
    mask = torch.zeros(B, 1, 4 * h, 4 * w)
    mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
    return feat, F.avg_pool2d(mask, 4, 4)


# ----------------------------------------------------------------------------- GPU: bands are invisible
@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "fp32", "fp32_direct"])
@pytest.mark.parametrize("h,w,B", [(64, 64, 2), (128, 102, 1), (256, 256, 1)])
def test_attention_bands_are_bit_identical(prec, h, w, B, attention_limit):
    from sketchedit_b200.engine import contextual_attention
    feat, mask_s = _cam_inputs(B, h, w, seed=h * w + 5, scale=0.15 if prec == "bf16" else 0.5)
    feat, mask_s = feat.cuda(), mask_s.cuda()
    attention_limit(0)
    one = contextual_attention(feat, mask_s, precision=prec)
    n_one = _launches()
    for lim in forced_limits(prec, B, h, w):
        attention_limit(lim)
        banded = contextual_attention(feat, mask_s, precision=prec)
        assert _launches() > n_one, (lim, _launches(), n_one)        # several bands ran
        assert torch.equal(banded, one), (prec, lim, float((banded - one).abs().max()))


@pytest.mark.gpu
def test_limit_below_one_band_fails_and_names_the_bytes(attention_limit):
    from sketchedit_b200._lib import SketchEditB200Error
    from sketchedit_b200.engine import contextual_attention
    feat, mask_s = _cam_inputs(1, 64, 64, seed=1)
    attention_limit(1024)
    with pytest.raises(SketchEditB200Error, match=str(bf16_row_bytes(1, 64, 64) * 17)):
        contextual_attention(feat.cuda(), mask_s.cuda(), precision="bf16")
    with pytest.raises(SketchEditB200Error, match=str(split_row_bytes(1, 64, 64) * 128)):
        contextual_attention(feat.cuda(), mask_s.cuda(), precision="fp32")
    with pytest.raises(SketchEditB200Error):
        attention_limit(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_inference_bands_are_bit_identical(prec, attention_limit):
    from sketchedit_b200 import synth
    from tests.util_parity import engine
    B, H, W = 2, 1024, 768
    img, sk = synth.synth_inputs(B, H, W, seed=31)
    img, sk = img.cuda(), sk.cuda()
    eng = engine()
    attention_limit(0)
    one, m_one, _ = eng.inference(img, sk, precision=prec)
    one, m_one, n_one = one.clone(), m_one.clone(), eng.launches()
    lim = forced_limits(prec, B, H // 4, W // 4)[-1]
    attention_limit(lim)
    for _ in range(3):                                   # eager, captured and replayed: the limit is part of the graph key
        banded, m_b, _ = eng.inference(img, sk, precision=prec)
        assert eng.launches() > n_one
        assert torch.equal(banded, one) and torch.equal(m_b, m_one)
    attention_limit(0)
    again, _, _ = eng.inference(img, sk, precision=prec)
    assert eng.launches() == n_one and torch.equal(again, one)


# ----------------------------------------------------------------------------- GPU: sizes whose L x L tensors do not fit
def _check_sampled(out, feat, mask_s, px, rel):
    ref = contextual_attention_at(feat, mask_s, px)
    got = torch.stack([out[b, :, y, x] for b, y, x in px]).double()
    tol = rel * torch.clamp(ref.abs(), min=1.0)
    bad = (got - ref).abs() > tol
    assert not bool(bad.any()), (int(bad.sum()), float((got - ref).abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("prec,h,w,rel", [("bf16", 750, 1000, 2e-2), ("fp32", 750, 1000, 1e-3), ("fp32_direct", 480, 480, 2e-4)])
def test_attention_beyond_the_single_band_size(prec, h, w, rel, attention_limit):
    """750 x 1000 is the map of a 3000 x 4000 image (L = 186,626 patches: P alone would be 72 GB in bf16). The split-half
    fp32 mode sums 186,626 keys per output in the tensor-core accumulators: its error there was 5.9e-4 relative (2e-4 holds
    at the smaller maps of test_gpu_ops.py), so it is held to 1e-3, the end-to-end bound of the fp32 modes. Two different
    band splits must still agree bit for bit."""
    from sketchedit_b200.engine import contextual_attention
    feat, mask_s = _cam_inputs(1, h, w, seed=7, scale=0.15 if prec == "bf16" else 0.5)
    attention_limit(8 * GiB)
    out = contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec)
    attention_limit(5 * GiB)
    assert torch.equal(contextual_attention(feat.cuda(), mask_s.cuda(), precision=prec), out)
    out = out.cpu()
    px = sample_pixels(1, h, w, 64, seed=h, extra=[(0, h // 2, w // 2 + 1), (0, h // 3, w // 2 + 3)])   # inside the hole too
    assert len(px) >= 256
    _check_sampled(out, feat, mask_s, px, rel)


@pytest.mark.gpu
def test_fp32_inference_at_1024_vs_oracle(attention_limit):
    """The split-half fp32 mode at 1024 x 1024 (L = 16,129) against the CPU oracle, with the mask rules of
    test_gpu_forward.py::test_inference_vs_oracle: netG and the outputs are compared with the oracle evaluated on OUR binarised
    mask. The threshold flips against the oracle's own mask come from netM (before the attention); at 64 x 64 there are none,
    at 1024 x 1024 there were 2 of 1,048,576 pixels, so they are bounded at 1e-5 of the pixels."""
    from sketchedit_b200 import synth
    from tests.util_parity import engine, maxdiff, weights
    WM, WG = weights()
    img, sk = synth.synth_inputs(1, 1024, 1024, seed=41)
    attention_limit(4 * GiB)
    composed, mask, ex = engine().inference(img.cuda(), sk.cuda(), precision="fp32", want=("coarse", "fine", "mask_bin"))
    ours_bin = ex["mask_bin"].cpu()
    with torch.no_grad():
        ref_mask, _ = O.netM_forward(WM, img, sk)
    assert int((ours_bin != (ref_mask > 0.5).float()).sum()) <= 1e-5 * ours_bin.numel()
    ref = O.inference(WM, WG, img, sk, mask_bin_override=ours_bin)
    assert maxdiff(mask.cpu(), ref["mask"]) <= 1e-3
    for k, t in (("coarse", ex["coarse"]), ("fine", ex["fine"]), ("composed", composed)):
        assert maxdiff(t.cpu(), ref[k]) <= 1e-3, (k, maxdiff(t.cpu(), ref[k]))


@pytest.mark.gpu
def test_demo_processor_on_a_12_megapixel_photo(attention_limit):
    from PIL import Image

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    limit = 8 * GiB
    attention_limit(limit)
    proc = DemoProcessor(_model("bf16"), max_batch=1, max_wait_ms=1.0)
    rs = np.random.RandomState(3)
    W, H = 4000, 3000
    img = Image.fromarray(rs.randint(0, 256, (H, W, 3), dtype=np.uint8))
    m = np.zeros((H, W), np.uint8)
    m[1000:1400, 1500:2600] = 255
    try:
        res = proc.process_image(img, Image.fromarray(m))
    finally:
        proc.close()
    assert res.size == (W, H)
    arr = np.array(res)
    assert arr.shape == (H, W, 3) and arr.std() > 0
    # the arena holds the attention band (<= limit) and linear activations, nothing L x L (P alone would be 72 GB)
    assert proc.engine.workspace_bytes() <= limit + 1024 * H * W


# ----------------------------------------------------------------------------- GPU: tensors beyond 2^31 bytes
@pytest.mark.gpu
def test_bf16_batch_48_at_1024(attention_limit):
    """Activations of 2.4 GB and more (a 24-channel full-resolution map at batch 48): the last image equals its batch-1 run."""
    from sketchedit_b200 import synth
    from tests.util_parity import engine
    img, sk = synth.synth_inputs(48, 1024, 1024, seed=48)
    attention_limit(4 * GiB)
    eng = engine()
    full, fm, _ = eng.inference(img.cuda(), sk.cuda(), precision="bf16")
    last, lm = full[47].cpu(), fm[47].cpu()
    del full, fm
    one, om, _ = eng.inference(img[47:].cuda(), sk[47:].cuda(), precision="bf16")
    assert torch.equal(one[0].cpu(), last) and torch.equal(om[0].cpu(), lm)

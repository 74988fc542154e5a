"""Every stage of the real forward against float64, on the forward's own stored intermediate tensors.

With activation taps on (se_taps_enable, Engine.set_taps) a forward records the stored bytes of every stage input. They are
decoded from DESIGN.md section 4's layouts (tests/util_taps.py) and every edge of the graph is checked with the
per-element bounds of tests/util_bounds.py (tests/util_stages.py): each gated conv / deconv / stem on its own stored input,
the packed network inputs bit for bit, the heads and their blends, the threshold, the global style pooling and its
broadcast into the concat, the pooled attention mask and the attention itself. Workloads: inference in all three
precisions at several shapes, bf16 at the bench shape, every reference-golden flag set, netG with separate x / x2 and
mask / mask2, with a soft mask, and with guide=None, and the uint8 entry point. Each check prints its max ratio.

Taps must not change results: a tapped forward equals the captured-and-replayed untapped one bit for bit, with the same
launch count.
"""
import glob
import os

import numpy as np
import pytest
import torch

from sketchedit_b200 import synth
from tests import util_stages as US
from tests.test_gpu_error_bounds import _netG_inputs
from tests.util_parity import engine
from tests.util_taps import decode_all

pytestmark = pytest.mark.gpu
PRECS = ["bf16", "fp32", "fp32_direct"]
WANT = ("coarse", "fine", "mask_bin", "mask_image")


def _tapped(eng, fn):
    eng.set_taps(True)
    try:
        out = fn()
        torch.cuda.synchronize()
        taps = eng.taps()
        torch.cuda.synchronize()
    finally:
        eng.set_taps(False)
    dec = decode_all(taps)
    T = {k: v[0] for k, v in dec.items()}
    pads = {k: v[1] for k, v in dec.items()}
    raw = {k: r.cpu() for k, (_, r) in taps.items()}
    return out, T, pads, raw


def _inference(prec, img, sk, flags):
    eng = engine(**flags)
    (composed, mask, ex), T, pads, raw = _tapped(eng, lambda: eng.inference(img.cuda(), sk.cuda(), precision=prec, want=WANT))
    io = dict(netM=True, x=img, x2=img, mask=ex["mask_bin"].cpu(), mask2=ex["mask_bin"].cpu(), guide=sk, soft=mask.cpu(),
              mask_bin=ex["mask_bin"].cpu(), composed=composed.cpu(), coarse=ex["coarse"].cpu(), fine=ex["fine"].cpu(),
              mask_image=ex["mask_image"].cpu())
    return T, pads, raw, io


def _report(label, res):
    for k in sorted(res):
        print("stage %s %s: max ratio %.3g" % (label, k, res[k]))
    print("stage %s per class: %s" % (label, {k: float("%.3g" % v) for k, v in US.summary(res).items()}))
    bad = {k: v for k, v in res.items() if not v <= 1.0}
    assert not bad, bad


def _check(label, T, pads, raw, io, flags, prec):
    _report(label, US.check_forward(T, pads, io, flags, prec, raw))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("B,H,W", [(2, 64, 64), (1, 24, 40), (1, 128, 104)])
def test_inference_stages(prec, B, H, W):
    img, sk = synth.synth_inputs(B, H, W, seed=H * 3 + W)
    T, pads, raw, io = _inference(prec, img, sk, {})
    _check("%s %dx%dx%d" % (prec, B, H, W), T, pads, raw, io, {}, prec)


def test_inference_stages_bench_shape_bf16():
    img, sk = synth.synth_inputs(1, 256, 256, seed=256)
    T, pads, raw, io = _inference("bf16", img, sk, {})
    _check("bf16 1x256x256", T, pads, raw, io, {}, "bf16")


def _golden_flag_sets():
    sets = {}
    for p in sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))):
        flags = dict(eval(str(np.load(p)["flags"])))
        sets.setdefault(tuple(sorted(flags.items())), os.path.basename(p)[:-4])
    return [dict(k) for k in sets]


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("flags", _golden_flag_sets(), ids=lambda f: "-".join("%s=%s" % kv for kv in sorted(f.items())) or "default")
def test_golden_flag_sets_stages(prec, flags):
    img, sk = synth.synth_inputs(1, 64, 64, seed=41)
    T, pads, raw, io = _inference(prec, img, sk, flags)
    _check("%s flags %s" % (prec, flags), T, pads, raw, io, flags, prec)


def _netG(prec, x, x2, m, m2, g, flags=None):
    eng = engine(**(flags or {}))
    cu = lambda t: None if t is None else t.cuda()
    xc, mc = cu(x), cu(m)
    x2c, m2c = xc if x2 is x else cu(x2), mc if m2 is m else cu(m2)   # one tensor for both: the paired path
    (s1, s2), T, pads, raw = _tapped(eng, lambda: eng.netG(xc, x2c, mc, m2c, cu(g), precision=prec))
    io = dict(netM=False, x=x, x2=x2, mask=m, mask2=m2, guide=g, coarse=s1.cpu(), fine=s2.cpu())
    return T, pads, raw, io


@pytest.mark.parametrize("prec", PRECS)
def test_netG_unpaired_stages(prec):
    """x != x2 and mask != mask2: the unpaired stems (bf16: two pack8 buffers, no stem pair)."""
    img, img2, mask, mask2, sk = _netG_inputs()
    T, pads, raw, io = _netG(prec, img, img2, mask, mask2, sk)
    if prec == "bf16":
        assert "in:G.conv1" in T and "in:G.wconv1" in T and "in:G.conv1+wconv1" not in T
    _check("%s netG unpaired" % prec, T, pads, raw, io, {}, prec)


@pytest.mark.parametrize("prec", PRECS)
def test_netG_soft_mask_stages(prec):
    """a mask of eighths (not binary): the coarse blend's (1 - m)^2 on the image, the stems' mask products and the pooled
    attention mask are all exercised off {0, 1}."""
    img, _, _, _, sk = _netG_inputs()
    yy, xx = torch.meshgrid(torch.arange(64), torch.arange(64), indexing="ij")
    m = (((yy // 4 + 3 * (xx // 4)) % 9).float() / 8.0).expand(2, 1, 64, 64).contiguous()
    T, pads, raw, io = _netG(prec, img, img, m, m, sk)
    _check("%s netG soft mask" % prec, T, pads, raw, io, {}, prec)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_netG_without_guide_stages(prec):
    img, img2, mask, mask2, _ = _netG_inputs()
    T, pads, raw, io = _netG(prec, img, img, mask, mask, None)
    _check("%s netG guide=None" % prec, T, pads, raw, io, {}, prec)


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_inference_u8_stem_inputs(prec):
    """the uint8 entry point's input codec: its packed stem inputs are bit for bit those of the float forward on the
    host-decoded inputs (reference data/testimage_dataset.py:89-103)."""
    rs = np.random.RandomState(5)
    img_u8 = torch.from_numpy(rs.randint(0, 256, (2, 64, 64, 3), dtype=np.uint8))
    _, sk = synth.synth_inputs(2, 64, 64, seed=5)
    sk_u8 = (sk[:, 0] * 255).to(torch.uint8)
    sk_u8[0, 10:14, 5:40] = 7
    image = img_u8.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5).contiguous()
    sketch = (sk_u8.float().div(255)[:, None] > 0).float()
    eng = engine()
    _, _, _, raw_u8 = _tapped(eng, lambda: eng.inference_u8(img_u8.cuda(), sk_u8.cuda(), precision=prec))
    _, _, _, raw_f = _tapped(eng, lambda: eng.inference(image.cuda(), sketch.cuda(), precision=prec))
    stems = [k for k in raw_f if k in ("in:M.conv1", "in:G.conv1+wconv1", "in:G.conv1", "in:G.wconv1")]
    assert "in:M.conv1" in stems and len(stems) >= 2, stems
    for k in stems:
        assert torch.equal(raw_u8[k], raw_f[k]), k


@pytest.mark.parametrize("prec", PRECS)
def test_eager_captured_replayed_and_tapped_agree(prec):
    """the first call of a signature runs eagerly, the second is captured into a CUDA graph, the third replays it; a
    tapped call runs eagerly again. All four give the same bytes, and taps add no kernel launch."""
    eng = engine()
    img, sk = synth.synth_inputs(2, 64, 64, seed=77)
    img, sk = img.cuda(), sk.cuda()
    out = (torch.empty(2, 3, 64, 64, device="cuda"), torch.empty(2, 1, 64, 64, device="cuda"))
    got, launches = [], []
    for _ in range(3):
        eng.inference(img, sk, precision=prec, out=out)
        torch.cuda.synchronize()
        got.append(tuple(t.cpu().clone() for t in out))
        launches.append(eng.launches())
    _, _, _, raw = _tapped(eng, lambda: eng.inference(img, sk, precision=prec, out=out))
    got.append(tuple(t.cpu().clone() for t in out))
    launches.append(eng.launches())
    assert len(raw) > 60
    for g in got[1:]:
        assert all(torch.equal(a, b) for a, b in zip(got[0], g))
    assert len(set(launches)) == 1, launches
    eng.set_taps(False)
    assert int(eng.lib.se_taps_count(eng.h)) == 0

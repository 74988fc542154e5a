"""Mask previews on the GPU: Engine.predict_mask_u8 is the forward's own netM mask, bit for bit, in every precision and batch
split, and Engine.inference_u8_with_soft_mask on it is inference_u8; the mask-only forward runs no netG launch; in edit
sessions of both flows, chains of propose / accept are chains of edits byte for byte, revised accepts are edits on the
corrected masks, predict_mask is process_image's mask, and proposals give their device memory back."""
import gc

import numpy as np
import pytest
import torch
from PIL import Image

from sketchedit_b200 import synth
from tests.test_gpu_c8_edges import C8Log
from tests.test_gpu_configs import _model
from tests.test_gpu_edit_session import _photo, _sketch
from tests.util_parity import engine

pytestmark = pytest.mark.gpu
PRECS = ("bf16", "fp32", "fp32_direct")


def _u8_inputs(B, H, W, seed):
    rs = np.random.RandomState(seed)
    img_u8 = torch.from_numpy(rs.randint(0, 256, (B, H, W, 3), dtype=np.uint8))
    _, sk = synth.synth_inputs(B, H, W, seed=seed)
    return img_u8.cuda(), (sk[:, 0] * 255).to(torch.uint8).cuda()


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("shape", [(3, 256, 256), (2, 512, 512), (3, 136, 200)])
def test_predicted_mask_is_the_forwards_and_reproduces_it(prec, shape):
    B, H, W = shape
    eng = engine()
    img, sk = _u8_inputs(B, H, W, seed=H + W)
    bgr, mk = eng.inference_u8(img, sk, precision=prec)
    soft, mk2 = eng.predict_mask_u8(img, sk, precision=prec)
    assert soft.shape == (B, 1, H, W) and soft.dtype == torch.float32
    assert torch.equal(mk2, mk)
    assert torch.equal(eng.inference_u8_with_soft_mask(img, sk, soft, precision=prec), bgr)
    # batch invariance: every split of the batch, and a batch mixing these images with others
    for a, b in ((0, 1), (1, B), (0, B - 1)):
        s1, m1 = eng.predict_mask_u8(img[a:b], sk[a:b], precision=prec)
        assert torch.equal(s1, soft[a:b]) and torch.equal(m1, mk[a:b]), (a, b)
        assert torch.equal(eng.inference_u8_with_soft_mask(img[a:b], sk[a:b], soft[a:b].contiguous(), precision=prec), bgr[a:b])
    oi, os_ = _u8_inputs(2, H, W, seed=H + W + 1)
    s2, _ = eng.predict_mask_u8(torch.cat([oi[:1], img, oi[1:]]), torch.cat([os_[:1], sk, os_[1:]]), precision=prec)
    assert torch.equal(s2[1:-1], soft)
    b2 = eng.inference_u8_with_soft_mask(torch.cat([img, oi]), torch.cat([sk, os_]), torch.cat([soft, s2[:1], s2[-1:]]), precision=prec)
    assert torch.equal(b2[:B], bgr)


@pytest.mark.parametrize("prec", PRECS)
def test_mask_only_forward_runs_no_netG_launch(prec):
    """Launches: predict + soft-mask forward = plain forward + the second input codec + the binarise of the edit mask; the
    conv_c8 record of the mask-only forward names netM layers only. Repeated calls are captured, then replayed, alike."""
    eng = engine()
    img, sk = _u8_inputs(2, 64, 64, seed=5)
    soft = torch.empty(2, 1, 64, 64, device="cuda")
    mk = torch.empty(2, 64, 64, device="cuda", dtype=torch.uint8)
    got, counts = [], []
    for _ in range(3):
        soft.fill_(-1.0)
        mk.fill_(7)
        eng.predict_mask_u8(img, sk, precision=prec, out=(soft, mk))
        counts.append(eng.launches())
        got.append((soft.clone(), mk.clone()))
    assert len(set(counts)) == 1 and all(torch.equal(a, got[0][0]) and torch.equal(b, got[0][1]) for a, b in got), counts
    bgr = eng.inference_u8_with_soft_mask(img, sk, soft, precision=prec)
    n_soft = eng.launches()
    bgr0, mk0 = eng.inference_u8(img, sk, precision=prec)
    n_plain = eng.launches()
    assert torch.equal(bgr, bgr0) and torch.equal(mk, mk0)
    assert counts[0] + n_soft == n_plain + 2, (counts[0], n_soft, n_plain)
    assert counts[0] < n_soft
    if prec != "fp32_direct":
        with C8Log() as log:
            eng.predict_mask_u8(img, sk, precision=prec)
        labels = {n for n, _ in log.recs}
        assert labels and all(n.startswith("M.") for n in labels), sorted(labels)
        assert not any("conv17" == n[2:] for n in labels)          # netM's image decoder does not run either


def test_either_output_may_be_omitted():
    import ctypes

    from sketchedit_b200 import _lib
    eng = engine()
    img, sk = _u8_inputs(1, 64, 64, seed=6)
    soft, mk = eng.predict_mask_u8(img, sk)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    s1, m1 = torch.empty_like(soft), torch.empty_like(mk)
    _lib.check(eng.lib.se_predict_mask_u8(eng.h, p(img), p(sk), 1, 64, 64, 0, p(s1), None, st))
    _lib.check(eng.lib.se_predict_mask_u8(eng.h, p(img), p(sk), 1, 64, 64, 0, None, p(m1), st))
    assert torch.equal(s1, soft) and torch.equal(m1, mk)
    assert eng.lib.se_predict_mask_u8(eng.h, p(img), p(sk), 1, 64, 64, 0, None, None, st) != 0
    assert b"mask or mask_u8" in eng.lib.se_last_error()


# ------------------------------------------------------------------------------------------ sessions
def _steps(w, h, rs, whole):
    """(mask, region, offset, feather, revised) steps: 'auto', 'strokes' with overlapping boxes, a list, None (``whole``),
    feather 0 and 32, a mask at an offset, and a revised accept."""
    sx, sy = w / 1000, h / 667
    r = lambda x0, y0, x1, y1: (int(x0 * sx), int(y0 * sy), int(x1 * sx), int(y1 * sy))
    three = [r(100, 100, 140, 160), r(330, 120, 370, 170), r(800, 500, 860, 560)]
    steps = [
        (_sketch(w, h, [r(300, 200, 330, 260)]), "auto", (0, 0), 0, False),
        (_sketch(w, h, three), "strokes", (0, 0), 32, False),
        (_sketch(w, h, three[:2]), [r(0, 0, 400, 300), r(100, 50, 500, 350)], (0, 0), 0, False),
        (_sketch(97, 61, [(10, 10, 40, 50), (60, 5, 90, 30)]), "auto", (int(500 * sx) + 3, int(300 * sy) + 5), 32, False),
        (_sketch(w, h, [three[0], three[2]]), "strokes", (0, 0), 32, True),      # two boxes apart: one M holds both
    ]
    if whole:
        steps += [(_sketch(w, h, three), None, (0, 0), 32, False), (_sketch(w, h, three[1:]), None, (0, 0), 0, True)]
    return steps


def _revision(p, rs):
    """Per box a correction of the proposal's mask: part of it cleared, part set to soft values."""
    out = []
    for m in p.masks:
        a = np.array(m)
        a[: a.shape[0] // 3] = 0
        a[-a.shape[0] // 4:, : a.shape[1] // 2] = rs.randint(0, 256, a[-a.shape[0] // 4:, : a.shape[1] // 2].shape)
        out.append(Image.fromarray(a))
    return out


@pytest.mark.parametrize("resize", ["device", "host"])
@pytest.mark.parametrize("prec", PRECS)
def test_propose_accept_chains_are_edit_chains(prec, resize):
    from sketchedit_b200.serving import DemoProcessor, _placed
    model = _model(prec)
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=2.0, resize=resize, region_size=(256, 256))
    rs = np.random.RandomState(17)
    try:
        for w, h in ((1000, 667), (4000, 2667)):
            img = _photo(w, h, rs)
            a, b = proc.open_session(img), proc.open_session(img)
            steps = _steps(w, h, rs, whole=(w == 1000 or prec == "bf16"))
            for k, (mask, region, off, feather, revised) in enumerate(steps):
                where = (w, h, k, region)
                p = a.propose(mask, region=region, offset=off, feather=feather)
                if region == "strokes" and not revised and w == 1000:
                    assert any(p.boxes[i][2] > p.boxes[j][0] and p.boxes[j][2] > p.boxes[i][0] and p.boxes[i][3] > p.boxes[j][1]
                               and p.boxes[j][3] > p.boxes[i][1] for i in range(len(p.boxes)) for j in range(i)), p.boxes
                if off == (0, 0):                            # the stateless preview of the same photo
                    assert np.array_equal(np.array(proc.predict_mask(a.image(), mask, region=region, feather=feather)),
                                          np.array(proc.process_image(a.image(), mask, region=region, return_mask=True,
                                                                      feather=feather)[1])), where
                if revised:
                    em = _revision(p, rs)
                    full = Image.new("L", mask.size if region is None else img.size, 0)
                    for box, m in zip(p.boxes, em):          # M with M.crop(box) == the box's correction (no overlaps here)
                        full.paste(m, box[:2])
                    assert all(np.array_equal(np.array(full.crop(box)), np.array(m)) for box, m in zip(p.boxes, em)), where
                    got = a.accept(p, edit_masks=em)
                    want = b.edit(_placed(mask, img.size, off), edit_mask=full, region=None if region is None else p.boxes,
                                  feather=feather)
                else:
                    got = a.accept(p, return_mask=True)
                    want = b.edit(mask, region=region, offset=off, feather=feather, return_mask=True)
                    assert p.boxes == want.boxes and len(p.masks) == len(want.masks), where
                    for x, y in zip(p.masks, want.masks):
                        assert np.array_equal(np.array(x), np.array(y)), where
                assert got.boxes == want.boxes, where
                for x, y in zip(got.patches + got.masks, want.patches + want.masks):
                    assert (x is None and y is None) or np.array_equal(np.array(x), np.array(y)), where
                assert np.array_equal(np.array(a.image()), np.array(b.image())), where
            assert a.jpeg() == b.jpeg()
            for _ in range(3):
                ua, ub = a.undo(), b.undo()
                assert ua[0] == ub[0] and all(np.array_equal(np.array(x), np.array(y)) for x, y in zip(ua[1], ub[1]))
                assert np.array_equal(np.array(a.image()), np.array(b.image()))
            a.close()
            b.close()
    finally:
        proc.close()


@pytest.mark.parametrize("resize", ["device", "host"])
def test_proposals_give_their_device_memory_back(resize):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(_model("bf16"), resize=resize, region_size=(256, 256))
    rs = np.random.RandomState(23)
    img = _photo(1000, 667, rs)
    mask = _sketch(1000, 667, [(100, 100, 140, 160), (330, 120, 370, 170), (800, 500, 860, 560)])

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)                   # graphs, tables and staging buffers
        for region in ("strokes", None):
            warm.accept(warm.propose(mask, region=region))
            warm.edit(mask, region=region)
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        base = allocated()
        p = s.propose(mask, region="strokes")
        assert allocated() - base >= len(p.boxes) * 256 * 256 * 4
        p.close()
        assert allocated() == base
        p = s.propose(mask, region="strokes")
        s.edit(mask, region="strokes")                  # invalidates p
        assert not p.open
        s.undo()
        assert allocated() == base
        p = s.propose(mask, region=None)
        s.accept(p)
        s.undo()
        assert allocated() == base
        s.propose(mask, region="strokes")
        s.propose(mask, region="auto")
        s.close()
        assert allocated() == start
    finally:
        proc.close()

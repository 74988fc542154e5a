"""Region-edit detail on the GPU: the export forward is each of the three uint8 region forwards bit for bit and returns its
own attention weights and hole; the detail kernels match the float64 restatement (tests/util_detail.py) within the stated
fp32 bound; the composite adds the plane as stated; and the serving flows keep their byte-for-byte properties with detail."""
import threading
import time

import numpy as np
import pytest
import torch
from PIL import Image

from sketchedit_b200.engine import contextual_attention, detail_u8_packed, resize_composite_u8_packed, resize_u8_packed
from tests import util_detail as U
from tests.test_gpu_configs import _model
from tests.test_gpu_edit_session import _photo, _sketch
from tests.test_gpu_mask_preview import _u8_inputs
from tests.util_parity import engine
from tests.util_taps import decode_all

pytestmark = pytest.mark.gpu
PRECS = ("bf16", "fp32", "fp32_direct")


@pytest.mark.parametrize("prec", PRECS)
def test_export_forward_is_each_region_forward(prec):
    eng = engine()
    img, sk = _u8_inputs(3, 256, 192, seed=11)
    bgr, mk = eng.inference_u8(img, sk, precision=prec)
    b2, m2, attn, hole = eng.inference_u8_export(img, sk, precision=prec)
    L = (256 // 8 - 1) * (192 // 8 - 1)
    assert torch.equal(b2, bgr) and torch.equal(m2, mk) and attn.shape == (3, L, L)
    soft, _ = eng.predict_mask_u8(img, sk, precision=prec)
    assert torch.equal(hole, (soft[:, 0] > 0.5).to(torch.uint8))
    # the weights are a softmax over the keys of every query
    assert torch.allclose(attn.sum(1), torch.ones(3, L, device="cuda"), atol=1e-2)
    em = (torch.arange(256 * 192, device="cuda").view(1, 256, 192) % 251).to(torch.uint8).expand(3, -1, -1).contiguous()
    b3, m3, _, h3 = eng.inference_u8_export(img, sk, edit_mask_u8=em, precision=prec)
    assert m3 is None and torch.equal(b3, eng.inference_with_mask_u8(img, sk, em, precision=prec))
    assert torch.equal(h3, (em >= 128).to(torch.uint8))
    b4, _, _, h4 = eng.inference_u8_export(img, sk, edit_mask=soft, precision=prec)
    assert torch.equal(b4, eng.inference_u8_with_soft_mask(img, sk, soft, precision=prec)) and torch.equal(h4, hole)
    # repeated calls (captured, then replayed) give the same bytes
    for _ in range(2):
        again = eng.inference_u8_export(img, sk, precision=prec)
        assert torch.equal(again[0], bgr) and torch.equal(again[2], attn) and torch.equal(again[3], hole)


@pytest.mark.parametrize("prec", PRECS)
def test_exported_attn_is_the_attention_on_its_own_input(prec):
    eng = engine()
    img, sk = _u8_inputs(2, 128, 96, seed=4)
    eng.set_taps(True)
    try:
        _, _, attn, _ = eng.inference_u8_export(img, sk, precision=prec)
        taps = decode_all(eng.taps())
    finally:
        eng.set_taps(False)
    feat = taps["in:G.cam.f32" if prec == "fp32" else "in:G.cam"][0].cuda().contiguous()
    mask_s = taps["in:G.cam.mask_s"][0].cuda().contiguous()
    _, ref = contextual_attention(feat, mask_s, precision=prec, want_attn=True)
    if prec == "fp32":   # the operator's attention map comes from the fp32 CUDA-core path; the forward's from split-half GEMMs
        assert torch.all((attn - ref).abs() <= _softmax_bound(feat, ref, "fp32") + _softmax_bound(feat, ref, "fp32_direct"))
    else:
        assert torch.equal(attn, ref)


def _softmax_bound(feat, P, prec):
    """Bound of P[b, k, q] against the exact softmax from the logit error model of tests/util_bounds.attention_err: logits off
    by at most E[q, k] = logit_rel * sum |10 q| |k| + logit_abs (m_l <= 1) move p_k by a factor within exp(+-(E_k + max_l E_l)),
    and the exponentials, the row sum and the normalisation add the model's 4 + L / 32 + 5 fp32 roundings."""
    from tests import util_bounds as UB
    B, C, h, w = feat.shape
    err = UB.attention_err(prec, C, h, w)
    f = feat.double()
    rn = 1.0 / f.pow(2).sum((2, 3)).sqrt().clamp_min(1e-30)                       # per (image, channel) plane
    q = f.unfold(2, 4, 2).unfold(3, 4, 2)                                          # [B, C, hs, ws, 4, 4]
    q = q.permute(0, 2, 3, 1, 4, 5).reshape(B, -1, C * 16)                         # [B, L, 16 C]
    k = (f * rn[:, :, None, None]).unfold(2, 4, 2).unfold(3, 4, 2).permute(0, 2, 3, 1, 4, 5).reshape(B, -1, C * 16)
    E = err["logit_rel"] * (10 * q.abs()) @ k.abs().transpose(1, 2) + err["logit_abs"]   # [B, q, k]
    E = E + E.amax(2, keepdim=True)
    L = P.shape[1]
    return (P.double() * (torch.expm1(E.transpose(1, 2)) + (4 + L / 32 + 5) * UB.U32 * 2) + 1e-30).float()


# (photo w, h, box (left, upper, right, lower)): scale 1, 19/8, a non-integer downscale, odd sizes, boxes on photo borders
BOXES = [(700, 650, (100, 120, 356, 376)), (700, 650, (40, 20, 648, 628)), (700, 650, (0, 450, 200, 650)),
         (700, 650, (399, 0, 700, 257)), (301, 257, (0, 0, 301, 257))]


@pytest.mark.parametrize("prec", PRECS)
def test_detail_kernels_against_float64(prec, capsys):
    eng = engine()
    Hn, Wn = 256, 256
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    near_total = 0
    for k, (w, h, box) in enumerate(BOXES):
        rs = np.random.RandomState(k)
        photo = np.asarray(_photo(w, h, rs))
        crop = np.ascontiguousarray(photo[box[1]:box[3], box[0]:box[2]])
        bh, bw = crop.shape[:2]
        ph = torch.from_numpy(photo).cuda()
        img = torch.from_numpy(np.asarray(Image.fromarray(crop).resize((Wn, Hn)))).cuda()[None].contiguous()
        sk = torch.zeros(1, Hn, Wn, dtype=torch.uint8, device="cuda")
        sk[0, 100:150, 90:180:3] = 255
        em = torch.zeros(1, Hn, Wn, dtype=torch.uint8, device="cuda")
        em[0, 70 + 5 * k:180, 60:200 - 7 * k] = 255
        _, _, attn, hole = eng.inference_u8_export(img, sk, edit_mask_u8=em, precision=prec)
        low, low_at = resize_u8_packed(img, [0], [(Hn, Wn)], [(bh, bw)], 3)
        D, d_at, agg = detail_u8_packed(ph, [(box[1] * w + box[0]) * 3], [w * 3], [(bh, bw)], (Hn, Wn), low, low_at, hole, [0], attn,
                                        [0], want_agg=True)
        low_np = U.low_of(crop, Hn, Wn)
        assert np.array_equal(low[low_at[0]:low_at[0] + bh * bw * 3].cpu().numpy().reshape(bh, bw, 3), low_np)
        A64, D64, inh = U.aggregate(crop, low_np, hole[0].cpu().numpy(), attn[0].cpu().numpy())
        A = agg[d_at[0] // 2:d_at[0] // 2 + bh * bw * 3].cpu().numpy().reshape(bh, bw, 3).astype(np.float64)
        Dg = D[d_at[0] // 2:d_at[0] // 2 + bh * bw * 3].cpu().numpy().reshape(bh, bw, 3).astype(np.int64)
        b = U.bound(L)
        assert inh.any() and (~inh).any()
        assert np.abs(A - A64).max() <= b, (box, np.abs(A - A64).max(), b)
        near = np.abs(np.abs(A64 - np.floor(A64)) - 0.5) <= b       # within the bound of a rounding boundary
        assert np.array_equal(Dg[~near], D64[~near]), box
        assert np.abs(Dg - D64).max() <= 1
        assert (Dg[~inh] == 0).all()
        assert (np.abs(D64).max() > 0) == ((bh, bw) != (Hn, Wn))   # a box of the working size has no residual
        near_total += int(near[inh].sum())
    with capsys.disabled():
        print("\n[detail %s] bytes within the bound of a rounding boundary: %d" % (prec, near_total))


def test_composite_adds_the_plane_then_pastes():
    """resize_composite_u8_packed(detail=...) = Pillow's paste of clamp(resize(res) + D, 0, 255) with the resized mask, boxes
    overlapping and composited in order, a box without a plane among them."""
    rs = np.random.RandomState(3)
    canvas = rs.randint(0, 256, (300, 320, 3), dtype=np.uint8)
    boxes = [((10, 20), (200, 180)), ((90, 100), (150, 160)), ((0, 0), (64, 64))]
    res = [rs.randint(0, 256, (64, 48, 3), dtype=np.uint8) for _ in boxes]
    msk = [rs.randint(0, 256, (64, 48), dtype=np.uint8) for _ in boxes]
    planes = [rs.randint(-300, 300, hw + (3,)).astype(np.int16) for _, hw in boxes]
    planes[2] = None
    ref = Image.fromarray(canvas)
    for (yx, hw), r, m, d in zip(boxes, res, msk, planes):
        up = np.asarray(Image.fromarray(r[..., ::-1].copy()).resize(hw[::-1])).astype(np.int64)
        if d is not None:
            up = np.clip(up + d, 0, 255)
        ref.paste(Image.fromarray(up.astype(np.uint8)), yx[::-1], Image.fromarray(m).resize(hw[::-1]))
    cv = torch.from_numpy(canvas.copy()).cuda().view(-1)
    rgb = torch.from_numpy(np.concatenate([r.reshape(-1) for r in res])).cuda()
    mk = torch.from_numpy(np.concatenate([m.reshape(-1) for m in msk])).cuda()
    dp = [p for p in planes if p is not None]
    dt = torch.from_numpy(np.concatenate([p.reshape(-1) for p in dp])).cuda()
    d_off = [0, dp[0].nbytes, -1]
    n = len(boxes)
    resize_composite_u8_packed(rgb, [i * 64 * 48 * 3 for i in range(n)], mk, [i * 64 * 48 for i in range(n)], [(64, 48)] * n, cv,
                               [0] * n, [320 * 3] * n, [b[0] for b in boxes], [b[1] for b in boxes], swap_rb=True, detail=dt,
                               detail_offsets=d_off)
    assert np.array_equal(cv.cpu().numpy().reshape(300, 320, 3), np.asarray(ref))


@pytest.fixture(scope="module")
def proc():
    from sketchedit_b200.serving import DemoProcessor
    p = DemoProcessor(_model("bf16"), max_batch=8, max_wait_ms=60.0, region_size=(256, 256))
    yield p
    p.close()


def test_box_of_the_working_size_adds_nothing(proc):
    rs = np.random.RandomState(7)
    img = _photo(600, 500, rs)
    sk = _sketch(600, 500, [(150, 150, 260, 260)])
    box = [(100, 100, 356, 356)]
    a = proc.process_image(img, sk, region=box)
    b = proc.process_image(img, sk, region=box, detail=True)
    assert np.array_equal(np.asarray(a), np.asarray(b))
    big = _sketch(600, 500, [(100, 100, 420, 400)])                 # an upscaled 600 x 500 box: detail changes bytes
    c = proc.process_image(img, big, region="auto", detail=True)
    assert not np.array_equal(np.asarray(c), np.asarray(proc.process_image(img, big, region="auto")))


def test_accept_is_edit_and_undo_restores(proc):
    rs = np.random.RandomState(9)
    img = _photo(1000, 667, rs)
    sk = _sketch(1000, 667, [(300, 200, 520, 420), (700, 450, 820, 600)])
    s1, s2 = proc.open_session(img), proc.open_session(img)
    try:
        r1 = s1.edit(sk, region="strokes", detail=True)
        p = s2.propose(sk, region="strokes")
        r2 = s2.accept(p, detail=True)
        assert r1.boxes == r2.boxes
        assert np.array_equal(np.asarray(s1.image()), np.asarray(s2.image()))
        plain = proc.process_image(img, sk, region="strokes")
        assert not np.array_equal(np.asarray(s1.image()), np.asarray(plain))
        assert np.array_equal(np.asarray(s1.image()), np.asarray(proc.process_image(img, sk, region="strokes", detail=True)))
        s1.undo()
        assert np.array_equal(np.asarray(s1.image()), np.asarray(img.convert("RGB")))
        assert s1.png() == s1.png() and len(s2.jpeg()) > 0
    finally:
        s1.close()
        s2.close()


def test_detail_bytes_do_not_depend_on_the_batch(proc):
    rs = np.random.RandomState(12)
    img = _photo(900, 700, rs)
    sk = _sketch(900, 700, [(200, 200, 420, 380)])
    alone = np.asarray(proc.process_image(img, sk, region="auto", detail=True))
    others = [(_photo(640, 480, np.random.RandomState(20 + i)), _sketch(640, 480, [(100 + 20 * i, 90, 260, 250)])) for i in range(3)]
    out, plain = {}, {}
    for i, (o, m) in enumerate(others):
        plain[i] = np.asarray(proc.process_image(o, m, region="auto"))

    def run(i, o, m, d):
        out[i] = np.asarray(proc.process_image(o, m, region="auto", detail=d))
    # submitted in this order within the batching window: the detail request is item 1 of one batch of 4
    ts = [threading.Thread(target=run, args=(0, *others[0], False)), threading.Thread(target=run, args=("me", img, sk, True))]
    ts += [threading.Thread(target=run, args=(i, o, m, False)) for i, (o, m) in enumerate(others) if i]
    n0 = len(proc.batcher.batches)
    for t in ts:
        t.start()
        time.sleep(0.004)
    for t in ts:
        t.join()
    assert np.array_equal(out["me"], alone)
    for i in plain:
        assert np.array_equal(out[i], plain[i]), i
    assert [n for _, n in proc.batcher.batches[n0:]] == [4]

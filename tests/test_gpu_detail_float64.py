"""Region-edit detail against float64 in the forms serving uses: se_detail_u8 with several boxes of different sizes per call
(the scratch reused at another size), photo windows with a pitch wider than the box and per-box photo tensors, offsets into a
batch's low, hole and attention buffers, at non-square, square, tiny and 512^2 working sizes, on the export forward's
weights in each precision and on synthetic ones; the paste with detail planes and feather together against Pillow; and the
serving flows with detail against the Pillow flow whose pastes add float64's plane.

Every box is held to tests/util_detail.violations: |A - A64| <= bound(L), D = D64 wherever A64 is farther than the bound from
a rounding boundary, |D - D64| <= 1, D = 0 outside the hole. Each check prints max |A - A64| / bound per working size and
the count of bytes within the bound of a rounding boundary."""
import threading
import time

import numpy as np
import pytest
import torch
from PIL import Image

from sketchedit_b200.engine import detail_u8_packed, resize_composite_u8_packed
from sketchedit_b200.serving import detail_box_ok, feather_mask, feather_widths
from tests import util_detail as U
from tests.test_gpu_configs import _model
from tests.test_gpu_edit_session import _photo, _sketch
from tests.util_parity import engine

pytestmark = pytest.mark.gpu
PRECS = ("bf16", "fp32", "fp32_direct")
PW, PH = 2600, 2200                           # the photo the boxes are cut from
HOLES = ("rect", "edges", "line", "empty", "whole")


def _min_side(n):
    """The smallest box side detail_box_ok accepts at working side n (its footprint is 3: every one clamps at the box's
    last column)."""
    return next(b for b in range(1, n + 1) if detail_box_ok((b, n), (n, n)))


# boxes of the same sizes at both orientations of a non-square working size, so a swapped Hn / Wn cannot hide
SHARED = [(101, 203, 801, 636), (1200, 900, 1210, 1010), (40, 1500, 1040, 1510)]


def _boxes(Hn, Wn):
    """PIL boxes (left, upper, right, lower) in the photo, large -> small -> large: an upscale of 8x where the photo holds
    it (else the whole photo), the smallest box flush with the photo's right and bottom edges, the working width with another
    height, a box flush with the right edge, one flush with the bottom, the least width and the least height."""
    mw, mh = _min_side(Wn), _min_side(Hn)
    uw, uh = min(8 * Wn, PW), min(8 * Hn, PH)
    boxes = [(0, 0, uw, uh), (PW - mw, PH - mh, PW, PH), (5, 7, 5 + Wn, 7 + Hn + 37), (PW - 301, 3, PW, 214),
             (11, PH - 190, 12 + 3 * Wn // 2, PH), (17, 19, 17 + mw, 22 + 2 * Hn), (23, 29, 28 + 2 * Wn, 29 + mh)]
    if sorted((Hn, Wn)) == [192, 320]:
        boxes += SHARED
    for b in boxes:
        assert detail_box_ok((b[2] - b[0], b[3] - b[1]), (Hn, Wn)), b
    return boxes


def _hole(kind, Hn, Wn):
    """An edit mask (uint8, hole where >= 128) of a kind: an interior rectangle, four bars each touching one edge of the
    working frame, a one-pixel line, no hole, the whole frame."""
    m = np.zeros((Hn, Wn), np.uint8)
    if kind == "rect":
        m[Hn // 4:3 * Hn // 4 + 1, Wn // 3:Wn - 5] = 255
    elif kind == "edges":
        m[:3, Wn // 4:Wn // 2] = 200
        m[Hn - 5:, Wn // 2:Wn - 1] = 255
        m[Hn // 3:Hn // 2 + 1, :4] = 128
        m[1:Hn // 3, Wn - 2:] = 255
    elif kind == "line":
        m[Hn // 2, 3:Wn - 3] = 255
    elif kind == "whole":
        m[:] = 255
    return m


def _setup(Hn, Wn):
    """Photo, boxes, crops, lows, and the edit masks of a batch of 6: image 0 a decoy, images 1-5 the HOLES."""
    photo = np.array(_photo(PW, PH, np.random.RandomState(Hn * 7 + Wn)))
    boxes = _boxes(Hn, Wn)
    crops = [np.ascontiguousarray(photo[b[1]:b[3], b[0]:b[2]]) for b in boxes]
    lows = [U.low_of(c, Hn, Wn) for c in crops]
    em = np.stack([_hole("rect", Hn, Wn)] + [_hole(k, Hn, Wn) for k in HOLES])
    return photo, boxes, crops, lows, em


def _run(photo, boxes, crops, lows, hole, attn, order, Hn, Wn, windows=True):
    """se_detail_u8 on the boxes in `order` (box i takes image 1 + i % 5 of the batch: nonzero offsets), photo windows of one
    tensor or one tensor per box; lows packed behind a 48-byte lead. Returns {box: (A, D)}."""
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    lead = np.zeros(48, np.uint8)
    low_buf = np.concatenate([lead] + [lows[i].reshape(-1) for i in order])
    low_at = list(np.cumsum([48] + [lows[i].size for i in order])[:-1])
    sizes = [crops[i].shape[:2] for i in order]
    if windows:
        src = torch.from_numpy(photo).cuda()
        offs = [(boxes[i][1] * PW + boxes[i][0]) * 3 for i in order]
        pitches = [PW * 3] * len(order)
    else:
        src = [torch.from_numpy(crops[i]).cuda() for i in order]
        offs, pitches = [0] * len(order), [crops[i].shape[1] * 3 for i in order]
    img_of = [1 + i % 5 for i in order]
    D, d_at, agg = detail_u8_packed(src, offs, pitches, sizes, (Hn, Wn), torch.from_numpy(low_buf).cuda(), low_at, hole,
                                    [j * Hn * Wn for j in img_of], attn, [j * L * L for j in img_of], want_agg=True)
    D, agg = D.cpu().numpy(), agg.cpu().numpy()
    out = {}
    for i, o, (bh, bw) in zip(order, d_at, sizes):
        n = bh * bw * 3
        out[i] = (agg[o // 2:o // 2 + n].reshape(bh, bw, 3).astype(np.float64), D[o // 2:o // 2 + n].reshape(bh, bw, 3).astype(np.int64))
    return out


def _check_all(tag, photo, boxes, crops, lows, hole, attn, Hn, Wn, exact=False):
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    n = len(boxes)
    got = _run(photo, boxes, crops, lows, hole, attn, list(range(n)), Hn, Wn)
    listed = _run(photo, boxes, crops, lows, hole, attn, list(range(n)), Hn, Wn, windows=False)
    back = _run(photo, boxes, crops, lows, hole, attn, list(range(n))[::-1], Hn, Wn)
    worst, near_total = 0.0, 0
    for i in range(n):
        A, D = got[i]
        for other in (listed[i], back[i]):           # the same planes whatever the order or the photo's form
            assert np.array_equal(other[0], A) and np.array_equal(other[1], D), (tag, boxes[i])
        j = 1 + i % 5
        A64, D64, inh = U.aggregate_vec(crops[i], lows[i], hole[j].cpu().numpy(), attn[j], device="cuda")
        v = U.violations(A, D, A64, D64, inh, L, exact=exact)
        assert not v, (tag, boxes[i], HOLES[j - 1], v, np.abs(A - A64).max())
        worst = max(worst, float(np.abs(A - A64).max(initial=0.0)) / U.bound(L))
        near_total += int(U.near_boundary(A64, L)[inh].sum())
    return worst, near_total


def _report(capsys, tag, L, worst, near):
    with capsys.disabled():
        print("\n[detail %s L=%d] max |A - A64| / bound %.3g, bytes within the bound of a rounding boundary: %d" % (tag, L, worst, near))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("Hn,Wn", [(192, 320), (320, 192), (272, 200), (512, 512), (64, 48), (16, 16)])
def test_detail_of_the_export_forward_against_float64(Hn, Wn, prec, capsys):
    eng = engine()
    photo, boxes, crops, lows, em = _setup(Hn, Wn)
    img = torch.from_numpy(np.stack([np.asarray(Image.fromarray(crops[(j - 1) % len(crops)]).resize((Wn, Hn))) for j in range(6)]))
    sk = torch.zeros(6, Hn, Wn, dtype=torch.uint8)
    sk[:, Hn // 3:Hn // 2, Wn // 4:Wn // 2:3] = 255
    _, _, attn, hole = eng.inference_u8_export(img.cuda(), sk.cuda(), edit_mask_u8=torch.from_numpy(em).cuda(), precision=prec)
    assert np.array_equal(hole.cpu().numpy(), (em >= 128).astype(np.uint8))
    worst, near = _check_all(prec, photo, boxes, crops, lows, hole, attn, Hn, Wn)
    _report(capsys, "%s %dx%d" % (prec, Hn, Wn), attn.shape[1], worst, near)


def _weights(kind, hole, rs):
    """Synthetic P [L keys, L queries] fp32 of one image: one-hot per query (on a valid key), uniform over the valid keys, or
    random with three dominant keys per query. A key is valid when more than 1/10 of its 16 x 16 patch is outside the hole
    (all keys when none is)."""
    Hn, Wn = hole.shape
    hs, ws = Hn // 8 - 1, Wn // 8 - 1
    L = hs * ws
    cover = np.array([hole[8 * (k // ws):8 * (k // ws) + 16, 8 * (k % ws):8 * (k % ws) + 16].mean() for k in range(L)])
    valid = np.nonzero(1 - cover > 0.1)[0]
    if valid.size == 0:
        valid = np.arange(L)
    P = np.zeros((L, L))
    if kind == "onehot":
        P[rs.choice(valid, L), np.arange(L)] = 1.0
    elif kind == "uniform":
        P[valid] = 1.0 / valid.size
    else:
        S = rs.randn(L, L)
        for q in range(L):
            S[rs.choice(L, min(3, L), replace=False), q] += 6.0
        P = np.exp(S - S.max(0))
        P /= P.sum(0)
    return torch.from_numpy(P.astype(np.float32))


@pytest.mark.parametrize("kind", ["onehot", "uniform", "dominant"])
def test_detail_of_synthetic_weights_against_float64(kind, capsys):
    """One-hot weights are exact in the fp16 hi half and R is exact, so the device's A and D equal float64's bit for bit with
    no boundary exemption."""
    Hn, Wn = 192, 320
    photo, boxes, crops, lows, em = _setup(Hn, Wn)
    hole = (em >= 128).astype(np.uint8)
    rs = np.random.RandomState(len(kind))
    attn = torch.stack([_weights(kind, h, rs) for h in hole]).cuda()
    worst, near = _check_all(kind, photo, boxes, crops, lows, torch.from_numpy(hole).cuda(), attn, Hn, Wn, exact=kind == "onehot")
    _report(capsys, "%s %dx%d" % (kind, Hn, Wn), attn.shape[1], worst, near)


def test_detail_of_a_whole_large_photo_against_float64(capsys):
    """A 4000 x 2667 photo as one box at 256^2: footprint 252 x 169, Np = 128,000 GEMM columns. Its scratch is about 1 GB:
    the residual operand (hi and lo halves, 4 Mp Np bytes) and the GEMM output (4 Mp Np) take 0.52 GB each at Mp = 1024,
    the P operand 4 MB."""
    Hn = Wn = 256
    eng = engine()
    photo = np.array(_photo(4000, 2667, np.random.RandomState(40)))
    assert (U.footprint(4000, Wn), U.footprint(2667, Hn)) == (252, 169)
    img = torch.from_numpy(np.array(Image.fromarray(photo).resize((Wn, Hn))))[None].cuda()
    sk = torch.zeros(1, Hn, Wn, dtype=torch.uint8, device="cuda")
    sk[0, 90:150, 80:200:3] = 255
    em = torch.zeros(1, Hn, Wn, dtype=torch.uint8, device="cuda")
    em[0, 60:200, 50:210] = 255
    _, _, attn, hole = eng.inference_u8_export(img, sk, edit_mask_u8=em, precision="bf16")
    low = U.low_of(photo, Hn, Wn)
    D, d_at, agg = detail_u8_packed(torch.from_numpy(photo).cuda(), [0], [4000 * 3], [(2667, 4000)], (Hn, Wn),
                                    torch.from_numpy(low.reshape(-1).copy()).cuda(), [0], hole, [0], attn, [0], want_agg=True)
    n = 2667 * 4000 * 3
    A = agg[d_at[0] // 2:d_at[0] // 2 + n].view(2667, 4000, 3).cpu().numpy().astype(np.float64)
    Dg = D[d_at[0] // 2:d_at[0] // 2 + n].view(2667, 4000, 3).cpu().numpy().astype(np.int64)
    del D, agg
    L = attn.shape[1]
    A64, D64, inh = U.aggregate_vec(photo, low, hole[0].cpu().numpy(), attn[0], device="cuda")
    v = U.violations(A, Dg, A64, D64, inh, L)
    assert inh.any() and not v, v
    _report(capsys, "bf16 256x256, 4000x2667 box", L, float(np.abs(A - A64).max()) / U.bound(L), int(U.near_boundary(A64, L)[inh].sum()))


# --------------------------------------------------------------------------------------------- paste: detail and feather
@pytest.mark.parametrize("swap_rb", [False, True])
def test_paste_with_detail_and_feather_is_pillows(swap_rb):
    """40 boxes on two canvases (more than one 32-box launch, overlapping boxes composited in order): each box pasted as
    Pillow pastes clamp(resize(rgb) + D, 0, 255) through feather_mask(resize(mask), widths); boxes with widths and no plane,
    with a plane and zero widths, and with both, on each side of the launch split."""
    rs = np.random.RandomState(17 + swap_rb)
    shapes = [(180, 240), (150, 200)]
    canvases = [rs.randint(0, 256, s + (3,), dtype=np.uint8) for s in shapes]
    n = 40
    boxes, srcs, widths, planes = [], [], [], []
    for i in range(n):
        c = i % 2
        Hc, Wc = shapes[c]
        h, w = rs.randint(6, 80), rs.randint(6, 100)
        boxes.append((c, (rs.randint(0, Hc - h + 1), rs.randint(0, Wc - w + 1)), (h, w)))
        srcs.append((rs.randint(4, 48), rs.randint(4, 48)))
        widths.append((0, 0, 0, 0) if i % 4 == 0 else
                      (rs.randint(0, w // 2 + 1), rs.randint(0, h // 2 + 1), rs.randint(0, w // 2 + 1), rs.randint(0, h // 2 + 1)))
        planes.append(None if i % 5 == 3 else rs.randint(-300, 301, (h, w, 3)).astype(np.int16))
    assert any(p is None and any(f) for p, f in zip(planes, widths)) and any(p is not None and not any(f) for p, f in zip(planes, widths))
    rgb = [rs.randint(0, 256, s + (3,), dtype=np.uint8) for s in srcs]
    msk = [rs.randint(0, 256, s, dtype=np.uint8) for s in srcs]
    ref = [Image.fromarray(c.copy()) for c in canvases]
    for (c, (y, x), (h, w)), r, m, f, d in zip(boxes, rgb, msk, widths, planes):
        up = np.asarray(Image.fromarray(r[..., ::-1].copy() if swap_rb else r).resize((w, h))).astype(np.int64)
        if d is not None:
            up = np.clip(up + d, 0, 255)
        pm = feather_mask(np.asarray(Image.fromarray(m).resize((w, h))), f)
        ref[c].paste(Image.fromarray(up.astype(np.uint8)), (x, y), Image.fromarray(pm))
    cv = torch.from_numpy(np.concatenate([c.reshape(-1) for c in canvases])).cuda()
    c_off = [0, canvases[0].size]
    r_off = list(np.cumsum([0] + [a.size for a in rgb])[:-1])
    m_off = list(np.cumsum([0] + [a.size for a in msk])[:-1])
    dp = [p for p in planes if p is not None]
    d_bytes = list(np.cumsum([0] + [p.nbytes for p in dp])[:-1])
    d_off, k = [], 0
    for p in planes:
        d_off.append(-1 if p is None else int(d_bytes[k]))
        k += p is not None
    resize_composite_u8_packed(torch.from_numpy(np.concatenate([a.reshape(-1) for a in rgb])).cuda(), r_off,
                               torch.from_numpy(np.concatenate([a.reshape(-1) for a in msk])).cuda(), m_off, srcs, cv,
                               [c_off[b[0]] for b in boxes], [shapes[b[0]][1] * 3 for b in boxes], [b[1] for b in boxes],
                               [b[2] for b in boxes], swap_rb=swap_rb, feather=widths,
                               detail=torch.from_numpy(np.concatenate([p.reshape(-1) for p in dp])).cuda(), detail_offsets=d_off)
    got = cv.cpu().numpy()
    for c in range(2):
        assert np.array_equal(got[c_off[c]:c_off[c] + canvases[c].size].reshape(canvases[c].shape), np.asarray(ref[c])), c


# --------------------------------------------------------------------------------------------- serving flows
def statement(proc, photo, sketch, boxes, feather, detail):
    """The Pillow flow of a region edit (the steps of DemoProcessor._region_host) with each box pasted as clamp(resize(res)
    + D64): D64 from the float64 aggregate on the attention and hole the export forward returns for the same working-size
    inputs (batch-independent, so one batch of the boxes gives the bytes serving's batch gives). Returns (bytes, where a
    byte may be one off: A64 within the bound of a rounding boundary under some box)."""
    Hn, Wn = proc.region_size
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    crops = [np.asarray(photo.crop(b)) for b in boxes]
    img = torch.from_numpy(np.stack([np.asarray(Image.fromarray(c).resize((Wn, Hn))) for c in crops])).cuda()
    sk = torch.from_numpy(np.stack([np.asarray(sketch.crop(b).resize((Wn, Hn))) for b in boxes])).cuda()
    bgr, pm, attn, hole = proc.engine.inference_u8_export(img, sk, precision=proc.precision)
    bgr, pm, hole = bgr.cpu().numpy(), pm.cpu().numpy(), hole.cpu().numpy()
    out = photo.copy()
    near = np.zeros((photo.size[1], photo.size[0]), bool)
    for i, b in enumerate(boxes):
        size = (b[2] - b[0], b[3] - b[1])
        up = np.asarray(Image.fromarray(bgr[i][..., ::-1].copy()).resize(size)).astype(np.int64)
        if detail:
            A64, D64, _ = U.aggregate_vec(crops[i], U.low_of(crops[i], Hn, Wn), hole[i], attn[i], device="cuda")
            up = np.clip(up + D64, 0, 255)
            near[b[1]:b[3], b[0]:b[2]] |= U.near_boundary(A64, L).any(-1)
        m = feather_mask(np.asarray(Image.fromarray(pm[i]).resize(size)), feather_widths(b, photo.size, feather))
        out.paste(Image.fromarray(up.astype(np.uint8)), b[:2], Image.fromarray(m))
    return np.asarray(out), near


def _agrees(got, want_near):
    want, near = want_near
    diff = np.abs(np.asarray(got).astype(np.int64) - want.astype(np.int64))
    assert diff.max(initial=0) <= 1 and not diff.max(-1)[~near].any(), (diff.max(), int((diff.max(-1) > 0).sum()), int(near.sum()))


@pytest.fixture(scope="module", params=[(256, 256), (192, 320)], ids=["256x256", "192x320"])
def proc(request):
    from sketchedit_b200.serving import DemoProcessor
    p = DemoProcessor(_model("bf16"), max_batch=8, max_wait_ms=60.0, region_size=request.param)
    yield p
    p.close()


def test_process_image_with_detail_is_the_statement(proc):
    rs = np.random.RandomState(31)
    img = _photo(1100, 800, rs)
    sk = _sketch(1100, 800, [(200, 150, 330, 300), (280, 260, 420, 380), (800, 500, 900, 640)])
    boxes = [(100, 80, 500, 420), (250, 230, 700, 600), (760, 430, 1100, 800)]      # the first two overlap
    _agrees(proc.process_image(img, sk, region=boxes, detail=True, feather=16), statement(proc, img, sk, boxes, 16, True))
    groups = proc._region_boxes(img.size, sk, None, "strokes")
    _agrees(proc.process_image(img, sk, region="strokes", detail=True), statement(proc, img, sk, groups, 0, True))


def test_batch_of_detail_and_plain_requests_is_the_statement(proc):
    reqs = [(_photo(900, 700, np.random.RandomState(50 + i)), _sketch(900, 700, [(150 + 40 * i, 200, 330, 380)]), d)
            for i, d in enumerate((True, False, True))]
    out = {}

    def run(i, img, sk, d):
        out[i] = proc.process_image(img, sk, region="auto", detail=d, feather=8)
    ts = [threading.Thread(target=run, args=(i,) + r) for i, r in enumerate(reqs)]
    n0 = len(proc.batcher.batches)
    for t in ts:
        t.start()
        time.sleep(0.004)
    for t in ts:
        t.join()
    assert [n for _, n in proc.batcher.batches[n0:]] == [3]
    for i, (img, sk, d) in enumerate(reqs):
        boxes = proc._region_boxes(img.size, sk, None, "auto")
        _agrees(out[i], statement(proc, img, sk, boxes, 8, d))


def test_session_edits_with_detail_are_the_statement(proc):
    rs = np.random.RandomState(61)
    img = _photo(1000, 667, rs)
    s = proc.open_session(img)
    try:
        for sk, region, feather in ((_sketch(1000, 667, [(300, 200, 520, 420), (700, 450, 820, 600)]), "strokes", 0),
                                    (_sketch(1000, 667, [(350, 250, 600, 500)]), "auto", 12)):
            before = s.image()
            r = s.edit(sk, region=region, feather=feather, detail=True)
            _agrees(s.image(), statement(proc, before, sk, list(r.boxes), feather, True))
    finally:
        s.close()

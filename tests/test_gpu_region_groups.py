"""Several regions per request on the GPU: se_resize_composite_feather_detail_u8 (engine.resize_composite_u8_packed) reproduces sequential
Pillow pastes bit for bit and writes nothing outside its boxes, and the device flow of DemoProcessor.process_image with
region="strokes" or a list of boxes returns exactly the Pillow flow's bytes."""
import threading

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import region_groups


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


# canvases (h, w) and their boxes in paste order: (canvas, (y, x), box (h, w), result (h', w')). Every axis is upscaled,
# downscaled or unchanged; widths are odd and even; boxes nest, repeat, overlap and touch the canvas edges. The boxes of
# canvases 0 and 1 interleave in the order.
CANVASES = [(300, 401), (97, 130), (64, 64)]
BOXES = [
    (0, (0, 0), (300, 401), (256, 256)),        # the whole canvas, both axes upscaled
    (1, (5, 3), (60, 77), (64, 96)),
    (0, (40, 37), (101, 133), (256, 256)),      # nested in the first
    (0, (40, 37), (101, 133), (64, 96)),        # the same box again, another result
    (1, (30, 50), (67, 80), (67, 80)),          # unchanged size, reaches the canvas's right and bottom edges
    (0, (150, 300), (150, 101), (150, 60)),     # height unchanged, width upscaled, bottom-right corner
    (0, (10, 141), (256, 256), (256, 256)),     # unchanged size, odd offset
    (0, (1, 2), (31, 45), (40, 52)),
    (1, (0, 0), (97, 1), (33, 7)),              # one column
    (0, (299, 0), (1, 401), (5, 7)),            # one row along the bottom edge
    (2, (8, 8), (48, 48), (256, 256)),          # a canvas of its own, aligned box
]


def _pillow(canvas, boxes, results, swap):
    out = Image.fromarray(canvas)
    for ((y, x), (h, w)), (rgb, mask) in zip(boxes, results):
        res = Image.fromarray(np.ascontiguousarray(rgb[..., ::-1]) if swap else rgb).resize((w, h))
        out.paste(res, (x, y, x + w, y + h), Image.fromarray(mask).resize((w, h)))
    return np.asarray(out)


def _result(src, seed):
    rs = np.random.RandomState(seed)
    rgb = rs.randint(0, 256, src + (3,), dtype=np.uint8)
    rgb[: src[0] // 3] = 255                                   # hard edges: both signs of every tap and both clamps
    mask = rs.randint(0, 256, src, dtype=np.uint8)
    mask[:, : src[1] // 4] = 0                                 # 0, 255 and soft values after the resize
    mask[:, src[1] // 4: src[1] // 2] = 255
    return rgb, mask


def _pack(arrays, align, start):
    offs, pos = [], start
    for a in arrays:
        offs.append(pos)
        pos += a.nbytes + (16 if align else 5 + pos % 3)
        if align:
            pos = (pos + 15) // 16 * 16
    buf = np.zeros(pos + 41, np.uint8)
    for a, o in zip(arrays, offs):
        buf[o:o + a.nbytes] = a.reshape(-1)
    return buf, offs


def _run(canvases, boxes, swap, aligned, seed):
    """Packs the canvases with guard bytes between rows and around them, runs the composite, returns (got, want, guards ok)."""
    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    rs = np.random.RandomState(seed)
    imgs = [rs.randint(0, 256, hw + (3,), dtype=np.uint8) for hw in canvases]
    pitches = [(3 * w + 15) // 16 * 16 if aligned else 3 * w + 7 for _, w in canvases]
    offs, pos = [], 16 if aligned else 9
    for (h, _), p in zip(canvases, pitches):
        offs.append(pos)
        pos = (pos + h * p + 64 + 15) // 16 * 16 + (0 if aligned else 3)
    buf = np.full(pos + 33, 0xA5, np.uint8)
    for img, o, p in zip(imgs, offs, pitches):
        rows = buf[o:o + img.shape[0] * p].reshape(img.shape[0], p)
        rows[:, :img.shape[1] * 3] = img.reshape(img.shape[0], -1)
    results = [_result(src, seed + 1 + i) for i, (_, _, _, src) in enumerate(boxes)]
    rgb, ro = _pack([r for r, _ in results], aligned, 0 if aligned else 3)
    msk, mo = _pack([m for _, m in results], aligned, 0 if aligned else 1)
    dev = torch.from_numpy(buf).cuda()
    resize_composite_u8_packed(torch.from_numpy(rgb).cuda(), ro, torch.from_numpy(msk).cuda(), mo, [b[3] for b in boxes], dev,
                               [offs[b[0]] for b in boxes], [pitches[b[0]] for b in boxes], [b[1] for b in boxes],
                               [b[2] for b in boxes], swap_rb=swap)
    got = dev.cpu().numpy()
    inside = np.zeros(got.size, bool)
    for c, (img, o, p) in enumerate(zip(imgs, offs, pitches)):
        h, w = img.shape[:2]
        idx = [i for i, b in enumerate(boxes) if b[0] == c]
        want = _pillow(img, [boxes[i][1:3] for i in idx], [results[i] for i in idx], swap)
        rows = got[o:o + h * p].reshape(h, p)
        assert np.array_equal(rows[:, :w * 3].reshape(h, w, 3), want), \
            "canvas %d: %d bytes differ (Pillow %s)" % (c, int((rows[:, :w * 3].reshape(h, w, 3) != want).sum()), PIL.__version__)
        for r in range(h):
            inside[o + r * p:o + r * p + w * 3] = True
    assert (got[~inside] == 0xA5).all()                                       # guard bytes: row ends and around every canvas


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("swap", [False, True])
def test_composite_matches_sequential_pastes(lib, swap, aligned):
    _run(CANVASES, BOXES, swap, aligned, seed=40)


@pytest.mark.gpu
def test_composite_continues_the_order_past_one_launch(lib):
    """70 boxes in one canvas, more than one launch's descriptors, overlapping in chains, and a second canvas between."""
    rs = np.random.RandomState(3)
    boxes = []
    for i in range(70):
        h, w = int(rs.randint(8, 90)), int(rs.randint(8, 120))
        boxes.append((0 if i % 9 else 1, (int(rs.randint(0, 200 - h)), int(rs.randint(0, 240 - w))), (h, w),
                      (int(rs.choice([h, 32, 64])), int(rs.choice([w, 32, 48])))))
    _run([(200, 240), (200, 240)], boxes, True, True, seed=90)


# ------------------------------------------------------------------------------------------ DemoProcessor region flows
def _photo(w, h, rs):
    a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    a[:, : w // 3] = 255 - a[:, : w // 3] // 4
    return Image.fromarray(a)


def _sketch(w, h, rects):
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1:3] = 255
    return Image.fromarray(m)


def _soft(w, h, rects, rs):
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1] = rs.randint(0, 256, (y1 - y0, x1 - x0), dtype=np.uint8)
    return Image.fromarray(m)


def _requests():
    """(photo, sketch, edit mask or None, return_mask, region) with 1, 2 and 3 stroke groups on 1000x667 and 4000x2667
    photos; the 3-group cases have two overlapping boxes."""
    rs = np.random.RandomState(29)
    one_k = [(300, 200, 330, 260)]
    two_k = [(100, 100, 140, 160), (800, 500, 860, 560)]
    three_k = [(100, 100, 140, 160), (330, 120, 370, 170), (800, 500, 860, 560)]
    one_4k = [(1200, 600, 1330, 900)]
    two_4k = [(600, 500, 760, 700), (3200, 1900, 3360, 2100)]
    three_4k = [(600, 500, 760, 700), (960, 500, 1120, 700), (3200, 1900, 3360, 2100)]
    p1, p4 = _photo(1000, 667, rs), _photo(4000, 2667, rs)
    reqs = []
    for p, groups in ((p1, (one_k, two_k, three_k)), (p4, (one_4k, two_4k, three_4k))):
        w, h = p.size
        for k, rects in enumerate(groups):
            reqs.append((p, _sketch(w, h, rects), None, k != 1, "strokes"))
        reqs.append((p, _sketch(w, h, groups[2]), _soft(w, h, groups[2], rs), True, "strokes"))
    reqs += [
        (p1, _sketch(1000, 667, two_k), None, True, [(0, 0, 400, 300), (100, 50, 500, 350), (0, 0, 400, 300)]),   # repeated
        (p1, _sketch(1000, 667, two_k), _soft(1000, 667, two_k, rs), False, [(600, 400, 1000, 667), (3, 5, 420, 333)]),
        (p4, _sketch(4000, 2667, two_4k), None, True, [(500, 400, 900, 800), (3000, 1700, 3500, 2250), (700, 450, 1300, 900)]),
    ]
    return reqs


def _boxes(req, region_size):
    _, sk, em, _, region = req
    if region == "strokes":
        return [b for _, b in region_groups(sk, em, region_size)]
    return region


def _serve(model, reqs, resize, region_size):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=50.0, resize=resize, region_size=region_size)
    got = [None] * len(reqs)

    def worker(i):
        img, sk, em, rm, region = reqs[i]
        got[i] = proc.process_image(img, sk, edit_mask=em, return_mask=rm, region=region)

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(reqs))]
    try:
        [t.start() for t in ts]
        [t.join() for t in ts]
    finally:
        proc.close()
    return got, proc.batcher.batches


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_device_flow_equals_the_pillow_flow(lib, precision):
    from tests.test_gpu_configs import _model
    model = _model(precision)
    reqs = _requests()
    counts = [len(_boxes(r, (256, 256))) for r in reqs]
    assert {1, 2, 3} <= set(counts)
    host, _ = _serve(model, reqs, "host", (256, 256))
    dev, batches = _serve(model, reqs, "device", (256, 256))
    assert sum(n for _, n in batches) == len(reqs) and len(batches) < len(reqs)
    for req, h, d in zip(reqs, host, dev):
        img, _, em, rm, region = req
        boxes = _boxes(req, (256, 256))
        if rm:
            (h, hm), (d, dm) = h, d
            if em is not None:
                assert hm is em and dm is em
            else:
                assert dm.mode == hm.mode == "L" and dm.size == img.size
                assert np.array_equal(np.array(hm), np.array(dm)), (img.size, boxes)
        hd, dd = np.array(h), np.array(d)
        assert d.size == img.size and np.array_equal(hd, dd), (img.size, boxes, int((hd != dd).sum()))
        outside = np.ones(dd.shape[:2], bool)
        for left, upper, right, lower in boxes:
            outside[upper:lower, left:right] = False
        assert np.array_equal(dd[outside], np.array(img)[outside]), (img.size, boxes)      # the photo's own bytes
        if rm and em is None:
            assert not np.array(dm)[outside].any()


@pytest.mark.gpu
def test_one_group_strokes_is_auto(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    rs = np.random.RandomState(5)
    img = _photo(4000, 2667, rs)
    sk = _sketch(4000, 2667, [(1200, 600, 1330, 900)])
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))
    try:
        a, am = proc.process_image(img, sk, return_mask=True, region="auto")
        s, sm = proc.process_image(img, sk, return_mask=True, region="strokes")
    finally:
        proc.close()
    assert np.array_equal(np.array(a), np.array(s)) and np.array_equal(np.array(am), np.array(sm))


@pytest.mark.gpu
def test_requests_with_different_box_counts_share_one_forward(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    rs = np.random.RandomState(8)
    img = _photo(1000, 667, rs)
    regions = [[(0, 0, 300, 300)], [(0, 0, 300, 300), (500, 300, 900, 667)], "strokes",
               [(0, 0, 300, 300), (100, 100, 400, 400), (200, 200, 500, 500), (600, 0, 1000, 300)]]
    sk = _sketch(1000, 667, [(100, 100, 140, 160), (330, 120, 370, 170), (800, 500, 860, 560)])
    proc = DemoProcessor(_model("bf16"), max_batch=16, max_wait_ms=200.0, region_size=(256, 256))
    got = [None] * len(regions)

    def worker(i):
        got[i] = proc.process_image(img, sk, region=regions[i])

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(regions))]
    try:
        [t.start() for t in ts]
        [t.join() for t in ts]
        alone = [proc.process_image(img, sk, region=r) for r in regions]
    finally:
        proc.close()
    assert proc.batcher.batches[0] == (("region", 256, 256), len(regions))
    for g, a in zip(got, alone):                                               # batching does not change a request's bytes
        assert np.array_equal(np.array(g), np.array(a))

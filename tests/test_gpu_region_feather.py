"""Feathered region pastes on the GPU: se_resize_composite_feather_detail_u8 and se_feather_u8 against the numpy statement bit for bit
(with guard bytes), zero widths against NULL widths, and the device flows of DemoProcessor.process_image
and EditSession.edit with feather > 0 against the Pillow flows."""
import gc
import threading

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import feather_mask
from tests.test_gpu_region_groups import BOXES, CANVASES, _pack, _requests, _result


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


@pytest.fixture(autouse=True)
def _release_device_memory():
    """The models of a test and the tensors torch caches go back to the device before the next test: later tests' engines
    allocate their arenas with cudaMalloc, which cannot use memory torch's allocator keeps."""
    yield
    gc.collect()
    try:
        import torch
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
    except ImportError:
        pass


# widths (left, top, right, bottom) of each box of BOXES: multiples of 4 and not, a box without bands among ones with them,
# bands that meet or cross in the middle of small boxes, the full side, the one-column and one-row boxes
FEATHER = [
    (13, 7, 0, 21),        # (300, 401)
    (3, 5, 2, 1),          # (60, 77)
    (33, 25, 33, 25),      # (101, 133)
    (4, 4, 8, 8),          # (101, 133) again
    (40, 34, 40, 33),      # (67, 80): the bands meet in the middle
    (12, 0, 7, 150),       # (150, 101), height unchanged: bottom band over the whole side
    (0, 0, 0, 0),          # (256, 256)
    (22, 15, 22, 15),      # (31, 45): the bands cross
    (1, 2, 0, 3),          # (97, 1)
    (100, 1, 3, 0),        # (1, 401)
    (16, 16, 16, 16),      # (48, 48)
]


def _canvas_buffer(canvases, aligned, seed):
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
    return imgs, offs, pitches, buf


def _composite(canvases, boxes, feather, swap, aligned, seed):
    """Runs one composite (engine.resize_composite_u8_packed) over canvases packed with guard bytes between rows and around
    them. Returns (device bytes, canvases, offsets, pitches, results)."""
    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    imgs, offs, pitches, buf = _canvas_buffer(canvases, aligned, seed)
    results = [_result(src, seed + 1 + i) for i, (_, _, _, src) in enumerate(boxes)]
    rgb, ro = _pack([r for r, _ in results], aligned, 0 if aligned else 3)
    msk, mo = _pack([m for _, m in results], aligned, 0 if aligned else 1)
    dev, rgb_d, msk_d = torch.from_numpy(buf).cuda(), torch.from_numpy(rgb).cuda(), torch.from_numpy(msk).cuda()
    resize_composite_u8_packed(rgb_d, ro, msk_d, mo, [b[3] for b in boxes], dev, [offs[b[0]] for b in boxes],
                               [pitches[b[0]] for b in boxes], [b[1] for b in boxes], [b[2] for b in boxes], swap_rb=swap,
                               feather=feather)
    return dev.cpu().numpy(), imgs, offs, pitches, results


def _check_statement(got, imgs, offs, pitches, boxes, results, feather, swap):
    """Each canvas against sequential Pillow pastes with m' = DIV255(m * ramp), and the guard bytes untouched."""
    inside = np.zeros(got.size, bool)
    for c, (img, o, p) in enumerate(zip(imgs, offs, pitches)):
        h, w = img.shape[:2]
        out = Image.fromarray(img)
        for i, ((_, (y, x), (bh, bw), _), (rgb, mask)) in enumerate(zip(boxes, results)):
            if boxes[i][0] != c:
                continue
            res = Image.fromarray(np.ascontiguousarray(rgb[..., ::-1]) if swap else rgb).resize((bw, bh))
            m = np.asarray(Image.fromarray(mask).resize((bw, bh)))
            if feather is not None:
                m = feather_mask(m, feather[i])
            out.paste(res, (x, y, x + bw, y + bh), Image.fromarray(m))
        rows = got[o:o + h * p].reshape(h, p)
        want = np.asarray(out)
        assert np.array_equal(rows[:, :w * 3].reshape(h, w, 3), want), \
            "canvas %d: %d bytes differ" % (c, int((rows[:, :w * 3].reshape(h, w, 3) != want).sum()))
        for r in range(h):
            inside[o + r * p:o + r * p + w * 3] = True
    assert (got[~inside] == 0xA5).all()


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("swap", [False, True])
def test_feathered_composite_matches_the_statement(lib, swap, aligned):
    got, imgs, offs, pitches, results = _composite(CANVASES, BOXES, FEATHER, swap, aligned, seed=40)
    _check_statement(got, imgs, offs, pitches, BOXES, results, FEATHER, swap)


@pytest.mark.gpu
def test_feathered_composite_past_one_launch(lib):
    """70 boxes with random widths in two canvases: more than one launch's descriptors, the order and the ramps carried on."""
    rs = np.random.RandomState(3)
    boxes, feather = [], []
    for i in range(70):
        h, w = int(rs.randint(8, 90)), int(rs.randint(8, 120))
        boxes.append((0 if i % 9 else 1, (int(rs.randint(0, 200 - h)), int(rs.randint(0, 240 - w))), (h, w),
                      (int(rs.choice([h, 32, 64])), int(rs.choice([w, 32, 48])))))
        feather.append(tuple(int(rs.randint(0, s + 1)) for s in (w, h, w, h)) if i % 5 else (0, 0, 0, 0))
    for aligned in (True, False):
        got, imgs, offs, pitches, results = _composite([(200, 240), (200, 240)], boxes, feather, True, aligned, seed=90)
        _check_statement(got, imgs, offs, pitches, boxes, results, feather, True)


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
def test_zero_widths_and_null_are_the_plain_composite(lib, aligned):
    plain = _composite(CANVASES, BOXES, None, True, aligned, seed=41)              # feather == NULL
    _check_statement(plain[0], *plain[1:4], BOXES, plain[4], None, True)
    got = _composite(CANVASES, BOXES, [(0, 0, 0, 0)] * len(BOXES), True, aligned, seed=41)[0]
    assert np.array_equal(got, plain[0])


@pytest.mark.gpu
def test_feather_u8_matches_numpy(lib):
    import torch

    from sketchedit_b200.engine import feather_u8_packed
    rs = np.random.RandomState(7)
    sizes, widths = [], []
    for i in range(45):                                       # more than one launch's descriptors
        h, w = int(rs.randint(1, 300)), int(rs.randint(1, 300))
        sizes.append((h, w))
        widths.append((0, 0, 0, 0) if i % 7 == 0 else tuple(int(rs.randint(0, s + 1)) for s in (w, h, w, h)))
    sizes += [(2667, 4000), (31, 45), (67, 80)]
    widths += [(32, 32, 32, 32), (22, 15, 22, 15), (40, 34, 40, 33)]
    imgs = [rs.randint(0, 256, hw, dtype=np.uint8) for hw in sizes]
    offs, pos = [], 5
    for a in imgs:
        offs.append(pos)
        pos += a.nbytes + 3 + pos % 5                         # odd offsets, guard bytes between the images
    buf = np.full(pos + 17, 0xA5, np.uint8)
    for a, o in zip(imgs, offs):
        buf[o:o + a.nbytes] = a.reshape(-1)
    want = buf.copy()
    for a, o, f in zip(imgs, offs, widths):
        want[o:o + a.nbytes] = feather_mask(a, f).reshape(-1)
    dev = torch.from_numpy(buf).cuda()
    feather_u8_packed(dev, offs, sizes, widths)
    got = dev.cpu().numpy()
    assert np.array_equal(got, want), int((got != want).sum())


# ------------------------------------------------------------------------------------------ DemoProcessor flows
FS = [16, 5, 32, 1, 64, 9]


def _serve(model, reqs, resize, feathers):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=50.0, resize=resize, region_size=(256, 256))
    got = [None] * len(reqs)

    def worker(i):
        img, sk, em, rm, region = reqs[i]
        got[i] = proc.process_image(img, sk, edit_mask=em, return_mask=rm, region=region, feather=feathers[i])

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(reqs))]
    try:
        [t.start() for t in ts]
        [t.join() for t in ts]
    finally:
        proc.close()
    return got, proc.batcher.batches


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_feathered_device_flow_equals_the_pillow_flow(lib, precision):
    from tests.test_gpu_configs import _model
    model = _model(precision)
    reqs = _requests()                                        # 'strokes' and box lists, edit masks, 1000x667 and 4000x2667
    reqs.append((reqs[0][0], reqs[0][1], None, True, "auto"))
    assert {r[0].size for r in reqs} == {(1000, 667), (4000, 2667)}
    feathers = [FS[i % len(FS)] for i in range(len(reqs))]
    host, _ = _serve(model, reqs, "host", feathers)
    dev, batches = _serve(model, reqs, "device", feathers)
    plain, _ = _serve(model, reqs, "device", [0] * len(reqs))
    assert sum(n for _, n in batches) == len(reqs)
    differ = 0
    for req, h, d, p in zip(reqs, host, dev, plain):
        img, _, em, rm, region = req
        if rm:
            (h, hm), (d, dm), (p, _) = h, d, p
            if em is not None:
                assert hm is em and dm is em
            else:
                assert dm.size == img.size and np.array_equal(np.array(hm), np.array(dm)), (img.size, region)
        hd, dd = np.array(h), np.array(d)
        assert np.array_equal(hd, dd), (img.size, region, int((hd != dd).sum()))
        differ += not np.array_equal(dd, np.array(p))
    assert differ >= len(reqs) // 2                            # the ramp is not a no-op (edit masks may be 0 at the edges)


@pytest.mark.gpu
def test_feather_0_and_16_share_one_forward(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_region_groups import _photo, _sketch
    rs = np.random.RandomState(8)
    img = _photo(1000, 667, rs)
    sk = _sketch(1000, 667, [(100, 100, 140, 160), (330, 120, 370, 170), (800, 500, 860, 560)])
    proc = DemoProcessor(_model("bf16"), max_batch=16, max_wait_ms=200.0, region_size=(256, 256))
    calls = [("strokes", 0), ("strokes", 16), ("auto", 16), ([(0, 0, 300, 300), (100, 100, 400, 400)], 0)]
    got = [None] * len(calls)

    def worker(i):
        got[i] = proc.process_image(img, sk, return_mask=True, region=calls[i][0], feather=calls[i][1])

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(calls))]
    try:
        [t.start() for t in ts]
        [t.join() for t in ts]
        alone = [proc.process_image(img, sk, return_mask=True, region=r, feather=f) for r, f in calls]
    finally:
        proc.close()
    assert proc.batcher.batches[0] == (("region", 256, 256), len(calls))
    for g, a in zip(got, alone):
        assert all(np.array_equal(np.array(x), np.array(y)) for x, y in zip(g, a))


def _chain(model, resize, img, steps):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=2.0, resize=resize, region_size=(256, 256))
    out = []
    try:
        s = proc.open_session(img)
        for k, (mask, em, region, off) in enumerate(steps):
            r = s.edit(mask, em, region=region, return_mask=True, offset=off, feather=FS[k % len(FS)])
            out.append((r, np.array(s.image())))
        for _ in range(len(steps)):
            boxes, patches = s.undo()
            out.append(((boxes, patches), np.array(s.image())))
    finally:
        proc.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_feathered_device_sessions_equal_host_sessions(lib, precision):
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo as photo
    from tests.test_gpu_edit_session import _steps
    model = _model(precision)
    rs = np.random.RandomState(31)
    for w, h in ((1000, 667), (4000, 2667)):
        img = photo(w, h, rs)
        steps = [st for st in _steps(w, h, rs) if st[2] is not None]   # region=None has no inner edges to feather
        host = _chain(model, "host", img, steps)
        dev = _chain(model, "device", img, steps)
        for k, ((hr, hi), (dr, di)) in enumerate(zip(host, dev)):
            assert np.array_equal(hi, di), (w, h, k, int((hi != di).sum()))
            if k < len(steps):
                assert hr.boxes == dr.boxes, (w, h, k)
                for a, b in zip(hr.patches + hr.masks, dr.patches + dr.masks):
                    assert (a is None and b is None) or np.array_equal(np.array(a), np.array(b)), (w, h, k)
            else:
                assert hr[0] == dr[0] and all(np.array_equal(np.array(a), np.array(b)) for a, b in zip(hr[1], dr[1]))
        assert np.array_equal(dev[-1][1], np.array(img))                 # undo walks back to the photo exactly

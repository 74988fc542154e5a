"""Region edits on the GPU: the composite with one box per canvas (engine.resize_composite_u8_packed) reproduces Pillow's
resize-and-paste bit for bit in ragged batches and writes nothing outside its destination slices, and the device flow of
DemoProcessor.process_image(..., region=...) returns exactly the Pillow flow's bytes."""
import threading

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import region_box

# (src (h, w), dst (h, w)): the height and the width each upscaled, downscaled or unchanged, odd widths
CASES = [
    ((256, 256), (608, 608)), ((256, 256), (100, 77)), ((256, 256), (256, 256)), ((256, 256), (256, 331)),
    ((256, 256), (256, 90)), ((256, 256), (401, 256)), ((256, 256), (97, 256)), ((64, 96), (300, 41)),
    ((64, 96), (17, 333)), ((64, 96), (64, 96)), ((31, 45), (31, 45)), ((1, 3), (5, 7)), ((40, 52), (1, 1)),
]


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _inputs(src, dst, seed):
    rs = np.random.RandomState(seed)
    rgb = rs.randint(0, 256, src + (3,), dtype=np.uint8)
    rgb[: src[0] // 3] = 255                                   # hard edges: both signs of every tap and both clamps
    rgb[src[0] // 3: src[0] // 2] = 0
    mask = rs.randint(0, 256, src, dtype=np.uint8)
    mask[:, : src[1] // 4] = 0                                 # 0, 255 and soft values after the resize
    mask[:, src[1] // 4: src[1] // 2] = 255
    base = rs.randint(0, 256, dst + (3,), dtype=np.uint8)
    return rgb, mask, base


def _pillow(rgb, mask, base, swap):
    h, w = base.shape[:2]
    res = Image.fromarray(np.ascontiguousarray(rgb[..., ::-1]) if swap else rgb).resize((w, h))
    out = Image.fromarray(base)
    out.paste(res, (0, 0), Image.fromarray(mask).resize((w, h)))
    return np.asarray(out)


def _pack(arrays, align, start, fill):
    """arrays packed into one uint8 buffer of canary bytes: 16-byte aligned offsets, or odd gaps (byte accesses)"""
    offs, pos = [], start
    for a in arrays:
        offs.append(pos)
        pos += a.nbytes + (16 if align else 5 + pos % 3)
        if align:
            pos = (pos + 15) // 16 * 16
    buf = np.full(pos + 41, fill, np.uint8)
    for a, o in zip(arrays, offs):
        buf[o:o + a.nbytes] = a.reshape(-1)
    return buf, offs


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("in_place", [False, True])
@pytest.mark.parametrize("swap_rb", [False, True])
def test_paste_matches_pillow_and_keeps_to_its_slices(lib, swap_rb, in_place, aligned):
    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    data = [_inputs(s, d, seed=400 + i) for i, (s, d) in enumerate(CASES)]
    rgb, rgb_offs = _pack([x[0] for x in data], aligned, 0 if aligned else 3, 0)
    msk, msk_offs = _pack([x[1] for x in data], aligned, 0 if aligned else 1, 0)
    base, base_offs = _pack([x[2] for x in data], aligned, 16 if aligned else 7, 0xA5)
    dev = {k: torch.from_numpy(v).cuda() for k, v in (("rgb", rgb), ("mask", msk), ("base", base))}
    if in_place:
        out, dst_offs = dev["base"], base_offs
    else:                                   # a separate destination: each base copied to its slice, then pasted over there
        _, dst_offs = _pack([x[2] for x in data], aligned, 32 if aligned else 9, 0x5A)
        out = torch.full((dst_offs[-1] + data[-1][2].nbytes + 77,), 0x5A, dtype=torch.uint8, device="cuda")
        for (_, _, b), bo, do in zip(data, base_offs, dst_offs):
            out[do:do + b.nbytes].copy_(dev["base"][bo:bo + b.nbytes])
    dst = [d for _, d in CASES]             # one box per canvas, filling it: at (0, 0), pitch 3 w
    resize_composite_u8_packed(dev["rgb"], rgb_offs, dev["mask"], msk_offs, [s for s, _ in CASES], out, dst_offs,
                               [3 * w for _, w in dst], [(0, 0)] * len(dst), dst, swap_rb=swap_rb)
    o = out.cpu().numpy()
    inside = np.zeros(o.size, bool)
    for (s, d), (r, m, b), off in zip(CASES, data, dst_offs):
        n = b.nbytes
        inside[off:off + n] = True
        want = _pillow(r, m, b, swap_rb).reshape(-1)
        got = o[off:off + n]
        assert np.array_equal(got, want), "%s -> %s: %d bytes differ (Pillow %s)" % (s, d, int((got != want).sum()), PIL.__version__)
    assert (o[~inside] == (0xA5 if in_place else 0x5A)).all()                 # guard bytes around every destination slice
    assert np.array_equal(dev["rgb"].cpu().numpy(), rgb) and np.array_equal(dev["mask"].cpu().numpy(), msk)
    if not in_place:
        assert np.array_equal(dev["base"].cpu().numpy(), base)


@pytest.mark.gpu
def test_paste_splits_long_batches(lib):
    """More than 32 canvases of one box each: the composite runs them in several launches with one scratch allocation."""
    import torch

    from sketchedit_b200.engine import resize_composite_u8_packed
    cases = [((32, 40), (50 + i, 29 + 2 * i)) for i in range(37)]
    data = [_inputs(s, d, seed=700 + i) for i, (s, d) in enumerate(cases)]
    rgb, ro = _pack([x[0] for x in data], True, 0, 0)
    msk, mo = _pack([x[1] for x in data], True, 0, 0)
    base, bo = _pack([x[2] for x in data], True, 0, 0)
    out = torch.from_numpy(base).cuda()
    resize_composite_u8_packed(torch.from_numpy(rgb).cuda(), ro, torch.from_numpy(msk).cuda(), mo, [s for s, _ in cases], out, bo,
                               [3 * d[1] for _, d in cases], [(0, 0)] * len(cases), [d for _, d in cases], swap_rb=True)
    o = out.cpu().numpy()
    for (r, m, b), off in zip(data, bo):
        assert np.array_equal(o[off:off + b.nbytes], _pillow(r, m, b, True).reshape(-1))


# ------------------------------------------------------------------------------------------ DemoProcessor region flows
def _requests():
    """(photo, sketch, edit mask or None, return_mask, region): photo sizes up to 4000x2667, boxes at the corners, an
    explicit box, a photo smaller than the working size, edit-mask requests and a whole-photo request alongside."""
    rs = np.random.RandomState(23)

    def photo(w, h):
        a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        a[:, : w // 3] = 255 - a[:, : w // 3] // 4
        return Image.fromarray(a)

    def sketch(w, h, x0, y0, x1, y1):
        m = np.zeros((h, w), np.uint8)
        m[y0:y1, x0:x1:3] = 255
        return Image.fromarray(m)

    def soft(w, h, x0, y0, x1, y1):
        m = np.zeros((h, w), np.uint8)
        m[y0:y1, x0:x1] = rs.randint(0, 256, (y1 - y0, x1 - x0), dtype=np.uint8)
        return Image.fromarray(m)

    return [
        (photo(4000, 2667), sketch(4000, 2667, 1200, 600, 1330, 900), None, False, "auto"),
        (photo(4000, 2667), sketch(4000, 2667, 3900, 2600, 3990, 2667), None, True, "auto"),           # bottom-right corner
        (photo(1000, 667), sketch(1000, 667, 0, 0, 40, 30), None, True, "auto"),                      # top-left corner
        (photo(641, 481), sketch(641, 481, 300, 200, 420, 230), None, False, (3, 5, 420, 333)),       # explicit, odd box
        (photo(300, 200), sketch(300, 200, 100, 50, 140, 60), None, True, "auto"),                    # smaller than the work size
        (photo(1000, 667), sketch(1000, 667, 600, 100, 640, 140), soft(1000, 667, 560, 80, 700, 190), True, "auto"),
        (photo(4000, 2667), sketch(4000, 2667, 10, 2500, 60, 2600), soft(4000, 2667, 0, 2400, 200, 2667), False,
         (0, 2300, 400, 2667)),                                                                        # bottom-left, edit mask
        (photo(1000, 667), sketch(1000, 667, 500, 300, 530, 360), None, False, None),                 # whole photo
    ]


def _box(req, region_size):
    img, sk, em, _, region = req
    if region != "auto":
        return region
    bbs = [b for b in (sk.getbbox(), em.getbbox() if em is not None else None) if b]
    return region_box((min(b[0] for b in bbs), min(b[1] for b in bbs), max(b[2] for b in bbs), max(b[3] for b in bbs)),
                      img.size, region_size)


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
@pytest.mark.parametrize("precision, region_size", [("bf16", (256, 256)), ("fp32_direct", (256, 256)), ("bf16", (192, 320))])
def test_device_region_flow_equals_the_pillow_flow(lib, precision, region_size):
    from tests.test_gpu_configs import _model
    model = _model(precision)
    reqs = _requests()
    host, _ = _serve(model, reqs, "host", region_size)
    dev, batches = _serve(model, reqs, "device", region_size)
    Hn, Wn = region_size
    n_region = sum(1 for r in reqs if r[4] is not None)
    region_batches = [(k, n) for k, n in batches if k[0] == "region"]
    assert sum(n for _, n in region_batches) == n_region and len(region_batches) < n_region     # photos of different sizes batch
    assert {k for k, _ in region_batches} == {("region", Hn, Wn), ("region", Hn, Wn, True)}
    for req, h, d in zip(reqs, host, dev):
        img, _, em, rm, region = req
        if rm:
            (h, hm), (d, dm) = h, d
            if em is not None:
                assert hm is em and dm is em
            else:
                assert dm.mode == hm.mode == "L" and dm.size == img.size
                assert np.array_equal(np.array(hm), np.array(dm)), (img.size, region)
        assert d.size == img.size and d.mode == h.mode == "RGB"
        hd, dd = np.array(h), np.array(d)
        assert np.array_equal(hd, dd), (img.size, region, int((hd != dd).sum()))
        if region is None:
            continue
        left, upper, right, lower = _box(req, region_size)
        outside = np.ones(dd.shape[:2], bool)
        outside[upper:lower, left:right] = False
        assert np.array_equal(dd[outside], np.array(img)[outside]), (img.size, region)       # the photo's own bytes
        if rm and em is None:
            assert not np.array(dm)[outside].any()

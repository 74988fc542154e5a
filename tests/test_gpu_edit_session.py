"""Edit sessions on the GPU: se_resize_window_u8 (engine.resize_window_u8_packed) is Image.crop(box).resize(size) bit for bit,
and DemoProcessor.open_session with the device flow returns the Pillow flow's bytes, undoes exactly, shares forwards with
other sessions and plain requests, and releases its device memory on close()."""
import gc
import threading

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


# sources (h, w, extra pitch bytes) and windows (source, (left, upper, right, lower), target (h, w)): every axis upscaled,
# downscaled or unchanged, odd widths, odd pitches, overlapping and repeated windows, windows at the source's edges.
SOURCES = [(300, 401, 0), (97, 130, 5), (64, 64, 64), (1, 33, 1)]
WINDOWS = [
    (0, (0, 0, 401, 300), (256, 256)),
    (0, (37, 40, 170, 141), (256, 256)),
    (0, (37, 40, 170, 141), (101, 133)),        # the same window again, unchanged size
    (0, (100, 90, 333, 250), (160, 77)),        # overlaps the two above
    (0, (300, 150, 401, 300), (150, 60)),       # height unchanged, width downscaled, bottom-right corner
    (1, (3, 5, 80, 65), (64, 96)),
    (1, (50, 30, 130, 97), (67, 80)),           # unchanged size, odd pitch
    (1, (0, 0, 1, 97), (33, 7)),                # one column
    (2, (8, 8, 56, 56), (256, 256)),
    (3, (2, 0, 31, 1), (1, 29)),                # one row, unchanged
    (0, (0, 299, 401, 300), (5, 7)),            # one row along the bottom edge
]


def _run_windows(channels, aligned, seed):
    import torch

    from sketchedit_b200.engine import resize_window_u8_packed
    rs = np.random.RandomState(seed)
    imgs, bufs, pitches = [], [], []
    for h, w, extra in SOURCES:
        a = rs.randint(0, 256, (h, w, channels) if channels == 3 else (h, w), dtype=np.uint8)
        a[: h // 3] = 255                                        # hard edges: both signs of every tap and both clamps
        p = w * channels + extra
        buf = np.full(h * p + 3, 0x5A, np.uint8)                 # the source's own row padding holds other bytes
        buf[:h * p].reshape(h, p)[:, :w * channels] = a.reshape(h, -1)
        imgs.append(a)
        bufs.append(torch.from_numpy(buf).cuda())
        pitches.append(p)
    offs, pos = [], 16 if aligned else 7
    for _, _, (th, tw) in WINDOWS:
        offs.append(pos)
        pos += th * tw * channels + (16 if aligned else 5)
        if aligned:
            pos = (pos + 15) // 16 * 16
    out = torch.full((pos + 29,), 0xA5, dtype=torch.uint8, device="cuda")
    srcs = [bufs[s] for s, _, _ in WINDOWS]
    starts = [b[1] * pitches[s] + b[0] * channels for s, b, _ in WINDOWS]
    sizes = [(b[3] - b[1], b[2] - b[0]) for _, b, _ in WINDOWS]
    resize_window_u8_packed(srcs, starts, [pitches[s] for s, _, _ in WINDOWS], sizes, [t for _, _, t in WINDOWS], channels,
                            out=out, dst_offsets=offs)
    got = out.cpu().numpy()
    inside = np.zeros(got.size, bool)
    for (s, box, (th, tw)), o in zip(WINDOWS, offs):
        want = np.asarray(Image.fromarray(imgs[s]).crop(box).resize((tw, th)))
        n = th * tw * channels
        assert np.array_equal(got[o:o + n].reshape(want.shape), want), \
            (box, (th, tw), int((got[o:o + n].reshape(want.shape) != want).sum()), PIL.__version__)
        inside[o:o + n] = True
    assert (got[~inside] == 0xA5).all()                          # guard bytes around every destination
    for buf, (h, w, extra), p in zip(bufs, SOURCES, pitches):      # the sources are only read
        assert (buf.cpu().numpy()[:h * p].reshape(h, p)[:, w * channels:] == 0x5A).all()


@pytest.mark.gpu
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("channels", [1, 3])
def test_window_resize_is_crop_then_resize(lib, channels, aligned):
    _run_windows(channels, aligned, seed=7 + channels)


@pytest.mark.gpu
def test_window_resize_of_more_than_one_call(lib):
    """40 windows of one photo, past one call's 32 images, against the crop-and-resize of each."""
    import torch

    from sketchedit_b200.engine import resize_window_u8_packed
    rs = np.random.RandomState(2)
    h, w = 200, 301
    a = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
    boxes, targets = [], []
    for _ in range(40):
        bh, bw = int(rs.randint(1, 120)), int(rs.randint(1, 150))
        y, x = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
        boxes.append((x, y, x + bw, y + bh))
        targets.append((int(rs.choice([bh, 48, 64])), int(rs.choice([bw, 40, 64]))))
    photo = torch.from_numpy(a).cuda().view(-1)
    out, offs = resize_window_u8_packed(photo, [(b[1] * w + b[0]) * 3 for b in boxes], [3 * w] * 40,
                                        [(b[3] - b[1], b[2] - b[0]) for b in boxes], targets, 3)
    got = out.cpu().numpy()
    for b, (th, tw), o in zip(boxes, targets, offs):
        want = np.asarray(Image.fromarray(a).crop(b).resize((tw, th)))
        assert np.array_equal(got[o:o + th * tw * 3].reshape(th, tw, 3), want), b


# ------------------------------------------------------------------------------------------ sessions
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


def _steps(w, h, rs):
    """A chain of (mask, edit mask, region, offset) on a w x h photo: every region form, edit masks, offset masks."""
    sx, sy = w / 1000, h / 667
    r = lambda x0, y0, x1, y1: (int(x0 * sx), int(y0 * sy), int(x1 * sx), int(y1 * sy))
    two = [r(100, 100, 140, 160), r(800, 500, 860, 560)]
    three = [r(100, 100, 140, 160), r(330, 120, 370, 170), r(800, 500, 860, 560)]
    small = _sketch(97, 61, [(10, 10, 40, 50), (60, 5, 90, 30)])
    return [
        (_sketch(w, h, [r(300, 200, 330, 260)]), None, "auto", (0, 0)),
        (_sketch(w, h, two), None, "strokes", (0, 0)),
        (_sketch(w, h, three), _soft(w, h, three, rs), "strokes", (0, 0)),
        (small, None, "strokes", (int(500 * sx) + 3, int(300 * sy) + 5)),
        (small, _soft(97, 61, [(0, 0, 97, 61)], rs), "auto", (w - 97, h - 61)),
        (_sketch(w, h, two), None, [r(0, 0, 400, 300), r(100, 50, 500, 350), r(0, 0, 400, 300)], (0, 0)),
        (_sketch(w, h, two), None, None, (0, 0)),
        (_sketch(w, h, two), _soft(w, h, two, rs), None, (0, 0)),
        (_sketch(w, h, three), None, r(600, 400, 1000, 667), (0, 0)),
    ]


def _chain(model, resize, img, steps):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=2.0, resize=resize, region_size=(256, 256))
    out = []
    try:
        s = proc.open_session(img)
        for mask, em, region, off in steps:
            r = s.edit(mask, em, region=region, return_mask=True, offset=off)
            out.append((r, np.array(s.image())))
        for _ in range(3):
            boxes, patches = s.undo()
            out.append(((boxes, patches), np.array(s.image())))
    finally:
        proc.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_device_sessions_equal_host_sessions(lib, precision):
    from tests.test_gpu_configs import _model
    model = _model(precision)
    rs = np.random.RandomState(31)
    for w, h in ((1000, 667), (4000, 2667)):
        img = _photo(w, h, rs)
        steps = _steps(w, h, rs)
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
        assert np.array_equal(dev[-1][1], np.array(_chain_state(img, steps, model)))


def _chain_state(img, steps, model):
    """The photo after len(steps) - 3 edits, by process_image fed its own result (the statement of a session)."""
    from sketchedit_b200.serving import DemoProcessor, _placed
    proc = DemoProcessor(model, region_size=(256, 256))
    cur = img.convert("RGB")
    try:
        for mask, em, region, off in steps[:-3]:
            cur = proc.process_image(cur, _placed(mask, img.size, off), _placed(em, img.size, off), region=region)
    finally:
        proc.close()
    return cur


@pytest.mark.gpu
def test_undo_restores_exact_bytes_and_memory_is_released(lib):
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    rs = np.random.RandomState(4)
    img = _photo(4000, 2667, rs)
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))
    steps = _steps(4000, 2667, rs)
    # Warm-up: graphs, tables and staging buffers of every step. The engine keeps buffers sized by its last forward, so the
    # warm-up and every measured stretch end with the same edit.
    last = lambda sess: sess.edit(*steps[1][:2], region="strokes")
    warm = proc.open_session(img)
    for mask, em, region, off in steps:
        warm.edit(mask, em, region=region, offset=off)
    last(warm)
    warm.close()

    def allocated():                                               # garbage of earlier tests is freed first
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    start = allocated()
    try:
        s = proc.open_session(img)
        states = [np.array(img)]
        for mask, em, region, off in steps:
            s.edit(mask, em, region=region, offset=off)
            states.append(np.array(s.image()))
        assert allocated() > start
        for k in range(len(steps), 0, -1):
            s.undo()
            assert np.array_equal(np.array(s.image()), states[k - 1]), k
        with pytest.raises(RuntimeError, match="nothing to undo"):
            s.undo()
        last(s)
        s.close()
        assert allocated() == start
        s2 = proc.open_session(img)
        last(s2)
    finally:
        proc.close()
    with pytest.raises(RuntimeError, match="closed"):
        s2.image()
    assert allocated() <= start                                    # the processor's close also frees its worker's buffers


@pytest.mark.gpu
def test_two_sessions_and_a_plain_request_share_one_forward(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    rs = np.random.RandomState(8)
    imgs = [_photo(1000, 667, rs), _photo(4000, 2667, rs), _photo(1000, 667, rs)]
    masks = [_sketch(1000, 667, [(100, 100, 140, 160), (800, 500, 860, 560)]),
             _sketch(4000, 2667, [(1200, 600, 1330, 900)]), _sketch(1000, 667, [(300, 200, 330, 260)])]
    proc = DemoProcessor(_model("bf16"), max_batch=16, max_wait_ms=300.0, region_size=(256, 256))
    try:
        sessions = [proc.open_session(imgs[0]), proc.open_session(imgs[1])]
        alone = [proc.open_session(imgs[0]), proc.open_session(imgs[1])]
        got = [None] * 3

        def worker(i):
            if i < 2:
                got[i] = sessions[i].edit(masks[i], region="strokes", return_mask=True)
            else:
                got[i] = proc.process_image(imgs[2], masks[2], return_mask=True, region="auto")

        n0 = len(proc.batcher.batches)
        ts = [threading.Thread(target=worker, args=(i,)) for i in range(3)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        assert proc.batcher.batches[n0:] == [(("region", 256, 256), 3)]
        want = [alone[i].edit(masks[i], region="strokes", return_mask=True) for i in range(2)]
        plain = proc.process_image(imgs[2], masks[2], return_mask=True, region="auto")
        for g, a, s, t in zip(got[:2], want, sessions, alone):        # batching does not change a session's bytes
            assert g.boxes == a.boxes
            for x, y in zip(g.patches + g.masks, a.patches + a.masks):
                assert np.array_equal(np.array(x), np.array(y))
            assert np.array_equal(np.array(s.image()), np.array(t.image()))
        assert all(np.array_equal(np.array(x), np.array(y)) for x, y in zip(got[2], plain))
    finally:
        proc.close()

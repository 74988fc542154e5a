"""Previews on the GPU: se_resize_reducing_u8 (engine.resize_reducing_u8_packed, engine.thumbnail_u8) equals Image.thumbnail
and its numpy restatement (tests/util_thumbnail.py) over the CPU matrix and 4000x2667 photos at the bounds a page uses; in
batches past one call of windows with odd pitches that overlap, with nothing written past each output, each equal to its
batch-1 result; EditSession.image/jpeg/png(size=...) equal the Pillow statements in both resize modes after edits and undo;
a size that already fits gives today's bytes; and the calls give their device memory back."""
import gc
import io

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build, engine
from tests import util_thumbnail as U
from tests.test_thumbnail import BAD_SIZES, THUMBS, _png, _random


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _pillow(a, size):
    im = Image.fromarray(a)
    im.thumbnail(size)
    return np.asarray(im)


@pytest.mark.gpu
def test_entry_is_pillow(lib):
    """The CPU matrix (random and photo-like) and 4000x2667 photo-like images at (640, 640), (256, 256), (1280, 1280) (a
    factor of 1: only the box-free resize runs) and (1, 1) (cells of 2000 x 1333 pixels), all in one call."""
    import torch
    cases = [(a, size) for hw, size in THUMBS for a in (_random(*hw, seed=hw[0] + hw[1]), U.photo_like(*hw, seed=7))]
    photo = U.photo_like(2667, 4000, seed=11)
    cases += [(photo, size) for size in ((640, 640), (256, 256), (1280, 1280), (1, 1))]
    srcs = [torch.from_numpy(a.reshape(-1)).cuda() for a, _ in cases]
    dst = []
    for a, size in cases:
        ts = engine.thumbnail_size(a.shape[1], a.shape[0], size)
        dst.append(a.shape[:2] if ts is None else (ts[1], ts[0]))
    out, offs = engine.resize_reducing_u8_packed(srcs, [0] * len(srcs), [3 * a.shape[1] for a, _ in cases],
                                                 [a.shape[:2] for a, _ in cases], dst)
    got = out.cpu().numpy()
    for (a, size), (h, w), o in zip(cases, dst, offs):
        want = _pillow(a, size)
        assert want.shape == (h, w, 3)
        g = got[o:o + h * w * 3].reshape(h, w, 3)
        assert np.array_equal(g, want), (a.shape, size, int((g != want).sum()), PIL.__version__)
        assert np.array_equal(g, U.thumbnail(a, size)), (a.shape, size)
    # thumbnail_u8 on the resident photo, one bound for the list
    t = torch.from_numpy(photo).cuda()
    for size in ((640, 640), (1, 1)):
        assert np.array_equal(engine.thumbnail_u8([t], size)[0].cpu().numpy(), _pillow(photo, size)), size


def _sources(rs):
    import torch
    sources, bufs, pitches = [], [], []
    for h, w, extra in ((1301, 977, 5), (64, 33, 1), (2100, 19, 2)):
        a = U.photo_like(h, w, seed=int(rs.randint(1000)))
        a[h // 2:, w // 2:] = rs.randint(0, 256, (h - h // 2, w - w // 2, 3))
        p = 3 * w + extra
        buf = np.full(h * p + 7, 0x5A, np.uint8)
        buf[:h * p].reshape(h, p)[:, :3 * w] = a.reshape(h, -1)
        sources.append(a)
        bufs.append(torch.from_numpy(buf).cuda())
        pitches.append(p)
    return sources, bufs, pitches


@pytest.mark.gpu
def test_windows_batches_and_guard_bytes(lib):
    """45 windows (past one call's 32) of three sources with odd pitches, overlapping and repeated, resized to thumbnails and
    to other sizes (upscales, one axis, the tall branch), into one buffer with odd gaps: each is Pillow's
    crop(box).resize(size, reducing_gap=2.0) and its own batch-1 result, every byte past an output is untouched, and the
    sources are only read."""
    import torch
    rs = np.random.RandomState(5)
    sources, bufs, pitches = _sources(rs)
    wins = [(0, (0, 0, 977, 1301), (100, 75)), (0, (0, 0, 977, 1301), (100, 75)), (1, (0, 0, 33, 64), (64, 33)),
            (2, (0, 0, 19, 2100), (1880, 17)), (2, (3, 7, 4, 2007), (19, 1)), (0, (970, 1290, 977, 1301), (1, 1)),
            (0, (5, 7, 960, 1250), (1, 1)), (1, (1, 1, 30, 60), (170, 20))]
    while len(wins) < 45:
        s = int(rs.randint(0, 3))
        h, w = sources[s].shape[:2]
        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
        y, x = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
        th, tw = max(1, bh // int(rs.randint(1, 40))), max(1, bw // int(rs.randint(1, 40)))
        if rs.rand() < 0.2:
            th = int(rs.randint(1, 2 * bh + 1))
        wins.append((s, (x, y, x + bw, y + bh), (th, tw)))
    offs, pos = [], 3
    for _, _, (th, tw) in wins:
        offs.append(pos)
        pos += th * tw * 3 + 5
    out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
    args = ([bufs[s] for s, _, _ in wins], [b[1] * pitches[s] + 3 * b[0] for s, b, _ in wins], [pitches[s] for s, _, _ in wins],
            [(b[3] - b[1], b[2] - b[0]) for _, b, _ in wins], [d for _, _, d in wins])
    engine.resize_reducing_u8_packed(*args, out=out, dst_offsets=offs)
    got = out.cpu().numpy()
    written = np.zeros(got.size, bool)
    for k, ((s, b, (th, tw)), o) in enumerate(zip(wins, offs)):
        crop = np.ascontiguousarray(sources[s][b[1]:b[3], b[0]:b[2]])
        want = np.asarray(Image.fromarray(crop).resize((tw, th), reducing_gap=2.0))
        g = got[o:o + th * tw * 3].reshape(th, tw, 3)
        assert np.array_equal(g, want), (k, b, (th, tw), int((g != want).sum()))
        assert np.array_equal(g, U.resize_reducing(crop, (th, tw))), (k, b)
        written[o:o + th * tw * 3] = True
        if k % 5 == 0:
            one, o1 = engine.resize_reducing_u8_packed(*(a[k:k + 1] for a in args))
            assert np.array_equal(one.cpu().numpy()[o1[0]:o1[0] + th * tw * 3].reshape(th, tw, 3), want), k
    assert (got[~written] == 0xA5).all()
    for buf, a, p in zip(bufs, sources, pitches):
        h, w = a.shape[:2]
        host = buf.cpu().numpy()
        assert (host[:h * p].reshape(h, p)[:, 3 * w:] == 0x5A).all() and (host[h * p:] == 0x5A).all()
        assert np.array_equal(host[:h * p].reshape(h, p)[:, :3 * w].reshape(h, w, 3), a)


def _jpeg(img, **kw):
    buf = io.BytesIO()
    img.save(buf, "JPEG", **kw)
    return buf.getvalue()


def _check(s, cur, box=None, size=(640, 640), host=False):
    """s.image/jpeg/png(size=..., box=...) against the Pillow statements on ``cur`` (the session's current photo)."""
    img = cur.crop(box) if box is not None else cur.copy()
    img.thumbnail(size)
    if box is None:
        assert np.array_equal(np.asarray(s.image(size=size)), np.asarray(img)), size
    for q, sub, opt, prog in ((75, 2, False, False), (90, 0, True, False), (85, 2, False, True)):
        try:
            want = _jpeg(img, quality=q, subsampling=sub, optimize=opt, progressive=prog)
        except OSError:                  # Pillow refuses optimized files past its buffer; the device writes them
            if host:
                with pytest.raises(OSError):
                    s.jpeg(q, sub, box=box, size=size, optimize=opt, progressive=prog)
            continue
        assert s.jpeg(q, sub, box=box, size=size, optimize=opt, progressive=prog) == want, (box, size, q, sub, opt, prog)
    assert s.png(box, size=size) == _png(img), (box, size)


@pytest.mark.gpu
def test_session_previews_are_pillow_after_edits_and_undo(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model("bf16")
    rs = np.random.RandomState(12)
    w, h = 1000, 667
    img = _photo(w, h, rs)
    steps = _steps(w, h, rs)
    for resize in ("device", "host"):
        proc = DemoProcessor(model, max_batch=4, resize=resize, region_size=(256, 256))
        try:
            s = proc.open_session(img)
            _check(s, s.image(), host=resize == "host")
            for k, (mask, em, region, off) in enumerate(steps[:6]):
                r = s.edit(mask, em, region=region, offset=off)
                cur = s.image()
                _check(s, cur, size=[(640, 640), (256, 256), (1, 1), (999, 20)][k % 4], host=resize == "host")
                _check(s, cur, box=r.boxes[0], size=(64, 64), host=resize == "host")
            boxes, _ = s.undo()
            _check(s, s.image(), box=boxes[0], size=(100, 33), host=resize == "host")
            s.undo()
            _check(s, s.image(), size=(320, 320), host=resize == "host")
        finally:
            proc.close()


@pytest.mark.gpu
def test_photo_previews_fitting_sizes_checks_and_memory(lib):
    """A 4000x2667 photo: previews at the page bounds equal Pillow, a size that fits gives today's bytes, bad sizes are
    ValueError in the device flow, and the calls give their device memory back."""
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    img = Image.fromarray(U.photo_like(2667, 4000, seed=3))
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)
        warm.jpeg(size=(640, 640))
        warm.png(size=(256, 256))
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        for size in ((640, 640), (256, 256), (1280, 1280), (1, 1)):
            _check(s, img, size=size)
        _check(s, img, box=(5, 7, 1001, 667), size=(np.int64(200), np.int32(200)))
        for size in ((4000, 2667), (5000, 2667), (4000, 9999)):
            assert np.array_equal(np.asarray(s.image(size=size)), np.asarray(img))
            assert s.jpeg(size=size) == s.jpeg() == _jpeg(img, quality=75, subsampling=2)
            assert s.png(size=size) == s.png()
        assert s.jpeg(box=(0, 0, 640, 427), size=(640, 427)) == s.jpeg(box=(0, 0, 640, 427))
        for bad in BAD_SIZES:
            for call in (lambda: s.image(size=bad), lambda: s.jpeg(size=bad), lambda: s.png(size=bad)):
                with pytest.raises(ValueError, match="size must be"):
                    call()
        s.close()
        assert allocated() == start
    finally:
        proc.close()

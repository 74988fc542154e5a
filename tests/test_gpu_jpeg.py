"""JPEG encoding on the GPU: se_jpeg_encode_u8 (engine.jpeg_encode_u8 / jpeg_encode_u8_packed) writes Pillow's bytes over
sizes, qualities, both subsamplings and contents, in mixed batches of windows with odd pitches that overlap, and nothing past
each file; EditSession.jpeg() is the Pillow statement on the session's photo after chains of edits and undos, and a session
gives its device memory back on close()."""
import gc
import io

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from tests import util_jpeg as J
from tests.test_jpeg import CONTENTS, QUALITIES, SIZES, content, pillow_jpeg


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


@pytest.mark.gpu
@pytest.mark.parametrize("subsampling", [0, 2])
def test_kernels_are_pillow(lib, subsampling):
    """Every size, content and quality of the CPU matrix, plus a 4000x2667 photo; one call per (size, quality) batch."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8
    rs = np.random.RandomState(17 + subsampling)
    for hw in SIZES + [(2667, 4000)]:
        imgs = [content(kind, *hw, rs) for kind in CONTENTS]
        dev = [torch.from_numpy(a).cuda() for a in imgs]
        for q in QUALITIES:
            got = jpeg_encode_u8(dev, q, subsampling)
            for kind, a, g in zip(CONTENTS, imgs, got):
                want = pillow_jpeg(a, q, subsampling)
                assert g == want, (hw, kind, q, subsampling, len(g), len(want), PIL.__version__)


@pytest.mark.gpu
def test_mixed_batches_overlapping_windows_and_guard_bytes(lib):
    """40 windows (past one call's 32) of two sources with odd pitches, overlapping and repeated, at mixed sizes, into one
    buffer with odd gaps: each file is Pillow's crop-and-save, and every byte past a file is untouched."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed
    rs = np.random.RandomState(3)
    sources, bufs, pitches = [], [], []
    for h, w, extra in ((301, 403, 5), (64, 33, 1)):
        a = content("places_11_512x408.npz", h, w, rs)
        a[h // 2:, w // 2:] = rs.randint(0, 256, (h - h // 2, w - w // 2, 3))
        p = 3 * w + extra
        buf = np.full(h * p + 7, 0x5A, np.uint8)
        buf[:h * p].reshape(h, p)[:, :3 * w] = a.reshape(h, -1)
        sources.append(a)
        bufs.append(torch.from_numpy(buf).cuda())
        pitches.append(p)
    wins = [(0, (0, 0, 403, 301)), (0, (0, 0, 403, 301)), (1, (0, 0, 33, 64)), (0, (400, 298, 403, 301)), (0, (5, 7, 6, 8))]
    for _ in range(35):
        s = int(rs.randint(0, 2))
        h, w = sources[s].shape[:2]
        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
        y, x = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
        wins.append((s, (x, y, x + bw, y + bh)))
    for sub, q in ((2, 75), (0, 90)):
        offs, pos = [], 3
        for s, b in wins:
            offs.append(pos)
            pos += J.max_bytes(b[3] - b[1], b[2] - b[0], sub) + 5
        out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
        _, _, nbytes = jpeg_encode_u8_packed([bufs[s] for s, _ in wins], [b[1] * pitches[s] + 3 * b[0] for s, b in wins],
                                             [pitches[s] for s, _ in wins], [(b[3] - b[1], b[2] - b[0]) for _, b in wins],
                                             quality=q, subsampling=sub, out=out, out_offsets=offs)
        got, lens = out.cpu().numpy(), nbytes.cpu().tolist()
        written = np.zeros(got.size, bool)
        for (s, b), o, n in zip(wins, offs, lens):
            want = pillow_jpeg(np.ascontiguousarray(sources[s][b[1]:b[3], b[0]:b[2]]), q, sub)
            assert got[o:o + n].tobytes() == want, (b, sub, n, len(want))
            written[o:o + n] = True
        assert (got[~written] == 0xA5).all()
        for buf, a, p in zip(bufs, sources, pitches):              # the sources are only read
            h, w = a.shape[:2]
            assert (buf.cpu().numpy()[:h * p].reshape(h, p)[:, 3 * w:] == 0x5A).all()


@pytest.mark.gpu
def test_strided_views_are_encoded_where_they_lie(lib):
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8
    rs = np.random.RandomState(9)
    a = content("face_602_256x256.npz", 300, 401, rs)
    t = torch.from_numpy(a).cuda()
    boxes = [(0, 0, 401, 300), (17, 3, 250, 77), (400, 0, 401, 300), (0, 299, 401, 300), (100, 100, 116, 116)]
    got = jpeg_encode_u8([t[b[1]:b[3], b[0]:b[2]] for b in boxes])
    for b, g in zip(boxes, got):
        assert g == pillow_jpeg(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2]])), b


def _pillow_of(img, quality=75, subsampling=2, box=None):
    buf = io.BytesIO()
    (img if box is None else img.crop(box)).save(buf, "JPEG", quality=quality, subsampling=subsampling)
    return buf.getvalue()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_session_jpeg_is_pillow_after_edits_and_undo(lib, precision):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model(precision)
    rs = np.random.RandomState(23)
    for w, h in ((1000, 667), (4000, 2667)):
        img = _photo(w, h, rs)
        steps = _steps(w, h, rs)
        for resize in ("device", "host"):
            proc = DemoProcessor(model, max_batch=4, resize=resize, region_size=(256, 256))
            try:
                s = proc.open_session(img)
                assert s.jpeg() == _pillow_of(s.image())
                for k, (mask, em, region, off) in enumerate(steps):
                    r = s.edit(mask, em, region=region, offset=off)
                    cur = s.image()
                    q, sub = (75, 2) if k % 2 == 0 else (90, 0)
                    assert s.jpeg(q, sub) == _pillow_of(cur, q, sub), (w, h, resize, k)
                    for b in r.boxes[:2]:                           # what the edit changed
                        assert s.jpeg(box=b) == _pillow_of(cur, box=b), (w, h, resize, k, b)
                for k in range(3):
                    boxes, _ = s.undo()
                    assert s.jpeg(95, 0, box=boxes[0]) == _pillow_of(s.image(), 95, 0, boxes[0]), (w, h, resize, k)
                assert s.jpeg(1, 2) == _pillow_of(s.image(), 1, 2)
            finally:
                proc.close()


@pytest.mark.gpu
def test_session_jpeg_checks_and_releases_memory(lib):
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo
    rs = np.random.RandomState(6)
    img = _photo(4000, 2667, rs)
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)
        warm.jpeg()
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        want = _pillow_of(img.convert("RGB"))
        assert s.jpeg() == want
        box = tuple(np.int64(v) for v in (5, 7, 1001, 667))         # numpy integers, as for quality
        assert s.jpeg(np.int64(90), np.int32(0), box=box) == _pillow_of(img.convert("RGB"), 90, 0, (5, 7, 1001, 667))
        for bad in [dict(quality=0), dict(quality=101), dict(subsampling=1), dict(quality=7.5), dict(box=(0, 0, 4001, 10)),
                    dict(box=(5, 5, 5, 10)), dict(box=(0, 0, 10)), dict(box=(False, 0, 10, 10)), dict(quality=True)]:
            with pytest.raises(ValueError):
                s.jpeg(**bad)
        s.close()
        assert allocated() == start
        with pytest.raises(RuntimeError, match="closed"):
            s.jpeg()
    finally:
        proc.close()

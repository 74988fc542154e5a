"""Progressive JPEG on the GPU: se_jpeg_encode_progressive_u8 (engine.jpeg_encode_u8(..., progressive=True)) writes Pillow's
``progressive=True`` bytes over sizes, qualities, both subsamplings and contents, at 4:2:0 sizes with dummy blocks, on a
4000x2667 photo and on content whose EOB runs are cut at 0x7FFF blocks and at the correction-bit limit; in mixed batches of
windows with odd pitches that overlap, past one call, with nothing written past each file, and each file equals its batch-1
encode; optimize makes no difference; files stay within their bound; EditSession.jpeg(progressive=True) is the Pillow
statement after edits and undos in both resize modes, and gives its transient device memory back."""
import gc
import io

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from tests import util_jpeg_progressive as P
from tests.test_gpu_jpeg_optimize import _sources
from tests.test_jpeg import CONTENTS, content
from tests.test_jpeg import SIZES as BASE_SIZES
from tests.test_jpeg_optimize import QUALITIES, SIZES
from tests.test_jpeg_progressive import EDGE_SIZES, corr_limit_image, pillow_jpeg_prog


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


@pytest.mark.gpu
@pytest.mark.parametrize("subsampling", [0, 2])
def test_kernels_are_pillow(lib, subsampling):
    """Every size, content and quality of the CPU matrices, the dummy-block sizes, plus a 4000x2667 photo; one call per
    (size, quality) batch."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8
    rs = np.random.RandomState(41 + subsampling)
    for hw in SIZES + BASE_SIZES + EDGE_SIZES + [(2667, 4000)]:
        imgs = [content(kind, *hw, rs) for kind in CONTENTS]
        dev = [torch.from_numpy(a).cuda() for a in imgs]
        for q in QUALITIES:
            got = jpeg_encode_u8(dev, q, subsampling, progressive=True)
            for kind, a, g in zip(CONTENTS, imgs, got):
                want = pillow_jpeg_prog(a, q, subsampling)
                assert g == want, (hw, kind, q, subsampling, len(g), len(want), PIL.__version__)


@pytest.mark.gpu
def test_run_limits_are_pillow(lib):
    """EOB runs cut at 0x7FFF blocks (a flat 1024x2048 image) and at the correction-bit limit (tests/test_jpeg_progressive.py),
    with 63 and with 8 correction bits per block, in one call with a photo between them."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8
    imgs = [np.full((1024, 2048, 3), (90, 120, 200), np.uint8), content("face_602_256x256.npz", 300, 200, np.random.RandomState(1)),
            corr_limit_image(), corr_limit_image(120, 640, 3), corr_limit_image(256, 1024, 5, ncoef=8)]
    for sub in (0, 2):
        for a in imgs[3:]:
            stats = {}
            P.encode(a, 100, sub, stats)
            assert stats["corr_limit"] > 0
        got = jpeg_encode_u8([torch.from_numpy(a).cuda() for a in imgs], 100, sub, progressive=True)
        for k, (a, g) in enumerate(zip(imgs, got)):
            assert g == pillow_jpeg_prog(a, 100, sub), (k, sub)


@pytest.mark.gpu
def test_mixed_batches_overlapping_windows_and_guard_bytes(lib):
    """40 windows (past one call's 32) of two sources with odd pitches, overlapping and repeated, at mixed sizes, into one
    buffer with odd gaps: each file is Pillow's crop-and-save with progressive=True and its own batch-1 encode, and every
    byte past a file is untouched."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed, jpeg_max_bytes
    sources, bufs, pitches, wins = _sources(np.random.RandomState(5))
    for sub, q in ((2, 75), (0, 90)):
        offs, pos = [], 3
        for s, b in wins:
            offs.append(pos)
            pos += jpeg_max_bytes(b[3] - b[1], b[2] - b[0], sub, progressive=True) + 5
        out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
        args = ([bufs[s] for s, _ in wins], [b[1] * pitches[s] + 3 * b[0] for s, b in wins], [pitches[s] for s, _ in wins],
                [(b[3] - b[1], b[2] - b[0]) for _, b in wins])
        _, _, nbytes = jpeg_encode_u8_packed(*args, quality=q, subsampling=sub, out=out, out_offsets=offs, progressive=True)
        got, lens = out.cpu().numpy(), nbytes.cpu().tolist()
        written = np.zeros(got.size, bool)
        for k, ((s, b), o, n) in enumerate(zip(wins, offs, lens)):
            want = pillow_jpeg_prog(np.ascontiguousarray(sources[s][b[1]:b[3], b[0]:b[2]]), q, sub)
            assert got[o:o + n].tobytes() == want, (b, sub, n, len(want))
            written[o:o + n] = True
            if k % 4 == 0:                                          # alone in its call
                one, _, nb1 = jpeg_encode_u8_packed(*(a[k:k + 1] for a in args), quality=q, subsampling=sub, progressive=True)
                assert one.cpu().numpy()[:int(nb1.cpu()[0])].tobytes() == want, (k, b)
        assert (got[~written] == 0xA5).all()
        for buf, a, p in zip(bufs, sources, pitches):              # the sources are only read
            h, w = a.shape[:2]
            assert (buf.cpu().numpy()[:h * p].reshape(h, p)[:, 3 * w:] == 0x5A).all()


@pytest.mark.gpu
def test_optimize_makes_no_difference_and_large_files(lib):
    """optimize=True and False give the same progressive file; files Pillow refuses (noise at quality 90, 4:4:4) are the ones
    it writes with a larger buffer; noise at quality 100, 4:4:4 stays within the bound."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8, jpeg_max_bytes
    rs = np.random.RandomState(8)
    a = content("places_11_512x408.npz", 301, 403, rs)
    t = torch.from_numpy(a).cuda()
    for sub in (0, 2):
        assert jpeg_encode_u8([t], 80, sub, optimize=True, progressive=True) == \
            jpeg_encode_u8([t], 80, sub, optimize=False, progressive=True)
    noise = rs.randint(0, 256, (300, 400, 3), dtype=np.uint8)
    with pytest.raises(OSError):
        Image.fromarray(noise).save(io.BytesIO(), "JPEG", quality=90, subsampling=0, progressive=True)
    assert jpeg_encode_u8([torch.from_numpy(noise).cuda()], 90, 0, progressive=True)[0] == pillow_jpeg_prog(noise, 90, 0)
    for h, w in ((64, 64), (200, 120), (517, 333)):
        n = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        g = jpeg_encode_u8([torch.from_numpy(n).cuda()], 100, 0, progressive=True)[0]
        assert g == pillow_jpeg_prog(n, 100, 0) and len(g) <= jpeg_max_bytes(h, w, 0, progressive=True)


def _pillow_of(img, quality=75, subsampling=2, box=None, buffer=True):
    """Pillow's progressive file of ``img`` (cropped to ``box``), with Pillow's buffer raised, or as Pillow saves it."""
    img = img if box is None else img.crop(box)
    if buffer:
        return pillow_jpeg_prog(np.asarray(img.convert("RGB")), quality, subsampling)
    buf = io.BytesIO()
    img.save(buf, "JPEG", quality=quality, subsampling=subsampling, progressive=True)
    return buf.getvalue()


def _check(s, resize, cur, quality=75, subsampling=2, box=None):
    want = _pillow_of(cur, quality, subsampling, box)
    if resize == "host":
        try:
            assert _pillow_of(cur, quality, subsampling, box, buffer=False) == want
        except OSError:
            with pytest.raises(OSError):
                s.jpeg(quality, subsampling, box=box, progressive=True)
            return
    assert s.jpeg(quality, subsampling, box=box, progressive=True) == want, (resize, quality, subsampling, box)


@pytest.mark.gpu
def test_session_jpeg_progressive_is_pillow_after_edits_and_undo(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model("bf16")
    rs = np.random.RandomState(33)
    for w, h in ((1000, 667), (4000, 2667)):
        img = _photo(w, h, rs)
        steps = _steps(w, h, rs)
        for resize in ("device", "host"):
            proc = DemoProcessor(model, max_batch=4, resize=resize, region_size=(256, 256))
            try:
                s = proc.open_session(img)
                _check(s, resize, s.image())
                for k, (mask, em, region, off) in enumerate(steps):
                    r = s.edit(mask, em, region=region, offset=off)
                    cur = s.image()
                    q, sub = (75, 2) if k % 2 == 0 else (90, 0)
                    _check(s, resize, cur, q, sub)
                    for b in r.boxes[:2]:
                        _check(s, resize, cur, box=b)
                boxes, _ = s.undo()
                _check(s, resize, s.image(), 95, 0, boxes[0])
                _check(s, resize, s.image())
                assert s.jpeg(optimize=True, progressive=True) == s.jpeg(progressive=True)
            finally:
                proc.close()


@pytest.mark.gpu
def test_session_jpeg_progressive_checks_and_releases_memory(lib):
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo
    img = _photo(4000, 2667, np.random.RandomState(7))
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)
        warm.jpeg(progressive=True)
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        assert s.jpeg(progressive=True) == _pillow_of(img.convert("RGB"))
        assert s.jpeg(90, 0, box=(5, 7, 1001, 667), progressive=np.bool_(True)) == _pillow_of(img.convert("RGB"), 90, 0,
                                                                                            (5, 7, 1001, 667))
        for bad in (1, 0, "yes", None):
            with pytest.raises(ValueError, match="progressive must be a bool"):
                s.jpeg(progressive=bad)
        s.close()
        assert allocated() == start
    finally:
        proc.close()

"""JPEG with optimal Huffman tables on the GPU: se_jpeg_encode_opt_u8 with optimize = 1 (engine.jpeg_encode_u8(...,
optimize=True)) writes Pillow's ``optimize=True`` bytes over sizes, qualities, both subsamplings and contents, in mixed
batches of windows with odd pitches that overlap, past one call, with nothing written past each file, and each file equals
its batch-1 encode; optimize = 0 is se_jpeg_encode_u8 byte for byte; EditSession.jpeg(optimize=True) is the Pillow statement
after edits and undos, and gives its transient device memory back."""
import ctypes
import gc
import io

import numpy as np
import PIL
import pytest

from sketchedit_b200 import _lib, build
from tests import util_jpeg as J
from tests.test_jpeg import CONTENTS, content
from tests.test_jpeg_optimize import QUALITIES, SIZES, pillow_jpeg_opt


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
    rs = np.random.RandomState(31 + subsampling)
    for hw in SIZES + [(2667, 4000)]:
        imgs = [content(kind, *hw, rs) for kind in CONTENTS]
        dev = [torch.from_numpy(a).cuda() for a in imgs]
        for q in QUALITIES:
            got = jpeg_encode_u8(dev, q, subsampling, optimize=True)
            for kind, a, g in zip(CONTENTS, imgs, got):
                want = pillow_jpeg_opt(a, q, subsampling)
                assert g == want, (hw, kind, q, subsampling, len(g), len(want), PIL.__version__)


def _sources(rs):
    import torch
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
    return sources, bufs, pitches, wins


@pytest.mark.gpu
def test_mixed_batches_overlapping_windows_and_guard_bytes(lib):
    """40 windows (past one call's 32) of two sources with odd pitches, overlapping and repeated, at mixed sizes, into one
    buffer with odd gaps: each file is Pillow's crop-and-save with optimize=True and its own batch-1 encode, and every byte
    past a file is untouched."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed
    sources, bufs, pitches, wins = _sources(np.random.RandomState(3))
    for sub, q in ((2, 75), (0, 90)):
        offs, pos = [], 3
        for s, b in wins:
            offs.append(pos)
            pos += J.max_bytes(b[3] - b[1], b[2] - b[0], sub) + 5
        out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
        args = ([bufs[s] for s, _ in wins], [b[1] * pitches[s] + 3 * b[0] for s, b in wins], [pitches[s] for s, _ in wins],
                [(b[3] - b[1], b[2] - b[0]) for _, b in wins])
        _, _, nbytes = jpeg_encode_u8_packed(*args, quality=q, subsampling=sub, out=out, out_offsets=offs, optimize=True)
        got, lens = out.cpu().numpy(), nbytes.cpu().tolist()
        written = np.zeros(got.size, bool)
        for k, ((s, b), o, n) in enumerate(zip(wins, offs, lens)):
            want = pillow_jpeg_opt(np.ascontiguousarray(sources[s][b[1]:b[3], b[0]:b[2]]), q, sub)
            assert got[o:o + n].tobytes() == want, (b, sub, n, len(want))
            written[o:o + n] = True
            if k % 4 == 0:                                          # alone in its call
                one, _, nb1 = jpeg_encode_u8_packed(*(a[k:k + 1] for a in args), quality=q, subsampling=sub, optimize=True)
                assert one.cpu().numpy()[:int(nb1.cpu()[0])].tobytes() == want, (k, b)
        assert (got[~written] == 0xA5).all()
        for buf, a, p in zip(bufs, sources, pitches):              # the sources are only read
            h, w = a.shape[:2]
            assert (buf.cpu().numpy()[:h * p].reshape(h, p)[:, 3 * w:] == 0x5A).all()


@pytest.mark.gpu
def test_optimize_0_is_se_jpeg_encode_u8(lib):
    """The new entry with optimize = 0 writes what se_jpeg_encode_u8 writes, on 32 of those windows in one call."""
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8_packed
    sources, bufs, pitches, wins = _sources(np.random.RandomState(4))
    ptrs = [bufs[s].data_ptr() + b[1] * pitches[s] + 3 * b[0] for s, b in wins][:32]
    hw = [v for _, b in wins[:32] for v in (b[3] - b[1], b[2] - b[0])]
    offs = list(np.cumsum([0] + [J.max_bytes(hw[2 * i], hw[2 * i + 1], 2) for i in range(32)])[:-1])
    n = len(ptrs)
    a_src, a_p = (ctypes.c_void_p * n)(*ptrs), (ctypes.c_longlong * n)(*[pitches[s] for s, _ in wins[:32]])
    a_hw, a_o = (ctypes.c_int * (2 * n))(*hw), (ctypes.c_longlong * n)(*[int(o) for o in offs])
    need = ctypes.c_longlong(0)
    assert lib.se_jpeg_encode_u8(a_src, a_p, a_hw, n, 80, 2, None, a_o, None, None, ctypes.byref(need), None) == 0
    scratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    out = torch.zeros(int(offs[-1]) + J.max_bytes(hw[-2], hw[-1], 2), dtype=torch.uint8, device="cuda")
    nb = torch.zeros(n, dtype=torch.int64, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.se_jpeg_encode_u8(a_src, a_p, a_hw, n, 80, 2, ctypes.c_void_p(out.data_ptr()), a_o, ctypes.c_void_p(nb.data_ptr()),
                                 ctypes.c_void_p(scratch.data_ptr()), ctypes.byref(need), stream) == 0
    got, _, nb2 = jpeg_encode_u8_packed([bufs[s] for s, _ in wins[:32]], [b[1] * pitches[s] + 3 * b[0] for s, b in wins[:32]],
                                        [pitches[s] for s, _ in wins[:32]], [(hw[2 * i], hw[2 * i + 1]) for i in range(n)],
                                        quality=80, subsampling=2, out=torch.zeros_like(out), out_offsets=[int(o) for o in offs],
                                        optimize=False)
    assert torch.equal(nb, nb2)
    for o, k in zip(offs, nb.cpu().tolist()):
        assert torch.equal(out[int(o):int(o) + k], got[int(o):int(o) + k])


@pytest.mark.gpu
def test_strided_views_are_encoded_where_they_lie(lib):
    import torch

    from sketchedit_b200.engine import jpeg_encode_u8
    rs = np.random.RandomState(9)
    a = content("face_602_256x256.npz", 300, 401, rs)
    t = torch.from_numpy(a).cuda()
    boxes = [(0, 0, 401, 300), (17, 3, 250, 77), (400, 0, 401, 300), (0, 299, 401, 300), (100, 100, 116, 116)]
    got = jpeg_encode_u8([t[b[1]:b[3], b[0]:b[2]] for b in boxes], optimize=True)
    for b, g in zip(boxes, got):
        assert g == pillow_jpeg_opt(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2]])), b


def _pillow_of(img, quality=75, subsampling=2, box=None, buffer=True):
    """Pillow's optimize=True file of ``img`` (cropped to ``box``); with ``buffer`` Pillow's output buffer is raised so that
    it can write files larger than max(64 KiB, w h) bytes (tests/test_jpeg_optimize.py, pillow_jpeg_opt)."""
    img = img if box is None else img.crop(box)
    if buffer:
        return pillow_jpeg_opt(np.asarray(img.convert("RGB")), quality, subsampling)
    buf = io.BytesIO()
    img.save(buf, "JPEG", quality=quality, subsampling=subsampling, optimize=True)
    return buf.getvalue()


def _check(s, resize, cur, quality=75, subsampling=2, box=None):
    """The device writes the statement's file; the host flow is Pillow's save as it stands, which raises OSError where the
    file does not fit Pillow's buffer."""
    want = _pillow_of(cur, quality, subsampling, box)
    if resize == "host":
        try:
            assert _pillow_of(cur, quality, subsampling, box, buffer=False) == want
        except OSError:
            with pytest.raises(OSError):
                s.jpeg(quality, subsampling, box=box, optimize=True)
            return
    assert s.jpeg(quality, subsampling, box=box, optimize=True) == want, (resize, quality, subsampling, box)


@pytest.mark.gpu
def test_session_jpeg_optimize_is_pillow_after_edits_and_undo(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model("bf16")
    rs = np.random.RandomState(29)
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
                assert s.jpeg(optimize=False) == s.jpeg()
            finally:
                proc.close()


@pytest.mark.gpu
def test_session_jpeg_optimize_checks_and_releases_memory(lib):
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo
    img = _photo(4000, 2667, np.random.RandomState(6))
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)
        warm.jpeg(optimize=True)
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        assert s.jpeg(optimize=True) == _pillow_of(img.convert("RGB"))
        assert s.jpeg(90, 0, box=(5, 7, 1001, 667), optimize=np.bool_(True)) == _pillow_of(img.convert("RGB"), 90, 0,
                                                                                        (5, 7, 1001, 667))
        for bad in (1, 0, "yes", None):
            with pytest.raises(ValueError, match="optimize must be a bool"):
                s.jpeg(optimize=bad)
        s.close()
        assert allocated() == start
    finally:
        proc.close()

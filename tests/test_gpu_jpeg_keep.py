"""JPEG files in the upload's own format on the GPU: se_jpeg_encode_tables_u8 (engine.jpeg_encode_tables_u8) writes Pillow's
bytes for per-call tables, 4:2:2 and APP1 / APP2 segments at each coding, over the CPU matrix and a 4000x2667 photo, in mixed
calls and on strided windows with the bytes around each file untouched; an edit session opened from a JPEG upload gives back
jpeg(quality="keep", exif=s.exif, icc_profile=s.icc_profile) as Pillow's statement in both resize modes, and its memory."""
import gc
import io

import numpy as np
import pytest
from PIL import Image, JpegImagePlugin

from sketchedit_b200 import _lib, build
from tests.test_jpeg import content
from tests.test_jpeg_keep import (CODING_IDS, CODINGS, SIZES_422, UPLOAD_QUALITIES, exif_orientation_6, icc_srgb, keep_statement,
                                  pillow, upload)


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("coding", CODINGS, ids=CODING_IDS)
def test_kernels_are_pillow(lib, coding):
    """4:2:2 sizes (every width mod 16), Pillow-saved uploads at each quality and sampling and a grayscale one, hand-made
    tables, metadata, and a 4000x2667 photo at 4:2:2."""
    from sketchedit_b200.engine import jpeg_encode_tables_u8
    rs = np.random.RandomState(11)
    qt = [list(rs.randint(1, 256, 64)) for _ in range(2)]
    sizes = SIZES_422 + [(w, h) for h in (8, 9) for w in range(1, 33)] + [(4000, 2667)]
    for w, h in sizes:
        imgs = [content(k, h, w, rs) for k in ("noise", "places_11_512x408.npz")]
        got = jpeg_encode_tables_u8([_dev(a) for a in imgs], qt, 1, **coding)
        for a, g in zip(imgs, got):
            assert g == pillow(a, qtables=qt, subsampling=1, **coding), (w, h)
    a = content("places_11_512x408.npz", 57, 83, rs)
    srcs = [upload(a, q, s) for q in UPLOAD_QUALITIES for s in (0, 1, 2)]
    srcs.append(Image.open(io.BytesIO(pillow(Image.fromarray(a).convert("L"), quality=80))))
    for src in srcs:
        sampling = JpegImagePlugin.get_sampling(src)
        assert jpeg_encode_tables_u8([_dev(a)], src.quantization, sampling, **coding)[0] == keep_statement(a, src, **coding)
    b = content("noise", 21, 37, rs)
    for n in (1, 2, 3, 4):
        for tabs in ([[1] * 64] * n, [[255] * 64] * n, [[0] + list(rs.randint(1, 256, 63)) for _ in range(n)]):
            for s in (0, 1, 2):
                assert jpeg_encode_tables_u8([_dev(b)], tabs, s, **coding)[0] == pillow(b, qtables=tabs, subsampling=s, **coding)
    metas = [dict(exif=b"abc"), dict(exif=bytes(65533)), dict(exif=exif_orientation_6()), dict(icc_profile=bytes(588)),
             dict(icc_profile=bytes(rs.randint(0, 256, 3 * 65519 + 7).astype(np.uint8))),
             dict(exif=exif_orientation_6(), icc_profile=bytes(65520))]
    for meta in metas:
        assert jpeg_encode_tables_u8([_dev(b)], qt, 1, **meta, **coding)[0] == pillow(b, qtables=qt, subsampling=1, **meta, **coding)


@pytest.mark.gpu
def test_mixed_sizes_and_samplings_strided_windows_and_guard_bytes(lib):
    """One photo's strided windows, 40 of them (past one call's 32), at each sampling: each file is Pillow's, written where
    it lies, with every byte around the files untouched; the source is only read."""
    import torch

    from sketchedit_b200 import engine
    rs = np.random.RandomState(12)
    a = content("places_11_512x408.npz", 301, 403, rs)
    a[150:, 200:] = rs.randint(0, 256, (151, 203, 3))
    buf = torch.full((301, 403 * 3 + 7), 0x5A, dtype=torch.uint8, device="cuda")
    buf[:, :403 * 3] = _dev(a.reshape(301, -1))
    photo = buf[:, :403 * 3].view(301, 403, 3)
    boxes = [(0, 0, 403, 301), (400, 298, 403, 301), (5, 7, 6, 8)]
    for _ in range(37):
        bh, bw = int(rs.randint(1, 302)), int(rs.randint(1, 404))
        y, x = int(rs.randint(0, 302 - bh)), int(rs.randint(0, 404 - bw))
        boxes.append((x, y, x + bw, y + bh))
    exif, icc = exif_orientation_6().tobytes(), icc_srgb()   # (a new profile carries a new creation time)
    seg = engine.jpeg_app_segments(exif, icc)
    for sub, coding in ((1, dict()), (0, dict(optimize=True)), (2, dict(progressive=True)), (1, dict(progressive=True))):
        qt = [list(rs.randint(1, 256, 64)) for _ in range(3)]
        got = engine.jpeg_encode_tables_u8([photo[b[1]:b[3], b[0]:b[2]] for b in boxes], qt, sub, exif=exif, icc_profile=icc,
                                           **coding)
        for b, g in zip(boxes, got):
            want = pillow(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2]]), qtables=qt, subsampling=sub, exif=exif, icc_profile=icc,
                          **coding)
            assert g == want, (b, sub, coding)
    assert (buf[:, 403 * 3:] == 0x5A).all()
    # the packed form with guard bytes: the files' slots at odd offsets in one buffer, each its bound apart
    lib_ = _lib.load()
    import ctypes
    sizes = [(b[3] - b[1], b[2] - b[0]) for b in boxes[:5]]
    offs, pos = [], 3
    for h, w in sizes:
        offs.append(pos)
        pos += engine.jpeg_tables_max_bytes(h, w, 1, 2, False, len(seg)) + 5
    out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
    nbytes = torch.empty(len(sizes), dtype=torch.int64, device="cuda")
    qt = [list(rs.randint(1, 256, 64)) for _ in range(2)]
    tabs = (ctypes.c_ushort * 128)(*[v for t in qt for v in t])
    segbuf = (ctypes.c_ubyte * len(seg)).from_buffer_copy(seg)
    ptrs = (ctypes.c_void_p * len(sizes))(*[photo[b[1]:b[3], b[0]:b[2]].data_ptr() for b in boxes[:5]])
    pitches = (ctypes.c_longlong * len(sizes))(*[photo.stride(0)] * len(sizes))
    hw = (ctypes.c_int * (2 * len(sizes)))(*[v for s in sizes for v in s])
    off = (ctypes.c_longlong * len(sizes))(*offs)
    need = ctypes.c_longlong(0)
    args = (ptrs, pitches, hw, len(sizes), tabs, 2, 1, 0, 0, segbuf, len(seg), ctypes.c_void_p(out.data_ptr()), off,
            ctypes.c_void_p(nbytes.data_ptr()))
    _lib.check(lib_.se_jpeg_encode_tables_u8(*args, None, ctypes.byref(need), None))
    scratch = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib_.se_jpeg_encode_tables_u8(*args, ctypes.c_void_p(scratch.data_ptr()), ctypes.byref(need),
                                             ctypes.c_void_p(stream)))
    host, lens = out.cpu().numpy(), nbytes.cpu().tolist()
    written = np.zeros(host.size, bool)
    for b, o, n in zip(boxes[:5], offs, lens):
        want = pillow(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2]]), qtables=qt, subsampling=1, exif=exif, icc_profile=icc)
        assert host[o:o + n].tobytes() == want, b
        written[o:o + n] = True
    assert (host[~written] == 0xA5).all()


def _statement(img, src, box=None, size=None, **kw):
    img = img if box is None else img.crop(box)
    if size is not None:
        img = img.copy()
        img.thumbnail(size)
    return keep_statement(img, src, **kw)


@pytest.mark.gpu
def test_session_keeps_the_upload_after_edits_and_undo(lib):
    """Sessions opened from JPEG uploads with EXIF and ICC ((92, 4:2:2), (95, 4:2:0), (85, 4:4:4) and grayscale), in both
    resize modes: after edits and undo, keep with box, size, optimize and progressive is the statement, s.jpeg() is still
    today's file, and the device memory comes back."""
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model("bf16")
    rs = np.random.RandomState(31)
    w, h = 1000, 667
    photo = _photo(w, h, rs)
    exif, icc = exif_orientation_6().tobytes(), icc_srgb()
    srcs = [upload(np.asarray(photo), q, s, exif=exif, icc_profile=icc) for q, s in ((92, 1), (95, 2), (85, 0))]
    srcs.append(Image.open(io.BytesIO(pillow(photo.convert("L"), quality=90, exif=exif, icc_profile=icc))))
    steps = _steps(w, h, rs)[:3]

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    for resize in ("device", "host"):
        proc = DemoProcessor(model, max_batch=4, resize=resize, region_size=(256, 256))
        try:
            warm = proc.open_session(srcs[0])
            warm.jpeg(quality="keep", exif=warm.exif, icc_profile=warm.icc_profile, progressive=True)
            warm.close()
            start = allocated()
            for src in srcs:
                s = proc.open_session(src)
                assert s.exif == exif and s.icc_profile == icc
                meta = dict(exif=s.exif, icc_profile=s.icc_profile)
                for k, (mask, em, region, off) in enumerate(steps):
                    r = s.edit(mask, em, region=region, offset=off)
                    cur = s.image()
                    b = r.boxes[0]
                    assert s.jpeg(quality="keep", **meta) == _statement(cur, src, **meta), (resize, src.mode, k)
                    assert s.jpeg(quality="keep", box=b, optimize=True, **meta) == _statement(cur, src, b, optimize=True, **meta)
                    assert s.jpeg(quality="keep", size=(320, 320), progressive=True, **meta) == \
                        _statement(cur, src, size=(320, 320), progressive=True, **meta)
                    assert s.jpeg() == pillow(cur, quality=75, subsampling=2)
                s.undo()
                cur = s.image()
                assert s.jpeg(quality="keep", box=(3, 5, 701, 400), size=(200, 100), **meta) == \
                    _statement(cur, src, (3, 5, 701, 400), (200, 100), **meta)
                assert s.jpeg(90, 0, **meta) == pillow(cur, quality=90, subsampling=0, **meta)
                assert s.jpeg(quality="keep") == _statement(cur, src)
                s.close()
            if resize == "device":
                assert allocated() == start
        finally:
            proc.close()

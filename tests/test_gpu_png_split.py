"""Large PNG files across the whole GPU: se_png_split_u8 (through engine.png_decode_u8_packed / png_decode_u8) gives Pillow's
pixels over the corpus of tests/util_png_decode.py cut into chunks of a few bytes, and at its default chunk spacing on large
files (4000x2667 photos saved by Pillow and by cv2, a flat 2048x2048 screenshot, every colour type and depth, 1xN and Nx1),
with the bytes around each output untouched; edit sessions opened from upload bytes equal sessions opened from Pillow
images, with the photo decoded on the device."""
import io

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build, pngfile
from tests import util_png_decode as U

INF_LINK = 12


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def pillow(f, mode):
    try:
        return np.asarray(Image.open(io.BytesIO(f)).convert(mode))
    except Exception as e:   # noqa: BLE001  (Pillow's exception is the expected result)
        return e


def _decode(files, modes, split, monkeypatch, chunk=None):
    """(pixels per file as numpy, status list) of one png_decode_u8_packed call over the files, all through the split
    decoder (chunks of `chunk` bytes, or the default spacing) or all through the one-warp decoder, into one buffer at odd
    offsets checked for guard bytes."""
    import torch

    from sketchedit_b200 import engine as E
    monkeypatch.setattr(E, "PNG_SPLIT_MIN_RAW", 0 if split else 1 << 62)
    if chunk is not None:
        monkeypatch.setattr(E, "PNG_SPLIT_MIN_CHUNK", chunk)
    heads = [pngfile.parse(f) for f in files]
    staging, offs, lens = E.png_stage(heads)
    sizes = [hd.h * hd.w * pngfile.MODES[m] for hd, m in zip(heads, modes)]
    out_offs, at = [], 3
    for s in sizes:
        out_offs.append(at)
        at += s + 5
    out = torch.full((at + 11,), 0xA5, dtype=torch.uint8, device="cuda")
    _, _, status = E.png_decode_u8_packed(staging.cuda(), offs, lens, heads, modes, out=out, out_offsets=out_offs)
    host = out.cpu().numpy()
    inside = np.zeros(host.size, bool)
    for o, s in zip(out_offs, sizes):
        inside[o:o + s] = True
    assert (host[~inside] == 0xA5).all()
    px = [host[o:o + s] for o, s in zip(out_offs, sizes)]
    return px, status.cpu().tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 5, 64, 4096])
def test_corpus_in_small_chunks(lib, monkeypatch, chunk):
    """Every corpus file and every malformed one through the split decoder cut every `chunk` bytes: status 0 gives Pillow's
    pixels, and is 0 wherever the one-warp decoder's is, apart from files the link rule refuses (named below)."""
    from sketchedit_b200 import engine as E
    named = U.corpus() + U.malformed()
    files = [f for _, f in named]
    modes = ["RGB" if k % 3 else "L" for k in range(len(files))]
    warp_px, warp_st = _decode(files, modes, False, monkeypatch)
    px, st = _decode(files, modes, True, monkeypatch, chunk)
    refused = []
    for (name, f), m, p, s, wp, ws in zip(named, modes, px, st, warp_px, warp_st):
        want = pillow(f, m)
        if s == 0:
            assert not isinstance(want, Exception) and np.array_equal(p, want.reshape(-1)), (name, chunk)
        elif ws == 0:
            assert s == INF_LINK, (name, chunk, s)
            refused.append(name)
        if ws == 0:
            assert np.array_equal(wp, want.reshape(-1)), name
    print("chunk %d: %d of %d files refused by the link rule: %s" % (chunk, len(refused), len(files), refused))
    assert len(refused) <= len(files) // 20
    assert all(s != 0 for s in st[len(files) - len(U.malformed()):])
    # through the wrapper with the fallback: always Pillow's
    monkeypatch.setattr(E, "PNG_SPLIT_MIN_RAW", 0)
    got = E.png_decode_u8([f for f in files if not isinstance(pillow(f, "RGB"), Exception)], "RGB")
    for g, f in zip(got, [f for f in files if not isinstance(pillow(f, "RGB"), Exception)]):
        assert np.array_equal(g.cpu().numpy(), pillow(f, "RGB"))


def _flat(h, w):
    """A screenshot-like image: flat panels, a few lines and some text-like noise."""
    a = np.full((h, w, 3), 240, np.uint8)
    a[: h // 12] = (40, 60, 90)
    a[h // 3: h // 2, w // 5: w // 2] = (255, 255, 255)
    a[::97] = 0
    rs = np.random.RandomState(4)
    for y in range(h // 10, h, h // 9):
        a[y:y + 12, 40:40 + w // 3] = rs.randint(0, 2, (12, w // 3, 1)) * 200
    return a


def large_files():
    import cv2
    rng = np.random.default_rng(21)
    ph = U.photo(2667, 4000, 9)
    out = [("pil_4000x2667", U.pil_png(ph)), ("cv2_4000x2667", cv2.imencode(".png", ph[..., ::-1])[1].tobytes()),
           ("flat_2048x2048", U.pil_png(_flat(2048, 2048)))]
    out.append(("rgba_1500x1200", U.pil_png(np.dstack([U.photo(1200, 1500, 3), rng.integers(0, 256, (1200, 1500, 1),
                                                                                              dtype=np.uint8)]))))
    out.append(("grey8_2000x1800", U.pil_png(U.photo(1800, 2000, 4)[..., 1])))
    for depth in (1, 2, 4, 8):
        v = (U.photo(1100, 1300, depth)[..., :1].astype(np.int32) >> (8 - depth))
        out.append(("grey%d_1300x1100" % depth, U.make_png(v, depth, 0, ftypes=(0, 1, 2, 3, 4), level=6)))
        out.append(("pal%d_1300x1100" % depth, U.make_png(v, depth, 3, palette=rng.integers(0, 256, (1 << depth, 3)),
                                                         level=6)))
    out.append(("row_1x65535", U.pil_png(U.photo(1, 65535, 5))))
    out.append(("column_65535x1", U.pil_png(U.photo(65535, 1, 6))))
    return out


@pytest.mark.gpu
def test_large_files_at_the_default_spacing(lib, monkeypatch):
    from sketchedit_b200 import engine as E
    named = large_files()
    for mode in ("RGB", "L"):
        files = [f for _, f in named]
        px, st = _decode(files, [mode] * len(files), True, monkeypatch)
        for (name, f), p, s in zip(named, px, st):
            assert s == 0, (name, mode, s, E.png_split_chunk_bytes(len(pngfile.parse(f).stream)))
            assert np.array_equal(p, pillow(f, mode).reshape(-1)), (name, mode)


def _gpu_proc():
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    return DemoProcessor(_model("bf16"), max_batch=4, resize="device", region_size=(256, 256))


@pytest.mark.gpu
@pytest.mark.parametrize("force_split", [False, True])
def test_session_from_bytes_is_session_from_pillow(lib, monkeypatch, force_split):
    """Device sessions opened from upload bytes (PNG: on the device when it is at least PNG_SPLIT_MIN_RAW, here forced, else
    by Pillow; a PNG the parser sends to Pillow; JPEG) equal sessions opened from Image.open of the same bytes after edits and undo, in image(), png() and
    jpeg(); garbage bytes and a PNG whose stream is damaged raise Pillow's exception."""
    import torch

    from sketchedit_b200 import engine as E
    from tests.test_gpu_edit_session import _photo, _steps
    if force_split:
        monkeypatch.setattr(E, "PNG_SPLIT_MIN_RAW", 0)
    rs = np.random.RandomState(7)
    w, h = 640, 427
    photo = np.asarray(_photo(w, h, rs))
    jpeg = io.BytesIO()
    Image.fromarray(photo).save(jpeg, "JPEG", quality=88)
    icc = io.BytesIO()
    Image.fromarray(photo).save(icc, "PNG", icc_profile=b"\0" * 200)
    uploads = {"png": U.pil_png(photo), "png_cv2": U.make_png(photo, 8, 2, level=9), "png_icc": icc.getvalue(),
               "png_grey": U.pil_png(photo[..., 0]), "jpeg": jpeg.getvalue()}
    calls = []
    decode_into = E.png_decode_into
    monkeypatch.setattr(E, "png_decode_into", lambda *a, **k: calls.append(1) or decode_into(*a, **k))
    steps = _steps(w, h, rs)[:2]
    proc = _gpu_proc()
    try:
        for name, data in uploads.items():
            calls.clear()
            a = proc.open_session(memoryview(data) if name == "png_grey" else data)
            on_device = force_split and name.startswith("png") and name != "png_icc"   # small files: Pillow is faster
            assert len(calls) == on_device, name
            b = proc.open_session(Image.open(io.BytesIO(data)))
            assert (a.size, a.exif, a.icc_profile) == (b.size, b.exif, b.icc_profile), name
            assert a.image().tobytes() == b.image().tobytes(), name
            for mask, em, region, off in steps:
                ra, rb = a.edit(mask, em, region=region, offset=off), b.edit(mask, em, region=region, offset=off)
                assert ra.boxes == rb.boxes and a.image().tobytes() == b.image().tobytes(), name
                assert a.png() == b.png() and a.jpeg(85) == b.jpeg(85), name
            if name == "jpeg":
                assert a.jpeg(quality="keep") == b.jpeg(quality="keep")
            else:
                with pytest.raises(ValueError, match="not a JPEG"):
                    a.jpeg(quality="keep")
            a.undo()
            b.undo()
            assert a.image().tobytes() == b.image().tobytes(), name
            a.close()
            b.close()
        # the device refuses a damaged stream; Pillow's exception comes out
        good = U.pil_png(photo[:40, :50])
        hd = pngfile.parse(good)
        bad = U.make_png(photo[:40, :50], 8, 2, stream=lambda r: hd.stream[:len(hd.stream) // 2])
        for data in (bad, b"\x89PNG\r\n\x1a\n" + bytes(30), b"not an image"):
            want = pillow(data, "RGB")
            assert isinstance(want, Exception)
            with pytest.raises(type(want)):
                proc.open_session(data)
        torch.cuda.synchronize()
    finally:
        proc.close()

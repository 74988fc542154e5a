"""JPEG files in the upload's own format, on the CPU: tests/util_jpeg_keep.py (per-call quantisation tables, 4:2:2, APP1 /
APP2 segments) is byte for byte Pillow 12.2 at each coding (baseline, optimize, progressive) over 4:2:2 sizes, Pillow-saved
uploads, hand-made tables and metadata; se_jpeg_tables_max_bytes bounds it; se_jpeg_encode_tables_u8 checks its arguments
on the host; and a resize='host' session's jpeg(quality="keep", exif=..., icc_profile=...) is the Pillow statement."""
import ctypes
import io

import numpy as np
import pytest
from PIL import Image, ImageCms, JpegImagePlugin

from sketchedit_b200 import _lib, build
from sketchedit_b200.engine import jpeg_app_segments, jpeg_quality_tables
from tests import util_jpeg_keep as K
from tests.test_jpeg import content

CODINGS = [dict(), dict(optimize=True), dict(progressive=True)]
CODING_IDS = ["baseline", "optimize", "progressive"]
SIZES_422 = [(1, 1), (9, 7), (16, 8), (17, 9), (33, 15), (31, 16), (23, 17), (641, 481)]   # (w, h)
UPLOAD_QUALITIES = [1, 10, 50, 75, 92, 95, 100]


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def pillow(img, **kw):
    buf = io.BytesIO()
    (img if isinstance(img, Image.Image) else Image.fromarray(img)).save(buf, "JPEG", **kw)
    return buf.getvalue()


def upload(rgb, quality, subsampling, **kw):
    """A Pillow-saved JPEG upload, opened as a user's would be."""
    return Image.open(io.BytesIO(pillow(rgb, quality=quality, subsampling=subsampling, **kw)))


def keep_statement(img, src, **kw):
    """The explicit form of ``src.save(quality="keep", ...)`` for the pixels of ``img``."""
    return pillow(img, qtables=src.quantization, subsampling=JpegImagePlugin.get_sampling(src), **kw)


def icc_srgb():
    return ImageCms.ImageCmsProfile(ImageCms.createProfile("sRGB")).tobytes()


def exif_orientation_6():
    e = Image.Exif()
    e[0x0112] = 6
    return e


@pytest.mark.parametrize("coding", CODINGS, ids=CODING_IDS)
def test_422_sizes_are_pillow(coding):
    """Every width 1..32 at heights 8 and 9 (each width mod 16: the MCU's second luma block real and a dummy) and the
    edge sizes, noise and a photo."""
    rs = np.random.RandomState(1)
    qt = [list(rs.randint(1, 256, 64)) for _ in range(2)]
    sizes = SIZES_422 + [(w, h) for h in (8, 9) for w in range(1, 33)]
    for w, h in sizes:
        for kind in ("noise", "places_11_512x408.npz"):
            a = content(kind, h, w, rs)
            assert K.encode(a, qt, 1, **coding) == pillow(a, qtables=qt, subsampling=1, **coding), (w, h, kind)


@pytest.mark.parametrize("coding", CODINGS, ids=CODING_IDS)
def test_uploads_are_kept_as_pillow_keeps_them(coding):
    """Pillow-saved uploads at each quality and sampling, and a grayscale one: the restatement with the upload's tables and
    sampling is Pillow's explicit statement, which is Pillow's own quality="keep"."""
    rs = np.random.RandomState(2)
    a = content("places_11_512x408.npz", 57, 83, rs)
    srcs = [upload(a, q, s) for q in UPLOAD_QUALITIES for s in (0, 1, 2)]
    srcs.append(Image.open(io.BytesIO(pillow(Image.fromarray(a).convert("L"), quality=80))))
    for src in srcs:
        want = keep_statement(a, src, **coding)
        if src.mode == "RGB":   # (Pillow keeps a grayscale upload grayscale; the session's photo is RGB)
            assert pillow(src, quality="keep", subsampling=0, **coding) == keep_statement(src, src, **coding)
        got = K.encode(a, src.quantization, JpegImagePlugin.get_sampling(src), **coding)
        assert got == want, (src.mode, JpegImagePlugin.get_sampling(src), len(src.quantization))
    assert JpegImagePlugin.get_sampling(srcs[-1]) == -1 and len(srcs[-1].quantization) == 1


@pytest.mark.parametrize("coding", CODINGS, ids=CODING_IDS)
def test_hand_made_tables_are_pillow(coding):
    """1 to 4 tables, entries all 1, all 255, one 0 (taken as 1) and random in 1..255, at each sampling."""
    rs = np.random.RandomState(3)
    a = content("noise", 21, 37, rs)
    kinds = {"ones": lambda: [1] * 64, "max": lambda: [255] * 64, "zero": lambda: [0] + list(rs.randint(1, 256, 63)),
             "random": lambda: list(rs.randint(1, 256, 64))}
    for n in (1, 2, 3, 4):
        for name, make in kinds.items():
            qt = [make() for _ in range(n)]
            for s in (0, 1, 2):
                assert K.encode(a, qt, s, **coding) == pillow(a, qtables=qt, subsampling=s, **coding), (n, name, s)


def test_quality_tables_are_the_quality_files():
    """save(quality=q) is save(qtables=jpeg_quality_tables(q)) for every quality, with metadata, at 4:4:4 and 4:2:0."""
    rs = np.random.RandomState(4)
    a = content("places_11_512x408.npz", 19, 26, rs)
    for q in range(1, 101):
        for s in (0, 2):
            want = pillow(a, quality=q, subsampling=s, exif=b"Exif\0\0x")
            assert pillow(a, qtables=jpeg_quality_tables(q), subsampling=s, exif=b"Exif\0\0x") == want, (q, s)
            assert K.encode(a, jpeg_quality_tables(q), s, segments=jpeg_app_segments(b"Exif\0\0x")) == want, (q, s)


@pytest.mark.parametrize("coding", CODINGS, ids=CODING_IDS)
def test_metadata_segments_are_pillow(coding):
    """EXIF of 0, 3 and 65533 bytes and an Image.Exif; ICC of 0 and 588 bytes (sRGB) and 65519, 65520 and 3 * 65519 + 7
    bytes (one, two and four APP2 segments); both together."""
    rs = np.random.RandomState(5)
    a = content("noise", 9, 17, rs)
    qt = [list(rs.randint(1, 256, 64)) for _ in range(2)]
    srgb = icc_srgb()
    assert len(srgb) == 588
    cases = [dict(exif=b""), dict(exif=b"abc"), dict(exif=bytes(rs.randint(0, 256, 65533).astype(np.uint8))),
             dict(exif=exif_orientation_6()), dict(icc_profile=b""), dict(icc_profile=srgb)]
    cases += [dict(icc_profile=bytes(rs.randint(0, 256, n).astype(np.uint8))) for n in (65519, 65520, 3 * 65519 + 7)]
    cases.append(dict(exif=exif_orientation_6(), icc_profile=srgb))
    for meta in cases:
        want = pillow(a, qtables=qt, subsampling=1, **meta, **coding)
        seg = jpeg_app_segments(**meta)
        assert K.encode(a, qt, 1, segments=seg, **coding) == want, {k: len(v) if v is not None and not isinstance(v, Image.Exif) else v
                                                                     for k, v in meta.items()}
    n = len(jpeg_app_segments(icc_profile=bytes(3 * 65519 + 7)))
    assert n == 3 * (4 + 14 + 65519) + (4 + 14 + 7)   # four APP2 segments
    with pytest.raises(ValueError, match="EXIF data is too long"):
        pillow(a, exif=bytes(65534))
    with pytest.raises(ValueError, match="EXIF data is too long"):
        jpeg_app_segments(exif=bytes(65534))


def test_keep_of_a_non_jpeg_is_refused_as_pillow_refuses_it():
    with pytest.raises(ValueError, match="Cannot use 'keep' when original image is not a JPEG"):
        pillow(Image.new("RGB", (8, 8)), quality="keep")


@pytest.mark.parametrize("progressive", [False, True])
def test_bound_holds(lib, progressive):
    """The library's bound is the restated one, and holds for noise at all-1 tables with metadata, at each sampling."""
    rs = np.random.RandomState(6)
    seg = jpeg_app_segments(b"Exif\0\0" + bytes(100), icc_profile=bytes(70000))
    for h, w in ((1, 1), (9, 17), (64, 48), (37, 129)):
        a = content("noise", h, w, rs)
        for s in (0, 1, 2):
            for n in (1, 2, 3, 4):
                bound = lib.se_jpeg_tables_max_bytes(h, w, s, n, int(progressive), len(seg))
                assert bound == K.max_bytes(h, w, s, n, progressive, len(seg))
                got = K.encode(a, [[1] * 64] * n, s, progressive=progressive, segments=seg)
                assert len(got) <= bound
    for s in (0, 2):   # the quality entries' bounds are the tables bound of their two tables
        assert lib.se_jpeg_max_bytes(480, 641, s) == lib.se_jpeg_tables_max_bytes(480, 641, s, 2, 0, 0)
        assert lib.se_jpeg_progressive_max_bytes(480, 641, s) == lib.se_jpeg_tables_max_bytes(480, 641, s, 2, 1, 0)
    for bad in ((0, 1, 0, 1, 0, 0), (1, 1, 3, 1, 0, 0), (1, 1, -1, 1, 0, 0), (1, 1, 0, 0, 0, 0), (1, 1, 0, 5, 0, 0),
                (1, 1, 0, 1, 2, 0), (1, 1, 0, 1, 0, -1), (1, 1, 0, 1, 0, (1 << 30) + 1)):
        assert lib.se_jpeg_tables_max_bytes(*bad) == -1


def _call(lib, qt, ntables=None, sub=1, optimize=0, progressive=0, seg=b"", hw=(8, 8), n=1, scratch=None):
    tabs = (ctypes.c_ushort * len(qt))(*qt) if qt is not None else None
    segbuf = (ctypes.c_ubyte * len(seg)).from_buffer_copy(seg) if seg else None
    hwa = (ctypes.c_int * 2)(*hw)
    pitch = (ctypes.c_longlong * 1)(3 * hw[1])
    off = (ctypes.c_longlong * 1)(0)
    size = ctypes.c_longlong(0)
    rc = lib.se_jpeg_encode_tables_u8(None, pitch, hwa, n, tabs, len(qt) // 64 if ntables is None else ntables, sub, optimize,
                                      progressive, segbuf, len(seg), None, off, None, scratch, ctypes.byref(size), None)
    return rc, size.value, (lib.se_last_error() or b"").decode()


def test_host_checks_and_scratch_query(lib):
    """Every argument is checked on the host; without scratch the call reports the scratch of the quality entries."""
    ok = [1] * 128
    rc, size, _ = _call(lib, ok)
    assert rc == 0 and size > 0
    for s in (0, 2):   # the same scratch as the quality entries at 4:4:4 and 4:2:0
        for prog in (0, 1):
            ref = ctypes.c_longlong(0)
            hwa, pitch, off = (ctypes.c_int * 2)(480, 641), (ctypes.c_longlong * 1)(3 * 641), (ctypes.c_longlong * 1)(0)
            entry = lib.se_jpeg_encode_progressive_u8 if prog else lib.se_jpeg_encode_u8
            assert entry(None, pitch, hwa, 1, 75, s, None, off, None, None, ctypes.byref(ref), None) == 0
            assert _call(lib, ok, sub=s, progressive=prog, hw=(480, 641))[1] == ref.value
    app1 = b"\xff\xe1\x00\x05abc"
    for kw, msg in [(dict(qt=ok, ntables=0), "ntables"), (dict(qt=[1] * 320, ntables=5), "ntables"),
                    (dict(qt=None, ntables=2), "qtables"), (dict(qt=[1] * 63 + [256] + [1] * 64), "entries"),
                    (dict(qt=ok, sub=3), "subsampling"), (dict(qt=ok, sub=-1), "subsampling"),
                    (dict(qt=ok, optimize=2), "optimize"), (dict(qt=ok, progressive=2), "progressive"),
                    (dict(qt=ok, seg=b"\xff\xe3\x00\x02"), "APP1"), (dict(qt=ok, seg=b"\xff\xe1\x00\x06abc"), "length"),
                    (dict(qt=ok, seg=b"\xff\xe1\x00\x01"), "length"), (dict(qt=ok, seg=app1 + b"\xff"), "cut short"),
                    (dict(qt=ok, seg=b"\xfe\xe1\x00\x02"), "APP1"), (dict(qt=ok, n=33), "n must"),
                    (dict(qt=ok, hw=(0, 8)), "sizes")]:
        rc, _, err = _call(lib, **kw)
        assert rc != 0 and msg in err, (kw, err)
    assert _call(lib, ok, seg=app1 + b"\xff\xe2\x00\x02")[0] == 0
    rc, _, err = _call(lib, ok, scratch=ctypes.c_void_p(1))
    assert rc != 0 and "scratch holds" in err


class _NoForward:
    precision = "bf16"

    def engine(self):
        return None


def _host_session(img):
    from sketchedit_b200.serving import DemoProcessor
    p = DemoProcessor(_NoForward(), resize="host", region_size=(64, 48))
    return p, p.open_session(img)


def test_host_session_keeps_the_upload():
    """resize='host': keep with box, size, optimize and progressive, metadata with a numeric quality, the session's exif and
    icc_profile, the argument checks, a non-JPEG upload and a closed session."""
    rs = np.random.RandomState(7)
    a = content("places_11_512x408.npz", 67, 93, rs)
    exif, icc = exif_orientation_6().tobytes(), icc_srgb()
    for q, sub in ((92, 1), (95, 2), (85, 0)):
        src = upload(a, q, sub, exif=exif, icc_profile=icc)
        p, s = _host_session(src)
        try:
            assert s.exif == exif and s.icc_profile == icc
            cur = s.image()
            assert s.jpeg() == pillow(cur, quality=75, subsampling=2)
            meta = dict(exif=s.exif, icc_profile=s.icc_profile)
            assert s.jpeg(quality="keep", **meta) == keep_statement(cur, src, **meta)
            assert s.jpeg(quality="keep", subsampling=0) == keep_statement(cur, src)   # Pillow's keep ignores subsampling
            for box, size, coding in (((3, 5, 60, 40), None, dict(optimize=True)), (None, (40, 40), dict(progressive=True)),
                                      ((1, 1, 90, 66), (30, 50), dict())):
                img = cur if box is None else cur.crop(box)
                if size is not None:
                    img = img.copy()
                    img.thumbnail(size)
                got = s.jpeg(quality="keep", box=box, size=size, **meta, **coding)
                assert got == keep_statement(img, src, **meta, **coding), (q, sub, box, size, coding)
                assert s.jpeg(90, 0, box=box, size=size, **meta, **coding) == pillow(img, quality=90, subsampling=0, **meta,
                                                                                     **coding)
            for bad in (dict(quality="keep", optimize=1), dict(quality="high"), dict(exif=bytes(65534)), dict(exif="x"),
                        dict(icc_profile=5), dict(quality=90, subsampling=1), dict(quality="keep", box=(0, 0, 94, 10))):
                with pytest.raises(ValueError):
                    s.jpeg(**bad)
            s.close()
            with pytest.raises(RuntimeError, match="closed"):
                s.jpeg(quality="keep")
        finally:
            p.close()
    p, s = _host_session(Image.fromarray(a))
    try:
        assert s.exif == b"" and s.icc_profile is None
        with pytest.raises(ValueError, match="Cannot use 'keep' when original image is not a JPEG"):
            s.jpeg(quality="keep")
    finally:
        p.close()

"""Region edits (DemoProcessor.process_image(..., region=...)) on the CPU: the box rule of serving.region_box, the validation
of region requests, the paste blend against Image.paste on every byte triple, and the host checks of the one-box-per-canvas
paste of se_resize_composite_feather_detail_u8."""
import ctypes

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import DemoProcessor, region_box

# (bbox, photo (w, h), working (Hn, Wn), expected box)
CASES = [
    ((1200, 600, 1330, 900), (4000, 2667), (256, 256), (961, 446, 1569, 1054)),     # s = 19/8
    ((0, 0, 40, 30), (1000, 667), (256, 256), (0, 0, 256, 256)),                     # corner sketch: shifted into the photo
    ((980, 300, 1000, 420), (1000, 667), (256, 256), (744, 232, 1000, 488)),         # right edge
    ((500, 300, 510, 305), (1000, 667), (256, 256), (377, 174, 633, 430)),           # tiny sketch: the working size, a pure crop
    ((0, 0, 1000, 667), (1000, 667), (256, 256), (0, 0, 1000, 667)),                 # spans the photo: the photo, clamped
    ((10, 10, 50, 50), (200, 150), (256, 256), (0, 0, 200, 150)),                    # photo smaller than the working size
    ((300, 200, 420, 230), (1000, 667), (256, 512), (104, 87, 616, 343)),            # non-square working size: s = 1
    ((300, 200, 700, 230), (1000, 667), (256, 512), (84, 7, 916, 423)),              # non-square, s = 13/8
]


@pytest.mark.parametrize("bbox, photo, work, want", CASES)
def test_region_box_cases(bbox, photo, work, want):
    assert region_box(bbox, photo, work) == want


def _check_invariants(bbox, photo, work):
    left, upper, right, lower = box = region_box(bbox, photo, work)
    w, h = photo
    Hn, Wn = work
    assert 0 <= left < right <= w and 0 <= upper < lower <= h, box
    assert left <= bbox[0] and upper <= bbox[1] and right >= bbox[2] and lower >= bbox[3], (bbox, box)
    bw, bh = right - left, lower - upper
    s8 = max(8, -(-16 * (bbox[2] - bbox[0]) // Wn), -(-16 * (bbox[3] - bbox[1]) // Hn))
    assert bw == min(w, s8 * Wn // 8) and bh == min(h, s8 * Hn // 8), (bbox, box)       # s is a multiple of 1/8
    if bw < w and bh < h:
        assert bw * Hn == bh * Wn, (bbox, box)                                          # the working aspect, unless clamped
    if bw < w:                                                                            # the strokes span at most half
        assert 2 * (bbox[2] - bbox[0]) <= bw
    if bh < h:
        assert 2 * (bbox[3] - bbox[1]) <= bh


def test_region_box_invariants():
    rs = np.random.RandomState(5)
    for _ in range(3000):
        w, h = int(rs.randint(16, 5000)), int(rs.randint(16, 5000))
        work = (8 * int(rs.randint(2, 80)), 8 * int(rs.randint(2, 80)))
        x0, y0 = int(rs.randint(0, w)), int(rs.randint(0, h))
        x1, y1 = int(rs.randint(x0 + 1, w + 1)), int(rs.randint(y0 + 1, h + 1))
        if rs.rand() < 0.7:                                                               # mostly local sketches
            x1, y1 = min(x1, x0 + int(rs.randint(1, 300))), min(y1, y0 + int(rs.randint(1, 300)))
        _check_invariants((x0, y0, x1, y1), (w, h), work)


def test_region_box_rejects_a_bbox_outside_the_photo():
    for bbox in ((0, 0, 0, 5), (10, 10, 5, 20), (-1, 0, 5, 5), (0, 0, 1001, 5)):
        with pytest.raises(ValueError):
            region_box(bbox, (1000, 667), (256, 256))


# ------------------------------------------------------------------------------------------ request validation (no forward)
class _NoForward:
    precision = "bf16"

    def engine(self):
        return None


@pytest.fixture
def proc():
    p = DemoProcessor(_NoForward(), region_size=(256, 256))
    yield p
    p.close()


def _photo(w=300, h=200, stroke=True):
    img = Image.fromarray(np.full((h, w, 3), 128, np.uint8))
    m = np.zeros((h, w), np.uint8)
    if stroke:
        m[50:60, 100:110] = 255
    return img, Image.fromarray(m)


def test_auto_region_needs_a_stroke(proc):
    img, m = _photo(stroke=False)
    with pytest.raises(ValueError, match="stroke"):
        proc.process_image(img, m, region="auto")
    with pytest.raises(ValueError, match="stroke"):
        proc.process_image(img, m, edit_mask=Image.new("L", img.size, 0), region="auto")


@pytest.mark.parametrize("region", [(0, 0, 0, 10), (5, 5, 4, 10), (-1, 0, 10, 10), (0, 0, 301, 10), (0, 0, 10, 201),
                                    (0, 0, 10.0, 10), (0, 0, 10), "box", [0, 0, 10, "10"]])
def test_explicit_boxes_are_validated(proc, region):
    img, m = _photo()
    with pytest.raises(ValueError):
        proc.process_image(img, m, region=region)


def test_region_masks_must_have_the_photo_size(proc):
    img, _ = _photo()
    with pytest.raises(ValueError, match="photo's size"):
        proc.process_image(img, Image.new("L", (150, 100), 255), region="auto")
    with pytest.raises(ValueError, match="photo's size"):
        proc.process_image(img, _photo()[1], edit_mask=Image.new("L", (150, 100), 255), region=(0, 0, 10, 10))


@pytest.mark.parametrize("size", [(255, 256), (256, 8), (0, 0), (256,)])
def test_region_size_is_validated(size):
    with pytest.raises(ValueError):
        DemoProcessor(_NoForward(), region_size=size)


# ------------------------------------------------------------------------------------------ the paste blend
def div255_blend(base, res, m):
    """Pillow's Image.paste(im, box, mask) per channel (libImaging/Paste.c): DIV255(base * (255 - m) + res * m)."""
    a = base.astype(np.int32) * (255 - m.astype(np.int32)) + res.astype(np.int32) * m.astype(np.int32) + 128
    return (((a >> 8) + a) >> 8).astype(np.uint8)


def test_div255_blend_equals_image_paste_on_every_byte_triple():
    """All 2^24 (base, result, mask) triples, 16 base values per 1024x1024 image so that memory stays small."""
    for b0 in range(0, 256, 16):
        p = np.arange(1 << 20, dtype=np.uint32).reshape(1024, 1024)
        b, r, m = (b0 + (p >> 16)).astype(np.uint8), ((p >> 8) & 255).astype(np.uint8), (p & 255).astype(np.uint8)
        base = np.stack([b, 255 - b, b], axis=-1)
        res = np.stack([r, r, 255 - r], axis=-1)
        im = Image.fromarray(base)
        im.paste(Image.fromarray(res), (0, 0), Image.fromarray(m))
        want = np.asarray(im)
        got = div255_blend(base, res, m[..., None])
        assert np.array_equal(got, want), (b0, int((got != want).any(axis=-1).sum()))


# ------------------------------------------------------------------------------------------ one box per canvas on the host
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _query(lib, src, dst, n=1, scratch=None, scratch_bytes=0, off=0):
    """se_resize_composite_feather_detail_u8 with n boxes, each filling its own canvas (at (0, 0), pitch 3 w), no feather."""
    k = max(n, 1)
    L, I = ctypes.c_longlong, ctypes.c_int
    offs = (L * k)(*([off] * k))
    coff, pitches = (L * k)(*range(off, off + 10 ** 6 * k, 10 ** 6)), (L * k)(*([3 * dst[1]] * k))
    shw, dhw, yx = (I * (2 * k))(*(src * k)), (I * (2 * k))(*(dst * k)), (I * (2 * k))(*([0, 0] * k))
    need = L(scratch_bytes)
    rc = lib.se_resize_composite_feather_detail_u8(None, offs, None, offs, shw, None, coff, pitches, yx, dhw, None, None, None, n, 1,
                                                   scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode()


def test_paste_scratch_query_with_null_detail(lib):
    r256 = lambda b: (b + 255) // 256 * 256
    assert _query(lib, (256, 256), (608, 608))[:2] == (0, r256(256 * 608 * 3) + r256(256 * 608))
    assert _query(lib, (256, 256), (608, 256))[:2] == (0, 0)           # width unchanged: the paste reads the result itself
    assert _query(lib, (256, 256), (256, 256))[:2] == (0, 0)
    assert _query(lib, (256, 256), (100, 77), n=3)[:2] == (0, 3 * (r256(256 * 77 * 3) + r256(256 * 77)))
    assert _query(lib, (256, 256), (100, 77), n=33)[:2] == (0, 33 * (r256(256 * 77 * 3) + r256(256 * 77)))   # no batch bound
    assert _query(lib, (256, 256), (100, 77), n=0)[:2] == (0, 0)


def test_paste_with_null_detail_validates_on_the_host_with_the_resize_messages(lib):
    cases = [
        (dict(src=(256, 256), dst=(64, 64), n=-1), "n must be >= 0 boxes"),
        (dict(src=(0, 256), dst=(64, 64)), "sizes must be in [1, 65535]"),
        (dict(src=(256, 256), dst=(64, 65536)), "sizes must be in [1, 65535]"),
        (dict(src=(8, 60000), dst=(8, 1)), "downscale factor too large"),
        (dict(src=(256, 256), dst=(64, 64), off=-1), "negative offset"),
        (dict(src=(256, 256), dst=(608, 608), scratch=1, scratch_bytes=100), "needs"),
    ]
    for kw, msg in cases:
        rc, _, err = _query(lib, **kw)
        assert rc != 0 and msg in err, (kw, err)
    # the shared checks say what the window resize says
    need = ctypes.c_longlong(0)
    off, hw = (ctypes.c_longlong * 1)(0), (ctypes.c_int * 2)(0, 256)
    assert lib.se_resize_window_u8(None, (ctypes.c_longlong * 1)(768), hw, None, off, (ctypes.c_int * 2)(64, 64), 1, 3, 0, None,
                                   ctypes.byref(need), None) != 0
    assert _query(lib, (0, 256), (64, 64))[2].split(" : ")[-1].split(" at ")[0] == \
        lib.se_last_error().decode().split(" : ")[-1].split(" at ")[0]
    hw = (ctypes.c_int * 2)(64, 64)
    assert lib.se_resize_composite_feather_detail_u8(None, None, None, None, hw, None, None, None, None, hw, None, None, None, 1, 0,
                                                     None, ctypes.byref(need), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()
    assert lib.se_resize_composite_feather_detail_u8(None, None, None, None, None, None, None, None, None, None, None, None, None, 0,
                                                     0, None, None, None) != 0

"""Feathered region pastes on the CPU: the width rule and the ramp of serving.feather_widths / feather_ramp, the host flow of
DemoProcessor with a fake forward against the Pillow statement, the property that the band never reaches a stroke of an
'auto' or 'strokes' box, the seam bound, host sessions with feather, and the host checks of se_resize_composite_feather_detail_u8 and
se_feather_u8."""
import ctypes

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import DemoProcessor, feather_mask, feather_ramp, feather_widths, region_box


def _div255(a):
    a = a + 128
    return ((a >> 8) + a) >> 8


def _ramp(bw, bh, widths):
    """The ramp as written: each side's band one line at a time, the least value kept."""
    fl, ft, fr, fb = widths
    r = np.full((bh, bw), 255, np.int64)
    for d in range(max(widths)):
        for f, sl in ((fl, np.s_[:, d]), (fr, np.s_[:, bw - 1 - d]), (ft, np.s_[d, :]), (fb, np.s_[bh - 1 - d, :])):
            if d < f:
                r[sl] = np.minimum(r[sl], 255 * (d + 1) // (f + 1))
    return r


# ------------------------------------------------------------------------------------------ the rule
@pytest.mark.parametrize("box, size, F, want", [
    ((100, 50, 300, 250), (1000, 667), 16, (16, 16, 16, 16)),        # every side inside the photo
    ((0, 50, 300, 250), (1000, 667), 16, (0, 16, 16, 16)),           # left on the border
    ((100, 0, 300, 250), (1000, 667), 16, (16, 0, 16, 16)),          # top on the border
    ((100, 50, 1000, 250), (1000, 667), 16, (16, 16, 0, 16)),        # right on the border
    ((100, 50, 300, 667), (1000, 667), 16, (16, 16, 16, 0)),         # bottom on the border
    ((0, 0, 1000, 667), (1000, 667), 16, (0, 0, 0, 0)),              # the whole photo
    ((100, 50, 140, 250), (1000, 667), 16, (10, 16, 10, 16)),        # the quarter cap: 40 // 4
    ((100, 50, 143, 69), (1000, 667), 99, (10, 4, 10, 4)),           # 43 // 4, 19 // 4
    ((100, 50, 103, 53), (1000, 667), 16, (0, 0, 0, 0)),             # bw < 4
    ((100, 50, 104, 55), (1000, 667), 16, (1, 1, 1, 1)),
    ((100, 50, 300, 250), (1000, 667), 0, (0, 0, 0, 0)),             # F = 0
    ((5, 7, 6, 8), (10, 10), 3, (0, 0, 0, 0)),                       # one pixel
])
def test_width_rule(box, size, F, want):
    assert feather_widths(box, size, F) == want


def test_hand_computed_ramps():
    r = feather_ramp((8, 1), (3, 0, 0, 0))
    assert r.tolist() == [[63, 127, 191, 255, 255, 255, 255, 255]]
    r = feather_ramp((8, 1), (0, 0, 3, 0))
    assert r.tolist() == [[255, 255, 255, 255, 255, 191, 127, 63]]
    # left f = 2: 85, 170; top f = 1: 127; bottom f = 3: 63, 127, 191 from the bottom row up; corners take the minimum
    r = feather_ramp((5, 5), (2, 1, 0, 3))
    assert r.tolist() == [[85, 127, 127, 127, 127],
                          [85, 170, 255, 255, 255],
                          [85, 170, 191, 191, 191],
                          [85, 127, 127, 127, 127],
                          [63, 63, 63, 63, 63]]
    for bw, bh, widths in [(7, 5, (1, 2, 1, 2)), (31, 45, (7, 11, 7, 11)), (12, 12, (6, 6, 6, 6)), (40, 3, (10, 0, 3, 0))]:
        assert np.array_equal(feather_ramp((bw, bh), widths), _ramp(bw, bh, widths)), (bw, bh, widths)


def test_div255_of_255m_is_m():
    m = np.arange(256)
    assert np.array_equal(_div255(255 * m), m)
    assert np.array_equal(feather_mask(m.astype(np.uint8)[None], (0, 0, 0, 0))[0], m)


# ------------------------------------------------------------------------------------------ the host flow, fake forward
class _NoForward:
    precision = "bf16"

    def engine(self):
        return None


def _fake_forward(img, sk, em):
    """The fake forward of tests/test_region_groups.py: a BGR result and a soft mask with 0, 255 and values between."""
    k, Hn, Wn = sk.shape
    yy, xx = np.mgrid[:Hn, :Wn]
    bgr = (255 - img[..., ::-1].astype(np.int32) + sk[..., None] // 3) % 256
    mk = em if em is not None else np.clip((xx * 7 + yy * 3)[None] % 400 - 70 + sk // 5, 0, 255)
    return bgr.astype(np.uint8), np.broadcast_to(mk, (k, Hn, Wn)).astype(np.uint8)


class _FakeProcessor(DemoProcessor):
    forward = staticmethod(_fake_forward)

    def _run_batch(self, key, payloads):
        out = []
        for img, sk, em, want in payloads:
            one = key[0] != "region"
            if one:
                img, sk, em = img[None], sk[None], em[None] if em is not None else None
            bgr, mk = self.forward(img, sk, em)
            rgb, mk = np.ascontiguousarray(bgr[..., ::-1]), mk if want and em is None else None
            out.append((rgb[0], mk[0] if mk is not None else None) if one else (rgb, mk))
        return out


@pytest.fixture
def fake():
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    yield p
    p.close()


def _statement(img, sk, em, boxes, Hn, Wn, F, forward=_fake_forward):
    """The statement: each box in order does out.paste(res_resized, box, Image.fromarray(m')), m' = DIV255(m * ramp), every
    crop taken from the photo; the returned mask is the largest m' over the boxes."""
    out, full = img.copy(), np.zeros(img.size[::-1], np.uint8)
    w, h = img.size
    for b in boxes:
        bw, bh = b[2] - b[0], b[3] - b[1]
        crop = np.array(img.crop(b).resize((Wn, Hn)))[None]
        s = ((np.array(sk.crop(b).resize((Wn, Hn))) > 0).astype(np.uint8) * 255)[None]
        e = np.array(em.crop(b).resize((Wn, Hn)))[None] if em is not None else None
        bgr, m = forward(crop, s, e)
        m = np.asarray(Image.fromarray(m[0]).resize((bw, bh))).astype(np.int64)
        widths = (0 if b[0] == 0 else min(F, bw // 4), 0 if b[1] == 0 else min(F, bh // 4),
                  0 if b[2] == w else min(F, bw // 4), 0 if b[3] == h else min(F, bh // 4))
        mp = _div255(m * _ramp(bw, bh, widths)).astype(np.uint8)
        out.paste(Image.fromarray(np.ascontiguousarray(bgr[0][..., ::-1])).resize((bw, bh)), b, Image.fromarray(mp))
        sub = full[b[1]:b[3], b[0]:b[2]]
        np.maximum(sub, mp, out=sub)
    return out, full


def _photo(w=300, h=200, seed=0):
    rs = np.random.RandomState(seed)
    img = Image.fromarray(rs.randint(0, 256, (h, w, 3), dtype=np.uint8))
    m = np.zeros((h, w), np.uint8)
    m[50:60, 100:110] = 255
    m[150:160, 250:262] = 255
    return img, Image.fromarray(m)


def _edit_mask():
    e = np.zeros((200, 300), np.uint8)
    e[40:80, 90:130] = np.arange(40 * 40).reshape(40, 40) % 256
    e[145:170, 240:270] = 200
    return Image.fromarray(e)


@pytest.mark.parametrize("F", [1, 5, 16, 1000])
@pytest.mark.parametrize("edit", [False, True])
def test_host_flow_equals_the_statement(fake, edit, F):
    img, m = _photo()
    em = _edit_mask() if edit else None
    regions = [
        (3, 7, 61, 51),                                                # one box
        "auto",
        "strokes",
        [(10, 10, 200, 150), (100, 50, 290, 190)],                     # overlapping
        [(10, 10, 200, 150), (100, 50, 290, 190), (10, 10, 200, 150)],  # repeated
        [(0, 0, 300, 200), (30, 20, 90, 80)],                          # the whole photo (no inner edge) and a nested box
        [(0, 13, 97, 200), (250, 0, 300, 77)],                         # boxes on the photo's borders
    ]
    changed = 0
    for region in regions:
        boxes = fake._region_boxes(img.size, m, em, region)
        got, gm = fake.process_image(img, m, edit_mask=em, return_mask=True, region=region, feather=F)
        want, wm = _statement(img, m, em, boxes, 64, 48, F)
        assert np.array_equal(np.array(got), np.array(want)), region
        if edit:
            assert gm is em                                             # a given edit mask comes back as given
        else:
            assert np.array_equal(np.array(gm), wm), region            # the largest feathered mask over the boxes
        changed += not np.array_equal(np.array(got), np.array(fake.process_image(img, m, edit_mask=em, region=region)))
    assert changed >= 3                                                 # the ramp is not a no-op


@pytest.mark.parametrize("region", [None, (3, 7, 61, 51), "auto", "strokes", [(10, 10, 200, 150), (100, 50, 290, 190)]])
def test_feather_0_is_no_feather(fake, region):
    img, m = _photo(seed=3)
    for em in (None, _edit_mask()):
        a, am = fake.process_image(img, m, edit_mask=em, return_mask=True, region=region)
        b, bm = fake.process_image(img, m, edit_mask=em, return_mask=True, region=region, feather=0)
        assert np.array_equal(np.array(a), np.array(b)) and np.array_equal(np.array(am), np.array(bm))
    if region is None:                                                  # no inner edges: feather has no effect
        c = fake.process_image(img, m, region=None, feather=16)
        assert np.array_equal(np.array(a), np.array(c))


@pytest.mark.parametrize("feather", [-1, 1.5, "16", True, None])
def test_feather_is_validated(fake, feather):
    img, m = _photo()
    for region in (None, "auto"):
        with pytest.raises(ValueError, match="feather"):
            fake.process_image(img, m, region=region, feather=feather)
    s = fake.open_session(img)
    with pytest.raises(ValueError, match="feather"):
        s.edit(m, feather=feather)
    with pytest.raises(RuntimeError, match="nothing to undo"):
        s.undo()
    s.close()


def test_the_band_never_reaches_a_stroke():
    """For 'auto' and 'strokes' boxes of random strokes and edit masks, and any F, the ramp is 255 at every stroke pixel and
    every non-zero edit-mask pixel inside the box."""
    rs = np.random.RandomState(17)
    proc = _FakeProcessor(_NoForward(), resize="host")
    try:
        checked = 0
        for trial in range(150):
            w, h = int(rs.randint(24, 500)), int(rs.randint(24, 400))
            proc.region_size = (8 * int(rs.randint(2, 16)), 8 * int(rs.randint(2, 16)))
            nz = np.zeros((h, w), bool)
            for _ in range(int(rs.randint(1, 7))):
                y, x = int(rs.randint(0, h)), int(rs.randint(0, w))
                for _ in range(int(rs.randint(1, 60))):
                    nz[y, x] = True
                    y, x = min(max(y + int(rs.randint(-3, 4)), 0), h - 1), min(max(x + int(rs.randint(-3, 4)), 0), w - 1)
            ez = np.zeros((h, w), bool)
            if trial % 3 == 0:
                y, x = int(rs.randint(0, h)), int(rs.randint(0, w))
                ez[y:y + int(rs.randint(1, 30)), x:x + int(rs.randint(1, 30))] = True
            m = Image.fromarray(nz.astype(np.uint8) * 255)
            em = Image.fromarray(ez.astype(np.uint8) * 7) if ez.any() else None
            for region in ("auto", "strokes"):
                for b in proc._region_boxes((w, h), m, em, region):
                    for F in (1, 3, int(rs.randint(1, 64)), 10 ** 6):
                        r = feather_ramp((b[2] - b[0], b[3] - b[1]), feather_widths(b, (w, h), F))
                        inside = (nz | ez)[b[1]:b[3], b[0]:b[2]]
                        assert (r[inside] == 255).all(), (trial, region, b, F, (w, h), proc.region_size)
                        checked += int(inside.sum())
        assert checked > 10000
    finally:
        proc.close()


def test_a_box_centred_on_a_half_size_bbox_keeps_a_quarter_margin():
    """The tightest cases of the cap: a bbox of exactly half the box, at both parities of the floored centring."""
    for work in ((16, 16), (24, 40), (256, 256)):
        for bw in range(1, 80):
            for left in (300, 301):
                bbox = (left, 300, left + bw, 300 + bw)
                box = region_box(bbox, (2000, 2000), work)
                r = feather_ramp((box[2] - box[0], box[3] - box[1]), feather_widths(box, (2000, 2000), 10 ** 6))
                assert (r[bbox[1] - box[1]:bbox[3] - box[1], bbox[0] - box[0]:bbox[2] - box[0]] == 255).all(), (work, bbox, box)


def _inverting_forward(img, sk, em):
    """The inverted crop as the result (BGR) and a paste mask of 255."""
    bgr = (255 - img[..., ::-1]).astype(np.uint8)
    return bgr, np.full(sk.shape, 255, np.uint8)


@pytest.mark.parametrize("F", [1, 4, 16])
def test_seam_bound_on_inner_edges(F):
    proc = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    proc.forward = staticmethod(_inverting_forward)
    rs = np.random.RandomState(F)
    a = np.zeros((200, 300, 3), np.uint8)                               # 0 along the box edges: the hard seam jumps by 255
    a[90:130, 120:200] = rs.randint(0, 256, (40, 80, 3))
    img = Image.fromarray(a)
    m = Image.new("L", img.size, 0)
    try:
        for box in [(40, 30, 240, 170), (0, 30, 240, 170), (41, 31, 99, 77)]:
            out = np.array(proc.process_image(img, m, region=box, feather=F)).astype(int)
            hard = np.array(proc.process_image(img, m, region=box)).astype(int)
            want, _ = _statement(img, m, None, [box], 64, 48, F, forward=_inverting_forward)
            assert np.array_equal(out, np.array(want))
            left, upper, right, lower = box
            fl, ft, fr, fb = feather_widths(box, img.size, F)
            edges = [(fl, np.s_[upper:lower, left]), (fr, np.s_[upper:lower, right - 1]),
                     (ft, np.s_[upper, left:right]), (fb, np.s_[lower - 1, left:right])]
            for f, sl in edges:
                if not f:
                    continue
                assert np.abs(out[sl] - a[sl]).max() <= 255 // (f + 1) + 1, (box, f)
                assert np.abs(hard[sl] - a[sl]).max() == 255, (box, f)
    finally:
        proc.close()


# ------------------------------------------------------------------------------------------ host sessions
def _mask(w, h, rects, soft=False, seed=0):
    rs = np.random.RandomState(seed)
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1] = rs.randint(0, 256, (y1 - y0, x1 - x0)) if soft else 255
    return Image.fromarray(m)


def _chain():
    m1 = _mask(300, 200, [(50, 50, 60, 70)])
    m2 = _mask(300, 200, [(20, 20, 30, 30), (250, 150, 262, 160)])
    m3 = _mask(300, 200, [(100, 40, 140, 90), (130, 80, 170, 120)])
    e3 = _mask(300, 200, [(90, 30, 150, 100)], soft=True, seed=3)
    return [
        (m1, None, "auto", 8),
        (m2, None, "strokes", 3),
        (m3, e3, "auto", 16),
        (m3, None, [(10, 10, 200, 150), (100, 50, 290, 190), (10, 10, 200, 150)], 12),
        (m1, None, None, 16),
        (m2, None, [(3, 7, 61, 51)], 0),
        (m1, None, (0, 0, 150, 120), 100),
    ]


def test_a_feathered_chain_is_chained_process_image(fake):
    rs = np.random.RandomState(0)
    img = Image.fromarray(rs.randint(0, 256, (200, 300, 3), dtype=np.uint8))
    s = fake.open_session(img)
    cur, states = img, [np.array(img)]
    for mask, em, region, F in _chain():
        prev = cur
        cur = fake.process_image(cur, mask, em, region=region, feather=F)
        r = s.edit(mask, em, region=region, return_mask=True, feather=F)
        assert np.array_equal(np.array(s.image()), np.array(cur)), region
        for b, p in zip(r.boxes, r.patches):
            assert np.array_equal(np.array(p), np.array(cur.crop(b)))
        if em is None:
            _, full = fake.process_image(prev, mask, em, return_mask=True, region=region, feather=F)
            want = np.zeros(cur.size[::-1], np.uint8)                   # the feathered per-box masks give process_image's
            for b, m in zip(r.boxes, r.masks):
                sub = want[b[1]:b[3], b[0]:b[2]]
                np.maximum(sub, np.asarray(m), out=sub)
            assert np.array_equal(want, np.array(full)), region
        else:
            assert r.masks == [None] * len(r.boxes)
        states.append(np.array(cur))
    for k in range(len(states) - 1, 0, -1):                             # undo is exact
        s.undo()
        assert np.array_equal(np.array(s.image()), states[k - 1]), k
    s.close()


# ------------------------------------------------------------------------------------------ the C entries on the host
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _composite(lib, src, dst, n=1, yx=(0, 0), feather=None, scratch=None, scratch_bytes=0):
    k = max(n, 1)
    L, I = ctypes.c_longlong, ctypes.c_int
    offs = (L * k)(*([0] * k))
    coff = (L * k)(*range(0, 10 ** 6 * k, 10 ** 6))
    pitches = (L * k)(*([3 * (yx[1] + dst[1])] * k))
    shw, dhw, byx = (I * (2 * k))(*(src * k)), (I * (2 * k))(*(dst * k)), (I * (2 * k))(*(yx * k))
    fw = (I * (4 * k))(*(list(feather) * k)) if feather is not None else None
    need = L(scratch_bytes)
    rc = lib.se_resize_composite_feather_detail_u8(None, offs, None, offs, shw, None, coff, pitches, byx, dhw, fw, None, None, n, 1,
                                                   scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode()


def test_composite_feather_scratch_query_is_the_composites_with_null_detail(lib):
    for src, dst, n in [((256, 256), (608, 608), 1), ((256, 256), (608, 256), 2), ((256, 256), (100, 77), 3),
                        ((256, 256), (100, 77), 70), ((256, 256), (100, 77), 0)]:
        want = _composite(lib, src, dst, n)                              # feather == NULL
        assert want[0] == 0
        for f in ((0, 0, 0, 0), (5, 7, dst[1], dst[0])):
            assert _composite(lib, src, dst, n, feather=f)[:2] == want[:2], (src, dst, n, f)


def test_composite_feather_with_null_detail_validates_on_the_host(lib):
    for f in [(-1, 0, 0, 0), (0, -1, 0, 0), (0, 0, -3, 0), (0, 0, 0, -1), (78, 0, 0, 0), (0, 101, 0, 0), (0, 0, 78, 0),
              (0, 0, 0, 101)]:
        rc, _, err = _composite(lib, (256, 256), (100, 77), feather=f)
        assert rc != 0 and "feather widths" in err and "must be in [0, the side's length]" in err, (f, err)
    assert _composite(lib, (256, 256), (100, 77), feather=(77, 100, 77, 100))[0] == 0
    rc, _, err = _composite(lib, (256, 256), (608, 608), feather=(1, 1, 1, 1), scratch=1, scratch_bytes=100)
    assert rc != 0 and "needs" in err
    rc, _, err = _composite(lib, (0, 256), (64, 64), feather=(1, 1, 1, 1))
    assert rc != 0 and "sizes must be in [1, 65535]" in err
    need = ctypes.c_longlong(0)
    hw = (ctypes.c_int * 2)(64, 64)
    fw = (ctypes.c_int * 4)(1, 1, 1, 1)
    assert lib.se_resize_composite_feather_detail_u8(None, None, None, None, hw, None, None, None, None, hw, fw, None, None, 1, 0,
                                                     None, ctypes.byref(need), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()
    rc, need_b, _ = _composite(lib, (256, 256), (64, 64), feather=(1, 1, 1, 1))
    assert rc == 0
    scratch = ctypes.c_longlong(max(need_b, 1))
    offs = (ctypes.c_longlong * 1)(0)
    assert lib.se_resize_composite_feather_detail_u8(None, offs, None, offs, (ctypes.c_int * 2)(256, 256), None, offs,
                                                     (ctypes.c_longlong * 1)(192), (ctypes.c_int * 2)(0, 0), hw, fw, None, None, 1, 0, 1,
                                                     ctypes.byref(scratch), None) != 0
    assert "null rgb / mask / canvas" in lib.se_last_error().decode()


def _feather(lib, hw, f, n=1, off=0, img=None, arrays=True):
    k = max(n, 1)
    L, I = ctypes.c_longlong, ctypes.c_int
    if not arrays:
        return lib.se_feather_u8(img, None, None, None, n, None), lib.se_last_error().decode()
    rc = lib.se_feather_u8(img, (L * k)(*([off] * k)), (I * (2 * k))(*(hw * k)), (I * (4 * k))(*(f * k)), n, None)
    return rc, lib.se_last_error().decode()


def test_feather_entry_validates_on_the_host(lib):
    cases = [
        (dict(hw=(10, 10), f=(0, 0, 0, 0), n=-1), "n must be >= 0"),
        (dict(hw=(10, 10), f=(0, 0, 0, 0), arrays=False), "null offset / size / feather array"),
        (dict(hw=(0, 10), f=(0, 0, 0, 0)), "sizes must be in [1, 65535]"),
        (dict(hw=(10, 65536), f=(0, 0, 0, 0)), "sizes must be in [1, 65535]"),
        (dict(hw=(10, 10), f=(0, 0, 0, 0), off=-1), "negative offset"),
        (dict(hw=(10, 12), f=(-1, 0, 0, 0)), "feather widths"),
        (dict(hw=(10, 12), f=(0, 0, 0, -2)), "feather widths"),
        (dict(hw=(10, 12), f=(13, 0, 0, 0)), "feather widths"),
        (dict(hw=(10, 12), f=(0, 11, 0, 0)), "feather widths"),
        (dict(hw=(10, 12), f=(0, 0, 13, 0)), "feather widths"),
        (dict(hw=(10, 12), f=(0, 0, 0, 11)), "feather widths"),
        (dict(hw=(10, 12), f=(12, 10, 12, 10)), "null img"),           # valid widths reach the pointer check
    ]
    for kw, msg in cases:
        rc, err = _feather(lib, **kw)
        assert rc != 0 and msg in err, (kw, err)
    assert _feather(lib, (10, 10), (0, 0, 0, 0), n=0, arrays=False)[0] == 0


def test_wrappers_check_their_arguments():
    torch = pytest.importorskip("torch")
    from sketchedit_b200.engine import feather_u8_packed, resize_composite_u8_packed
    t = torch.empty(100, dtype=torch.uint8)
    with pytest.raises(_lib.SketchEditB200Error, match="same length"):
        feather_u8_packed(t, [0], [(3, 10)], [])
    with pytest.raises(_lib.SketchEditB200Error, match="CUDA uint8"):
        feather_u8_packed(t, [0], [(3, 10)], [(1, 1, 1, 1)])
    with pytest.raises(_lib.SketchEditB200Error, match="CUDA uint8"):
        resize_composite_u8_packed(t, [0], t, [0], [(3, 3)], t, [0], [9], [(0, 0)], [(3, 3)], feather=[(0, 0, 0, 0)])

"""Several regions per request on the CPU: the grouping rule of serving.region_groups (region="strokes"), the validation of box
lists, the host flow of DemoProcessor against the Pillow statement with a fake forward, and the host checks of
se_resize_composite_feather_detail_u8 without feather widths."""
import ctypes
from collections import deque

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import DemoProcessor, region_box, region_groups

W4K, H4K = 4000, 2667


def _strokes(w, h, rects):
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1] = 255
    return Image.fromarray(m)


# ------------------------------------------------------------------------------------------ the grouping rule
def test_one_group_is_the_auto_box():
    m = _strokes(W4K, H4K, [(1200, 600, 1330, 900)])
    assert region_groups(m) == [((1200, 600, 1330, 900), region_box((1200, 600, 1330, 900), (W4K, H4K), (256, 256)))]


def test_two_faces_stay_apart():
    m = _strokes(W4K, H4K, [(600, 500, 760, 700), (3200, 1900, 3360, 2100)])
    assert region_groups(m) == [((600, 500, 760, 700), (472, 392, 888, 808)), ((3200, 1900, 3360, 2100), (3072, 1792, 3488, 2208))]


def test_eyes_and_mouth_of_one_face_merge():
    m = _strokes(W4K, H4K, [(600, 500, 640, 515), (700, 500, 740, 515), (640, 600, 700, 610)])   # two eyes and a mouth
    want = (600, 500, 740, 610)
    assert region_groups(m) == [(want, region_box(want, (W4K, H4K), (256, 256)))]


def test_a_stroke_inside_a_ring_merges():
    m = np.zeros((667, 1000), np.uint8)
    m[100:300, 100:102] = m[100:300, 298:300] = m[100:102, 100:300] = m[298:300, 100:300] = 255
    m[199:201, 199:201] = 255                                                   # a dot inside: its own cell component
    assert region_groups(Image.fromarray(m)) == [((100, 100, 300, 300), region_box((100, 100, 300, 300), (1000, 667), (256, 256)))]


def test_chained_merges():
    """Merges repeat to a fixpoint: three strokes whose boxes reach their neighbours, then a chain of five."""
    rects = [(100, 100, 110, 110), (330, 100, 340, 110), (215, 100, 225, 110)]
    got = region_groups(_strokes(1000, 667, rects))
    assert [g for g, _ in got] == [(100, 100, 340, 110)]
    rects = [(100, 100, 110, 110), (600, 100, 610, 110), (225, 150, 235, 160), (350, 150, 360, 160), (475, 150, 485, 160)]
    got = region_groups(_strokes(1000, 667, rects))
    assert [g for g, _ in got] == [(100, 100, 610, 160)]


def test_strokes_touching_the_photo_edge():
    m = _strokes(1000, 667, [(0, 0, 5, 40), (990, 650, 1000, 667)])
    assert region_groups(m) == [((0, 0, 5, 40), (0, 0, 256, 256)), ((990, 650, 1000, 667), (744, 411, 1000, 667))]


def test_an_edit_mask_only_group():
    m = _strokes(1000, 667, [(100, 100, 140, 140)])
    e = np.zeros((667, 1000), np.uint8)
    e[500:560, 800:830] = 1
    got = region_groups(m, Image.fromarray(e))
    assert [g for g, _ in got] == [(100, 100, 140, 140), (800, 500, 830, 560)]
    assert got[1][1] == region_box((800, 500, 830, 560), (1000, 667), (256, 256))


def test_order_is_upper_then_left():
    m = _strokes(2000, 2000, [(1500, 100, 1510, 110), (100, 900, 110, 910), (100, 100, 110, 110)])
    assert [g[:2] for g, _ in region_groups(m)] == [(100, 100), (1500, 100), (100, 900)]


def _groups_by_definition(nz, work):
    """The rule as written: 8-connected components of the 8x8 cells by breadth-first search, then pairwise merges."""
    h, w = nz.shape
    H8, W8 = -(-h // 8), -(-w // 8)
    cells = np.zeros((H8, W8), bool)
    for y, x in zip(*np.nonzero(nz)):
        cells[y // 8, x // 8] = True
    seen, groups = np.zeros_like(cells), []
    for cy, cx in zip(*np.nonzero(cells)):
        if seen[cy, cx]:
            continue
        seen[cy, cx] = True
        q, pix = deque([(cy, cx)]), []
        while q:
            a, b = q.popleft()
            ys, xs = np.nonzero(nz[a * 8:a * 8 + 8, b * 8:b * 8 + 8])
            pix += [(a * 8 + y, b * 8 + x) for y, x in zip(ys, xs)]
            for da in (-1, 0, 1):
                for db in (-1, 0, 1):
                    u, v = a + da, b + db
                    if 0 <= u < H8 and 0 <= v < W8 and cells[u, v] and not seen[u, v]:
                        seen[u, v] = True
                        q.append((u, v))
        ys, xs = zip(*pix)
        groups.append((min(xs), min(ys), max(xs) + 1, max(ys) + 1))
    hits = lambda a, b: a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]
    box = lambda g: region_box(g, (w, h), work)
    while True:
        pair = next(((i, j) for i in range(len(groups)) for j in range(len(groups))
                     if i != j and hits(groups[j], box(groups[i]))), None)
        if pair is None:
            break
        a, b = groups[pair[0]], groups[pair[1]]
        groups = [g for k, g in enumerate(groups) if k not in pair] + \
            [(min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3]))]
    return sorted((g, box(g)) for g in groups)


def test_invariants_over_random_strokes():
    rs = np.random.RandomState(11)
    hits = lambda a, b: a[0] < b[2] and b[0] < a[2] and a[1] < b[3] and b[1] < a[3]
    for trial in range(60):
        w, h = int(rs.randint(40, 400)), int(rs.randint(40, 300))
        work = (8 * int(rs.randint(2, 12)), 8 * int(rs.randint(2, 12)))
        nz = np.zeros((h, w), bool)
        for _ in range(int(rs.randint(1, 8))):                  # strokes: short random walks, some of them single pixels
            y, x = int(rs.randint(0, h)), int(rs.randint(0, w))
            for _ in range(int(rs.randint(1, 40))):
                nz[y, x] = True
                y, x = min(max(y + int(rs.randint(-2, 3)), 0), h - 1), min(max(x + int(rs.randint(-2, 3)), 0), w - 1)
        m = Image.fromarray(nz.astype(np.uint8) * 255)
        got = region_groups(m, region_size=work)
        assert sorted(got) == _groups_by_definition(nz, work), trial
        assert [(g[1], g[0]) for g, _ in got] == sorted((g[1], g[0]) for g, _ in got)
        covered = np.zeros_like(nz)
        for i, (g, box) in enumerate(got):
            assert box[0] <= g[0] and box[1] <= g[1] and box[2] >= g[2] and box[3] >= g[3]         # its strokes are in its box
            sub = nz[g[1]:g[3], g[0]:g[2]]
            assert sub[0].any() and sub[-1].any() and sub[:, 0].any() and sub[:, -1].any()        # the exact pixel bbox
            covered[g[1]:g[3], g[0]:g[2]] = True
            for j, (g2, _) in enumerate(got):
                assert i == j or not hits(g2, box), (trial, g, box, g2)                          # no other group's stroke
        assert not (nz & ~covered).any()
        if len(got) == 1:
            assert got[0][1] == region_box(m.getbbox(), (w, h), work)


# ------------------------------------------------------------------------------------------ request validation (no forward)
class _NoForward:
    precision = "bf16"

    def engine(self):
        return None


@pytest.fixture
def proc():
    p = DemoProcessor(_NoForward(), region_size=(64, 64))
    yield p
    p.close()


def _photo(w=300, h=200):
    rs = np.random.RandomState(w * h)
    img = Image.fromarray(rs.randint(0, 256, (h, w, 3), dtype=np.uint8))
    m = np.zeros((h, w), np.uint8)
    m[50:60, 100:110] = 255
    m[150:160, 250:262] = 255
    return img, Image.fromarray(m)


@pytest.mark.parametrize("region", [[], [(0, 0, 10, 10), (0, 0, 0, 10)], [(0, 0, 10, 10), (0, 0, 301, 10)],
                                    [(0, 0, 10, 10), "box"], [(0, 0, 10, 10), (0, 0, 10)], [(0, 0, 10, 10), (0, 0, 10.0, 10)],
                                    "stroke"])
def test_box_lists_are_validated(proc, region):
    img, m = _photo()
    with pytest.raises(ValueError):
        proc.process_image(img, m, region=region)


def test_strokes_needs_a_stroke_and_masks_of_the_photo_size(proc):
    img, m = _photo()
    with pytest.raises(ValueError, match="stroke"):
        proc.process_image(img, Image.new("L", img.size, 0), region="strokes")
    with pytest.raises(ValueError, match="photo's size"):
        proc.process_image(img, Image.new("L", (150, 100), 255), region="strokes")
    with pytest.raises(ValueError, match="photo's size"):
        proc.process_image(img, m, edit_mask=Image.new("L", (150, 100), 255), region=[(0, 0, 10, 10), (5, 5, 20, 20)])
    with pytest.raises(ValueError, match="one size"):
        region_groups(m, Image.new("L", (150, 100), 255))


# ------------------------------------------------------------------------------------------ the host flow, fake forward
def _fake_forward(img, sk, em):
    """A deterministic stand-in for the forward on [k,Hn,Wn] items: a BGR result and a soft mask with 0, 255 and values
    between, so the paste blends."""
    k, Hn, Wn = sk.shape
    yy, xx = np.mgrid[:Hn, :Wn]
    bgr = (255 - img[..., ::-1].astype(np.int32) + sk[..., None] // 3) % 256
    mk = em if em is not None else np.clip((xx * 7 + yy * 3)[None] % 400 - 70 + sk // 5, 0, 255)
    return bgr.astype(np.uint8), np.broadcast_to(mk, (k, Hn, Wn)).astype(np.uint8)


class _FakeProcessor(DemoProcessor):
    def _run_batch(self, key, payloads):
        out = []
        for img, sk, em, want in payloads:
            bgr, mk = _fake_forward(img, sk, em)
            out.append((np.ascontiguousarray(bgr[..., ::-1]), mk if want and em is None else None))
        return out


def _statement(img, sk, em, boxes, Hn, Wn):
    """The Pillow statement of a region edit with several boxes, with the fake forward."""
    out, full = img.copy(), np.zeros(img.size[::-1], np.uint8)
    for b in boxes:
        size = (b[2] - b[0], b[3] - b[1])
        crop = np.array(img.crop(b).resize((Wn, Hn)))[None]
        s = ((np.array(sk.crop(b).resize((Wn, Hn))) > 0).astype(np.uint8) * 255)[None]
        e = np.array(em.crop(b).resize((Wn, Hn)))[None] if em is not None else None
        bgr, m = _fake_forward(crop, s, e)
        mk = Image.fromarray(m[0]).resize(size)
        out.paste(Image.fromarray(np.ascontiguousarray(bgr[0][..., ::-1])).resize(size), b, mk)
        sub = full[b[1]:b[3], b[0]:b[2]]
        np.maximum(sub, np.asarray(mk), out=sub)
    return out, full


@pytest.fixture
def fake():
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    yield p
    p.close()


@pytest.mark.parametrize("edit", [False, True])
def test_host_flow_equals_the_pillow_statement(fake, edit):
    img, m = _photo()
    em = None
    if edit:
        e = np.zeros((200, 300), np.uint8)
        e[40:80, 90:130] = np.arange(40 * 40).reshape(40, 40) % 256
        em = Image.fromarray(e)
    lists = [
        [(10, 10, 200, 150), (100, 50, 290, 190)],                     # overlapping: the second blends over the first
        [(100, 50, 290, 190), (10, 10, 200, 150)],                     # the same boxes in the other order
        [(10, 10, 200, 150), (100, 50, 290, 190), (10, 10, 200, 150)],  # a repeated box
        [(0, 0, 300, 200), (30, 20, 90, 80)],                          # nested
        [(3, 7, 61, 51)],
    ]
    results = []
    for boxes in lists:
        got, gm = fake.process_image(img, m, edit_mask=em, return_mask=True, region=boxes)
        want, wm = _statement(img, m, em, boxes, 64, 48)
        assert np.array_equal(np.array(got), np.array(want)), boxes
        if edit:
            assert gm is em
        else:
            assert np.array_equal(np.array(gm), wm), boxes
        results.append(np.array(got))
    assert not np.array_equal(results[0], results[1])                  # order matters where boxes overlap
    one = fake.process_image(img, m, edit_mask=em, region=(3, 7, 61, 51))
    assert np.array_equal(np.array(one), results[-1])                  # a one-box list is the single box


def test_host_flow_strokes_uses_the_groups(fake):
    img, m = _photo()
    boxes = [box for _, box in region_groups(m, region_size=(64, 48))]
    assert len(boxes) == 2
    got = fake.process_image(img, m, region="strokes")
    assert np.array_equal(np.array(got), np.array(_statement(img, m, None, boxes, 64, 48)[0]))
    assert fake.batcher.batches[-1] == (("region", 64, 48), 1)         # a request's boxes run in one forward


# ------------------------------------------------------------------------------------------ the composite on the host
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _query(lib, src, dst, n=1, yx=(0, 0), pitch=None, canvas_off=None, scratch=None, scratch_bytes=0, off=0):
    k = max(n, 1)
    L, I = ctypes.c_longlong, ctypes.c_int
    offs = (L * k)(*([off] * k))
    coff = (L * k)(*(canvas_off if canvas_off is not None else range(0, 10**6 * k, 10**6)))
    pitches = (L * k)(*(pitch if isinstance(pitch, list) else [pitch if pitch is not None else 3 * (yx[1] + dst[1])] * k))
    shw, dhw, byx = (I * (2 * k))(*(src * k)), (I * (2 * k))(*(dst * k)), (I * (2 * k))(*(yx * k))
    need = L(scratch_bytes)
    rc = lib.se_resize_composite_feather_detail_u8(None, offs, None, offs, shw, None, coff, pitches, byx, dhw, None, None, None, n, 1,
                                                   scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode()


def test_composite_scratch_query_with_null_detail(lib):
    r256 = lambda b: (b + 255) // 256 * 256
    assert _query(lib, (256, 256), (608, 608))[:2] == (0, r256(256 * 608 * 3) + r256(256 * 608))
    assert _query(lib, (256, 256), (608, 256))[:2] == (0, 0)           # width unchanged: the paste reads the result itself
    assert _query(lib, (256, 256), (100, 77), n=3)[:2] == (0, 3 * (r256(256 * 77 * 3) + r256(256 * 77)))
    assert _query(lib, (256, 256), (100, 77), n=70, yx=(5, 9))[:2] == (0, 70 * (r256(256 * 77 * 3) + r256(256 * 77)))
    assert _query(lib, (256, 256), (100, 77), n=0)[:2] == (0, 0)


def test_composite_with_null_detail_validates_on_the_host(lib):
    cases = [
        (dict(src=(256, 256), dst=(64, 64), n=-1), "boxes"),
        (dict(src=(0, 256), dst=(64, 64)), "sizes must be in [1, 65535]"),
        (dict(src=(256, 256), dst=(64, 65536)), "sizes must be in [1, 65535]"),
        (dict(src=(8, 60000), dst=(8, 1)), "downscale factor too large"),
        (dict(src=(256, 256), dst=(64, 64), off=-1), "negative offset"),
        (dict(src=(256, 256), dst=(64, 64), yx=(-1, 0)), "negative offset"),
        (dict(src=(256, 256), dst=(64, 64), yx=(0, 3), pitch=3 * 66), "narrower than the box"),
        (dict(src=(256, 256), dst=(64, 64), n=2, canvas_off=[0, 0], pitch=[3 * 64, 3 * 80]), "one pitch"),
        (dict(src=(256, 256), dst=(608, 608), scratch=1, scratch_bytes=100), "needs"),
    ]
    for kw, msg in cases:
        rc, _, err = _query(lib, **kw)
        assert rc != 0 and msg in err, (kw, err)
    need = ctypes.c_longlong(0)
    off, hw = (ctypes.c_longlong * 1)(0), (ctypes.c_int * 2)(0, 256)
    assert lib.se_resize_window_u8(None, (ctypes.c_longlong * 1)(768), hw, None, off, (ctypes.c_int * 2)(64, 64), 1, 3, 0, None,
                                   ctypes.byref(need), None) != 0
    assert _query(lib, (0, 256), (64, 64))[2].split(" : ")[-1].split(" at ")[0] == \
        lib.se_last_error().decode().split(" : ")[-1].split(" at ")[0]        # the shared checks say what the window resize says
    hw = (ctypes.c_int * 2)(64, 64)
    assert lib.se_resize_composite_feather_detail_u8(None, None, None, None, hw, None, None, None, None, hw, None, None, None, 1, 0,
                                                     None, ctypes.byref(need), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()

"""Edit sessions on the CPU: DemoProcessor.open_session with the Pillow flow and a fake forward against chained process_image
calls, undo and its history limit, masks placed at an offset, the validation, and the host checks of se_resize_window_u8."""
import ctypes
import re

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import DemoProcessor, region_groups


class _NoForward:
    precision = "bf16"

    def engine(self):
        return None


def _fake_forward(img, sk, em):
    """A deterministic stand-in for the forward on [k,H,W] items: a BGR result and a soft mask with 0, 255 and values
    between, so the paste blends."""
    k, H, W = sk.shape
    yy, xx = np.mgrid[:H, :W]
    bgr = (255 - img[..., ::-1].astype(np.int32) + sk[..., None] // 3) % 256
    mk = em if em is not None else np.clip((xx * 7 + yy * 3)[None] % 400 - 70 + sk // 5, 0, 255)
    return bgr.astype(np.uint8), np.broadcast_to(mk, (k, H, W)).astype(np.uint8)


class _FakeProcessor(DemoProcessor):
    def _run_batch(self, key, payloads):
        out = []
        for img, sk, em, want in payloads:
            one = key[0] != "region"                    # a whole-photo item has no box axis
            if one:
                img, sk, em = img[None], sk[None], em[None] if em is not None else None
            bgr, mk = _fake_forward(img, sk, em)
            rgb, mk = np.ascontiguousarray(bgr[..., ::-1]), mk if want and em is None else None
            out.append((rgb[0], mk[0] if mk is not None else None) if one else (rgb, mk))
        return out


@pytest.fixture
def proc():
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    yield p
    p.close()


def _photo(w=300, h=200, seed=0):
    rs = np.random.RandomState(seed)
    return Image.fromarray(rs.randint(0, 256, (h, w, 3), dtype=np.uint8))


def _mask(w, h, rects, soft=False, seed=0):
    rs = np.random.RandomState(seed)
    m = np.zeros((h, w), np.uint8)
    for x0, y0, x1, y1 in rects:
        m[y0:y1, x0:x1] = rs.randint(0, 256, (y1 - y0, x1 - x0)) if soft else 255
    return Image.fromarray(m)


def _chain():
    """(mask, edit mask or None, region) steps on a 300x200 photo: every region form, with and without edit masks."""
    m1 = _mask(300, 200, [(50, 50, 60, 70)])
    m2 = _mask(300, 200, [(20, 20, 30, 30), (250, 150, 262, 160)])
    m3 = _mask(300, 200, [(100, 40, 140, 90), (130, 80, 170, 120)])
    e3 = _mask(300, 200, [(90, 30, 150, 100)], soft=True, seed=3)
    e2 = _mask(300, 200, [(240, 140, 270, 170)], soft=True, seed=4)
    return [
        (m1, None, "auto"),
        (m2, None, "strokes"),
        (m3, e3, "auto"),
        (m2, e2, "strokes"),
        (m1, None, (10, 10, 200, 150)),
        (m3, None, [(10, 10, 200, 150), (100, 50, 290, 190), (10, 10, 200, 150)]),
        (m1, None, None),
        (m3, e3, None),
        (m2, None, [(3, 7, 61, 51)]),
    ]


def _boxes(proc, size, mask, em, region):
    if region is None:
        return [(0, 0) + size]
    return proc._region_boxes(size, mask, em, region)


def test_a_chain_of_edits_is_chained_process_image(proc):
    img = _photo()
    s = proc.open_session(img)
    cur = img.convert("RGB")
    for mask, em, region in _chain():
        prev = cur
        cur = proc.process_image(cur, mask, em, region=region)
        r = s.edit(mask, em, region=region, return_mask=True)
        assert r.boxes == _boxes(proc, img.size, mask, em, region)
        assert np.array_equal(np.array(s.image()), np.array(cur)), region
        assert [p.mode for p in r.patches] == ["RGB"] * len(r.boxes)
        for b, p in zip(r.boxes, r.patches):
            assert np.array_equal(np.array(p), np.array(cur.crop(b))), b
        outside = np.ones(cur.size[::-1], bool)
        for left, upper, right, lower in r.boxes:
            outside[upper:lower, left:right] = False
        assert np.array_equal(np.array(cur)[outside], np.array(prev)[outside])
        if em is not None:
            assert r.masks == [None] * len(r.boxes)
        else:
            assert [m.size for m in r.masks] == [(b[2] - b[0], b[3] - b[1]) for b in r.boxes]
            _, full = proc.process_image(prev, mask, em, return_mask=True, region=region)
            want = np.zeros(cur.size[::-1], np.uint8)     # the per-box masks give process_image's returned mask
            for b, m in zip(r.boxes, r.masks):
                sub = want[b[1]:b[3], b[0]:b[2]]
                np.maximum(sub, np.asarray(m), out=sub)
            assert np.array_equal(want, np.array(full)), region
    assert s.edit(_chain()[0][0]).masks == [None]          # return_mask=False
    s.close()


def test_undo_walks_back_to_the_original(proc):
    img = _photo(seed=1)
    s = proc.open_session(img)
    states = [np.array(img)]
    for mask, em, region in _chain():
        s.edit(mask, em, region=region)
        states.append(np.array(s.image()))
    assert len({st.tobytes() for st in states}) == len(states)
    for k in range(len(states) - 1, 0, -1):
        boxes, patches = s.undo()
        cur = np.array(s.image())
        assert np.array_equal(cur, states[k - 1]), k
        for b, p in zip(boxes, patches):
            assert np.array_equal(np.array(p), cur[b[1]:b[3], b[0]:b[2]])
    with pytest.raises(RuntimeError, match="nothing to undo"):
        s.undo()
    s.edit(*_chain()[0][:2], region="auto")                # edits continue after undo
    s.close()


def test_history_bytes_evicts_oldest_first(proc):
    img = _photo(seed=2)
    m = _mask(300, 200, [(50, 50, 60, 70)])
    box = proc._region_boxes(img.size, m, None, "auto")[0]
    nbytes = (box[2] - box[0]) * (box[3] - box[1]) * 3
    s = proc.open_session(img, history_bytes=2 * nbytes)
    states = [np.array(img)]
    for _ in range(4):
        s.edit(m, region="auto")
        states.append(np.array(s.image()))
    s.undo()
    s.undo()
    assert np.array_equal(np.array(s.image()), states[2])
    with pytest.raises(RuntimeError, match="nothing to undo"):
        s.undo()
    s.close()
    s = proc.open_session(img, history_bytes=nbytes - 1)    # a snapshot larger than the limit is not kept
    s.edit(m, region="auto")
    with pytest.raises(RuntimeError, match="nothing to undo"):
        s.undo()
    s.close()


@pytest.mark.parametrize("region", ["auto", "strokes", (0, 0, 150, 120), [(100, 50, 290, 190), (10, 10, 200, 150)]])
@pytest.mark.parametrize("edit", [False, True])
def test_an_offset_mask_is_the_zero_padded_mask(proc, region, edit):
    img = _photo(seed=5)
    a, b = proc.open_session(img), proc.open_session(img)
    for off in [(61, 37), (0, 0), (5, 3), (300 - 97, 200 - 53)]:      # cell-aligned and not, touching the photo's edges
        small = _mask(97, 53, [(3, 4, 12, 20), (70, 30, 80, 45)], seed=off[0])
        em = _mask(97, 53, [(0, 0, 40, 30)], soft=True, seed=off[1]) if edit else None
        full, efull = Image.new("L", img.size, 0), None
        full.paste(small, off)
        if edit:
            efull = Image.new("L", img.size, 0)
            efull.paste(em, off)
        ra = a.edit(small, em, region=region, return_mask=True, offset=off)
        rb = b.edit(full, efull, region=region, return_mask=True)
        assert ra.boxes == rb.boxes, off
        for x, y in zip(ra.patches + ra.masks, rb.patches + rb.masks):
            assert (x is None and y is None) or np.array_equal(np.array(x), np.array(y))
        assert np.array_equal(np.array(a.image()), np.array(b.image())), off
    a.close()
    b.close()


def test_region_groups_of_a_placed_mask():
    rs = np.random.RandomState(13)
    for trial in range(30):
        w, h = int(rs.randint(60, 400)), int(rs.randint(60, 300))
        mw, mh = int(rs.randint(8, w + 1)), int(rs.randint(8, h + 1))
        ox, oy = int(rs.randint(0, w - mw + 1)), int(rs.randint(0, h - mh + 1))
        nz = np.zeros((mh, mw), np.uint8)
        for _ in range(int(rs.randint(1, 6))):
            y, x = int(rs.randint(0, mh)), int(rs.randint(0, mw))
            nz[y:y + int(rs.randint(1, 9)), x:x + int(rs.randint(1, 9))] = 255
        small = Image.fromarray(nz)
        full = Image.new("L", (w, h), 0)
        full.paste(small, (ox, oy))
        work = (8 * int(rs.randint(2, 8)), 8 * int(rs.randint(2, 8)))
        assert region_groups(small, region_size=work, photo_size=(w, h), offset=(ox, oy)) == \
            region_groups(full, region_size=work), trial


def test_validation_and_use_after_close(proc):
    img = _photo()
    s = proc.open_session(img)
    m = _mask(300, 200, [(50, 50, 60, 70)])
    small = _mask(40, 30, [(5, 5, 10, 10)])
    cases = [
        (dict(mask=m.convert("RGB")), "'L' mask"),
        (dict(mask=m, edit_mask=small), "one size"),
        (dict(mask=small, offset=(280, 0)), "does not fit"),
        (dict(mask=small, offset=(-1, 0)), "does not fit"),
        (dict(mask=small, offset=(1.5, 0)), "offset must be"),
        (dict(mask=small, region=None), "region=None needs"),
        (dict(mask=m, region=None, offset=(1, 0)), "region=None needs"),
        (dict(mask=Image.new("L", img.size, 0)), "needs a sketch stroke"),
        (dict(mask=m, region=(0, 0, 301, 10)), "region"),
        (dict(mask=m, region=[]), "empty"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=re.escape(msg)):
            s.edit(**kw)
    with pytest.raises(RuntimeError, match="nothing to undo"):
        s.undo()                                                       # failed edits leave no snapshot
    tiny = proc.open_session(_photo(15, 40))
    with pytest.raises(ValueError, match="16x16"):
        tiny.edit(_mask(15, 40, [(1, 1, 5, 5)]), region=None)
    s.edit(m)
    s.close()
    s.close()
    for call in (lambda: s.edit(m), s.undo, s.image):
        with pytest.raises(RuntimeError, match="closed"):
            call()
    with pytest.raises(ValueError, match="history_bytes"):
        proc.open_session(img, history_bytes=-1)


def test_processor_close_closes_its_sessions():
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    s = p.open_session(_photo())
    p.close()
    with pytest.raises(RuntimeError, match="closed"):
        s.image()
    with pytest.raises(RuntimeError, match="closed"):
        p.open_session(_photo())


# ------------------------------------------------------------------------------------------ se_resize_window_u8 on the host
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _query(lib, src, dst, n=1, channels=3, pitch=None, off=0, scratch=None, scratch_bytes=0, ptrs=None):
    k = max(n, 1)
    L, I = ctypes.c_longlong, ctypes.c_int
    pitches = (L * k)(*([pitch if pitch is not None else src[1] * channels] * k))
    shw, dhw, offs = (I * (2 * k))(*(src * k)), (I * (2 * k))(*(dst * k)), (L * k)(*([off] * k))
    need = L(scratch_bytes)
    rc = lib.se_resize_window_u8(ptrs, pitches, shw, None, offs, dhw, n, channels, 0, scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode()


def test_window_scratch_query(lib):
    r256 = lambda b: (b + 255) // 256 * 256
    for src, dst, n, c, per_image in [((667, 1000), (256, 256), 1, 3, r256(667 * 256 * 3)),   # both axes: ih x ow x C
                                      ((256, 256), (608, 256), 3, 3, 0),                     # one axis: no intermediate
                                      ((256, 256), (256, 77), 2, 1, 0),
                                      ((2667, 4000), (256, 256), 32, 1, r256(2667 * 256)),
                                      ((33, 45), (33, 45), 4, 3, 0), ((10, 10), (20, 20), 0, 3, r256(10 * 20 * 3))]:
        assert _query(lib, src, dst, n, c)[:2] == (0, n * per_image), (src, dst, n, c)
    assert _query(lib, (667, 1000), (256, 256), pitch=12000)[:2] == (0, r256(667 * 256 * 3))   # the pitch needs no scratch


def test_window_validates_on_the_host(lib):
    cases = [
        (dict(src=(256, 256), dst=(64, 64), n=33), "n must be in [0, 32]"),
        (dict(src=(256, 256), dst=(64, 64), channels=2), "channels must be 1 or 3"),
        (dict(src=(0, 256), dst=(64, 64)), "sizes must be in [1, 65535]"),
        (dict(src=(256, 256), dst=(64, 65536)), "sizes must be in [1, 65535]"),
        (dict(src=(8, 60000), dst=(8, 1)), "downscale factor too large"),
        (dict(src=(256, 256), dst=(64, 64), off=-1), "negative offset"),
        (dict(src=(256, 256), dst=(64, 64), pitch=767), "pitch of 767 bytes is narrower than its row of 768 bytes"),
        (dict(src=(256, 256), dst=(64, 64), channels=1, pitch=255), "narrower"),
        (dict(src=(256, 256), dst=(608, 608), scratch=1, scratch_bytes=100), "needs"),
    ]
    for kw, msg in cases:
        rc, _, err = _query(lib, **kw)
        assert rc != 0 and msg in err, (kw, err)
    assert _query(lib, (256, 256), (64, 64), pitch=1 << 40)[0] == 0      # any pitch at least the row
    rc, _, err = _query(lib, (256, 256), (64, 64), scratch=1, scratch_bytes=1 << 20)
    assert rc != 0 and "null src / dst" in err
    need = ctypes.c_longlong(0)
    hw = (ctypes.c_int * 2)(64, 64)
    assert lib.se_resize_window_u8(None, None, hw, None, None, hw, 1, 3, 0, None, ctypes.byref(need), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()


def test_window_wrapper_checks_bounds():
    torch = pytest.importorskip("torch")
    from sketchedit_b200.engine import resize_window_u8_packed
    t = torch.empty(100, dtype=torch.uint8)                 # a CPU tensor is refused before any bound
    with pytest.raises(_lib.SketchEditB200Error, match="CUDA uint8"):
        resize_window_u8_packed(t, [0], [30], [(3, 10)], [(5, 5)], 3)
    with pytest.raises(_lib.SketchEditB200Error, match="same length"):
        resize_window_u8_packed([t, t], [0], [30], [(3, 10)], [(5, 5)], 3)

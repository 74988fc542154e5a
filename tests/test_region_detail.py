"""Region-edit detail on the CPU: the geometry of the restatement (tests/util_detail.py), its properties, the argument checks
of the serving flows and of se_detail_u8, and that detail and plain region requests share batches."""
import ctypes

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build
from sketchedit_b200.serving import _check_detail, detail_box_ok
from tests import util_detail as U
from tests.test_region_feather import _FakeProcessor, _NoForward, _photo


@pytest.mark.parametrize("b,n", [(256, 256), (608, 256), (200, 256), (301, 256), (257, 192), (1000, 512), (17, 64), (64, 64)])
def test_geometry(b, n):
    ax = U.anchors(b, n)
    fw = U.footprint(b, n)
    if b == n:
        assert np.array_equal(ax, 8 * np.arange(n // 8 - 1))
    u = U.work_of(np.arange(b), b, n)
    assert u.min() >= 0 and u.max() < n
    for x in range(b):
        qs = U.covering(int(u[x]), n)
        assert 1 <= len(qs) <= 2            # per axis: nq = product, 1 to 4
        for p in qs:
            assert 8 * p <= u[x] < 8 * p + 16
            assert 0 <= x - ax[p] < fw
    # the anchor is the least box column whose centre reaches the patch
    for p, a in enumerate(ax):
        assert u[a] >= 8 * p and (a == 0 or u[a - 1] < 8 * p)


def _case(bh, bw, Hn, Wn, seed):
    rs = np.random.RandomState(seed)
    crop = rs.randint(0, 256, (bh, bw, 3), dtype=np.uint8)
    hole = np.zeros((Hn, Wn), np.uint8)
    hole[Hn // 4:3 * Hn // 4, Wn // 3:Wn - 5] = 1
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    P = rs.rand(L, L)
    return crop, U.low_of(crop, Hn, Wn), hole, P / P.sum(0)


def test_box_of_the_working_size_has_no_residual():
    crop, low, hole, P = _case(64, 48, 64, 48, 1)
    assert np.array_equal(low, crop)
    A, D, inh = U.aggregate(crop, low, hole, P)
    assert inh.any() and not A.any() and not D.any()


def test_empty_hole_adds_nothing():
    crop, low, hole, P = _case(97, 83, 64, 48, 2)
    A, D, inh = U.aggregate(crop, low, np.zeros_like(hole), P)
    assert not inh.any() and not D.any()


def test_one_hot_weights_copy_the_chosen_patch():
    bh, bw, Hn, Wn = 152, 120, 64, 48     # scale 19/8 and 5/2
    crop, low, hole, _ = _case(bh, bw, Hn, Wn, 3)
    hs, ws = Hn // 8 - 1, Wn // 8 - 1
    L = hs * ws
    key = 0                                # patch (0, 0): outside the hole
    P = np.zeros((L, L))
    P[key] = 1.0
    A, D, inh = U.aggregate(crop, low, hole, P)
    R, _ = U.residual(crop, low, hole)
    ax, ay = U.anchors(bw, Wn), U.anchors(bh, Hn)
    u, v = U.work_of(np.arange(bw), bw, Wn), U.work_of(np.arange(bh), bh, Hn)
    ys, xs = np.nonzero(inh)
    for y, x in zip(ys[::37], xs[::37]):
        qs = [(py, px) for py in U.covering(v[y], Hn) for px in U.covering(u[x], Wn)]
        want = sum(R[min(ay[0] + y - ay[py], bh - 1), min(ax[0] + x - ax[px], bw - 1)] for py, px in qs) / len(qs)
        assert np.allclose(A[y, x], want)
    assert np.abs(D).max() > 0 and not D[~inh].any()


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.bool_(True)])
def test_detail_must_be_a_bool(bad):
    with pytest.raises(ValueError):
        _check_detail(bad, False, False)


def test_argument_checks():
    assert _check_detail(False, True, True) is False
    with pytest.raises(ValueError, match="region"):
        _check_detail(True, True, False)
    with pytest.raises(ValueError, match="resize='device'"):
        _check_detail(True, False, True)
    p = _FakeProcessor(_NoForward(), resize="host", region_size=(64, 48))
    try:
        img, sk = _photo()
        with pytest.raises(ValueError):
            p.process_image(img, sk, region="auto", detail=True)
        with pytest.raises(ValueError):
            p.process_image(img, sk, detail=True)
        with pytest.raises(ValueError):
            p.process_image(img, sk, region="auto", detail=1)
        s = p.open_session(img)
        with pytest.raises(ValueError):
            s.edit(sk, region="auto", detail=True)
        with pytest.raises(ValueError):
            s.accept(s.propose(sk), detail=True)
        s.close()
    finally:
        p.close()


def test_detail_and_plain_requests_share_batches():
    """The batch key of a region request does not depend on detail: both kinds queue under one key."""
    import threading

    p = _Keys()
    img, sk = _photo()
    ts = [threading.Thread(target=p.process_image, args=(img, sk), kwargs=dict(region="auto", detail=d)) for d in (True, False, True)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    p.batcher.close()
    assert len(p.keys) == 1 and sorted(p.keys[0][1]) == [False, True, True]

@pytest.mark.parametrize("n", [16, 64, 256, 512])
def test_detail_box_ok_is_where_every_patch_has_an_anchor(n):
    for b in range(1, n // 8 + 3):
        u = U.work_of(np.arange(b), b, n)
        every = all((u >= 8 * p).any() for p in range(n // 8 - 1))
        assert detail_box_ok((b, n), (n, n)) == every == detail_box_ok((n, b), (n, n)), (b, n)
        if every:
            U.anchors(b, n)


class _Keys:
    """A device-flow DemoProcessor whose batches are recorded instead of run: (key, detail flags) per batch."""

    def __new__(cls, use_cam=True, region_size=(64, 48)):
        import types

        from sketchedit_b200 import serving

        class Keys(serving.DemoProcessor):
            def __init__(self):
                self.region_size, self.resize, self.keys = region_size, "device", []
                self.engine = types.SimpleNamespace(use_cam=use_cam)
                self.batcher = serving.RequestBatcher(self._collect, max_batch=8, max_wait_ms=200.0)

            def _collect(self, key, payloads):
                self.keys.append((key, [p[8] for p in payloads]))
                return [[(np.zeros((b[3] - b[1], b[2] - b[0], 3), np.uint8), None) for b in p[4]] for p in payloads]

        return Keys()


def test_no_detail_on_a_model_without_attention():
    """A model without the contextual attention has no weights to aggregate with: detail=True is refused before it is queued,
    so it cannot fail the plain requests it would share a batch with."""
    p = _Keys(use_cam=False)
    try:
        img, sk = _photo()
        with pytest.raises(ValueError, match="use_cam"):
            p.process_image(img, sk, region="auto", detail=True)
        assert p.process_image(img, sk, region="auto").size == img.size
        assert [d for _, d in p.keys] == [[False]]
    finally:
        p.batcher.close()
    with pytest.raises(ValueError, match="use_cam"):
        _check_detail(True, False, False, has_attention=False)
    assert _check_detail(False, False, False, has_attention=False) is False


def test_no_detail_on_boxes_without_anchors():
    p = _Keys(region_size=(256, 256))
    try:
        img, sk = _photo()
        with pytest.raises(ValueError, match="1/32"):
            p.process_image(img, sk, region=[(10, 10, 17, 120)], detail=True)   # 7 px < 256 / 32
        p.process_image(img, sk, region=[(10, 10, 18, 120)], detail=True)
        assert [d for _, d in p.keys] == [[True]]
    finally:
        p.batcher.close()


# ------------------------------------------------------------------------------------------ se_detail_u8's host checks
@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _scratch_need(bh, bw, Hn, Wn):
    """se_detail_u8's scratch for one box: the P operand, the residual operand and the GEMM's output, each rounded to 256 B."""
    r = lambda v: -(-v // 256) * 256
    Mp = r((Hn // 8 - 1) * (Wn // 8 - 1))
    Np = r(U.footprint(bw, Wn) * U.footprint(bh, Hn) * 3)
    return r(4 * Mp * Mp) + r(4 * Np * Mp) + r(4 * Mp * Np)


def _call(lib, hw, pitch, n=1, size=(64, 64), offs=(0, 0, 0, 0), agg=None, agg_off=0, scratch=None, need=None, photo=None):
    need = need if need is not None else ctypes.c_longlong(0)
    k = max(n, 1)
    L = ctypes.c_longlong
    arr = lambda v: (L * k)(*([v] * k))
    low_off, hole_off, attn_off, d_off = offs
    rc = lib.se_detail_u8(photo, arr(pitch), (ctypes.c_int * (2 * k))(*(list(hw) * k)), n, size[0], size[1], None, arr(low_off), None,
                          arr(hole_off), None, arr(attn_off), None, arr(d_off), agg, arr(agg_off) if agg_off is not None else None,
                          scratch, ctypes.byref(need), None)
    return rc, need.value, lib.se_last_error().decode() if rc else ""


def test_host_checks_and_scratch_query(lib):
    assert _call(lib, (64, 64), 192)[:2] == (0, _scratch_need(64, 64, 64, 64))
    assert _call(lib, (608, 400), 1200, size=(256, 256))[:2] == (0, _scratch_need(608, 400, 256, 256))
    assert _call(lib, (64, 64), 192, n=3)[:2] == (0, _scratch_need(64, 64, 64, 64))   # the boxes take turns with one scratch
    assert _call(lib, (64, 64), 192, n=0)[:2] == (0, 0)
    for hw, pitch, kw, msg in [((64, 64), 192, dict(n=-1), "n must be >= 0"),
                               ((64, 64), 192, dict(size=(60, 64)), "multiples of 8 and >= 16"),
                               ((64, 64), 192, dict(size=(8, 64)), "multiples of 8 and >= 16"),
                               ((64, 64), 192, dict(agg=ctypes.c_void_p(256), agg_off=None), "agg needs agg_off"),
                               ((0, 64), 192, {}, "box 0: sizes must be in [1, 65535]"),
                               ((64, 65536), 3 * 65536, {}, "box 0: sizes must be in [1, 65535]"),
                               ((64, 64), 191, {}, "box 0: the photo pitch is narrower than the box's row"),
                               ((7, 120), 360, dict(size=(256, 256)), "box 0: 7 x 120 is below 1/32 of the working size"),
                               ((64, 64), 192, dict(offs=(-1, 0, 0, 0)), "box 0: offsets must be >= 0 and aligned"),
                               ((64, 64), 192, dict(offs=(0, -1, 0, 0)), "box 0: offsets must be >= 0 and aligned"),
                               ((64, 64), 192, dict(offs=(0, 0, 2, 0)), "box 0: offsets must be >= 0 and aligned"),
                               ((64, 64), 192, dict(offs=(0, 0, 0, 1)), "box 0: offsets must be >= 0 and aligned"),
                               ((64, 64), 192, dict(agg=ctypes.c_void_p(256), agg_off=2), "box 0: offsets must be >= 0 and aligned")]:
        rc, _, err = _call(lib, hw, pitch, **kw)
        assert rc != 0 and msg in err, (hw, pitch, kw, err)
    hw = (ctypes.c_int * 2)(64, 64)
    assert lib.se_detail_u8(None, None, hw, 1, 64, 64, None, None, None, None, None, None, None, None, None, None, None,
                            ctypes.byref(ctypes.c_longlong(0)), None) != 0
    assert "null size / offset array" in lib.se_last_error().decode()
    # past the query: scratch too small or misaligned, then null pointers, all refused before anything is enqueued
    need = _scratch_need(64, 64, 64, 64)
    rc, _, err = _call(lib, (64, 64), 192, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(1))
    assert rc != 0 and "scratch holds 1 bytes, needs %d" % need in err
    rc, _, err = _call(lib, (64, 64), 192, scratch=ctypes.c_void_p(16), need=ctypes.c_longlong(need))
    assert rc != 0 and "scratch must be 256 B aligned" in err
    rc, _, err = _call(lib, (64, 64), 192, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(need))
    assert rc != 0 and "null photo / low / hole / attn / D" in err
    assert _call(lib, (64, 64), 192, n=0, scratch=ctypes.c_void_p(256), need=ctypes.c_longlong(0))[0] == 0

"""Mask previews on the CPU: DemoProcessor.predict_mask and EditSession.propose / accept with the Pillow flow and a fake
forward, against process_image(return_mask=True) and chains of plain edits; proposal lifetimes, argument errors and the
batch keys of the mask-only and soft-mask forwards."""
import threading

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200.serving import PREDICT, SOFT, Proposal
from tests.test_edit_session import _FakeProcessor, _fake_forward, _mask, _NoForward, _photo


class _PreviewFake(_FakeProcessor):
    """The fake forward of test_edit_session, plus its mask-only form (the soft mask is its bytes / 255, on the host here)
    and its form on soft masks (the result does not depend on the mask)."""

    def _run_batch(self, key, payloads):
        if key[-1] == PREDICT:
            out = []
            for img, sk in payloads:
                _, mk = _fake_forward(img, sk, None)
                out.append((mk[:, None].astype(np.float32) / 255, mk))
            return out
        if key[-1] == SOFT:
            return [np.ascontiguousarray(_fake_forward(img, sk, None)[0][..., ::-1]) for img, sk, _ in payloads]
        return super()._run_batch(key, payloads)


@pytest.fixture
def proc():
    p = _PreviewFake(_NoForward(), resize="host", region_size=(64, 48))
    yield p
    p.close()


M1 = [(50, 50, 60, 70)]
M2 = [(20, 20, 30, 30), (250, 150, 262, 160)]
M3 = [(100, 40, 140, 90), (130, 80, 170, 120)]
REGIONS = ["auto", "strokes", [(10, 10, 200, 150), (100, 50, 290, 190)], (3, 7, 61, 51), None]


def _same(a, b):
    return a.size == b.size and np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.parametrize("feather", [0, 8])
@pytest.mark.parametrize("region", REGIONS, ids=str)
def test_predict_mask_is_process_images_mask(proc, region, feather):
    img, mask = _photo(), _mask(300, 200, M3)
    want = proc.process_image(img, mask, region=region, return_mask=True, feather=feather)[1]
    assert _same(proc.predict_mask(img, mask, region=region, feather=feather), want)


@pytest.mark.parametrize("feather", [0, 8])
def test_propose_accept_chain_is_the_edit_chain(proc, feather):
    """propose gives edit's boxes and paste masks; accept makes edit's photo, result and undo snapshot."""
    img = _photo()
    a, b = proc.open_session(img), proc.open_session(img)
    steps = [(_mask(300, 200, rects), region) for rects in (M1, M2, M3) for region in REGIONS]
    for mask, region in steps:
        p = a.propose(mask, region=region, feather=feather)
        r = b.edit(mask, region=region, return_mask=True, feather=feather)
        assert isinstance(p, Proposal) and p.open and p.boxes == r.boxes, region
        assert all(_same(x, y) for x, y in zip(p.masks, r.masks)) and len(p.masks) == len(r.masks)
        got = a.accept(p, return_mask=True)
        assert not p.open and got.boxes == r.boxes
        assert all(_same(x, y) for x, y in zip(got.patches, r.patches))
        assert all(_same(x, y) for x, y in zip(got.masks, r.masks))
        assert _same(a.image(), b.image()) and a.jpeg() == b.jpeg()
    for _ in range(3):
        ua, ub = a.undo(), b.undo()
        assert ua[0] == ub[0] and all(_same(x, y) for x, y in zip(ua[1], ub[1]))
        assert _same(a.image(), b.image())
    assert a.accept(a.propose(_mask(300, 200, M1))).masks == [None]      # return_mask=False


def test_revised_accept_is_edit_with_the_edit_mask(proc):
    img = _photo()
    a, b = proc.open_session(img), proc.open_session(img)
    mask = _mask(300, 200, M3)
    em = _mask(300, 200, [(90, 30, 150, 100)], soft=True, seed=3)
    for region in ("strokes", None, "auto"):
        p = a.propose(mask, region=region, feather=8)
        got = a.accept(p, edit_masks=[em.crop(bx) for bx in p.boxes])
        r = b.edit(mask, edit_mask=em, region=p.boxes if region is not None else None, feather=8)
        assert got.boxes == r.boxes and got.masks == [None] * len(r.boxes)
        assert all(_same(x, y) for x, y in zip(got.patches, r.patches))
        assert _same(a.image(), b.image())


def test_masks_at_an_offset(proc):
    img = _photo()
    a, b = proc.open_session(img), proc.open_session(img)
    small = _mask(80, 60, [(10, 10, 30, 25)])
    p = a.propose(small, region="auto", offset=(150, 100), feather=4)
    r = b.edit(small, region="auto", offset=(150, 100), feather=4, return_mask=True)
    assert p.boxes == r.boxes and all(_same(x, y) for x, y in zip(p.masks, r.masks))
    a.accept(p)
    assert _same(a.image(), b.image())


@pytest.mark.parametrize("how", ["edit", "undo", "accept", "close"])
def test_proposals_are_invalidated(proc, how):
    s = proc.open_session(_photo())
    mask = _mask(300, 200, M1)
    s.edit(mask)
    p, q = s.propose(mask), s.propose(mask, region=None)
    assert p.open and q.open
    if how == "edit":
        s.edit(mask)
    elif how == "undo":
        s.undo()
    elif how == "accept":
        s.accept(q)
    else:
        s.close()
    assert not p.open and not q.open and p._soft is None and not s._proposals
    with pytest.raises(RuntimeError, match="closed"):
        s.accept(p)


def test_closing_a_proposal_leaves_the_others_open(proc):
    s = proc.open_session(_photo())
    mask = _mask(300, 200, M1)
    p, q = s.propose(mask), s.propose(mask, region=None)
    p.close()
    p.close()                                        # idempotent
    assert not p.open and p._soft is None and q.open and s._proposals == {q}
    with pytest.raises(RuntimeError, match="proposal is closed"):
        s.accept(p)
    s.accept(q)
    assert not q.open and not s._proposals


def test_a_proposal_is_accepted_once(proc):
    s = proc.open_session(_photo())
    p = s.propose(_mask(300, 200, M1))
    s.accept(p)
    with pytest.raises(RuntimeError, match="proposal is closed"):
        s.accept(p)


def test_argument_errors(proc):
    s, t = proc.open_session(_photo()), proc.open_session(_photo())
    mask = _mask(300, 200, M2)
    p = s.propose(mask, region="strokes")
    assert len(p.boxes) == 2
    with pytest.raises(TypeError, match="Proposal"):
        s.accept(p.boxes)
    with pytest.raises(ValueError, match="another session"):
        t.accept(p)
    with pytest.raises(ValueError, match="one per box"):
        s.accept(p, edit_masks=[mask.crop(p.boxes[0])])
    with pytest.raises(ValueError, match="one per box"):
        s.accept(p, edit_masks=mask)
    with pytest.raises(ValueError, match=r"edit_masks\[1\] must be an 'L' image of its box's size"):
        s.accept(p, edit_masks=[mask.crop(p.boxes[0]), Image.new("L", (5, 5))])
    with pytest.raises(ValueError, match=r"edit_masks\[0\]"):
        s.accept(p, edit_masks=[mask.crop(b).convert("RGB") for b in p.boxes])
    assert p.open                                    # a refused accept leaves the proposal open
    with pytest.raises(ValueError, match="feather"):
        s.propose(mask, feather=-1)
    with pytest.raises(ValueError, match="region"):
        s.propose(mask, region="nowhere")
    with pytest.raises(ValueError, match="does not fit"):
        s.propose(_mask(80, 60, M1), offset=(250, 0))
    with pytest.raises(ValueError, match="photo's size"):
        proc.predict_mask(_photo(), _mask(100, 100, M1), region="auto")
    with pytest.raises(ValueError, match="16x16"):
        proc.predict_mask(_photo(12, 40), _mask(12, 40, [(1, 1, 3, 3)]))
    s.close()
    with pytest.raises(RuntimeError, match="EditSession is closed"):
        s.propose(mask)


def test_mask_forwards_have_their_own_batch_keys(proc):
    img, mask = _photo(), _mask(300, 200, M3)
    s = proc.open_session(img)
    proc.process_image(img, mask, region="auto", return_mask=True)
    proc.process_image(img, mask, return_mask=True)
    s.edit(mask, region="strokes")
    s.edit(mask, edit_mask=mask, region=None)
    proc.predict_mask(img, mask, region="auto")
    proc.predict_mask(img, mask)
    s.accept(s.propose(mask, region="strokes"))
    s.accept(s.propose(mask, region=None))
    keys = [k for k, _ in proc.batcher.batches]
    assert keys[:4] == [("region", 64, 48), (200, 296), ("region", 64, 48), (200, 296, True)]
    assert keys[4:] == [("region", 64, 48, PREDICT), (200, 296, PREDICT), ("region", 64, 48, PREDICT),
                        ("region", 64, 48, SOFT), (200, 296, PREDICT), (200, 296, SOFT)]


def test_predicts_of_several_sessions_share_a_forward():
    proc = _PreviewFake(_NoForward(), resize="host", region_size=(64, 48), max_batch=3, max_wait_ms=10_000.0)
    img, mask = _photo(), _mask(300, 200, M3)
    ss = [proc.open_session(img) for _ in range(2)]
    got = [None] * 3

    def run(i):
        got[i] = ss[i].propose(mask, region="strokes") if i < 2 else proc.predict_mask(img, mask, region="strokes")

    ts = [threading.Thread(target=run, args=(i,)) for i in range(3)]
    [t.start() for t in ts]
    [t.join(timeout=10.0) for t in ts]
    assert proc.batcher.batches == [(("region", 64, 48, PREDICT), 3)]        # one forward, dispatched full
    assert got[0].boxes == got[1].boxes and _same(got[2], proc.process_image(img, mask, region="strokes", return_mask=True)[1])
    proc.close()
    assert not got[0].open and not got[1].open                               # closing the processor closes the sessions


def test_soft_masks_of_a_revised_accept_are_dropped(proc):
    s = proc.open_session(_photo())
    mask = _mask(300, 200, M1)
    p = s.propose(mask)
    s.accept(p, edit_masks=[Image.new("L", (b[2] - b[0], b[3] - b[1]), 200) for b in p.boxes])
    assert not p.open and not s._proposals

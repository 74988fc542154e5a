"""conv_c8_kernel at its tile edges and tile-walk geometries, against float64 with the per-element bounds of
tests/util_bounds.py, with the launch record (se_c8_log_enable) saying which form each launch ran.

A tile is 16 rows x 8 columns. Checked in bf16 and split-half fp32:

* Per operator, every gated conv / deconv of test_gpu_ops.py LAYER_CASES on tile grids of Ho in {1, 9, 15, 16, 17} rows
  and Wo in {1, 2, 3, 6, 7, 9} columns (the output grid; the input grid of a deconv): every partial-column residue the
  epilogue's column mask and the right-edge TMA fill meet. Every one of these sizes is accepted. The caller's output
  starts as a canary that the call must overwrite completely. This checks the entry's own output path, not the kernel:
  conv_c8 writes into a workspace buffer that the entry converts into the caller's tensor, so a pixel the kernel fails
  to write shows as a stale workspace value, and the bound check is what catches it.
* Per operator, walk geometries chosen against the device's SM count: a 1 x 1 tile grid with more than 2 x SMs images
  (a resident layer on two teams, a streamed layer on clusters), more column tiles than the grid has CTAs, a grid that is
  an exact multiple of an image's tiles, a step whose x, y and image coordinates all carry at once (found with the CPU
  model of tests/test_c8_tile_walk.py), and a phantom CTA on a wrapped cluster walk, with the 96->192 layer and with a
  one-box-per-tap layer. Every layer with a two-team form also runs two teams, in each precision its form exists for.
  The launch record must show the form and geometry a case is written for. A case that does not reach it is skipped
  with the reason, never passed.
* Through the forward: the stage checks of tests/util_stages.py on tapped forwards at eight sizes whose 1/2- and
  1/4-resolution maps reach every row residue mod 16 and column residue mod 8 the forward can produce, and one batch per
  mode large enough for every two-team form its plans allow, walking across images. These are the bound checks of the
  channel-blocked and space-to-depth epilogues, of outputs at a channel offset in a wider concat buffer and of the stem
  pair's split output.
* Coverage: some of the bound-checked cases above are re-run with the record on. These are the 17 x 9 edge grid of every
  layer, every walk case, the big batch and the 72 x 40 forward, with the same shapes and inputs. Together they must run
  every kC8Insts instantiation and both forms of every instantiation that has a two-team form. They must also reach a
  clustered launch with a phantom, one box per tap (also with 64-channel chunks), fused classes (2 and 4), every output
  layout, a channel offset and the stem pair's split.

Each bound check prints its max ratio.
"""
import ctypes
import math

import pytest
import torch

from sketchedit_b200 import _lib, synth
from sketchedit_b200.arch import layer_map, out_channels_after_gate
from sketchedit_b200.engine import _ptr, _stream
from tests import util_bounds as UB
from tests.test_c8_tile_walk import plan as walk_plan, walk as model_walk
from tests.test_gpu_forward_stages import _check, _inference
from tests.test_gpu_ops import LAYER_CASES
from tests.util_parity import engine

pytestmark = pytest.mark.gpu
PRECS = ["bf16", "fp32"]
GATED = [(n, l) for n, l, _, _ in LAYER_CASES if layer_map(n)[l].act is not None]
EDGE_HO = (1, 9, 15, 16, 17)
EDGE_WO = (1, 2, 3, 6, 7, 9)
CANARY = -12345.678


# --------------------------------------------------------------------------------------------- launch record
class C8Log:
    """with C8Log() as log: ... -> log.recs = [(label, {field: value})] of the conv_c8 launches inside (process-wide)."""

    def __enter__(self):
        self.lib = _lib.load()
        _lib.check(self.lib.se_c8_log_enable(1))
        self.recs = []
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        name = ctypes.create_string_buffer(128)
        rec = (ctypes.c_int * len(_lib.C8_REC))()
        for i in range(self.lib.se_c8_log_count()):
            _lib.check(self.lib.se_c8_log_get(i, name, len(name), rec))
            self.recs.append((name.value.decode(), dict(zip(_lib.C8_REC, list(rec)))))
        _lib.check(self.lib.se_c8_log_enable(0))
        return False

    def of(self, label):
        return [r for n, r in self.recs if n == label]


def instantiations():
    lib = _lib.load()
    info = (ctypes.c_int * len(_lib.C8_INST))()
    out = []
    for i in range(lib.se_c8_inst_count()):
        _lib.check(lib.se_c8_inst_info(i, info))
        out.append(dict(zip(_lib.C8_INST, list(info))))
    return out


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# --------------------------------------------------------------------------------------------- per operator
def _out_hw(spec, H, W):
    if spec.kind == "deconv":
        return 2 * H, 2 * W
    return (H + spec.stride - 1) // spec.stride, (W + spec.stride - 1) // spec.stride


def conv_canary(net, name, x, prec):
    """se_gated_conv_forward into an output filled with CANARY: the output, or None when the entry rejects the size. A call
    that succeeds must overwrite the whole output, and a rejected call must write none of it. This checks the entry's
    conversion into the caller's tensor. The kernel writes a workspace buffer that the entry then converts in full, so an
    output pixel conv_c8 drops shows up as a stale workspace value, which the bound check catches."""
    eng = engine()
    spec = layer_map(net)[name]
    B, _, H, W = x.shape
    Ho, Wo = _out_hw(spec, H, W)
    y = torch.full((B, out_channels_after_gate(spec), Ho, Wo), CANARY, device="cuda")
    xc = x.cuda().contiguous()
    try:
        _lib.check(eng.lib.se_gated_conv_forward(eng.h, net.encode(), name.encode(), _ptr(xc), B, H, W, _lib.PREC[prec],
                                                 _ptr(y), _stream()))
    except _lib.SketchEditB200Error:
        torch.cuda.synchronize()
        assert bool((y == CANARY).all()), (net, name, prec, H, W, "a rejected call wrote its output")
        return None
    y = y.cpu()
    assert not bool((y == CANARY).any()), (net, name, prec, H, W, "output elements left unwritten")
    return y


def grid_input(spec, Ho, Wo):
    """layer input whose tile grid is Ho x Wo (the output grid; a deconv's grid is its input)."""
    return (Ho, Wo) if spec.kind == "deconv" else UB.thin_input(spec, Ho, Wo)


def edge_input(net, name, Ho, Wo):
    spec = layer_map(net)[name]
    H, W = grid_input(spec, Ho, Wo)
    return UB.conv_input(net, name, 2, H, W, "unit", UB.stable_seed(net, name, "edge", Ho, Wo))


def walk_input(net, name, B, Ho, Wo):
    spec = layer_map(net)[name]
    H, W = grid_input(spec, Ho, Wo)
    return UB.conv_input(net, name, B, H, W, "unit", UB.stable_seed(net, name, "walk", B, Ho, Wo))


def bound_ratio(net, name, x, y, prec):
    r = UB.reference(net, name, x, prec)
    assert y.shape == r["Y"].shape, (y.shape, r["Y"].shape)
    return UB.max_ratio(y, r["Y"], UB.gated_bound(r, prec))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("net,name", GATED)
def test_tile_edges_within_bound(net, name, prec):
    worst, rejected = (0.0, None), []
    for Ho in EDGE_HO:
        for Wo in EDGE_WO:
            x = edge_input(net, name, Ho, Wo)
            with C8Log() as log:
                y = conv_canary(net, name, x, prec)
            if y is None:
                rejected.append((Ho, Wo))
                continue
            recs = log.recs
            assert recs and all(r["Ho"] == Ho and r["Wo"] == Wo and r["tiles_x"] == math.ceil(Wo / 8) for _, r in recs), recs
            worst = max(worst, (bound_ratio(net, name, x, y, prec), (Ho, Wo)))
    print("bound %s %s.%s tile edges: max ratio %.3g at %s" % (prec, net, name, worst[0], worst[1]))
    assert not rejected, (net, name, prec, "the entry rejects tile grids", rejected)
    assert worst[0] <= 1.0, (net, name, prec, worst)


def _divisor_grid(sms):
    """(tiles_x, tiles_y) of an image whose tile count divides sms (> 1 tile)."""
    for tx in range(2, sms + 1):
        if sms % tx == 0 and tx <= 64:
            return tx, 1
    return sms, 1


# one layer per instantiation with a two-team form, in each precision where it has one (split-half: 24->24 and the stems)
TEAM_LAYERS = {
    "bf16": [("M", "conv16"), ("M", "conv1"), ("M", "conv3"), ("G", "xconv3"), ("M", "conv2_downsample"),
             ("G", "xconv2_downsample"), ("M", "conv15_upsample_conv"), ("G", "xconv1"), ("G", "conv1")],
    "fp32": [("M", "conv16"), ("M", "conv1"), ("G", "xconv1"), ("G", "conv1")],
}


def walk_cases(sms, prec):
    """[(id, net, layer, B, Ho, Wo, check(rec) -> reason it missed or None)] of the walk geometries on an sms-SM device."""
    two = lambda r: None if r["teams"] == 2 else "one team"
    clus = lambda r: None if r["cluster"] == 2 else "not clustered"
    tx, ty = _divisor_grid(sms)
    per = tx * ty

    def all_of(*fs):
        def f(r):
            for g in fs:
                why = g(r)
                if why:
                    return why
            return None
        return f

    def one_tile(r):
        return None if r["tiles_x"] == r["tiles_y"] == 1 and r["N"] > 2 * sms else "not a 1 x 1 grid over > 2 x SMs images"

    def wide(r):
        return None if r["tiles_x"] > r["grid"] else "tiles_x %d <= grid %d" % (r["tiles_x"], r["grid"])

    def multiple(r):
        p = r["tiles_x"] * r["tiles_y"]
        return None if r["grid"] % p == 0 and r["grid"] >= p else "grid %d is not a multiple of %d tiles" % (r["grid"], p)

    def xyimg(r):
        ev = set()
        p = walk_plan("teams" if r["teams"] == 2 else "cluster" if r["cluster"] == 2 else "one", r["N"], r["tiles_x"],
                      r["tiles_y"], sms)
        if (p["grid"], p["teams"]) != (r["grid"], r["teams"]):
            return "the model plans grid %d / %d teams" % (p["grid"], p["teams"])
        model_walk(p, a_bufs=r["a_bufs"], ncls=r["ncls"], events=ev)
        return None if "xyimg_carry" in ev else "no step carries x, y and img at once"

    def phantom(r):
        return None if r["phantom"] and r["total_tiles"] > r["grid"] else "no phantom on a wrapped walk"

    def pertap(r):
        return None if r["mode"] == 1 else "not one box per tap"

    # 3 x 72 x 140: 5 x 18 tiles an image, 270 in all (two or three tiles a CTA on 132 SMs)
    teams = [("teams_%s_%s" % (n, l), n, l, 3, 72, 140, two) for n, l in TEAM_LAYERS[prec]]
    return teams + [
        ("one_tile_teams", "M", "conv16", 2 * sms + 3, 13, 7, all_of(two, one_tile)),
        ("one_tile_cluster", "M", "conv5", 2 * sms + 3, 3, 2, all_of(clus, one_tile)),
        ("wide_teams", "M", "conv16", 1, 17, 8 * (sms + 3) + 5, all_of(two, wide)),
        ("wide_cluster", "M", "conv5", 1, 17, 8 * (sms + 3) + 5, all_of(clus, wide)),
        ("multiple_teams", "M", "conv16", 3 * sms // per + 1, 16 * ty - 3, 8 * tx - 1, all_of(two, multiple)),
        ("xyimg_teams", "M", "conv16", 20, 16 * 3 - 5, 8 * 5 - 3, all_of(two, xyimg)),
        ("xyimg_s2d", "G", "xconv2_downsample", 20, 16 * 3 - 5, 8 * 5 - 3, xyimg),
        ("phantom_cluster", "M", "conv5", 5, 16, 8 * 53 - 1, all_of(clus, phantom)),
        ("phantom_pertap", "M", "conv9_atrous", 5, 13, 8 * 53 - 1, all_of(clus, phantom, pertap)),
    ]


WALK_IDS = [(c[0], prec) for prec in PRECS for c in walk_cases(132, prec)]


@pytest.mark.parametrize("case,prec", WALK_IDS)
def test_walk_geometries_within_bound(case, prec):
    _, net, name, B, Ho, Wo, check = {c[0]: c for c in walk_cases(sm_count(), prec)}[case]
    x = walk_input(net, name, B, Ho, Wo)
    with C8Log() as log:
        y = conv_canary(net, name, x, prec)
    assert y is not None, (case, prec, "rejected")
    recs = log.of(net + "." + name)
    assert recs, log.recs
    missed = [check(r) for r in recs]
    if any(missed):
        pytest.skip("%s %s did not run its form on %d SMs: %s" % (case, prec, sm_count(), missed))
    q = bound_ratio(net, name, x, y, prec)
    print("bound %s %s %s.%s B%d %dx%d: max ratio %.3g; %s" % (prec, case, net, name, B, Ho, Wo, q,
          [{k: r[k] for k in ("grid", "teams", "cluster", "tiles_x", "tiles_y", "N", "phantom", "mode")} for r in recs]))
    assert q <= 1.0, (case, prec, q)


# --------------------------------------------------------------------------------------------- through the forward
# H / 8 runs through every residue mod 8 and W / 8 through every residue mod 4: at 1/2 resolution (H / 2 rows, W / 2
# columns) and 1/4 resolution every row residue mod 16 and column residue mod 8 a forward can produce occurs
FORWARD_SHAPES = [(72, 40), (80, 48), (88, 56), (96, 64), (104, 40), (112, 48), (120, 56), (128, 64)]
BIG_BATCH = (5, 256, 256)   # 1/4 resolution: 32 tiles an image, 160 a launch; stems 2560


def forward_inputs(B, H, W):
    return synth.synth_inputs(B, H, W, seed=H * 5 + W + B)


def _forward_stages(prec, B, H, W):
    img, sk = forward_inputs(B, H, W)
    with C8Log() as log:
        T, pads, raw, io = _inference(prec, img, sk, {})
    _check("%s %dx%dx%d" % (prec, B, H, W), T, pads, raw, io, {}, prec)
    return log


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("H,W", FORWARD_SHAPES)
def test_forward_tile_residues_stages(prec, H, W):
    log = _forward_stages(prec, 1, H, W)
    assert {r["out_c8"] for _, r in log.recs} >= {1, 2}


@pytest.mark.parametrize("prec", PRECS)
def test_forward_big_batch_stages(prec):
    log = _forward_stages(prec, *BIG_BATCH)
    teams = sorted({n for n, r in log.recs if r["teams"] == 2})
    print("two-team launches %s: %s" % (prec, teams))
    # two teams walking across the images of the batch; in bf16 also with a step longer than one image (the 1/2- and
    # 1/4-resolution layers; split-half runs two teams on the full-resolution stems and 24->24 layers only)
    assert any(r["teams"] == 2 and r["N"] == BIG_BATCH[0] and r["total_tiles"] > r["grid"] for _, r in log.recs)
    if prec == "bf16":
        assert any(r["teams"] == 2 and r["grid"] > r["tiles_x"] * r["tiles_y"] for _, r in log.recs)
        assert any(r["teams"] == 2 for r in log.of("G.conv1+wconv1")), log.of("G.conv1+wconv1")


# --------------------------------------------------------------------------------------------- coverage
def test_every_instantiation_and_form_runs():
    # only shapes (and inputs) that the tests above hold to their bounds: the form of a launch depends on its shape alone
    insts = instantiations()
    sms = sm_count()
    with C8Log() as log:
        for prec in PRECS:
            for net, name in GATED:
                assert conv_canary(net, name, edge_input(net, name, 17, 9), prec) is not None
            for _, net, name, B, Ho, Wo, _ in walk_cases(sms, prec):
                assert conv_canary(net, name, walk_input(net, name, B, Ho, Wo), prec) is not None
            for shape in (BIG_BATCH, (1,) + FORWARD_SHAPES[0]):
                img, sk = forward_inputs(*shape)
                engine().inference(img.cuda(), sk.cuda(), precision=prec)
    recs = [r for _, r in log.recs]
    ran = {}
    for r in recs:
        ran.setdefault(r["inst"], set()).add(r["teams"])
    missing = []
    for i, k in enumerate(insts):
        want = {1, 2} if k["teams"] == 2 else {1}
        if ran.get(i, set()) != want:
            missing.append((i, k, sorted(ran.get(i, set()))))
    forms = {
        "clustered with a phantom": any(r["cluster"] == 2 and r["phantom"] for r in recs),
        "one box per tap": any(r["mode"] == 1 for r in recs),
        "one box per 64-channel chunk": any(r["mode"] == 1 and r["cpt"] > 1 for r in recs),
        "two fused classes": any(r["ncls"] == 2 for r in recs),
        "four fused classes": any(r["ncls"] == 4 for r in recs),
        "NHWC output": any(r["out_c8"] == 0 for r in recs),
        "channel-blocked output": any(r["out_c8"] == 1 for r in recs),
        "space-to-depth output": any(r["out_c8"] == 2 for r in recs),
        "channel offset": any(r["choff"] > 0 for r in recs),
        "stem pair split": any(r["blk_split"] > 0 for r in recs),
    }
    print("instantiations run: %s" % {i: sorted(t) for i, t in sorted(ran.items())})
    print("forms: %s" % forms)
    assert not missing, missing
    assert all(forms.values()), [k for k, v in forms.items() if not v]

"""The stage checks of tests/util_stages.py catch glue bugs that the end-to-end tolerances miss (CPU only).

Stage tensors are built from the oracle's intermediate tensors (oracle netG_forward / inference taps) with each mode's
storage emulated: bf16 round to nearest, the split-half pair, or fp32; the gated convs through the emulations of
tests/test_error_bounds.py. Unmutated, every check passes. Each mutation below, a plausible bug in a glue kernel, exceeds
its check. The same hi-only mutations, propagated through the fp32 oracle, move netG's outputs by far less than the 1e-3
end-to-end tolerance of the fp32 modes: only the stage checks can see them.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from tests import util_bounds as UB
from tests import util_stages as US
from tests.test_error_bounds import emulate
from tests.util_parity import weights

PRECS = ["bf16", "fp32", "fp32_direct"]


def hi_only(v):
    """a split-half store that drops the lo half: fp16 precision."""
    return UB.f16((v.float() * UB.ACT_SCALE).clamp(-65000.0, 65000.0)) / UB.ACT_SCALE


def truncate_bf16(v):
    return (v.float().contiguous().view(torch.int32) & -65536).view(torch.float32)


def _soft_mask(B, H, W):
    """a mask of eighths: the blends and products see values off {0, 1}."""
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    return (((yy // 4 + 3 * (xx // 4)) % 9).float() / 8.0).expand(B, 1, H, W).contiguous()


_RUN = {}


def _oracle_run():
    """inference at 64 x 64, batch 2, netG fed a soft mask (mask_bin_override), with every layer's output."""
    if not _RUN:
        WM, WG = weights()
        img, sk = synth.synth_inputs(2, 64, 64, seed=12)
        m = _soft_mask(2, 64, 64)
        taps = {}
        r = O.inference(WM, WG, img, sk, mask_bin_override=m, taps=taps)
        _RUN.update(img=img, sk=sk, m=m, taps=taps, r=r)
    return _RUN


def _store(v, prec, how=None):
    if how == "hi_only":
        return hi_only(v)
    if how == "truncate":
        return truncate_bf16(v)
    return US.store(v, prec)


def _head(net, name, x):
    _, w, b = UB.layer(net, name)
    return F.conv2d(x, w.float(), b.float(), padding=1)


def stages(prec, mutation=None, flags=None):
    """(T, pads, io) of the emulated forward; `mutation` names the glue bug."""
    flags = flags or {}
    R = _oracle_run()
    img, sk, m, taps = R["img"], R["sk"], R["m"], R["taps"]
    T, pads = {}, {}
    io = dict(netM=False, x=img, x2=img, mask=m, mask2=m, guide=sk)
    # packed network input of the coarse encoder
    e = US.packed_expect(io, flags, "in:G.conv1")
    T["in:G.conv1"] = _store(e, prec, {"pack8_hi_only": "hi_only", "pack8_bf16_truncate": "truncate"}.get(mutation))
    pads["in:G.conv1"] = torch.zeros(16)
    # the style stem on its input (the sketch channel zeroed under joint_train_inp; the mutation feeds the sketch)
    x_style = US.stem_inputs(io, flags)["G", "wconv1"]
    if mutation == "style_stem_sketch":
        x_style = torch.cat([x_style[:, :3], sk, x_style[:, 4:]], 1)
    T["in:G.wconv2_downsample"] = emulate("G", "wconv1", x_style, prec)
    # global pooling of the stored style map, broadcast into concat blocks 12-23
    T["in:G.pool"] = US.store(taps["netG.wconv10_atrous"], prec)
    v = T["in:G.pool"]
    pooled = v.mean((2, 3), keepdim=True) if flags.get("pool_type") == "avg" else v.amax((2, 3), keepdim=True)
    how = {"pool_hi_only": "hi_only", "broadcast_bf16_truncate": "truncate"}.get(mutation)
    bc = _store(pooled, prec, how).expand_as(v)
    enc = US.store(taps["netG.conv10_atrous"], prec)
    T["in:G.conv11"] = torch.cat([bc, enc] if mutation == "broadcast_swapped_halves" else [enc, bc], 1)
    # coarse head on its stored input, then the packed stage-2 input
    T["in:G.conv17"] = US.store(taps["netG.conv16"], prec)
    coarse = torch.tanh(_head("G", "conv17", UB.bf16(T["in:G.conv17"]) if prec == "bf16" else T["in:G.conv17"]))
    io["coarse"] = coarse
    if flags.get("no_mask_coarse"):
        blend = coarse
    elif mutation == "xnow_one_minus_m_once":
        blend = coarse * m + img * (1 - m)
    else:
        blend = coarse * m + img * (1 - m) * (1 - m)
    how = {"xnow_hi_only": "hi_only", "xnow_bf16_truncate": "truncate"}.get(mutation)
    T["in:G.xconv1"] = torch.cat([_store(blend, prec, how), torch.zeros(2, 5, 64, 64)], 1)
    pads["in:G.xconv1"] = torch.zeros(16)
    # contextual attention on the stored feature map and the pooled mask (float64, then stored)
    T["in:G.cam"] = US.store(taps["netG.pmconv6"], prec)
    T["in:G.cam.mask_s"] = F.avg_pool2d(m, 4)
    att = O.contextual_attention(T["in:G.cam"].double(), T["in:G.cam.mask_s"].double())[0].float()
    T["in:G.pmconv9"] = hi_only(att) if mutation == "attention_hi_only" else US.store(att, prec)
    if prec == "fp32":
        T["in:G.cam.f32"], T["out:G.cam.f32"] = T["in:G.cam"], att
    return T, pads, io


def _checks(prec, mutation=None, flags=None):
    flags = flags or {}
    T, pads, io = stages(prec, mutation, flags)
    return {"pack8": US.check_pack8(T, pads, io, flags, prec)["in:G.conv1"],
            "stem:G.wconv1": US.conv_ratio("G", "wconv1", US.stem_inputs(io, flags)["G", "wconv1"], T["in:G.wconv2_downsample"], prec),
            "pool": US.check_pool(T, flags, prec),
            "xnow": US.check_xnow(T, pads, io, flags, prec),
            **(US.check_attention(T, io, prec) if prec != "bf16" else {})}


@pytest.mark.parametrize("flags", [{}, {"pool_type": "avg"}])
@pytest.mark.parametrize("prec", PRECS)
def test_unmutated_stages_within_checks(prec, flags):
    q = _checks(prec, flags=flags)
    print("unmutated %s %s: %s" % (prec, flags, q))
    assert all(v <= 1.0 for v in q.values()), q


# (mutation, precision, check, flags)
MUTATIONS = [
    ("pool_hi_only", "fp32", "pool", {}),
    ("xnow_hi_only", "fp32", "xnow", {}),
    ("attention_hi_only", "fp32", "attention_glue", {}),
    ("pack8_hi_only", "fp32", "pack8", {}),
    ("pack8_bf16_truncate", "bf16", "pack8", {}),
    ("xnow_bf16_truncate", "bf16", "xnow", {}),
    ("broadcast_bf16_truncate", "bf16", "pool", {"pool_type": "avg"}),
    ("broadcast_swapped_halves", "bf16", "pool", {}),
    ("broadcast_swapped_halves", "fp32", "pool", {}),
    ("style_stem_sketch", "bf16", "stem:G.wconv1", {}),
    ("style_stem_sketch", "fp32", "stem:G.wconv1", {}),
    ("xnow_one_minus_m_once", "bf16", "xnow", {}),
    ("xnow_one_minus_m_once", "fp32", "xnow", {}),
    ("xnow_one_minus_m_once", "fp32_direct", "xnow", {}),
]


@pytest.mark.parametrize("mutation,prec,check,flags", MUTATIONS, ids=["%s-%s" % (m[0], m[1]) for m in MUTATIONS])
def test_mutation_exceeds_stage_check(mutation, prec, check, flags):
    q = _checks(prec, mutation, flags)
    print("%s (%s): %s max ratio %.3g" % (mutation, prec, check, q[check]))
    assert q[check] > 1.0, (mutation, q)


def test_threshold_at_half():
    """mask_bin = (mask > 0.5): a soft mask of exactly 0.5 stays 0; a `>=` threshold sets it."""
    soft = _oracle_run()["r"]["mask"].clone()
    soft[0, 0, 3, 5] = 0.5
    soft[1, 0, 60, 2] = 0.5
    assert US.check_threshold(soft, (soft > 0.5).float()) == 0.0
    assert US.check_threshold(soft, (soft >= 0.5).float()) > 1.0


def test_heads_emulated_within_checks():
    """fp32 heads on the oracle's stored decoder outputs satisfy the head bounds in every mode, and the public mask is
    the sigmoid of its head."""
    R = _oracle_run()
    taps, img, m = R["taps"], R["img"], R["m"]
    for prec in PRECS:
        T = {"in:M.conv_mask_17": US.store(taps["netM.conv_mask_16"], prec), "in:M.conv17": US.store(taps["netM.conv16"], prec),
             "in:G.conv17": US.store(taps["netG.conv16"], prec), "in:G.allconv17": US.store(taps["netG.allconv16"], prec)}
        op = lambda k: UB.bf16(T[k]) if prec == "bf16" else T[k]
        soft = torch.sigmoid(_head("M", "conv_mask_17", op("in:M.conv_mask_17")))
        fine = torch.tanh(_head("G", "allconv17", op("in:G.allconv17")))
        io = dict(netM=True, x=img, soft=soft, mask_bin=(soft > 0.5).float(),
                  mask_image=torch.tanh(_head("M", "conv17", op("in:M.conv17"))),
                  coarse=torch.tanh(_head("G", "conv17", op("in:G.conv17"))), fine=fine, composed=fine * soft + img * (1 - soft))
        q = US.check_heads(T, io, {}, prec)
        print("heads %s: %s" % (prec, q))
        assert all(v <= 1.0 for v in q.values()), (prec, q)
        io["composed"] = fine * soft + img * (1 - soft) * 1.0001
        assert US.check_heads(T, io, {}, prec)["composed"] > 1.0


# --------------------------------------------------------------------------------------------- what the end-to-end check sees
def _netG_hooked(WG, x, mask, guide, hook):
    """oracle netG_forward (default flags, x = x2, mask = mask2) with `hook(stage, tensor)` applied to the pooled style
    vector, the stage-2 input xnow and the attention output."""
    run = lambda names, t: O._chain("G", WG, names, t)
    xin = x * (1 - mask)
    a = run(US.ENC, torch.cat([xin, guide, mask], 1))
    s = run(["w" + n for n in US.ENC], torch.cat([x * mask, guide * 0, mask], 1))
    pooled = hook("pool", F.max_pool2d(s, kernel_size=s.shape[2:]))
    z = run(["conv" + n for n in US.DEC], torch.cat([a, pooled.expand_as(s)], 1))
    coarse = torch.tanh(z)
    xnow = hook("xnow", coarse * mask + xin * (1 - mask))
    xh = run(["x" + n for n in US.ENC], xnow)
    pm = run(US.PM, xnow)
    pm = hook("cam", O.contextual_attention(pm, F.avg_pool2d(mask, 4))[0])
    pm = run(["pmconv9", "pmconv10"], pm)
    fine = torch.tanh(run(["allconv" + n for n in US.DEC], torch.cat([xh, pm], 1)))
    return coarse, fine


def test_hi_only_glue_passes_end_to_end_tolerance():
    """netG 64 x 64, batch 2 (test_gpu_forward.test_netG's inputs): each split-half glue output stored hi-only moves the
    coarse and fine outputs by less than the fp32 modes' 1e-3, while its stage check above fails."""
    _, WG = weights()
    img, sk = synth.synth_inputs(2, 64, 64, seed=12)
    mask = torch.zeros(2, 1, 64, 64)
    mask[0, :, 16:40, 8:50] = 1
    mask[1, :, 30:60, 20:44] = 1
    with torch.no_grad():
        c0, f0 = _netG_hooked(WG, img, mask, sk, lambda k, t: t)
        r1, r2 = O.netG_forward(WG, img, img, mask, mask, sk)
        assert float((c0 - r1).abs().max()) == 0.0 and float((f0 - r2).abs().max()) == 0.0   # the restatement is the oracle
        for stage in ("pool", "xnow", "cam"):
            c, f = _netG_hooked(WG, img, mask, sk, lambda k, t: hi_only(t) if k == stage else t)
            dc, df = float((c - c0).abs().max()), float((f - f0).abs().max())
            print("%s stored hi-only: max change coarse %.2g, fine %.2g" % (stage, dc, df))
            assert max(dc, df) < 1e-3, (stage, dc, df)
            assert max(dc, df) > 0

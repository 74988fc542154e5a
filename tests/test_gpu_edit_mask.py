"""The forward on a caller-supplied edit mask (Engine.inference_with_mask / inference_with_mask_u8, se_forward_with_mask*) on
the GPU: identity with the plain forward on netM's own mask, parity with the oracle on unrelated masks, the uint8 codec,
batch independence and CUDA graphs, the module surface (forward, inference_stream, test.py) and the demo."""
import ctypes

import numpy as np
import pytest
import torch

from sketchedit_b200 import _lib, synth
from tests.test_gpu_configs import TOL, _model
from tests.util_edit_mask import inference_with_mask
from tests.util_parity import engine, maxdiff, weights

pytestmark = pytest.mark.gpu
PRECS = ("bf16", "fp32", "fp32_direct")
WANT = ("coarse", "fine", "mask_image", "mask_bin")
FLAG_SETS = {"avg_nocam": {"use_cam": False, "pool_type": "avg"},
             "nomask_flags": {"no_mask_cc": True, "no_mask_coarse": True, "joint_train_inp": False}}


def _identity(eng, prec, B, H, W, seed):
    img, sk = synth.synth_inputs(B, H, W, seed=seed)
    img, sk = img.cuda(), sk.cuda()
    comp, mask, ex = eng.inference(img, sk, precision=prec, want=WANT)
    comp2, ex2 = eng.inference_with_mask(img, sk, mask, precision=prec, want=WANT)
    assert torch.equal(comp2, comp)
    for k in WANT:
        assert torch.equal(ex2[k], ex[k]), k


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("shape", [(2, 64, 64), (1, 24, 40), (1, 128, 104)])
def test_netM_own_mask_reproduces_the_plain_forward(prec, shape):
    _identity(engine(), prec, *shape, seed=sum(shape))


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("flags", sorted(FLAG_SETS))
def test_netM_own_mask_reproduces_the_plain_forward_flag_sets(prec, flags):
    _identity(engine(**FLAG_SETS[flags]), prec, 1, 64, 64, seed=9)


def _blobs(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    m = torch.zeros(B, 1, H, W)
    for b in range(B):
        for _ in range(3):
            cy, cx = float(torch.rand(1, generator=g)) * H, float(torch.rand(1, generator=g)) * W
            r = 4 + float(torch.rand(1, generator=g)) * H / 4
            m[b, 0] = torch.maximum(m[b, 0], torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r)))
    return m


def _masks(B, H, W):
    half = torch.full((B, 1, H, W), 0.5)
    up, down = float(np.nextafter(np.float32(0.5), np.float32(1))), float(np.nextafter(np.float32(0.5), np.float32(0)))
    half[..., :, : W // 3] = up
    half[..., :, W // 3: 2 * W // 3] = down
    half[..., : H // 4, :] = 0.5
    return {"blobs": _blobs(B, H, W, 5), "zeros": torch.zeros(B, 1, H, W), "ones": torch.ones(B, 1, H, W), "half_ulp": half}


_ORACLE = {}


def _oracle(img, sk, name, em):
    if name not in _ORACLE:
        WM, WG = weights()
        _ORACLE[name] = inference_with_mask(WM, WG, img, sk, em)
    return _ORACLE[name]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", ["blobs", "zeros", "ones", "half_ulp"])
def test_oracle_parity_on_unrelated_masks(prec, name):
    img, sk = synth.synth_inputs(2, 64, 64, seed=21)
    em = _masks(2, 64, 64)[name]
    ref = _oracle(img, sk, name, em)
    comp, ex = engine().inference_with_mask(img.cuda(), sk.cuda(), em.cuda(), precision=prec, want=WANT)
    assert torch.equal(ex["mask_bin"].cpu(), (em > 0.5).float())                       # zero threshold flips, strict >
    for ours, k in ((comp, "composed"), (ex["coarse"], "coarse"), (ex["fine"], "fine"), (ex["mask_image"], "mask_image")):
        assert maxdiff(ours.cpu(), ref[k]) <= TOL[prec], (k, maxdiff(ours.cpu(), ref[k]))


def _u8_inputs(B, H, W, seed):
    rs = np.random.RandomState(seed)
    img_u8 = torch.from_numpy(rs.randint(0, 256, (B, H, W, 3), dtype=np.uint8))
    _, sk = synth.synth_inputs(B, H, W, seed=seed)
    sk_u8 = (sk[:, 0] * 255).to(torch.uint8)
    image = img_u8.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5)
    sketch = (sk_u8.float().div(255)[:, None] > 0).float()
    return img_u8, sk_u8, image, sketch


@pytest.mark.parametrize("prec", PRECS)
def test_uint8_entry_is_the_float_entry_on_decoded_inputs(prec):
    from oracle import sketchedit_oracle as O
    img_u8, sk_u8, image, sketch = _u8_inputs(2, 64, 96, 7)
    rs = np.random.RandomState(8)
    em_u8 = torch.from_numpy(rs.randint(0, 256, (2, 64, 96), dtype=np.uint8))
    em_u8[0, :8, :32] = torch.arange(256, dtype=torch.uint8).reshape(8, 32)             # every byte value present
    em_u8[1, 20:40, 30:70] = 255
    eng = engine()
    bgr = eng.inference_with_mask_u8(img_u8.cuda(), sk_u8.cuda(), em_u8.cuda(), precision=prec)
    em = em_u8.float().div(255)[:, None]
    comp, _ = eng.inference_with_mask(image.cuda(), sketch.cuda(), em.cuda(), precision=prec)
    g, _ = O.to_uint8_outputs(comp.cpu(), em)
    assert np.array_equal(bgr.cpu().numpy(), g.transpose(0, 2, 3, 1)[..., ::-1])
    # feeding back the mask inference_u8 wrote: the float entry on its decode v/255
    _, mk = eng.inference_u8(img_u8.cuda(), sk_u8.cuda(), precision=prec)
    bgr2 = eng.inference_with_mask_u8(img_u8.cuda(), sk_u8.cuda(), mk, precision=prec)
    comp2, _ = eng.inference_with_mask(image.cuda(), sketch.cuda(), mk.float().div(255)[:, None], precision=prec)
    g2, _ = O.to_uint8_outputs(comp2.cpu(), mk.cpu().float().div(255)[:, None])
    assert np.array_equal(bgr2.cpu().numpy(), g2.transpose(0, 2, 3, 1)[..., ::-1])


def test_batch_independence_256_bf16():
    B = 32
    img, sk = synth.synth_inputs(B, 256, 256, seed=90)
    em = _blobs(B, 256, 256, 91).cuda()
    img, sk = img.cuda(), sk.cuda()
    eng = engine()
    comp, ex = eng.inference_with_mask(img, sk, em, precision="bf16", want=("fine",))
    bad = []
    for i in range(B):
        c1, e1 = eng.inference_with_mask(img[i:i + 1], sk[i:i + 1], em[i:i + 1], precision="bf16", want=("fine",))
        if not (torch.equal(c1[0], comp[i]) and torch.equal(e1["fine"][0], ex["fine"][i])):
            bad.append(i)
    assert not bad, bad


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
def test_eager_captured_and_replayed_calls_agree(prec):
    """The same call signature three times runs eagerly, is captured into a CUDA graph, then replays it: same bytes and the
    same launch count each time, and fewer launches than the plain forward."""
    eng = engine()
    img_u8, sk_u8, image, sketch = _u8_inputs(2, 64, 64, 12)
    img_u8, sk_u8 = img_u8.cuda(), sk_u8.cuda()
    em_u8 = torch.from_numpy(np.random.RandomState(13).randint(0, 256, (2, 64, 64), dtype=np.uint8)).cuda()
    out = torch.empty(2, 64, 64, 3, device="cuda", dtype=torch.uint8)
    got, counts = [], []
    for _ in range(3):
        out.fill_(0)
        eng.inference_with_mask_u8(img_u8, sk_u8, em_u8, precision=prec, out=out)
        counts.append(eng.launches())
        got.append(out.cpu())
    assert all(torch.equal(g, got[0]) for g in got) and len(set(counts)) == 1, counts
    eng.inference_u8(img_u8, sk_u8, precision=prec)
    assert counts[0] < eng.launches(), (counts[0], eng.launches())
    # float entry through the C ABI with fixed buffers (so the call signature repeats)
    image, sketch, em = image.cuda(), sketch.cuda(), em_u8.float().div(255)[:, None]
    comp = torch.empty(2, 3, 64, 64, device="cuda")
    fine = torch.empty_like(comp)
    res, fcounts = [], []
    for _ in range(3):
        comp.zero_(); fine.zero_()
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        _lib.check(eng.lib.se_forward_with_mask(eng.h, p(image), p(sketch), p(em), 2, 64, 64, _lib.PREC[prec], p(comp), None, p(fine),
                                                None, None, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        fcounts.append(eng.launches())
        res.append((comp.cpu(), fine.cpu()))
    assert all(torch.equal(a, res[0][0]) and torch.equal(b, res[0][1]) for a, b in res) and len(set(fcounts)) == 1, fcounts
    eng.inference(image, sketch, precision=prec)
    assert fcounts[0] < eng.launches()


# ------------------------------------------------------------------------------------------------ module surface
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_module_forward_with_edit_mask(prec):
    img, sk = synth.synth_inputs(2, 64, 96, seed=31)
    em = _blobs(2, 64, 96, 32)
    model = _model(prec)
    with torch.no_grad():
        comp, m = model({"image": img, "mask": sk, "edit_mask": em}, mode="inference")
        vis = model({"image": img, "mask": sk, "edit_mask": em}, mode="visualize")
        _, _, plain = model.engine().inference(img.cuda(), sk.cuda(), precision=prec, want=("mask_image",))
    assert m.is_cuda and torch.equal(m.cpu(), em)
    want, _ = model.engine().inference_with_mask(img.cuda(), sk.cuda(), em.cuda(), precision=prec)
    assert torch.equal(comp, want)
    assert sorted(vis) == ["coarse", "composed", "fine", "mask", "maskim"]
    assert torch.equal(vis["mask"].cpu(), (em > 0.5).float())
    assert torch.equal(vis["composed"], comp)
    assert torch.equal(vis["maskim"], plain["mask_image"])
    assert maxdiff(vis["composed"].cpu(), (vis["fine"].cpu() * em + img * (1 - em))) <= 1e-6


def test_stream_mixing_edit_masks_equals_blocking_calls():
    model = _model("bf16")
    eng = model.engine()
    batches = []
    for i, b in enumerate((2, 2, 1, 2, 2)):
        img_u8, sk_u8, _, _ = _u8_inputs(b, 64, 64, 50 + i)
        d = {"image_u8": img_u8.pin_memory(), "mask_u8": sk_u8.pin_memory(), "tag": i}
        if i % 2 == 0:
            d["edit_mask_u8"] = torch.from_numpy(np.random.RandomState(i).randint(0, 256, (b, 64, 64), dtype=np.uint8)).pin_memory()
        batches.append(d)
    with torch.no_grad():
        want = []
        for d in batches:
            if "edit_mask_u8" in d:
                bgr = eng.inference_with_mask_u8(d["image_u8"].cuda(), d["mask_u8"].cuda(), d["edit_mask_u8"].cuda(), precision="bf16")
                want.append((bgr.cpu(), d["edit_mask_u8"].clone()))
            else:
                want.append(tuple(t.cpu() for t in eng.inference_u8(d["image_u8"].cuda(), d["mask_u8"].cuda(), precision="bf16")))
        got = [(a.clone(), b.clone(), d["tag"]) for a, b, d in model.inference_stream(iter(batches), uint8=True, with_data=True)]
        with pytest.raises(ValueError, match="uint8 mode only"):
            img, sk = synth.synth_inputs(1, 64, 64, seed=1)
            list(model.inference_stream(iter([{"image": img, "mask": sk, "edit_mask": torch.zeros(1, 1, 64, 64)}])))
    assert [t for _, _, t in got] == [0, 1, 2, 3, 4]
    for (ga, gb, _), (wa, wb) in zip(got, want):
        assert torch.equal(ga, wa) and torch.equal(gb, wb)


def test_test_py_round_trip_through_edit_mask_dir(tmp_path):
    """test.py writes masks with --output_mask_dir; a second run with --edit_mask_dir pointing at them writes PNGs equal to
    inference_with_mask_u8 on the dataset's tensors."""
    import cv2
    from PIL import Image

    import test as test_entry
    from options.test_options import TestOptions
    import data
    from tests.test_host_surface import _script_args
    idir, mdir, odir, omdir, odir2, cdir = (tmp_path / n for n in ("images", "edges", "out", "out_mask", "out2", "ckpt"))
    idir.mkdir(); mdir.mkdir(); (cdir / "celeb").mkdir(parents=True)
    WM, WG = weights()
    torch.save(WM, cdir / "celeb" / "latest_net_M.pth")
    torch.save(WG, cdir / "celeb" / "latest_net_G.pth")
    names = []
    for j, (H, W) in enumerate(((64, 64), (64, 64), (96, 64))):
        img, sk = synth.synth_inputs(1, H, W, seed=140 + j)
        Image.fromarray(((img[0].permute(1, 2, 0) + 1) / 2 * 255).round().clamp(0, 255).to(torch.uint8).numpy()).save(idir / ("im_%d.png" % j))
        Image.fromarray((sk[0, 0] * 255).to(torch.uint8).numpy()).save(mdir / ("im_%d.png" % j))
        names.append("im_%d" % j)
    (tmp_path / "list.txt").write_text("".join(n + ".png\n" for n in names))
    base = _script_args("test_celeb.sh") + ["--image_dirs", str(idir), "--mask_dirs", str(mdir), "--image_lists", str(tmp_path / "list.txt"),
                                            "--checkpoints_dir", str(cdir), "--precision", "bf16", "--nThreads", "0"]
    test_entry.main(base + ["--output_dir", str(odir), "--output_mask_dir", str(omdir)])
    argv2 = base + ["--output_dir", str(odir2), "--edit_mask_dir", str(omdir)]
    test_entry.main(argv2)
    eng = engine()
    for item in data.create_dataloader(TestOptions().parse(argv2)):
        n = item["path"][0]
        bgr = eng.inference_with_mask_u8(item["image_u8"].cuda(), item["mask_u8"].cuda(), item["edit_mask_u8"].cuda(), precision="bf16")
        got = cv2.imread(str(odir2 / n), cv2.IMREAD_COLOR)
        assert np.array_equal(got, bgr[0].cpu().numpy()), n
        assert np.array_equal(item["edit_mask_u8"][0].numpy(), cv2.imread(str(omdir / n), cv2.IMREAD_GRAYSCALE)), n


def test_demo_device_and_host_flows_agree():
    from PIL import Image

    from sketchedit_b200.serving import DemoProcessor
    model = _model("bf16")
    rs = np.random.RandomState(17)
    photo = Image.fromarray(rs.randint(0, 256, (481, 641, 3), dtype=np.uint8))
    sk = np.zeros((481, 641), np.uint8)
    sk[100:300, 200:204] = 255
    sketch = Image.fromarray(sk)
    edit = Image.fromarray(rs.randint(0, 256, (97, 131), dtype=np.uint8))   # not the floored size: resized like the sketch
    outs = {}
    for flow in ("device", "host"):
        proc = DemoProcessor(model, resize=flow, max_batch=4, max_wait_ms=1.0)
        try:
            plain, mk = proc.process_image(photo, sketch, return_mask=True)
            edited, mk_e = proc.process_image(photo, sketch, edit_mask=edit, return_mask=True)
            edited_only = proc.process_image(photo, sketch, edit_mask=edit)
        finally:
            proc.close()
        assert plain.size == edited.size == mk.size == (641, 481) and mk.mode == "L" and mk_e is edit
        assert np.array_equal(np.asarray(edited), np.asarray(edited_only))
        outs[flow] = [np.asarray(plain), np.asarray(mk), np.asarray(edited)]
    for a, b in zip(outs["device"], outs["host"]):
        assert np.array_equal(a, b)
    assert not np.array_equal(outs["device"][0], outs["device"][2])                   # the edit mask did change the result

"""CPU-side checks of the forward on a caller-supplied edit mask: the C ABI's error paths that need no device, the oracle
composition, the dataset's --edit_mask_dir and DemoProcessor's keying / return_mask with a fake forward."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sketchedit_oracle as O
from sketchedit_b200 import _lib, build, synth
from tests.test_host_surface import _script_args
from tests.util_edit_mask import inference_with_mask


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _err(lib):
    return lib.se_last_error().decode()


def test_abi_entry_points_reject_null_arguments_and_models(lib):
    p = ctypes.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    assert lib.se_forward_with_mask(None, p, p, None, 1, 64, 64, 0, p, None, None, None, None, None) != 0
    assert "null tensor" in _err(lib)
    assert lib.se_forward_with_mask(None, p, p, p, 1, 64, 64, 0, None, None, None, None, None, None) != 0
    assert "null tensor" in _err(lib)
    assert lib.se_forward_with_mask(None, p, p, p, 1, 64, 64, 0, p, None, None, None, None, None) != 0
    assert "model not finalized" in _err(lib)
    assert lib.se_forward_with_mask(None, p, p, p, 1, 60, 64, 0, p, None, None, None, None, None) != 0
    assert "multiples of 8" in _err(lib)
    assert lib.se_forward_with_mask_u8(None, p, p, None, 1, 64, 64, 0, p, None) != 0
    assert "null tensor" in _err(lib)
    assert lib.se_forward_with_mask_u8(None, p, p, p, 1, 64, 64, 0, None, None) != 0
    assert "null tensor" in _err(lib)
    h = ctypes.c_void_p()
    assert lib.se_model_create(ctypes.byref(h)) == 0
    assert lib.se_forward_with_mask_u8(h, p, p, p, 1, 64, 64, 0, p, None) != 0
    assert "model not finalized" in _err(lib)
    lib.se_model_destroy(h)


def test_engine_methods_reject_host_tensors(lib):
    from sketchedit_b200.engine import Engine
    eng = Engine()
    x = torch.zeros(1, 3, 64, 64)
    with pytest.raises(_lib.SketchEditB200Error, match="image must be a CUDA float32"):
        eng.inference_with_mask(x, x[:, :1], x[:, :1])
    u8 = torch.zeros(1, 64, 64, dtype=torch.uint8)
    with pytest.raises(_lib.SketchEditB200Error, match="image_u8 must be a contiguous CUDA uint8"):
        eng.inference_with_mask_u8(torch.zeros(1, 64, 64, 3, dtype=torch.uint8), u8, u8)


@pytest.mark.parametrize("flags", [{}, {"use_cam": False, "pool_type": "avg"},
                                   {"no_mask_cc": True, "no_mask_coarse": True, "joint_train_inp": False}])
def test_oracle_on_netM_own_mask_is_the_plain_forward(flags):
    WM, WG = synth.synth_state_dict("M"), synth.synth_state_dict("G")
    img, sk = synth.synth_inputs(1, 32, 48, seed=3)
    ref = O.inference(WM, WG, img, sk, **flags)
    got = inference_with_mask(WM, WG, img, sk, ref["mask"], **flags)
    forced = O.inference(WM, WG, img, sk, mask_bin_override=got["mask_bin"], **flags)
    for k in ("composed", "mask_bin", "coarse", "fine", "mask_image"):
        assert torch.equal(got[k], ref[k]) and torch.equal(got[k], forced[k]), k


def test_uint8_edit_mask_codec_round_trips():
    """v/255 (the decode of an edit mask byte) truncates back to v under the output codec (int)(m * 255), and it is above
    the 0.5 threshold exactly for v >= 128."""
    v = np.arange(256, dtype=np.float32)
    m = v / np.float32(255)
    assert np.array_equal((m * np.float32(255)).astype(np.int32), v.astype(np.int32))
    assert np.array_equal(m > np.float32(0.5), v >= 128)


def _dataset_args(tmp_path, sizes, edit_dir):
    from PIL import Image
    idir, mdir = tmp_path / "images", tmp_path / "edges"
    idir.mkdir(); mdir.mkdir()
    rng = np.random.RandomState(1)
    for n, (h, w) in sizes.items():
        Image.fromarray(rng.randint(0, 256, (h, w, 3), dtype=np.uint8)).save(idir / (n + ".png"))
        Image.fromarray(np.zeros((h, w), np.uint8)).save(mdir / (n + ".png"))
    (tmp_path / "list.txt").write_text("".join(n + ".png\n" for n in sizes))
    return _script_args("test_celeb.sh") + ["--gpu_ids", "-1", "--image_dirs", str(idir), "--mask_dirs", str(mdir),
                                            "--image_lists", str(tmp_path / "list.txt"), "--output_dir", str(tmp_path / "out"),
                                            "--batchSize", "1", "--nThreads", "0", "--edit_mask_dir", str(edit_dir)]


def test_dataset_reads_and_resizes_edit_masks(tmp_path):
    from PIL import Image
    from options.test_options import TestOptions
    import data
    edir = tmp_path / "edit"
    edir.mkdir()
    rng = np.random.RandomState(2)
    same = rng.randint(0, 256, (64, 48), dtype=np.uint8)
    small = rng.randint(0, 256, (20, 30), dtype=np.uint8)
    Image.fromarray(same).save(edir / "a.png")
    Image.fromarray(small).save(edir / "b.png")
    opt = TestOptions().parse(_dataset_args(tmp_path, {"a": (64, 48), "b": (40, 56)}, edir))
    items = {it["path"][0]: it for it in data.create_dataloader(opt)}
    want = {"a.png": same, "b.png": np.array(Image.fromarray(small).resize((56, 40)))}
    for name, it in items.items():
        assert torch.equal(it["edit_mask_u8"][0], torch.from_numpy(want[name]))
        assert it["edit_mask"].shape == (1, 1) + want[name].shape
        assert torch.equal(it["edit_mask"][0, 0], torch.from_numpy(want[name]).float().div(255))
    assert sorted(items) == ["a.png", "b.png"]


def test_dataset_names_a_missing_edit_mask(tmp_path):
    from options.test_options import TestOptions
    import data
    edir = tmp_path / "edit"
    edir.mkdir()
    opt = TestOptions().parse(_dataset_args(tmp_path, {"a": (64, 48)}, edir))
    with pytest.raises(FileNotFoundError, match=str(edir / "a.png")):
        next(iter(data.create_dataloader(opt)))


class _FakeModel:
    precision = "bf16"

    def engine(self):
        return None


def _fake_processor():
    """DemoProcessor whose forward (host flow) is replaced by a stand-in: the result is the resized photo itself and the
    predicted mask is a ramp, so shapes and routing can be checked without a device."""
    from sketchedit_b200.serving import DemoProcessor

    class Fake(DemoProcessor):
        def _run_batch(self, key, payloads):
            self.seen.append((key, [p[2] is not None for p in payloads]))
            H, W = key[:2]
            ramp = (np.arange(H * W) % 256).astype(np.uint8).reshape(H, W)
            return [(p[0].copy(), ramp if (p[3] and len(key) == 2) else None) for p in payloads]

    Fake.seen = []
    return Fake(_FakeModel(), resize="host", max_batch=4, max_wait_ms=1.0)


def test_demo_processor_keys_and_return_mask_with_a_fake_forward():
    from PIL import Image
    proc = _fake_processor()
    rng = np.random.RandomState(4)
    photo = Image.fromarray(rng.randint(0, 256, (481, 641, 3), dtype=np.uint8))
    sketch = Image.fromarray(np.zeros((481, 641), np.uint8))
    edit = Image.fromarray(rng.randint(0, 256, (100, 90), dtype=np.uint8))
    try:
        res = proc.process_image(photo, sketch)
        assert isinstance(res, Image.Image) and res.size == (641, 481)
        res, mk = proc.process_image(photo, sketch, return_mask=True)
        assert res.size == (641, 481) and mk.mode == "L" and mk.size == (641, 481)
        ramp = (np.arange(480 * 640) % 256).astype(np.uint8).reshape(480, 640)
        assert np.array_equal(np.asarray(mk), np.asarray(Image.fromarray(ramp).resize((641, 481))))
        res, mk = proc.process_image(photo, sketch, edit_mask=edit, return_mask=True)
        assert res.size == (641, 481) and mk is edit
        assert proc.process_image(photo, sketch, edit_mask=edit).size == (641, 481)
    finally:
        proc.close()
    assert [k for k, _ in proc.seen] == [(480, 640), (480, 640), (480, 640, True), (480, 640, True)]
    assert [e for _, e in proc.seen] == [[False], [False], [True], [True]]

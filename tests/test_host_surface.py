"""Host-side mirror of the reference's inference surface (no GPU): the test_celeb.sh command line parses, the module /
class / attribute names the reference's checkpoints and scripts rely on exist, and the dataset reads the reference's
list format."""
import os
import re
import shlex

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script_args(name):
    txt = open(os.path.join(ROOT, name)).read().replace("\\\n", " ")
    argv = shlex.split(txt)
    assert argv[:2] == ["python", "test.py"]
    return argv[2:]


def test_reference_command_lines_parse():
    from options.test_options import TestOptions
    for script in ("test_celeb.sh", "test_places.sh"):
        opt = TestOptions().parse(_script_args(script) + ["--gpu_ids", "-1"])
        assert opt.model == "editline2" and opt.netG == "deepfillc2" and opt.use_cam and opt.pool_type == "max"
        assert opt.isTrain is False and opt.gpu_ids == [] and opt.precision in ("bf16", "fp32")


def test_module_surface_and_state_dict_keys():
    """Same class names / constructor path / parameter names as the reference (strict checkpoint loading depends on it)."""
    from options.test_options import TestOptions
    import models
    from sketchedit_b200 import synth
    from sketchedit_b200.arch import NET_LAYERS
    opt = TestOptions().parse(_script_args("test_celeb.sh") + ["--gpu_ids", "-1"])
    opt.isSkip = True                                   # the reference's own escape hatch: do not look for checkpoints
    model = models.create_model(opt)
    assert type(model).__name__ == "EditLine2Model"
    assert type(model.netM).__name__ == "MDGenerator" and type(model.netG).__name__ == "DeepFillC2Generator"
    for net, mod in (("M", model.netM), ("G", model.netG)):
        keys = set(mod.state_dict().keys())
        want = set()
        for L in NET_LAYERS[net]:
            want |= {L.name + ".weight", L.name + ".bias"}
        assert keys == want, (net, sorted(keys ^ want)[:6])
        # the synthetic checkpoints load strictly into the UNMODIFIED reference (oracle/make_golden.py): same key set
        assert keys == set(synth.synth_state_dict(net).keys())
    for attr in ("forward", "inference_stream", "engine", "preprocess_input", "initialize_networks"):
        assert callable(getattr(model, attr))


def test_inference_requires_the_gpu_path():
    """No CPU fallback behind the module surface either."""
    import pytest
    from argparse import Namespace
    import models
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    opt = Namespace(gpu_ids=[], isTrain=False, isSkip=True, netG="deepfillc2", init_type="xavier", init_variance=0.02, use_cam=True,
                    pool_type="max", no_mask_cc=False, no_mask_coarse=False, joint_train_inp=True, model="editline2", precision="bf16")
    model = models.create_model(opt)
    data = {"image": torch.zeros(1, 3, 64, 64), "mask": torch.zeros(1, 1, 64, 64)}
    with pytest.raises(Exception):
        model(data, mode="inference")


def test_testimage_dataset_reads_the_reference_list_format(tmp_path):
    """data.create_dataloader on a list file: [-1,1] RGB image, sketch resized to the image and binarised with > 0,
    output name = list entry (reference data/testimage_dataset.py:60-111)."""
    import numpy as np
    from PIL import Image
    from options.test_options import TestOptions
    import data
    idir, mdir, odir = tmp_path / "images", tmp_path / "edges", tmp_path / "out"
    idir.mkdir(); mdir.mkdir()
    rng = np.random.RandomState(0)
    names = ["a_00", "b_01", "c_02"]
    imgs = {}
    for n in names:
        imgs[n] = rng.randint(0, 256, (64, 48, 3), dtype=np.uint8)
        Image.fromarray(imgs[n]).save(idir / (n + ".png"))
        edge = np.zeros((32, 24), np.uint8)               # half resolution: must be resized to the image size
        edge[8:12, 4:20] = 255
        Image.fromarray(edge).save(mdir / (n + ".png"))
    (tmp_path / "list.txt").write_text("".join(n + ".png\n" for n in names))
    argv = _script_args("test_celeb.sh") + ["--gpu_ids", "-1", "--image_dirs", str(idir), "--mask_dirs", str(mdir),
                                            "--image_lists", str(tmp_path / "list.txt"), "--output_dir", str(odir), "--batchSize", "1"]
    opt = TestOptions().parse(argv)
    loader = data.create_dataloader(opt)
    seen = []
    for item in loader:
        assert item["image"].shape == (1, 3, 64, 48) and item["mask"].shape == (1, 1, 64, 48)
        n = item["path"][0].replace(".png", "")
        want = torch.from_numpy(imgs[n]).permute(2, 0, 1).float().div(255).sub(0.5).div(0.5)
        assert torch.equal(item["image"][0], want)
        assert set(item["mask"].unique().tolist()) <= {0.0, 1.0} and item["mask"].sum() > 0
        seen.append(n)
    assert seen == names                                  # serial_batches: list order
    assert os.path.isdir(odir)


def test_bench_roofline_math_from_class_table():
    """bench.py's roofline block is recomputable from its per-class rows: frac = sum(algorithmic FLOPs of the tensor-core classes) / sum(their
    time) / peak; a class is 'hbm' bound when its bytes / HBM peak exceed its FLOPs / tensor peak; per-layer frac = sum(ideal) / sum(time)."""
    import bench
    peaks = {"hbm_gbs": 6000.0, "bf16_tflops": 1700.0, "bf16_tflops_sustained": 1500.0}
    classes = [
        {"name": "conv_c8_kernel|big", "tensor": 1, "launches": 20, "ms": 2 * 1.0, "flops_alg": 2 * 1.2e12, "flops_exec": 2 * 1.0e12, "bytes_alg": 2 * 1.0e8},
        {"name": "conv_c8_kernel|small", "tensor": 1, "launches": 4, "ms": 2 * 0.5, "flops_alg": 2 * 0.03e12, "flops_exec": 2 * 0.03e12, "bytes_alg": 2 * 1.2e9},
        {"name": "pack8_kernel|glue", "tensor": 0, "launches": 2, "ms": 2 * 0.1, "flops_alg": 0.0, "flops_exec": 0.0, "bytes_alg": 2 * 3.0e8},
    ]
    roof, rows = bench.roofline_from_classes(classes, 2, peaks, "test", 2.0)
    by = {r["class"]: r for r in rows}
    assert by["conv_c8_kernel|big"]["bound"] == "tensor" and abs(by["conv_c8_kernel|big"]["frac"] - 1.2e12 / 1500e12 / 1e-3) < 1e-9
    assert by["conv_c8_kernel|small"]["bound"] == "hbm" and abs(by["conv_c8_kernel|small"]["frac"] - (1.2e9 / 6000e9) / 0.5e-3) < 1e-9
    assert by["pack8_kernel|glue"]["bound"] == "hbm"
    tc_ms = 1.0 + 0.5
    assert abs(roof["achieved"] - (1.2e12 + 0.03e12) / (tc_ms * 1e-3) / 1e12) < 1e-6
    assert abs(roof["frac"] - roof["achieved"] / 1500.0) < 1e-12 and roof["peak"] == 1500.0
    assert abs(roof["kernel_share_of_step"] - tc_ms / 2.0) < 1e-12
    ideal = 1.2e12 / 1500e12 * 1e3 + 1.2e9 / 6000e9 * 1e3 + 3.0e8 / 6000e9 * 1e3
    assert abs(roof["per_layer_roofline_frac"] - ideal / 1.6) < 1e-9
    assert roof["dominant"]["class"] == "conv_c8_kernel|big"

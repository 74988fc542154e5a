"""CPU-side checks of the C ABI: the library loads without a GPU and exports every symbol
include/sketchedit_b200.h declares; the Python binding lists the same set."""
import ctypes
import os
import re

import pytest

from sketchedit_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    return build.build(verbose=False)


def _declared():
    src = open(os.path.join(ROOT, "include", "sketchedit_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(se_[A-Za-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert _declared() == sorted(_lib.SIGNATURES)


def test_library_exports_every_symbol(lib_path):
    lib = ctypes.CDLL(lib_path)
    for name in _declared():
        assert hasattr(lib, name), name


def test_abi_version_3_and_error_string(lib_path):
    lib = _lib.load()
    assert lib.se_abi_version() == 3
    assert isinstance(lib.se_last_error(), bytes)


def test_shape_validation_without_gpu(lib_path):
    """se_model_set_layer validates against the architecture table on the host (no device needed)."""
    import numpy as np
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.se_model_create(ctypes.byref(h)) == 0
    w = np.zeros((48, 4, 5, 5), np.float32)
    b = np.zeros((48,), np.float32)
    assert lib.se_model_set_layer(h, b"M", b"conv1", w.ctypes.data, b.ctypes.data, 48, 4, 5) == 0
    assert lib.se_model_set_layer(h, b"M", b"conv1", w.ctypes.data, b.ctypes.data, 48, 5, 5) != 0
    assert b"shape mismatch" in lib.se_last_error()
    assert lib.se_model_set_layer(h, b"M", b"nope", w.ctypes.data, b.ctypes.data, 48, 4, 5) != 0
    lib.se_model_destroy(h)


def test_taps_without_gpu(lib_path):
    """the activation-tap calls are host-side: a model that never ran a forward has no taps, with taps on or off, and an
    index past the end is an error."""
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.se_model_create(ctypes.byref(h)) == 0
    assert lib.se_taps_count(h) == 0
    assert lib.se_taps_enable(h, 1) == 0
    assert lib.se_taps_count(h) == 0
    assert lib.se_tap_info(h, 0, None, 0, None, None) != 0
    assert b"tap index" in lib.se_last_error()
    assert lib.se_taps_enable(h, 0) == 0
    lib.se_model_destroy(h)
    assert lib.se_taps_count(None) == -1


def test_c8_launch_record_without_gpu(lib_path):
    """the conv_c8 launch record and the instantiation table are host-side: empty with the record on or off, an index past
    the end is an error, and the table lists its 23 instantiations, nine with a two-team form, in both precisions."""
    lib = _lib.load()
    assert len(_lib.C8_REC) == 26 and len(_lib.C8_INST) == 6
    for on in (1, 0):
        assert lib.se_c8_log_enable(on) == 0
        assert lib.se_c8_log_count() == 0
        assert lib.se_c8_log_get(0, None, 0, None) != 0
        assert b"launch record index" in lib.se_last_error()
    info = (ctypes.c_int * len(_lib.C8_INST))()
    insts = []
    for i in range(lib.se_c8_inst_count()):
        assert lib.se_c8_inst_info(i, info) == 0
        insts.append(dict(zip(_lib.C8_INST, list(info))))
    assert lib.se_c8_inst_info(len(insts), info) != 0
    assert len(insts) == 23
    assert sum(k["teams"] == 2 for k in insts) == 9
    assert {k["f16"] for k in insts} == {0, 1} and all(k["teams"] in (1, 2) for k in insts)
    assert len({(k["nt"], k["f16"], k["r64"], k["m64"], k["r32"]) for k in insts}) == 23


def test_no_cpu_fallback(lib_path):
    """Without a CUDA device finalize must fail loudly, never fall back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from sketchedit_b200 import synth
    from sketchedit_b200.engine import Engine
    with pytest.raises(_lib.SketchEditB200Error):
        Engine.from_state_dicts(synth.synth_state_dict("M"), synth.synth_state_dict("G"))

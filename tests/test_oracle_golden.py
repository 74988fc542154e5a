"""Pin the CPU oracle against outputs of the UNMODIFIED reference (tests/golden/*.npz,
made by oracle/make_golden.py from the reference checkout; large arrays stored as a fixed sample)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import sketchedit_oracle as O
from sketchedit_b200 import synth
from tests.util_parity import golden

TOL = 2e-5   # fp32 vs fp32, different op order (attention form vs grouped conv)


def _load(path):
    z = np.load(path)
    if "image" in z:
        image, sketch = torch.from_numpy(z["image"]), torch.from_numpy(z["sketch"])
    else:   # uint8 inputs: reference data/testimage_dataset.py:89-103 preprocessing
        image = torch.from_numpy(z["image_u8"]).permute(2, 0, 1).float().div(255).sub(0.5).div(0.5)[None]
        sketch = (torch.from_numpy(z["sketch_u8"]).float().div(255) > 0).float()[None, None]
    flags = dict(eval(str(z["flags"])))
    return z, image, sketch, flags


@pytest.fixture(scope="module")
def weights():
    return synth.synth_state_dict("M"), synth.synth_state_dict("G")


@pytest.mark.parametrize("name", sorted(os.path.basename(p)[:-4] for p in
                                        glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz"))))
def test_oracle_matches_reference(name, weights, golden_dir):
    WM, WG = weights
    z, image, sketch, flags = _load(os.path.join(golden_dir, name + ".npz"))
    taps = {}
    r = O.inference(WM, WG, image, sketch, taps=taps, **flags)
    # the binarised mask must agree exactly (otherwise nothing downstream is comparable)
    ours_bin, ref_mask = golden(z, "mask", r["mask_bin"])
    assert int(((ref_mask > 0.5) != (ours_bin > 0.5)).sum()) == 0
    for key in ("composed", "mask", "coarse", "fine"):
        if key in z:
            ours, ref = golden(z, key, r[key])
            d = float((ours - ref).abs().max())
            assert d <= TOL, (name, key, d)
    for key in z.files:
        if key.startswith("tap:") and not key.endswith("@idx"):
            ours, ref = golden(z, key, taps[key[4:]])
            d = float((ours - ref).abs().max())
            scale = max(1.0, float(ref.abs().max()))
            assert d <= TOL * scale * 4, (name, key, d)


def test_uint8_conversion_truncates():
    """test.py:25-27: (x+1)/2*255 -> astype(uint8) truncates; mask*255 likewise."""
    comp = torch.tensor([[[[-1.0, 0.0, 0.999, 1.0]]]]).expand(1, 3, 1, 4)
    mask = torch.tensor([[[[0.0, 0.5, 0.999, 1.0]]]])
    g, m = O.to_uint8_outputs(comp, mask)
    assert g[0, 0, 0].tolist() == [0, 127, 254, 255]
    assert m[0, 0].tolist() == [0, 127, 254, 255]

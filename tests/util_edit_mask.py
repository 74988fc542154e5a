"""CPU oracle of the forward on a caller-supplied edit mask (Engine.inference_with_mask), composed from the oracle's
netM_forward / netG_forward: generate_fake (reference models/editline2_model.py:338-370) with netM's soft mask replaced by
the caller's.

    mask_inpaint = (edit_mask > 0.5)
    coarse, fine = netG(image, image, mask_inpaint, mask_inpaint, sketch)
    composed     = fine * edit_mask + image * (1 - edit_mask)
"""
import torch

from oracle import sketchedit_oracle as O


def inference_with_mask(WM, WG, image, sketch, edit_mask, **flags):
    """Returns dict(composed, mask_bin, coarse, fine, mask_image); mask_image is netM's image head (mode='visualize')."""
    with torch.no_grad():
        _, mask_image = O.netM_forward(WM, image, sketch)
        mask_bin = (edit_mask > 0.5).float()
        coarse, fine = O.netG_forward(WG, image, image, mask_bin, mask_bin, sketch, **flags)
        composed = fine * edit_mask + image * (1 - edit_mask)
    return dict(composed=composed, mask_bin=mask_bin, coarse=coarse, fine=fine, mask_image=mask_image)

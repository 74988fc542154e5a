"""List-file test dataset (reference data/testimage_dataset.py:13-111): each line of ``--image_lists`` names
an image under ``--image_dirs`` and a sketch under ``--mask_dirs``. The image becomes a [-1,1] RGB tensor,
the sketch an 'L' image resized to the image size and binarised with ``> 0``. Several ';'-separated
dir/list triples may be given. With ``--edit_mask_dir`` each item also carries the edit mask stored there under its
output name ('edit_mask_u8' [H,W] uint8, 'edit_mask' [1,H,W] = v/255), resized to the image like the sketch."""
import os

import numpy as np
import torch
import torch.utils.data
from PIL import Image


class TestImageDataset(torch.utils.data.Dataset):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        # same required flags and defaults as the reference (data/testimage_dataset.py:16-32)
        parser.add_argument("--image_dirs", type=str, required=True)
        parser.add_argument("--mask_dirs", type=str, required=True)
        parser.add_argument("--image_lists", type=str, required=True)
        parser.add_argument("--image_postfix", type=str, default=".jpg")
        parser.add_argument("--mask_postfix", type=str, default=".png")
        parser.add_argument("--output_labels", type=str, required=False, help="';'-separated prefixes for output names")
        parser.add_argument("--output_dir", type=str, required=True)
        parser.add_argument("--output_mask_dir", type=str, required=False)
        parser.add_argument("--edit_mask_dir", type=str, required=False,
                            help="run on these edit masks instead of the predicted ones: <dir>/<output name> as an 'L' image "
                                 "(what --output_mask_dir wrote), v/255, inpainted where v >= 128")
        return parser

    def initialize(self, opt):
        self.opt = opt
        os.makedirs(opt.output_dir, exist_ok=True)
        if opt.output_mask_dir is not None:
            os.makedirs(opt.output_mask_dir, exist_ok=True)
        labels = opt.output_labels.split(";") if opt.output_labels else None
        self.items = []
        for i, (idir, mdir, lst) in enumerate(zip(opt.image_dirs.split(";"), opt.mask_dirs.split(";"),
                                                  opt.image_lists.split(";"))):
            with open(lst) as f:
                stems = [ln.strip("\n").replace(opt.image_postfix, "") for ln in f]                   # every line is an entry, like the reference (:74-76)
            for s in stems:
                out = (labels[i] + "_" if labels else "") + s + opt.image_postfix
                self.items.append((os.path.join(idir, s + opt.image_postfix), os.path.join(mdir, s + opt.mask_postfix), out))

    def __len__(self):
        return len(self.items)

    def __getitem__(self, index):
        ipath, mpath, out = self.items[index]
        img = Image.open(ipath).convert("RGB")
        w, h = img.size
        image_u8 = torch.from_numpy(np.asarray(img, dtype=np.uint8).copy())
        image = image_u8.permute(2, 0, 1).float().div(255)
        image = (image - 0.5) / 0.5                                   # ToTensor + Normalize(0.5, 0.5)
        sk = Image.open(mpath).convert("L").resize((w, h))
        mask_u8 = torch.from_numpy(np.asarray(sk, dtype=np.uint8).copy())
        sketch = (mask_u8.float().div(255)[None] > 0).float()
        # 'image_u8' / 'mask_u8': the same pixels before ToTensor / Normalize, for the device-side codec path
        # (models.EditLine2Model.inference_stream(uint8=True)): 4x fewer bytes to copy
        item = {"image": image, "gt": image, "mask": sketch, "path": out, "image_u8": image_u8, "mask_u8": mask_u8}
        edir = getattr(self.opt, "edit_mask_dir", None)
        if edir is not None:
            # the mask a previous run wrote under --output_mask_dir (possibly corrected by hand) replaces netM's prediction
            epath = os.path.join(edir, out)
            if not os.path.isfile(epath):
                raise FileNotFoundError("edit mask %s not found (--edit_mask_dir expects one file per output name)" % epath)
            em = Image.open(epath).convert("L")
            if em.size != (w, h):
                em = em.resize((w, h))
            item["edit_mask_u8"] = torch.from_numpy(np.asarray(em, dtype=np.uint8).copy())
            item["edit_mask"] = item["edit_mask_u8"].float().div(255)[None]
        return item

"""List-file test dataset (reference data/testimage_dataset.py:13-111): each line of ``--image_lists`` names
an image under ``--image_dirs`` and a sketch under ``--mask_dirs``. The image becomes a [-1,1] RGB tensor,
the sketch an 'L' image resized to the image size and binarised with ``> 0``. Several ';'-separated
dir/list triples may be given. With ``--edit_mask_dir`` each item also carries the edit mask stored there under its
output name ('edit_mask_u8' [H,W] uint8, 'edit_mask' [1,H,W] = v/255), resized to the image like the sketch.

``files = True`` (test.py, when every input is a PNG) makes items carry the files instead of pixels, for the device
decoder of ``EditLine2Model.inference_stream(uint8=True)``; ``collate_files`` packs them into batches."""
import io
import os
from collections import namedtuple

import numpy as np
import torch
import torch.utils.data
from PIL import Image


class TestImageDataset(torch.utils.data.Dataset):
    files = False   # items carry the photo, sketch and edit-mask files (bytes) and their sizes, not pixels

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

    def edit_path(self, out):
        epath = os.path.join(self.opt.edit_mask_dir, out)
        if not os.path.isfile(epath):
            raise FileNotFoundError("edit mask %s not found (--edit_mask_dir expects one file per output name)" % epath)
        return epath

    def __getitem__(self, index):
        ipath, mpath, out = self.items[index]
        if self.files:
            item = {"path": out, "photo": _file(ipath), "sketch": _file(mpath)}
            if getattr(self.opt, "edit_mask_dir", None) is not None:
                item["edit"] = _file(self.edit_path(out))
            return item
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
            em = Image.open(self.edit_path(out)).convert("L")
            if em.size != (w, h):
                em = em.resize((w, h))
            item["edit_mask_u8"] = torch.from_numpy(np.asarray(em, dtype=np.uint8).copy())
            item["edit_mask"] = item["edit_mask_u8"].float().div(255)[None]
        return item


def _file(path):
    """(bytes, (h, w)) of an image file: the size from a PNG's IHDR, else from Pillow's header read."""
    with open(path, "rb") as f:
        data = f.read()
    from sketchedit_b200 import pngfile
    hw = pngfile.size(data)
    if hw is None:
        w, h = Image.open(io.BytesIO(data)).size
        hw = (h, w)
    return data, hw


PngFile = namedtuple("PngFile", "target index head offset length size data")
PngFile.__doc__ = """One file of a files-mode batch: target 'img', 'line' or 'edit'; index, its item in the batch; head, the
``pngfile.PngHead`` without its stream (None when the parser sends the file to Pillow); offset and length of its stream in
the batch's png_streams (its palette follows the stream); size, its (h, w); data, the file's bytes, which Pillow decodes
when the parser or the device decoder refuses the file."""


def collate_files(items):
    """A batch of files-mode items for ``inference_stream(uint8=True)``: 'path' as usual; 'png_size', the photos' (H, W);
    'png_streams', the joined IDAT payloads (and palette) of every file ``pngfile.parse`` sends to the device, packed in one
    uint8 tensor (the DataLoader pins it); 'png', a ``PngFile`` per file: photos, then sketches, then edit masks."""
    from sketchedit_b200 import pngfile
    sizes = {it["photo"][1] for it in items}
    if len(sizes) != 1:
        raise RuntimeError("the photos of a batch must have one size, got %s" % sorted(sizes))
    files = []
    for target, key in (("img", "photo"), ("line", "sketch"), ("edit", "edit")):
        for b, it in enumerate(items):
            if key not in it:
                continue
            data, hw = it[key]
            try:
                hd = pngfile.parse(data)
            except pngfile.Host:
                hd = None
            files.append((target, b, hd, hw, data))
    packed, offs, lens = pngfile.stage([f[2] for f in files if f[2] is not None], lambda n: torch.empty(n, dtype=torch.uint8))
    staged = iter(zip(offs, lens))
    files = [PngFile(t, b, None, 0, 0, hw, data) if hd is None else PngFile(t, b, hd._replace(stream=b""), *next(staged), hw, data)
             for t, b, hd, hw, data in files]
    return {"path": [it["path"] for it in items], "png_size": sizes.pop(), "png_streams": packed, "png": files}

"""Batch inference entry point -- same command line as the reference's test.py (reference test.py:12-37,
test_celeb.sh, test_places.sh): build the dataloader and the model from the flags, run
``model(data, mode='inference')`` per batch on the CUDA kernels, convert to uint8 (truncating, like
``astype(np.uint8)``), RGB->BGR, and write PNGs to --output_dir (masks to --output_mask_dir). PNG files are encoded on the
device, byte for byte as cv2.imwrite writes them.

``--edit_mask_dir D`` runs every entry on the mask ``D/<output name>`` instead of netM's prediction: write the masks with
--output_mask_dir, correct the wrong ones by hand, and rerun with --edit_mask_dir pointing at them."""
import os

import cv2
import torch

import data
import models
from options.test_options import TestOptions

# PNG inputs are decoded on the device only where tools/png_decode_bench.py measured it faster than the host loader at both
# 1 and 8 workers (H100 80GB HBM3, 700 W, steady images/s): 256² batch 16 (338 and 332 against 72 and 241), 256² batch 128
# (1203 and 1493 against 111 and 1381), 512² batch 16 (102 and 96 against 24 and 80). It lost at batch 4 with 8 workers
# (87 against 105 at 256², 26 against 44 at 512², 8.7 against 19.5 at 1024²) and at batch 1 (23 against 42): one warp
# decodes each file, so small batches and large photos leave most of the GPU idle while a file decodes serially.
PNG_DECODE_MIN_BATCH = 16
PNG_DECODE_MAX_PIXELS = 512 * 512


def _png_inputs(dataset, opt):
    """Whether test.py's loader hands the device decoder the files: every photo, sketch and edit mask is a PNG by its name
    (any case), batches hold PNG_DECODE_MIN_BATCH images or more, and no photo's IHDR is larger than PNG_DECODE_MAX_PIXELS."""
    from sketchedit_b200 import pngfile
    items = getattr(dataset, "items", None)
    edits = getattr(opt, "edit_mask_dir", None) is not None   # an edit mask is named like its output, items' third entry
    if not items or opt.batchSize < PNG_DECODE_MIN_BATCH or not all(
            p.lower().endswith(".png") for it in items for p in (it if edits else it[:2])):
        return False
    for ipath, _, _ in items:
        with open(ipath, "rb") as f:
            hw = pngfile.size(f.read(24))
        if hw is None or hw[0] * hw[1] > PNG_DECODE_MAX_PIXELS:
            return False
    return True


def main(argv=None):
    opt = TestOptions().parse(argv)
    dataloader = data.create_dataloader(opt)
    if _png_inputs(dataloader.dataset, opt):   # decoded on the device, pixel for pixel as Pillow opens them
        dataloader = data.loader_of(dataloader.dataset, opt, files=True)
    model = models.create_model(opt)
    model.eval()

    def batches():
        for i, batch in enumerate(dataloader):
            if i * opt.batchSize >= opt.how_many:
                break
            yield batch

    # the reference loop (test.py:20-37: model(data_i, mode='inference') -> uint8 -> BGR -> imwrite), pipelined: copies of the
    # neighbouring batches overlap the forward, and both codecs (normalise / binarise in, (x+1)/2*255 -> uint8 HWC BGR out) run
    # on the device, so 4 bytes per pixel cross PCIe in each direction instead of 16
    # When every output is a PNG, the files are encoded on the device too (byte for byte what cv2.imwrite writes) and only
    # they are downloaded; cv2 picks its encoder by the extension, case-insensitively, and stays the writer of other formats.
    mask_dir = getattr(opt, "output_mask_dir", None)
    png = None
    if all(out.lower().endswith(".png") for _, _, out in getattr(dataloader.dataset, "items", [("", "", "")])):
        png = ("image", "mask") if mask_dir is not None else ("image",)
    with torch.no_grad():
        for res, mk, batch in model.inference_stream(batches(), uint8=True, with_data=True, png=png):
            if png is None:
                res, mk = res.numpy(), mk.numpy()
            for b, path in enumerate(batch["path"]):
                print("process image... %s" % path)
                if png is None:
                    assert cv2.imwrite(os.path.join(opt.output_dir, path), res[b])
                else:
                    _write(os.path.join(opt.output_dir, path), res[b])
                if mask_dir is not None:
                    if png is None:
                        assert cv2.imwrite(os.path.join(mask_dir, path), mk[b])
                    else:
                        _write(os.path.join(mask_dir, path), mk[b])


def _write(path, data):
    with open(path, "wb") as f:
        f.write(data)


if __name__ == "__main__":
    main()

"""Batch inference entry point -- same command line as the reference's test.py (reference test.py:12-37,
test_celeb.sh, test_places.sh): build the dataloader and the model from the flags, run
``model(data, mode='inference')`` per batch on the CUDA kernels, convert to uint8 (truncating, like
``astype(np.uint8)``), RGB->BGR, and write PNGs to --output_dir (masks to --output_mask_dir).

``--edit_mask_dir D`` runs every entry on the mask ``D/<output name>`` instead of netM's prediction: write the masks with
--output_mask_dir, correct the wrong ones by hand, and rerun with --edit_mask_dir pointing at them."""
import os

import cv2
import torch

import data
import models
from options.test_options import TestOptions


def main(argv=None):
    opt = TestOptions().parse(argv)
    dataloader = data.create_dataloader(opt)
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
    with torch.no_grad():
        for bgr, mk, batch in model.inference_stream(batches(), uint8=True, with_data=True):
            bgr, mk = bgr.numpy(), mk.numpy()
            for b, path in enumerate(batch["path"]):
                print("process image... %s" % path)
                assert cv2.imwrite(os.path.join(opt.output_dir, path), bgr[b])
                if getattr(opt, "output_mask_dir", None) is not None:
                    assert cv2.imwrite(os.path.join(opt.output_mask_dir, path), mk[b])


if __name__ == "__main__":
    main()

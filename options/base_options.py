"""Command-line surface of test.py (reference options/base_options.py:16-186, options/test_options.py:5-19).

Same two-pass scheme as the reference: the base flags are parsed first with parse_known_args so that
``--model`` / ``--dataset_mode`` can inject their own flags (models.get_option_setter,
data.get_option_setter), then everything is parsed strictly. ``--gpu_ids`` is turned into a list and the
first id becomes the current CUDA device. The flags of the SPADE code base that nothing on this path reads
are still accepted so that existing command lines keep working."""
import argparse
import sys

import torch

import data
import models

_VESTIGIAL = {  # accepted and ignored (defaults inherited by the reference from the SPADE code base)
    "--norm_G": "spectralinstance", "--norm_D": "spectralinstance", "--norm_E": "spectralinstance",
    "--preprocess_mode": "scale_width_and_crop", "--dataroot": "./datasets/cityscapes/", "--ngf": 64, "--nef": 16,
    "--z_dim": 256, "--label_nc": 182, "--output_nc": 3, "--load_size": 256, "--crop_size": 256, "--aspect_ratio": 1.0,
    "--display_winsize": 256, "--max_dataset_size": sys.maxsize,
}
_VESTIGIAL_FLAGS = ["--contain_dontcare_label", "--no_flip", "--load_from_opt_file", "--cache_filelist_write",
                    "--cache_filelist_read", "--no_instance", "--use_vae"]


class BaseOptions:
    isTrain = False

    def initialize(self, parser):
        parser.add_argument("--name", type=str, default="label2coco", help="experiment name = checkpoint sub-directory")
        parser.add_argument("--joint_train_inp", action="store_true", help="zero the sketch channel of the style encoder")
        parser.add_argument("--gpu_ids", type=str, default="0", help="e.g. 0 or 0,1; the GPU path needs at least one GPU")
        parser.add_argument("--checkpoints_dir", type=str, default="./checkpoints")
        parser.add_argument("--model", type=str, default="pix2pix")
        parser.add_argument("--phase", type=str, default="train")
        parser.add_argument("--batchSize", type=int, default=1)
        parser.add_argument("--serial_batches", action="store_true")
        parser.add_argument("--nThreads", default=0, type=int, help="# dataloader workers")
        parser.add_argument("--netG", type=str, default="spade", help="generator class prefix (deepfillc2)")
        parser.add_argument("--init_type", type=str, default="xavier")
        parser.add_argument("--init_variance", type=float, default=0.02)
        for flag, default in _VESTIGIAL.items():
            parser.add_argument(flag, type=type(default), default=default, help=argparse.SUPPRESS)
        for flag in _VESTIGIAL_FLAGS:
            parser.add_argument(flag, action="store_true", help=argparse.SUPPRESS)
        return parser

    def gather_options(self, argv=None):
        if argv is not None:      # option setters re-parse sys.argv (like the reference): keep them consistent
            sys.argv = [sys.argv[0]] + list(argv)
        parser = argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)
        parser = self.initialize(parser)
        opt, _ = parser.parse_known_args(argv)
        parser = models.get_option_setter(opt.model)(parser, self.isTrain)
        opt, _ = parser.parse_known_args(argv)
        parser = data.get_option_setter(opt.dataset_mode)(parser, self.isTrain)
        self.parser = parser
        return parser.parse_args(argv)

    def print_options(self, opt):
        lines = ["----------------- Options ---------------"]
        for k, v in sorted(vars(opt).items()):
            default = self.parser.get_default(k)
            note = "" if v == default else "\t[default: %s]" % str(default)
            lines.append("{:>25}: {:<30}{}".format(str(k), str(v), note))
        lines.append("----------------- End -------------------")
        print("\n".join(lines))

    def parse(self, argv=None):
        opt = self.gather_options(argv)
        opt.isTrain = self.isTrain
        self.print_options(opt)
        ids = [int(s) for s in opt.gpu_ids.split(",") if int(s) >= 0]
        opt.gpu_ids = ids
        if ids:
            torch.cuda.set_device(ids[0])
        assert not ids or opt.batchSize % len(ids) == 0, \
            "Batch size %d is wrong. It must be a multiple of # GPUs %d." % (opt.batchSize, len(ids))
        self.opt = opt
        return opt

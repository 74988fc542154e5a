"""Dataset factory (reference data/__init__.py:12-49): ``--dataset_mode X`` -> class ``XDataset`` in
``data/X_dataset.py``; ``create_dataloader`` wraps it in a torch DataLoader (no shuffle at test time)."""
import importlib

import torch.utils.data


def find_dataset_using_name(dataset_name):
    module = importlib.import_module("data.%s_dataset" % dataset_name)
    wanted = (dataset_name.replace("_", "") + "dataset").lower()
    for attr, obj in vars(module).items():
        if attr.lower() == wanted and isinstance(obj, type) and issubclass(obj, torch.utils.data.Dataset):
            return obj
    raise ValueError("data/%s_dataset.py defines no Dataset subclass named like %r" % (dataset_name, wanted))


def get_option_setter(dataset_name):
    return find_dataset_using_name(dataset_name).modify_commandline_options


def create_dataloader(opt):
    dataset = find_dataset_using_name(opt.dataset_mode)()
    dataset.initialize(opt)
    print("dataset [%s] of size %d was created" % (type(dataset).__name__, len(dataset)))
    return loader_of(dataset, opt)


def loader_of(dataset, opt, files=False):
    """The DataLoader of ``dataset`` under opt's settings. files=True puts a TestImageDataset in its files mode (items carry
    the PNG files, batches come from ``collate_files``), for the device decoder of ``inference_stream(uint8=True)``."""
    collate = None
    if files:
        from data.testimage_dataset import collate_files
        dataset.files, collate = True, collate_files
    return torch.utils.data.DataLoader(dataset, batch_size=opt.batchSize, shuffle=not opt.serial_batches,
                                       num_workers=int(opt.nThreads), drop_last=opt.isTrain,
                                       pin_memory=True, collate_fn=collate)

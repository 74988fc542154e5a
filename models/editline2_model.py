"""EditLine2Model, inference subset (reference models/editline2_model.py:49-147, 184-242, 338-370).

``forward(data, mode)`` with mode 'inference' returns ``(composed_image, mask)`` exactly like the
reference: netM predicts the edit mask from (image, sketch), the mask is binarised at 0.5, netG inpaints,
and the result is blended with the SOFT mask. All of it is one C-ABI call (``se_forward_inference``) on the
CUDA kernels; tensors in ``data`` may live on the CPU (they are copied to the GPU like the reference's
``preprocess_input`` does) and the outputs are CUDA tensors. Training modes are out of scope.

An optional ``data['edit_mask']`` [B,1,H,W] replaces netM's prediction (mask revising): 'inference' then returns
``(composed, edit_mask)`` and 'visualize' the same five keys with ``mask`` = (edit_mask > 0.5)."""
import torch

import models.networks as networks
import util.util as util


class EditLine2Model(torch.nn.Module):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        networks.modify_commandline_options(parser, is_train)
        parser.add_argument("--precision", default="bf16", choices=("bf16", "fp32", "fp32_direct"),
                            help="GPU arithmetic: bf16 tensor-core path, fp32-parity arithmetic on the tensor cores (split-half fp16), "
                                 "or its fp32 CUDA-core cross-check")
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        if getattr(opt, "isTrain", False):
            raise NotImplementedError("only the inference path is implemented on the GPU")
        self.precision = getattr(opt, "precision", "bf16")
        self.netM, self.netG, self.netD = self.initialize_networks(opt)
        self._engine = None
        self._engine_key = None

    def use_gpu(self):
        return len(self.opt.gpu_ids) > 0

    def initialize_networks(self, opt):
        netG = networks.define_G(opt)
        saved = opt.netG
        opt.netG = "MD"
        netM = networks.define_G(opt)
        opt.netG = saved
        if not hasattr(opt, "isSkip"):           # same escape hatch as the reference (:195)
            netG = util.load_network(netG, "G", opt.which_epoch, opt)
            netM = util.load_network(netM, "M", opt.which_epoch, opt)
        return netM, netG, None

    def engine(self):
        from sketchedit_b200.engine import Engine
        key = self.netM._weights_key() + self.netG._weights_key()
        if self._engine is None or key != self._engine_key:
            eng = Engine()
            eng.load_state_dict("M", self.netM.state_dict())
            eng.load_state_dict("G", self.netG.state_dict())
            self.netG._configure_engine(eng)
            eng.finalize()
            self._engine, self._engine_key = eng, key
        return self._engine

    def preprocess_input(self, data):
        dev = torch.device("cuda")
        image = data["image"].to(dev, torch.float32, non_blocking=True)
        line = data["mask"].to(dev, torch.float32, non_blocking=True)
        return image, line

    def forward(self, data, mode, is_real_im=True):
        image, line = self.preprocess_input(data)
        if mode not in ("inference", "visualize"):
            raise ValueError("|mode| is invalid or training-only: %r" % (mode,))
        want = ("coarse", "fine", "mask_image", "mask_bin") if mode == "visualize" else ()
        if data.get("edit_mask") is None:
            composed, mask, ex = self.engine().inference(image, line, precision=self.precision, want=want)
        else:
            # data['mask'] is the sketch, as in the reference: netG inpaints edit_mask > 0.5 and the result is blended with
            # edit_mask itself
            mask = data["edit_mask"].to(image.device, torch.float32, non_blocking=True)
            composed, ex = self.engine().inference_with_mask(image, line, mask, precision=self.precision, want=want)
        if mode == "inference":
            return composed, mask
        # reference :134-145 -- 'mask' is the BINARISED mask netG inpaints (mask_inpaint), 'composed' is blended
        # with the SOFT mask exactly like mode='inference'
        return {"mask": ex["mask_bin"], "maskim": ex["mask_image"], "coarse": ex["coarse"], "fine": ex["fine"],
                "composed": composed}

    def inference_stream(self, loader, depth=2, pinned_ring=True, gather=None, uint8=False, with_data=False, png=None):
        """Pipelined form of ``for data in loader: model(data, mode='inference')`` for throughput serving.

        Yields ``(composed, mask)`` per batch, in order, as PINNED CPU tensors (views of one packed [B,4,H,W] host
        buffer). The host->device copy of batch i+1 and the device->host copy of batch i-1 run on their own CUDA
        streams while batch i computes (``depth`` device buffers per tensor), so a step costs max(copy, compute)
        instead of their sum. Batches whose input tensors are in pinned memory (DataLoader(pin_memory=True)) overlap fully.

        uint8=True: the reference's host-side codecs run on the device (``Engine.inference_u8``): a batch supplies
        ``data['image_u8']`` [B,H,W,3] RGB uint8 and ``data['mask_u8']`` [B,H,W] uint8 (what the dataset holds before
        ToTensor/Normalize, reference data/testimage_dataset.py:89-103) and the results are ``(bgr_u8 [B,H,W,3], mask_u8
        [B,H,W])`` exactly as test.py:25-35 writes them: 4x fewer bytes over PCIe in each direction. A batch that also
        carries ``data['edit_mask_u8']`` [B,H,W] uint8 runs on that mask instead of netM's prediction
        (``Engine.inference_with_mask_u8``) and its mask result is a copy of the supplied bytes; batches with and without
        one may be mixed. Float mode rejects batches that carry an edit mask.

        uint8 mode also takes batches of PNG files (``data.testimage_dataset.collate_files``: 'png_streams', 'png', 'png_size'
        in place of the pixels): their compressed streams are uploaded from pinned memory and decoded on the input stream
        into the batch's input buffers (``engine.png_decode_u8_packed``), sketches and edit masks of another size than their
        photo resized to it as Pillow's ``.resize`` does. The host reads the decoder's per-file status once the decode is
        done (the previous batch's forward is already queued by then) and uploads Pillow's pixels of the files the parser or
        the decoder sent to it before the batch's forward.

        with_data=True: yield ``(out0, out1, data)`` (test.py needs the batch's output paths).

        png=("image",) or ("image", "mask") (uint8 mode): each batch's BGR results (and masks) are encoded on the device after
        the forward, on the compute stream (``engine.png_encode_u8_packed``), and only the files are downloaded: each result is
        a list of ``bytes`` per image, ``cv2.imencode(".png", x)[1]`` of the array uint8 mode yields, and the mask result is
        None without "mask". The lengths leave the device with the batch; the bytes are downloaded when the batch is drawn,
        while later batches compute.

        pinned_ring=True (default): results are views of a ring of ``depth + 2`` pinned buffers handed out round robin. The
        copy of batch i + depth - 1 is already in flight when result i is drawn, so a result stays intact while at most
        ``depth`` further results are drawn (you may hold the newest ``depth + 1``; consume or ``.clone()`` older ones);
        pinned_ring=False allocates fresh pinned tensors for every batch (a cudaHostAlloc per batch when the host
        allocator cannot recycle, which costs more than the copy itself).

        gather: a ``sketchedit_b200.parallel.OutputGather`` (data-parallel serving, one process per GPU; float mode): every
        batch's packed outputs are written into this rank's slice of the gather buffer and all-gathered over NCCL (async, in
        place) before this rank's shard is copied to the host; all ranks must feed equal batch sizes."""
        import collections

        from sketchedit_b200 import engine as E
        eng = self.engine()
        if png is not None:
            png = tuple(png)
            if not uint8 or png not in (("image",), ("image", "mask")):
                raise ValueError('png= needs uint8=True and is ("image",) or ("image", "mask") (got %r)' % (png,))
        if gather is not None and (gather.depth != depth or uint8):
            raise ValueError("gather= needs float mode and a ring depth equal to the stream depth (%d)" % depth)
        dev = torch.device("cuda")
        cur = torch.cuda.current_stream()
        s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()
        s_files = torch.cuda.Stream() if png else None   # file downloads: behind nothing but the batch's own encode
        slots = [None] * depth
        pending = collections.deque()
        ring = {}        # (B, H, W) -> [buffers, results handed out so far]

        def new_host(B, H, W):
            if uint8:
                return (torch.empty(B, H, W, 3, dtype=torch.uint8, pin_memory=True), torch.empty(B, H, W, dtype=torch.uint8, pin_memory=True))
            packed = torch.empty(B, 4, H, W, pin_memory=True)
            return (packed,)

        def host_out(B, H, W):
            if not pinned_ring:
                return new_host(B, H, W)
            entry = ring.setdefault((B, H, W), [[], 0])
            bufs, count = entry
            if len(bufs) < depth + 2:
                bufs.append(new_host(B, H, W))
            entry[1] = count + 1
            return bufs[count % (depth + 2)]       # strict round robin per shape: 0, 1, .., depth+1, 0, 1, ..

        def drain_one():
            host, ev, data = pending.popleft()
            ev.synchronize()
            if png:   # host: (files buffer, offsets, pinned lengths, images)
                out, offs, lens, B = host
                with torch.cuda.stream(s_files):
                    files = E.download_files(out, offs, lens.tolist())
                res = (files[:B], files[B:] if len(png) == 2 else None)
            else:
                res = (host[0], host[1]) if uint8 else (host[0][:, :3], host[0][:, 3:4])
            return res + (data,) if with_data else res

        in_keys = ("image_u8", "mask_u8") if uint8 else ("image", "mask")
        for i, data in enumerate(loader):
            files = data.get("png") if uint8 else None
            if files is not None:
                B, (H, W) = len(data["path"]), data["png_size"]
                edit_h = True if any(f.target == "edit" for f in files) else None
            else:
                img_h, line_h = data[in_keys[0]], data[in_keys[1]]
                edit_h = data.get("edit_mask_u8") if uint8 else None
                B, H, W = (img_h.shape[0], img_h.shape[1], img_h.shape[2]) if uint8 else (img_h.shape[0], img_h.shape[2], img_h.shape[3])
            if not uint8 and (data.get("edit_mask") is not None or data.get("edit_mask_u8") is not None):
                raise ValueError("inference_stream runs batches with an edit mask in uint8 mode only (uint8=True, data['edit_mask_u8'])")
            if not uint8 and data.get("png") is not None:
                raise ValueError("inference_stream runs batches of PNG files in uint8 mode only (uint8=True)")
            slot = slots[i % depth]
            fresh = slot is None or slot["shape"] != (B, H, W) or (edit_h is not None and "edit" not in slot)
            if slot is None or slot["shape"] != (B, H, W):
                if slot is not None:   # shape change (ragged last batch): let the old buffers' users finish first
                    slot["ev_comp"].synchronize()
                    slot["ev_out"].synchronize()
                if uint8:
                    u8 = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.uint8)
                    bufs = {"img": u8(B, H, W, 3), "line": u8(B, H, W), "out": (u8(B, H, W, 3), u8(B, H, W))}
                    if png:   # the files of the batch: images, then masks
                        offs, total = E._aligned_offsets([E.png_max_bytes(H, W, 3)] * B + [E.png_max_bytes(H, W, 1)] * B * (len(png) - 1))
                        bufs["png"] = (u8(total), offs)
                else:
                    f32 = lambda c: torch.empty(B, c, H, W, device=dev, dtype=torch.float32)
                    bufs = {"img": f32(3), "line": f32(1), "out": None if gather is not None else (f32(4),)}
                slot = dict(bufs, shape=(B, H, W), ev_in=torch.cuda.Event(), ev_comp=torch.cuda.Event(), ev_out=torch.cuda.Event())
                slots[i % depth] = slot
            if edit_h is not None and "edit" not in slot:
                slot["edit"] = torch.empty(B, H, W, device=dev, dtype=torch.uint8)
            if fresh:
                # new buffers come from the compute stream's pool, so queued compute-stream work may still use their memory
                # (the PNG encode's freed scratch, for one): the copies into them wait for it
                s_in.wait_stream(cur)
            s_in.wait_event(slot["ev_comp"])           # the previous user of these input buffers has been computed
            if edit_h is not None:
                s_in.wait_event(slot["ev_out"])        # ... and the edit mask, which is also an output, has left the device
            with torch.cuda.stream(s_in):
                if files is not None:
                    _decode_png_batch(data, slot, B, H, W, dev)
                else:
                    slot["img"].copy_(img_h, non_blocking=True)
                    slot["line"].copy_(line_h, non_blocking=True)
                    if edit_h is not None:
                        slot["edit"].copy_(edit_h, non_blocking=True)
                slot["ev_in"].record(s_in)
            cur.wait_event(slot["ev_in"])
            cur.wait_event(slot["ev_out"])             # ... and its outputs have left the device buffers
            if gather is not None:
                if (B, H, W) != (gather.B,) + tuple(gather.bufs[0].shape[2:]):
                    raise ValueError("with gather= every batch must be [%d,*,%d,%d]" % ((gather.B,) + tuple(gather.bufs[0].shape[2:])))
                out = gather.next_slot()               # (waits, on `cur`, for the collective that last used this buffer)
                eng.inference_packed(slot["img"], slot["line"], precision=self.precision, out=out)
                k = gather.launch()
                slot["ev_comp"].record(cur)            # inputs are free again; the outputs follow the collective:
                with torch.cuda.stream(s_out):
                    gather.wait(k)                     # s_out waits for the all-gather of this batch
                    src = (gather.bufs[k][gather.rank * B:(gather.rank + 1) * B],)
            else:
                src = slot["out"]
                if edit_h is not None:
                    eng.inference_with_mask_u8(slot["img"], slot["line"], slot["edit"], precision=self.precision, out=slot["out"][0])
                    src = (slot["out"][0], slot["edit"])   # the mask result is the mask the batch ran on
                elif uint8:
                    eng.inference_u8(slot["img"], slot["line"], precision=self.precision, out=slot["out"])
                else:
                    eng.inference_packed(slot["img"], slot["line"], precision=self.precision, out=slot["out"][0])
                if png:
                    # the drain of the batch that last used this files buffer has already downloaded it
                    files, offs = slot["png"]
                    lens = [E.png_encode_u8_packed(t, [b * t[0].numel() for b in range(B)], [W * c] * B, [(H, W)] * B, c,
                                                   swap_rb=True, out=files, out_offsets=offs[k * B:(k + 1) * B])[2]
                            for k, (t, c) in enumerate(zip(src[:len(png)], (3, 1)))]
                slot["ev_comp"].record(cur)
                s_out.wait_event(slot["ev_comp"])
            with torch.cuda.stream(s_out):
                if png:
                    n_files = B * len(png)
                    lens_h = torch.empty(n_files, dtype=torch.int64, pin_memory=True)
                    for k, l in enumerate(lens):
                        lens_h[k * B:(k + 1) * B].copy_(l, non_blocking=True)
                        l.record_stream(s_out)
                    host = (slot["png"][0], slot["png"][1][:n_files], lens_h, B)
                else:
                    host = host_out(B, H, W)
                    for h_t, d_t in zip(host, src):
                        h_t.copy_(d_t, non_blocking=True)
                slot["ev_out"].record(s_out)
                done = torch.cuda.Event()
                done.record(s_out)
            pending.append((host, done, data))
            if len(pending) >= depth:
                yield drain_one()
        while pending:
            yield drain_one()


def _decode_png_batch(data, slot, B, H, W, dev):
    """Enqueues on the current stream the decode of a batch of PNG files (``collate_files``) into slot['img'], ['line'] and
    ['edit'] (``engine.png_decode_into``: Pillow's pixels wherever the parser or the decoder refuses a file). Files of another
    size than the photo go to a staging buffer and are resized into them, as Pillow's ``.resize`` does."""
    from sketchedit_b200 import engine as E
    files = data["png"]
    chans = {"img": 3, "line": 1, "edit": 1}
    mode = {"img": "RGB", "line": "L", "edit": "L"}
    sized = [k for k, f in enumerate(files) if tuple(f.size) != (H, W)]   # sketches / edit masks to resize (photos set H, W)
    aux_offs, aux_total = E._aligned_offsets([files[k].size[0] * files[k].size[1] for k in sized])
    aux = torch.empty(max(aux_total, 1), device=dev, dtype=torch.uint8)
    where = {k: (aux, o) for k, o in zip(sized, aux_offs)}   # file -> (buffer, byte offset) of its decoded pixels
    for k, f in enumerate(files):
        if k not in where:
            where[k] = (slot[f.target].view(-1), f.index * H * W * chans[f.target])
    parsed = [f for f in files if f.head is not None]
    E.png_decode_into((data["png_streams"], [f.offset for f in parsed], [f.length for f in parsed]), [f.head for f in files],
                      [mode[f.target] for f in files], [f.data for f in files], [where[k] + (f.size,) for k, f in enumerate(files)],
                      [data["path"][f.index] for f in files], dev)
    for target in ("line", "edit"):
        ks = [k for k in sized if files[k].target == target]
        if ks:
            E.resize_u8_packed(aux, [where[k][1] for k in ks], [files[k].size for k in ks], [(H, W)] * len(ks), 1,
                               out=slot[target].view(-1), dst_offsets=[files[k].index * H * W for k in ks])

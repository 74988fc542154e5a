"""Torch-tensor front end of the C ABI: owns an ``se_model`` (packed weights on the GPU) and
exposes the reference's call surface for the generator forward pass with CUDA tensors in and out.

    eng = Engine.from_state_dicts(sd_M, sd_G, use_cam=True, pool_type="max", joint_train_inp=True)
    composed, mask = eng.inference(image_cuda, sketch_cuda, precision="bf16")

PyTorch is plumbing here (device memory + current stream); all compute is in libsketchedit_b200.so.
"""
import array
import ctypes
import math
import numbers

import numpy as np
import torch

from . import _lib, pngfile
from .arch import NET_LAYERS, layer_map, out_channels_after_gate


# fields of a tap descriptor, in the order of SE_TAP_LAYOUT .. SE_TAP_PADL (include/sketchedit_b200.h)
TAP_DESC = ("layout", "dtype", "B", "C", "H", "W", "ld", "cb_off", "Wp", "padl")


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _chk_in(t, shape_tail=None, name="tensor"):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32):
        raise _lib.SketchEditB200Error("%s must be a CUDA float32 tensor (got %r)" % (name, getattr(t, "device", type(t))))
    return t.contiguous()


def _chk_out(t, shape, name, dtype=torch.float32):
    """Caller-owned output or uint8 input (shape None: any): the kernels use its pointer, so .contiguous() is not an option."""
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise _lib.SketchEditB200Error("%s must be a contiguous CUDA %s tensor" % (name, str(dtype)[len("torch."):]))
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise _lib.SketchEditB200Error("%s must have shape %r (got %r)" % (name, tuple(shape), tuple(t.shape)))
    return t


def _f32(*shape, like):
    return torch.empty(*shape, device=like.device, dtype=torch.float32)


class Engine:
    def __init__(self):
        self.lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(self.lib.se_model_create(ctypes.byref(h)))
        self.h = h
        self.finalized = False
        self.use_cam = True              # the library's default options run the contextual attention

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.se_model_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # -------------------------------------------------------------------------------- weights
    def set_layer(self, net, name, weight, bias):
        w = weight.detach().to("cpu", torch.float32).contiguous()
        b = bias.detach().to("cpu", torch.float32).contiguous()
        cout, cin, k, k2 = w.shape
        assert k == k2
        _lib.check(self.lib.se_model_set_layer(self.h, net.encode(), name.encode(), ctypes.c_void_p(w.data_ptr()),
                                               ctypes.c_void_p(b.data_ptr()), cout, cin, k))

    def load_state_dict(self, net, sd):
        """sd: reference-format state_dict ('<layer>.weight', '<layer>.bias'; optional 'module.' prefix,
        stripped like reference util/util.py:221-222). Strict: every layer of the net must be present."""
        sd = {(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()}
        expect = set()
        for l in NET_LAYERS[net]:
            expect.add(l.name + ".weight")
            expect.add(l.name + ".bias")
        missing, extra = expect - set(sd), set(sd) - expect
        if missing or extra:
            raise KeyError("state_dict mismatch for net%s: missing %s unexpected %s" % (net, sorted(missing), sorted(extra)))
        for l in NET_LAYERS[net]:
            self.set_layer(net, l.name, sd[l.name + ".weight"], sd[l.name + ".bias"])

    def set_options(self, use_cam=True, pool_type="max", no_mask_cc=False, no_mask_coarse=False, joint_train_inp=True):
        if pool_type not in ("max", "avg"):
            raise NotImplementedError(pool_type)          # reference editline_g.py:164-165
        for key, val in (("use_cam", use_cam), ("pool_avg", pool_type == "avg"), ("no_mask_cc", no_mask_cc),
                         ("no_mask_coarse", no_mask_coarse), ("joint_train_inp", joint_train_inp)):
            _lib.check(self.lib.se_model_set_option(self.h, _lib.OPT[key], int(bool(val))))
        self.use_cam = bool(use_cam)     # whether the forward has attention weights to export (inference_u8_export)

    def finalize(self):
        if not torch.cuda.is_available():
            raise _lib.SketchEditB200Error("sketchedit_b200 needs a CUDA device (sm_90a, H100); there is no CPU fallback")
        _lib.check(self.lib.se_model_finalize(self.h))
        self.finalized = True
        self.device = torch.device("cuda", torch.cuda.current_device())   # weights + workspace live here

    def _on_device(self, *tensors):
        for t in tensors:
            if t is not None and t.device != self.device:
                raise _lib.SketchEditB200Error("tensor on %s but this engine was finalized on %s" % (t.device, self.device))

    @classmethod
    def from_state_dicts(cls, sd_M, sd_G, **options):
        e = cls()
        if sd_M is not None:
            e.load_state_dict("M", sd_M)
        if sd_G is not None:
            e.load_state_dict("G", sd_G)
        e.set_options(**options)
        e.finalize()
        return e

    # -------------------------------------------------------------------------------- forward
    def _forward_tensors(self, dtype, ins, outs, out=None, want=()):
        """Checked (name, tensor) inputs, image first (fp32: made contiguous, an edit mask [B,1,H,W]; uint8: [B,H,W,3] then
        [B,H,W]), the results of ``outs`` channels (the caller's ``out``, one tensor for one result, or new) and the ``want``
        extras: (B, H, W, inputs, results, extras)."""
        names = [n for n, _ in ins]
        if dtype == torch.uint8:
            ins = [_chk_out(t, None, n, torch.uint8) for n, t in ins]
            B, H, W, C = ins[0].shape
            if C != 3 or any(tuple(t.shape) != (B, H, W) for t in ins[1:]):
                raise _lib.SketchEditB200Error(", ".join(["image_u8 must be [B,H,W,3]"] + names[1:-1]) + " and %s [B,H,W]" % names[-1])
            shape = lambda c: (B, H, W, 3) if c == 3 else (B, H, W)
        else:
            ins = [_chk_in(t, name=n) for n, t in ins]
            B, _, H, W = ins[0].shape
            shape = lambda c: (B, c, H, W)
            for n, t in zip(names[2:], ins[2:]):
                _chk_out(t, shape(1), n)
        one = len(outs) == 1
        res = [torch.empty(shape(c), device=ins[0].device, dtype=dtype) if out is None else
               _chk_out(out if one else out[i], shape(c), "out" if one else "out[%d]" % i, dtype) for i, c in enumerate(outs)]
        extra = {k: _f32(B, 1 if k == "mask_bin" else 3, H, W, like=ins[0]) for k in want}
        self._on_device(*ins, *res)
        return B, H, W, ins, res, extra

    def inference(self, image, sketch, precision="bf16", want=(), mask_bin=None, out=None):
        """EditLine2Model.forward(mode='inference'): returns (composed, mask) and, in a dict, any of
        want = ('coarse', 'fine', 'mask_image', 'mask_bin'). ``out=(composed, mask)`` writes into caller-owned
        fp32 CUDA tensors of shape [B,3,H,W] / [B,1,H,W] instead of allocating (pipelined callers)."""
        B, H, W, (image, sketch), (composed, mask), extra = self._forward_tensors(
            torch.float32, (("image", image), ("sketch", sketch)), (3, 1), out, want)
        mb_in = _chk_in(mask_bin, name="mask_bin") if mask_bin is not None else None
        self._on_device(mb_in)
        _lib.check(self.lib.se_forward_inference(
            self.h, _ptr(image), _ptr(sketch), B, H, W, _lib.PREC[precision], _ptr(composed), _ptr(mask),
            _ptr(extra.get("coarse")), _ptr(extra.get("fine")), _ptr(extra.get("mask_image")), _ptr(mb_in),
            _ptr(extra.get("mask_bin")), _stream()))
        return composed, mask, extra

    def inference_packed(self, image, sketch, precision="bf16", out=None):
        """Same forward, ONE packed output [B,4,H,W] (channels 0-2 composed, channel 3 the soft mask) = the layout of the
        data-parallel output all-gather: ``out`` may be this rank's slice of the gather buffer (parallel.OutputGather)."""
        B, H, W, (image, sketch), (packed,), _ = self._forward_tensors(torch.float32, (("image", image), ("sketch", sketch)), (4,), out)
        _lib.check(self.lib.se_forward_inference_packed(self.h, _ptr(image), _ptr(sketch), B, H, W, _lib.PREC[precision], _ptr(packed),
                                                        _stream()))
        return packed

    def inference_u8(self, image_u8, sketch_u8, precision="bf16", out=None):
        """Forward with the reference's host-side codecs on the device: image_u8 [B,H,W,3] RGB uint8 and sketch_u8 [B,H,W]
        uint8 (reference data/testimage_dataset.py:89-103 up to ToTensor) -> (bgr_u8 [B,H,W,3], mask_u8 [B,H,W]) exactly as
        test.py:25-35 writes them. ``out=(bgr, mask)`` writes into caller-owned uint8 CUDA tensors."""
        B, H, W, (image_u8, sketch_u8), (bgr, mk), _ = self._forward_tensors(
            torch.uint8, (("image_u8", image_u8), ("sketch_u8", sketch_u8)), (3, 1), out)
        _lib.check(self.lib.se_forward_inference_u8(self.h, _ptr(image_u8), _ptr(sketch_u8), B, H, W, _lib.PREC[precision], _ptr(bgr), _ptr(mk),
                                                    _stream()))
        return bgr, mk

    def inference_with_mask(self, image, sketch, edit_mask, precision="bf16", want=()):
        """The forward on a caller-supplied edit mask [B,1,H,W] instead of netM's prediction: netG inpaints
        (edit_mask > 0.5) and composed = fine * edit_mask + image * (1 - edit_mask); values are used as given. Returns
        (composed, extra) with any of want = ('coarse', 'fine', 'mask_image', 'mask_bin') in the dict. netM runs only
        for 'mask_image'. Given the soft mask ``inference`` returned, every output equals that call's bit for bit."""
        B, H, W, (image, sketch, edit_mask), (composed,), extra = self._forward_tensors(
            torch.float32, (("image", image), ("sketch", sketch), ("edit_mask", edit_mask)), (3,), None, want)
        _lib.check(self.lib.se_forward_with_mask(
            self.h, _ptr(image), _ptr(sketch), _ptr(edit_mask), B, H, W, _lib.PREC[precision], _ptr(composed),
            _ptr(extra.get("coarse")), _ptr(extra.get("fine")), _ptr(extra.get("mask_image")), _ptr(extra.get("mask_bin")),
            _stream()))
        return composed, extra

    def inference_with_mask_u8(self, image_u8, sketch_u8, edit_mask_u8, precision="bf16", out=None):
        """``inference_u8`` on a caller-supplied edit mask: edit_mask_u8 [B,H,W] uint8 means v/255 (inpainted where
        v >= 128). Returns bgr_u8 [B,H,W,3]; ``out`` is a caller-owned contiguous CUDA uint8 tensor of that shape."""
        B, H, W, (image_u8, sketch_u8, edit_mask_u8), (bgr,), _ = self._forward_tensors(
            torch.uint8, (("image_u8", image_u8), ("sketch_u8", sketch_u8), ("edit_mask_u8", edit_mask_u8)), (3,), out)
        _lib.check(self.lib.se_forward_with_mask_u8(self.h, _ptr(image_u8), _ptr(sketch_u8), _ptr(edit_mask_u8), B, H, W,
                                                    _lib.PREC[precision], _ptr(bgr), _stream()))
        return bgr

    def predict_mask_u8(self, image_u8, sketch_u8, precision="bf16", out=None):
        """netM's edit mask alone, on ``inference_u8``'s input codec (``se_predict_mask_u8``; netG does not run): returns
        (mask_f32 [B,1,H,W], mask_u8 [B,H,W]), the soft mask bit for bit as netM computes it inside ``inference_u8`` on the
        same bytes, and its bytes as that call writes them. ``out=(mask_f32, mask_u8)`` writes into caller-owned CUDA
        tensors (float32 and uint8)."""
        B, H, W, (image_u8, sketch_u8), (mk,), _ = self._forward_tensors(
            torch.uint8, (("image_u8", image_u8), ("sketch_u8", sketch_u8)), (1,), out[1] if out is not None else None)
        soft = _f32(B, 1, H, W, like=mk) if out is None else _chk_out(out[0], (B, 1, H, W), "out[0]")
        self._on_device(soft)
        _lib.check(self.lib.se_predict_mask_u8(self.h, _ptr(image_u8), _ptr(sketch_u8), B, H, W, _lib.PREC[precision], _ptr(soft),
                                               _ptr(mk), _stream()))
        return soft, mk

    def inference_u8_with_soft_mask(self, image_u8, sketch_u8, edit_mask, precision="bf16", out=None):
        """``inference_u8`` on a caller's fp32 edit mask [B,1,H,W] (``se_forward_u8_with_soft_mask``; netM does not run):
        netG inpaints edit_mask > 0.5 and the result is blended with edit_mask as given. Given the mask_f32 of
        ``predict_mask_u8``, the returned bgr_u8 [B,H,W,3] is ``inference_u8``'s bit for bit. ``out``: a caller-owned
        contiguous CUDA uint8 tensor of that shape."""
        B, H, W, (image_u8, sketch_u8), (bgr,), _ = self._forward_tensors(
            torch.uint8, (("image_u8", image_u8), ("sketch_u8", sketch_u8)), (3,), out)
        _chk_out(edit_mask, (B, 1, H, W), "edit_mask")
        self._on_device(edit_mask)
        _lib.check(self.lib.se_forward_u8_with_soft_mask(self.h, _ptr(image_u8), _ptr(sketch_u8), _ptr(edit_mask), B, H, W,
                                                         _lib.PREC[precision], _ptr(bgr), _stream()))
        return bgr

    def inference_u8_export(self, image_u8, sketch_u8, edit_mask_u8=None, edit_mask=None, precision="bf16"):
        """One of ``inference_u8`` (no edit mask), ``inference_with_mask_u8`` (``edit_mask_u8``) or
        ``inference_u8_with_soft_mask`` (``edit_mask``, fp32 [B,1,H,W]), with netG's attention exported for region-edit detail
        (``se_forward_u8_export``). Returns (bgr_u8 [B,H,W,3], mask_u8 [B,H,W] or None with an edit mask, attn fp32 [B,L,L],
        hole_u8 [B,H,W]): bgr_u8 and mask_u8 are the chosen call's bit for bit; attn holds the attention's softmax weights as
        the forward used them, [key][query] like ``contextual_attention(..., want_attn=True)``, L = (H/8 - 1)(W/8 - 1); hole_u8
        is the mask netG inpaints as 0 / 1. attn takes 4 L^2 bytes per image: 3.7 MB at 256 x 256, 63 MB at 512 x 512. To return
        it whole, the attention runs in one band of query rows: its L x L workspace (bf16: P at 2 L^2 bytes per image;
        fp32_direct: S and P at 8 L^2) is then not held to ``set_attention_workspace_limit``. A model without the attention
        (``use_cam=False``) has no weights to export: the call raises."""
        if edit_mask_u8 is not None and edit_mask is not None:
            raise _lib.SketchEditB200Error("give at most one of edit_mask_u8 and edit_mask")
        ins = (("image_u8", image_u8), ("sketch_u8", sketch_u8)) + ((("edit_mask_u8", edit_mask_u8),) if edit_mask_u8 is not None else ())
        B, H, W, ins, (bgr,), _ = self._forward_tensors(torch.uint8, ins, (3,), None)
        predicted = edit_mask_u8 is None and edit_mask is None
        mk = torch.empty(B, H, W, device=bgr.device, dtype=torch.uint8) if predicted else None
        if edit_mask is not None:
            _chk_out(edit_mask, (B, 1, H, W), "edit_mask")
            self._on_device(edit_mask)
        L = (H // 8 - 1) * (W // 8 - 1)
        attn = _f32(B, L, L, like=bgr)
        hole = torch.empty(B, H, W, device=bgr.device, dtype=torch.uint8)
        _lib.check(self.lib.se_forward_u8_export(self.h, _ptr(ins[0]), _ptr(ins[1]), _ptr(ins[2]) if len(ins) > 2 else None,
                                                 _ptr(edit_mask), B, H, W, _lib.PREC[precision], _ptr(bgr), _ptr(mk), _ptr(attn),
                                                 _ptr(hole), _stream()))
        return bgr, mk, attn, hole

    def netM(self, x, guide, precision="bf16", want_image=True):
        B, H, W, (x, guide), (mask1,), ex = self._forward_tensors(torch.float32, (("tensor", x), ("tensor", guide)), (1,), None,
                                                                  ("x_stage1",) if want_image else ())
        _lib.check(self.lib.se_netM_forward(self.h, _ptr(x), _ptr(guide), B, H, W, _lib.PREC[precision], _ptr(mask1),
                                            _ptr(ex.get("x_stage1")), _stream()))
        return mask1, ex.get("x_stage1")

    def netG(self, x, x2, mask, mask2, guide, precision="bf16"):
        x, x2, mask, mask2 = _chk_in(x), _chk_in(x2), _chk_in(mask), _chk_in(mask2)
        guide = _chk_in(guide) if guide is not None else None
        B, _, H, W = x.shape
        self._on_device(x, x2, mask, mask2, guide)
        s1 = _f32(B, 3, H, W, like=x)
        s2 = _f32(B, 3, H, W, like=x)
        _lib.check(self.lib.se_netG_forward(self.h, _ptr(x), _ptr(x2), _ptr(mask), _ptr(mask2), _ptr(guide), B, H, W,
                                            _lib.PREC[precision], _ptr(s1), _ptr(s2), _stream()))
        return s1, s2

    def gated_conv(self, net, name, x, precision="bf16"):
        x = _chk_in(x)
        spec = layer_map(net)[name]
        B, cin, H, W = x.shape
        if cin != spec.cin:
            raise _lib.SketchEditB200Error("%s expects %d input channels, got %d" % (name, spec.cin, cin))
        if spec.kind == "deconv":
            Ho, Wo = 2 * H, 2 * W
        else:
            Ho, Wo = (H + spec.stride - 1) // spec.stride, (W + spec.stride - 1) // spec.stride
        self._on_device(x)
        y = _f32(B, out_channels_after_gate(spec), Ho, Wo, like=x)
        _lib.check(self.lib.se_gated_conv_forward(self.h, net.encode(), name.encode(), _ptr(x), B, H, W, _lib.PREC[precision],
                                                  _ptr(y), _stream()))
        return y

    def set_taps(self, on):
        """Record the stored input of every stage of each following forward (include/sketchedit_b200.h, se_taps_enable);
        those forwards run eagerly."""
        _lib.check(self.lib.se_taps_enable(self.h, int(bool(on))))

    def taps(self):
        """{name: (desc, uint8 CUDA tensor of the raw bytes)} of the last forward; desc is a dict with the keys of TAP_DESC."""
        out = {}
        name = ctypes.create_string_buffer(256)
        desc = (ctypes.c_int * len(TAP_DESC))()
        nbytes = ctypes.c_longlong(0)
        for i in range(int(self.lib.se_taps_count(self.h))):
            _lib.check(self.lib.se_tap_info(self.h, i, name, len(name), desc, ctypes.byref(nbytes)))
            raw = torch.empty(nbytes.value, device=self.device, dtype=torch.uint8)
            _lib.check(self.lib.se_tap_copy(self.h, i, _ptr(raw), _stream()))
            out[name.value.decode()] = (dict(zip(TAP_DESC, list(desc))), raw)
        return out

    def launches(self):
        return int(self.lib.se_last_launch_count())

    def workspace_bytes(self):
        return int(self.lib.se_workspace_bytes(self.h))


def contextual_attention(feat, mask_s, precision="bf16", want_attn=False):
    """cam_2(cam_1(f, f, mask_s), f, mask_s, {})[0] of netG (reference editline_g.py:203-207)."""
    lib = _lib.load()
    feat, mask_s = _chk_in(feat), _chk_in(mask_s)
    B, C, h, w = feat.shape
    out = _f32(*feat.shape, like=feat)
    attn = None
    if want_attn:
        hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
        attn = _f32(B, hs * ws, hs * ws, like=feat)
    _lib.check(lib.se_contextual_attention_forward(_ptr(feat), _ptr(mask_s), B, C, h, w, _lib.PREC[precision], _ptr(out), _ptr(attn),
                                                   _stream()))
    return (out, attn) if want_attn else out


def set_attention_workspace_limit(nbytes):
    """Bytes the contextual attention's L x L temporaries may take (process-wide; 0 = the default of 16 GiB). Larger
    inputs run the attention in bands of query rows that fit; the results do not depend on the band split."""
    _lib.check(_lib.load().se_set_attention_workspace_limit(int(nbytes)))


RESIZE_MAX_BATCH = 32    # images per se_resize_window_u8 call; the wrappers split longer lists into calls of this size


# ---- plumbing shared by the uint8 image wrappers below
def _chk_u8(*named):
    """(tensor, name) pairs: contiguous CUDA uint8 tensors, whose pointers the kernels use as they are."""
    for t, name in named:
        _chk_out(t, None, name, torch.uint8)


def _device(*named):
    """The one device of the (tensor, name) pairs."""
    devs = {t.device for t, _ in named}
    if len(devs) > 1:
        names = ", ".join(dict.fromkeys(nm for _, nm in named))
        raise _lib.SketchEditB200Error("%s must be on one device (got %s)" % (names, ", ".join(sorted(map(str, devs)))))
    return named[0][0].device


def _check_windows(what, bufs, offsets, pitches, sizes, bpp):
    """Window i is sizes[i] = (h, w) rows of w * bpp bytes, row r at byte offsets[i] + r * pitches[i] of bufs[i] (of bufs
    itself when it is one tensor): its pitch must hold its row and the window must lie inside its buffer. Sizes below 1 are
    left to the C entry, which names them."""
    nbytes = [bufs.numel()] * len(sizes) if isinstance(bufs, torch.Tensor) else [t.numel() for t in bufs]
    for i, (n, o, p, (h, w)) in enumerate(zip(nbytes, offsets, pitches, sizes)):
        if p < w * bpp:
            raise _lib.SketchEditB200Error("%s %d: the pitch of %d bytes is narrower than its row of %d bytes" % (what, i, p, w * bpp))
        if o < 0 or (h >= 1 and w >= 1 and o + (h - 1) * p + w * bpp > n):
            raise _lib.SketchEditB200Error("%s %d (%dx%d at %d, pitch %d) is outside the %d-byte buffer" % (what, i, h, w, o, p, n))


def _aligned_offsets(nbytes, align=16):
    """Offsets of blocks of nbytes[i] bytes packed at align-byte aligned offsets, and the bytes they span."""
    offs, total = [], 0
    for n in nbytes:
        offs.append(total)
        total += (n + align - 1) // align * align
    return offs, total


def _out(out, offsets, nbytes, device, name):
    """(out, offsets) of a wrapper's output slices of nbytes[i] bytes: the caller's, checked, or without ``out`` a new tensor
    holding them at 16-byte aligned offsets. ``name`` is the offsets argument's name."""
    if out is None:
        if offsets is not None:
            raise _lib.SketchEditB200Error("%s needs out" % name)
        offsets, total = _aligned_offsets(nbytes)
        return torch.empty(total, device=device, dtype=torch.uint8), offsets
    if offsets is None or len(offsets) != len(nbytes):
        raise _lib.SketchEditB200Error("out needs one %s entry per image" % name)
    offsets = [int(o) for o in offsets]
    _check_windows("out", out, offsets, nbytes, [(1, b) for b in nbytes], 1)
    return out, offsets


def _hw(pairs):
    return [(int(a), int(b)) for a, b in pairs]


def _longs(values):
    return (ctypes.c_longlong * len(values))(*values)


def _ints(rows):
    """The int tuples ``rows`` flattened into one C array."""
    flat = [v for r in rows for v in r]
    return (ctypes.c_int * len(flat))(*flat)


def _run_chunks(n, per_call, device, chunk):
    """Calls a scratch-taking C entry over n images, per_call images per call, on the current stream of ``device``.
    ``chunk(sl)`` returns for the images of slice sl a function f(scratch, scratch_bytes, stream) that makes the call;
    f(None, ...) is its scratch query. One scratch allocation, the largest query, serves every call."""
    _run_calls([chunk(slice(c0, c0 + per_call)) for c0 in range(0, n, per_call)], device)


def _run_calls(calls, device):
    """``_run_chunks`` over the call functions ``calls``, in order."""
    with torch.cuda.device(device):
        need = 0
        for f in calls:
            size = ctypes.c_longlong(0)
            _lib.check(f(None, ctypes.byref(size), None))
            need = max(need, size.value)
        scratch = torch.empty(max(need, 1), device=device, dtype=torch.uint8)
        for f in calls:
            _lib.check(f(_ptr(scratch), ctypes.byref(ctypes.c_longlong(scratch.numel())), _stream()))


def resize_u8_packed(src, src_offsets, src_sizes, dst_sizes, channels, swap_rb=False, out=None, dst_offsets=None):
    """PIL.Image.resize(size) (BICUBIC, its default) of a batch of uint8 HWC images, bit for bit, on the device.

    Image i is the ``src_sizes[i] = (h, w)`` x ``channels`` bytes at byte ``src_offsets[i]`` of the contiguous CUDA uint8 tensor
    ``src``; it is resized to ``dst_sizes[i]`` and written at ``dst_offsets[i]`` of ``out``. Without ``out`` the results are
    packed into a new tensor at 16-byte aligned offsets. ``swap_rb`` reverses the channel order of the output (channels 3).
    Returns ``(out, dst_offsets)``. Only enqueues work on the current stream, except that the first resize between a pair of
    lengths uploads its coefficient table. This is ``resize_window_u8_packed`` with packed rows (pitch ``w * channels``)."""
    return resize_window_u8_packed(src, src_offsets, [int(w) * channels for _, w in src_sizes], src_sizes, dst_sizes, channels,
                                   swap_rb=swap_rb, out=out, dst_offsets=dst_offsets)


def resize_window_u8_packed(src, src_offsets, src_pitches, src_sizes, dst_sizes, channels, swap_rb=False, out=None,
                            dst_offsets=None):
    """``resize_u8_packed`` of windows of larger images (``se_resize_window_u8``): image i is the ``src_sizes[i] = (h, w)``
    window whose row r starts at byte ``src_offsets[i] + r * src_pitches[i]`` of its source, with ``src_pitches[i] >= w *
    channels``. ``src`` is one contiguous CUDA uint8 tensor, or a list of them with one per image. With the offset of a box's
    top-left pixel in an [H,W,C] photo and the pitch ``W * C`` the window is ``Image.crop(box)``, so the result is
    ``Image.crop(box).resize(size)`` bit for bit, without the crop. Windows may overlap; ``out`` must not overlap any of them.
    ``out``, ``dst_offsets``, ``swap_rb`` and the return value are those of ``resize_u8_packed``."""
    lib = _lib.load()
    return _resize_windows(src, src_offsets, src_pitches, src_sizes, dst_sizes, channels, out, dst_offsets,
                           lambda a: lambda scratch, size, stream: lib.se_resize_window_u8(*a, channels, int(bool(swap_rb)),
                                                                                           scratch, size, stream))


def _resize_windows(src, src_offsets, src_pitches, src_sizes, dst_sizes, channels, out, dst_offsets, call):
    """The body of ``resize_window_u8_packed`` and ``resize_reducing_u8_packed``: checks the windows, allocates ``out`` when
    it is None and runs ``call(a)`` over chunks of RESIZE_MAX_BATCH windows, ``a`` being the chunk's entry arguments up to n."""
    n = len(src_sizes)
    listed = isinstance(src, (list, tuple))
    srcs = list(src) if listed else [src] * n
    if not (len(srcs) == len(src_offsets) == len(src_pitches) == len(dst_sizes) == n):
        raise _lib.SketchEditB200Error("src (as a list), src_offsets, src_pitches, src_sizes and dst_sizes must have the same length")
    named = [(t, "src") for t in (srcs if listed else [src])] + ([(out, "out")] if out is not None else [])
    _chk_u8(*named)
    if not named:
        return out, dst_offsets
    dev = _device(*named)
    src_sizes, dst_sizes = _hw(src_sizes), _hw(dst_sizes)
    src_offsets, src_pitches = [int(o) for o in src_offsets], [int(p) for p in src_pitches]
    _check_windows("window", srcs if listed else src, src_offsets, src_pitches, src_sizes, channels)
    out, dst_offsets = _out(out, dst_offsets, [h * w * channels for h, w in dst_sizes], dev, "dst_offsets")
    ptrs = [t.data_ptr() + o for t, o in zip(srcs, src_offsets)] if listed else [src.data_ptr() + o for o in src_offsets]

    def chunk(sl):
        k = len(ptrs[sl])
        return call(((ctypes.c_void_p * k)(*ptrs[sl]), _longs(src_pitches[sl]), _ints(src_sizes[sl]), _ptr(out),
                     _longs(dst_offsets[sl]), _ints(dst_sizes[sl]), k))

    _run_chunks(n, RESIZE_MAX_BATCH, dev, chunk)
    return out, dst_offsets


def resize_composite_u8_packed(rgb, rgb_offsets, mask, mask_offsets, src_sizes, canvas, canvas_offsets, canvas_pitches,
                               box_offsets, box_sizes, swap_rb=False, feather=None, detail=None, detail_offsets=None):
    """Resize back and paste boxes in order into canvases (``se_resize_composite_feather_detail_u8``), bit for bit as sequential
    Pillow pastes, in place:

        for each box i in order:  canvas_i.paste(Image.fromarray(rgb_i).resize((w, h)), (x, y), Image.fromarray(mask_i).resize((w, h)))

    Box i's result [h',w',3] is at byte ``rgb_offsets[i]`` of ``rgb`` and its mask [h',w'] at ``mask_offsets[i]`` of
    ``mask``, with ``src_sizes[i] = (h', w')``. Its canvas starts at byte ``canvas_offsets[i]`` of ``canvas`` with
    ``canvas_pitches[i]`` bytes per row; ``box_offsets[i] = (y, x)`` is its top-left pixel there and ``box_sizes[i] = (h, w)``
    its size. Boxes with the same canvas offset share that canvas, so a later box blends over an earlier one where they
    overlap. ``swap_rb`` reverses the result's channel order first (the forward writes BGR). All tensors are contiguous CUDA
    uint8 on one device; only the boxes' canvas pixels are read and written. To paste into a copy instead, copy the canvas
    first. ``feather``: None, or per box its ramp widths ``(left, top, right, bottom)`` in box pixels: the box's resized mask
    becomes ``DIV255(m * ramp)`` before the blend, with the ramp of ``serving.feather_ramp``. ``detail``: None, or a contiguous
    CUDA int16 tensor holding at byte ``detail_offsets[i]`` box i's detail plane [h,w,3] (RGB, from ``detail_u8_packed``; an
    offset < 0: none), added to the resized result with a clamp to [0, 255] before the blend. Returns ``canvas``. Only enqueues work on the current stream, except that the
    first resize between a pair of lengths uploads its coefficient table."""
    n = len(src_sizes)
    if not (len(rgb_offsets) == len(mask_offsets) == len(canvas_offsets) == len(canvas_pitches) == len(box_offsets)
            == len(box_sizes) == n):
        raise _lib.SketchEditB200Error("rgb_offsets, mask_offsets, src_sizes, canvas_offsets, canvas_pitches, box_offsets and "
                                       "box_sizes must have the same length")
    if feather is not None:
        feather = [tuple(int(v) for v in f) for f in feather]
        if len(feather) != n or any(len(f) != 4 for f in feather):
            raise _lib.SketchEditB200Error("feather needs 4 widths (left, top, right, bottom) per box")
    named = [(rgb, "rgb"), (mask, "mask"), (canvas, "canvas")]
    _chk_u8(*named)
    dev = _device(*named)
    if detail is not None:
        _chk_out(detail, None, "detail", torch.int16)
        _device(*named, (detail, "detail"))
        if detail_offsets is None or len(detail_offsets) != n:
            raise _lib.SketchEditB200Error("detail needs one detail_offsets entry per box")
        detail_offsets = [int(o) for o in detail_offsets]
        for i, o in enumerate(detail_offsets):
            h, w = int(box_sizes[i][0]), int(box_sizes[i][1])
            if o >= 0 and (o % 2 or o + h * w * 6 > detail.numel() * 2):
                raise _lib.SketchEditB200Error("detail %d at byte %d is outside the detail tensor or not 2-byte aligned" % (i, o))
    src_sizes, box_sizes, box_offsets = _hw(src_sizes), _hw(box_sizes), _hw(box_offsets)
    rgb_offsets, mask_offsets = [int(o) for o in rgb_offsets], [int(o) for o in mask_offsets]
    canvas_offsets, canvas_pitches = [int(o) for o in canvas_offsets], [int(p) for p in canvas_pitches]
    _check_windows("rgb", rgb, rgb_offsets, [3 * w for _, w in src_sizes], src_sizes, 3)
    _check_windows("mask", mask, mask_offsets, [w for _, w in src_sizes], src_sizes, 1)
    for i, (y, x) in enumerate(box_offsets):
        if y < 0 or x < 0:
            raise _lib.SketchEditB200Error("box %d at (%d, %d) is outside the canvas" % (i, y, x))
    # box i lies inside the window of its canvas's first y + h rows and first x + w pixels
    _check_windows("box", canvas, canvas_offsets, canvas_pitches,
                   [(y + h, x + w) for (y, x), (h, w) in zip(box_offsets, box_sizes)], 3)
    lib = _lib.load()
    a = (_ptr(rgb), _longs(rgb_offsets), _ptr(mask), _longs(mask_offsets), _ints(src_sizes), _ptr(canvas), _longs(canvas_offsets),
         _longs(canvas_pitches), _ints(box_offsets), _ints(box_sizes), _ints(feather) if feather is not None else None,
         _ptr(detail), _longs(detail_offsets) if detail is not None else None, n, int(bool(swap_rb)))
    call = lambda scratch, size, stream: lib.se_resize_composite_feather_detail_u8(*a, scratch, size, stream)
    # one call: the entry keeps the boxes' order across its launches
    _run_chunks(n, max(n, 1), dev, lambda sl: call)
    return canvas


def detail_u8_packed(photo, photo_offsets, photo_pitches, box_sizes, region_size, low, low_offsets, hole, hole_offsets, attn,
                     attn_offsets, want_agg=False):
    """Region-edit detail planes (``se_detail_u8``; DESIGN.md section 7b): for box i of ``box_sizes[i] = (bh, bw)`` edited at
    ``region_size = (Hn, Wn)``, the RGB window of the photo whose row r starts at byte ``photo_offsets[i] + r * photo_pitches[i]``
    of ``photo`` (one contiguous CUDA uint8 tensor, or a list with one per box), ``low``'s [bh,bw,3] at byte ``low_offsets[i]``
    (the window resized to the working size and back), the forward's hole_u8 [Hn,Wn] at byte ``hole_offsets[i]`` of ``hole`` and
    its attn [L,L] at element ``attn_offsets[i]`` of the fp32 tensor ``attn``. Returns ``(D, d_offsets, agg)``: D a CUDA int16
    tensor holding box i's plane [bh,bw,3] at byte ``d_offsets[i]``, for ``resize_composite_u8_packed(..., detail=D,
    detail_offsets=d_offsets)``; agg (``want_agg``) a CUDA float32 tensor holding box i's aggregate A [bh,bw,3] at element
    ``d_offsets[i] // 2``, else None. Only enqueues work on the current stream. Transient device memory: one box's scratch at
    a time, 4 Mp^2 + 8 Mp Np bytes (Mp = L rounded up to 256; Np = 3 fw fh rounded up to 256, fw = ceil(16 bw / Wn) + 2):
    about 44 MB for a 608 x 608 box at 256 x 256."""
    n = len(box_sizes)
    listed = isinstance(photo, (list, tuple))
    srcs = list(photo) if listed else [photo] * n
    if not (len(srcs) == len(photo_offsets) == len(photo_pitches) == len(low_offsets) == len(hole_offsets) == len(attn_offsets) == n):
        raise _lib.SketchEditB200Error("photo (as a list), photo_offsets, photo_pitches, box_sizes, low_offsets, hole_offsets and "
                                       "attn_offsets must have the same length")
    Hn, Wn = (int(v) for v in region_size)
    L = (Hn // 8 - 1) * (Wn // 8 - 1)
    named = [(t, "photo") for t in (srcs if listed else [photo])] + [(low, "low"), (hole, "hole")]
    _chk_u8(*named)
    _chk_out(attn, None, "attn")
    dev = _device(*named, (attn, "attn"))
    sizes = _hw(box_sizes)
    photo_offsets, photo_pitches = [int(o) for o in photo_offsets], [int(p) for p in photo_pitches]
    low_offsets, hole_offsets, attn_offsets = [int(o) for o in low_offsets], [int(o) for o in hole_offsets], [int(o) for o in attn_offsets]
    _check_windows("window", srcs if listed else photo, photo_offsets, photo_pitches, sizes, 3)
    _check_windows("low", low, low_offsets, [3 * w for _, w in sizes], sizes, 3)
    _check_windows("hole", hole, hole_offsets, [Wn] * n, [(Hn, Wn)] * n, 1)
    for i, o in enumerate(attn_offsets):
        if o < 0 or o + L * L > attn.numel():
            raise _lib.SketchEditB200Error("attn %d at element %d is outside the attn tensor" % (i, o))
    d_offs, total = _aligned_offsets([h * w * 3 * 4 for h, w in sizes])   # room for A (fp32) at the same element index as D
    D = torch.empty(max(total // 4, 1), device=dev, dtype=torch.int16)     # plane i at byte d_offs[i] // 2, 6 bh bw bytes
    agg = torch.empty(max(total // 4, 1), device=dev, dtype=torch.float32) if want_agg else None
    d_offs = [o // 2 for o in d_offs]
    ptrs = [t.data_ptr() + o for t, o in zip(srcs, photo_offsets)]
    lib = _lib.load()
    a = ((ctypes.c_void_p * n)(*ptrs), _longs(photo_pitches), _ints(sizes), n, Hn, Wn, _ptr(low), _longs(low_offsets), _ptr(hole),
         _longs(hole_offsets), _ptr(attn), _longs([4 * o for o in attn_offsets]), _ptr(D), _longs(d_offs), _ptr(agg),
         _longs([2 * o for o in d_offs]) if want_agg else None)
    _run_chunks(n, max(n, 1), dev, lambda sl: lambda scratch, size, stream: lib.se_detail_u8(*a, scratch, size, stream))
    return D, d_offs, agg


def feather_u8_packed(buf, offsets, sizes, feather):
    """The feather of ``resize_composite_u8_packed(..., feather=...)`` on 'L' images alone, in place (``se_feather_u8``):
    image i is the ``sizes[i] = (h, w)`` bytes at byte ``offsets[i]`` of the contiguous CUDA uint8 tensor ``buf``, and each
    byte m becomes ``DIV255(m * ramp)`` with the ramp of ``feather[i] = (left, top, right, bottom)``. Images whose four widths
    are 0 are not touched. Returns ``buf``; only enqueues work on the current stream."""
    n = len(sizes)
    if len(offsets) != n or len(feather) != n:
        raise _lib.SketchEditB200Error("offsets, sizes and feather must have the same length")
    _chk_u8((buf, "buf"))
    sizes, offsets = _hw(sizes), [int(o) for o in offsets]
    feather = [tuple(int(v) for v in f) for f in feather]
    if any(len(f) != 4 for f in feather):
        raise _lib.SketchEditB200Error("feather needs 4 widths (left, top, right, bottom) per image")
    _check_windows("image", buf, offsets, [w for _, w in sizes], sizes, 1)
    with torch.cuda.device(buf.device):
        _lib.check(_lib.load().se_feather_u8(_ptr(buf), _longs(offsets), _ints(sizes), _ints(feather), n, _stream()))
    return buf


def set_resize_table_cache_limit(nbytes):
    """Bytes of coefficient tables the resize keeps per device (process-wide; 0 = the default of 256 MiB). Past the limit the
    device's tables are dropped, after a device synchronise, before the next call that needs a new one."""
    _lib.check(_lib.load().se_resize_set_table_cache_limit(int(nbytes)))


def resize_table_cache_bytes():
    """Bytes of coefficient tables cached for the current device."""
    return int(_lib.load().se_resize_table_cache_bytes())


def resize_u8(images, sizes, swap_rb=False):
    """List form of ``resize_u8_packed``: ``images`` are CUDA uint8 tensors [h,w,3] or [h,w] (one channel count for the
    list), ``sizes`` the target ``(h, w)`` of each. Returns the resized images, views of one packed tensor. The inputs are
    first packed into one buffer; callers that already hold packed data use ``resize_u8_packed`` and skip that copy."""
    if len(images) != len(sizes):
        raise _lib.SketchEditB200Error("one target size per image")
    if not images:
        return []
    chans = {1 if t.dim() == 2 else t.shape[-1] for t in images}
    C = chans.pop()
    if chans or C not in (1, 3) or any(t.dim() not in (2, 3) for t in images):
        raise _lib.SketchEditB200Error("images must all be [h,w] or all be [h,w,3]")
    offs, total = [], 0
    for t in images:
        offs.append(total)
        total += t.numel()
    src = torch.cat([t.reshape(-1) for t in images]) if len(images) > 1 else images[0].reshape(-1).contiguous()
    out, dst_offs = resize_u8_packed(src, offs, [tuple(t.shape[:2]) for t in images], sizes, C, swap_rb=swap_rb)
    shape = (lambda h, w: (h, w)) if images[0].dim() == 2 else (lambda h, w: (h, w, C))
    return [out[o:o + h * w * C].view(*shape(int(h), int(w))) for o, (h, w) in zip(dst_offs, sizes)]


def check_thumbnail_size(size):
    """A thumbnail bound ``(width, height)`` as a tuple of Python ints, or ValueError: two Python or numpy integers >= 1,
    not bools."""
    if not (isinstance(size, (tuple, list)) and len(size) == 2 and all(_is_int(v) and v >= 1 for v in size)):
        raise ValueError("size must be None or (width, height) of integers >= 1, got %r" % (size,))
    return int(size[0]), int(size[1])


def thumbnail_size(w, h, size):
    """The size ``(tw, th)`` that Pillow 12.2's ``Image.thumbnail(size)`` gives a ``w x h`` image, or None when the image
    already fits ``size = (width, height)`` (thumbnail never enlarges). The aspect ratio is kept, each side rounded to
    whichever of floor and ceil keeps it closer, and no side goes below 1."""
    x, y = (math.floor(v) for v in size)
    if x >= w and y >= h:
        return None
    aspect = w / h

    def round_aspect(number, key):
        return max(min(math.floor(number), math.ceil(number), key=key), 1)

    if x / y >= aspect:
        x = round_aspect(y * aspect, key=lambda n: abs(aspect - n / y))
    else:
        y = round_aspect(x / aspect, key=lambda n: 0 if n == 0 else abs(aspect - x / n))
    return x, y


def resize_reducing_u8_packed(src, src_offsets, src_pitches, src_sizes, dst_sizes, out=None, dst_offsets=None):
    """``Image.crop(box).resize(size, reducing_gap=2.0)`` (BICUBIC) of RGB windows, bit for bit, on the device
    (``se_resize_reducing_u8``): Pillow reduces each window by the integer factors ``(int(w / w' / 2) or 1, ...)`` with
    ``Image.reduce`` and resamples the reduced image with a fractional box. This is the resize of ``Image.thumbnail``, whose
    size rule is ``thumbnail_size``. Windows, ``out``, ``dst_offsets`` and the return value are those of
    ``resize_window_u8_packed`` with 3 channels; a window whose size does not change is copied. Only enqueues work on the
    current stream, except that the first resize with a new table uploads it. Scratch (allocated per call, freed on
    return): the reduced images and one pass intermediate each, about 5.3 MB for a 4000x2667 window to 640x427."""
    lib = _lib.load()
    return _resize_windows(src, src_offsets, src_pitches, src_sizes, dst_sizes, 3, out, dst_offsets,
                           lambda a: lambda scratch, size, stream: lib.se_resize_reducing_u8(*a, scratch, size, stream))


def thumbnail_u8(images, size):
    """``Image.thumbnail(size)`` of CUDA uint8 [h, w, 3] RGB images (Pillow 12.2: BICUBIC, reducing_gap=2.0), bit for bit:
    each is resized to ``thumbnail_size(w, h, size)`` by ``resize_reducing_u8_packed``, and an image that already fits is
    copied. An image may be a strided view (a box of a larger photo: pixels packed along a row, rows ``stride(0)`` bytes
    apart); it is read where it lies. Returns the thumbnails, views of one packed tensor."""
    size = check_thumbnail_size(size)
    images = list(images)
    for t in images:
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3):
            raise _lib.SketchEditB200Error("images must be CUDA uint8 [h, w, 3] tensors")
        if t.stride(2) != 1 or (t.stride(1) != 3 and t.shape[1] > 1) or t.stride(0) < 3 * t.shape[1]:
            raise _lib.SketchEditB200Error("an image's pixels must be packed along its rows (got strides %r)" % (t.stride(),))
    if not images:
        return []
    src_sizes = [(int(t.shape[0]), int(t.shape[1])) for t in images]
    dst_sizes = []
    for h, w in src_sizes:
        ts = thumbnail_size(w, h, size)
        dst_sizes.append((h, w) if ts is None else (ts[1], ts[0]))
    # each window as the flat bytes it spans, from its first pixel on
    spans = [t.as_strided(((h - 1) * t.stride(0) + 3 * w,), (1,)) for t, (h, w) in zip(images, src_sizes)]
    out, dst_offs = resize_reducing_u8_packed(spans, [0] * len(spans), [t.stride(0) for t in images], src_sizes, dst_sizes)
    return [out[o:o + h * w * 3].view(h, w, 3) for o, (h, w) in zip(dst_offs, dst_sizes)]


JPEG_MAX_BATCH = 32      # images per se_jpeg_encode_opt_u8 call; the wrappers split longer lists into calls of this size
JPEG_SUBSAMPLING = (0, 2)   # Pillow's subsampling values the encoder takes: 4:4:4 and 4:2:0


def _max_bytes(entry, *args):
    """The file bound ``entry(*args)`` (se_jpeg_max_bytes, se_png_max_bytes), or ValueError with the library's message."""
    n = int(entry(*(int(a) for a in args)))
    if n < 0:
        raise ValueError(_lib.load().se_last_error().decode())
    return n


def jpeg_max_bytes(h, w, subsampling=2, progressive=False):
    """A true upper bound of the JPEG file of an h x w image (``se_jpeg_max_bytes``, or ``se_jpeg_progressive_max_bytes``
    with ``progressive=True``, about 2.2 times as large)."""
    lib = _lib.load()
    return _max_bytes(lib.se_jpeg_progressive_max_bytes if progressive else lib.se_jpeg_max_bytes, h, w, subsampling)


def _is_int(v):
    """An integer argument of the JPEG calls: a Python or numpy integer, not a bool."""
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def _check_jpeg_args(quality, subsampling, optimize=False, progressive=False):
    """(quality, subsampling) as Python ints, or ValueError; ``optimize`` and ``progressive`` must be bools (Python or
    numpy)."""
    if not _is_int(quality) or not 1 <= quality <= 100:
        raise ValueError("quality must be an integer in [1, 100], got %r" % (quality,))
    if not _is_int(subsampling) or subsampling not in JPEG_SUBSAMPLING:
        raise ValueError("subsampling must be 0 (4:4:4) or 2 (4:2:0), got %r" % (subsampling,))
    if not isinstance(optimize, (bool, np.bool_)):
        raise ValueError("optimize must be a bool, got %r" % (optimize,))
    if not isinstance(progressive, (bool, np.bool_)):
        raise ValueError("progressive must be a bool, got %r" % (progressive,))
    return int(quality), int(subsampling)


def _encode(codec, ptrs, pitches, sizes, dev, out=None, out_offsets=None):
    """The encoder ``codec`` over windows already checked, its batch size per call, on the current stream of ``dev``.
    ``codec = (entry, per_call, args, max_bytes)``: the C entry's name (se_jpeg_encode_opt_u8, se_png_encode_u8), images per
    call, its format arguments after n, and the file bound of an h x w window. Returns ``(out, out_offsets, out_bytes)``."""
    entry, per_call, args, max_bytes = codec
    entry = getattr(_lib.load(), entry)
    out, out_offsets = _out(out, out_offsets, [max_bytes(h, w) for h, w in sizes], dev, "out_offsets")
    out_bytes = torch.empty(len(sizes), device=dev, dtype=torch.int64)

    def chunk(sl):
        k = len(ptrs[sl])
        a = ((ctypes.c_void_p * k)(*ptrs[sl]), _longs(pitches[sl]), _ints(sizes[sl]), k, *args, _ptr(out), _longs(out_offsets[sl]),
             ctypes.c_void_p(out_bytes.data_ptr() + 8 * sl.start))
        return lambda scratch, size, stream: entry(*a, scratch, size, stream)

    _run_chunks(len(sizes), per_call, dev, chunk)
    return out, out_offsets, out_bytes


def _encode_packed(codec, channels, src, src_offsets, src_pitches, sizes, out, out_offsets):
    """The body of ``jpeg_encode_u8_packed`` and ``png_encode_u8_packed`` for ``codec`` (``_encode``) on windows of
    ``channels`` bytes per pixel."""
    n = len(sizes)
    srcs = list(src) if isinstance(src, (list, tuple)) else [src] * n
    if not (len(srcs) == len(src_offsets) == len(src_pitches) == n):
        raise _lib.SketchEditB200Error("src (as a list), src_offsets, src_pitches and sizes must have the same length")
    named = [(t, "src") for t in srcs] + ([(out, "out")] if out is not None else [])
    _chk_u8(*named)
    if n == 0:
        return out, out_offsets, None
    dev = _device(*named)
    sizes = _hw(sizes)
    src_offsets, src_pitches = [int(o) for o in src_offsets], [int(p) for p in src_pitches]
    for i, (h, w) in enumerate(sizes):
        if not (1 <= h <= 65535 and 1 <= w <= 65535):
            raise _lib.SketchEditB200Error("window %d: sizes must be in [1, 65535], got %dx%d" % (i, h, w))
    _check_windows("window", srcs, src_offsets, src_pitches, sizes, channels)
    return _encode(codec, [t.data_ptr() + o for t, o in zip(srcs, src_offsets)], src_pitches, sizes, dev, out, out_offsets)


def _encode_list(codec, channels, images):
    """The body of ``jpeg_encode_u8`` and ``png_encode_u8`` for ``codec`` (``_encode``) on a non-empty list of CUDA uint8
    images of ``channels`` bytes per pixel ([h, w, 3], or [h, w] for 1): their files as ``bytes``."""
    shape = "[h, w, 3]" if channels == 3 else "[h, w]"
    for t in images:
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.uint8 and
                (t.dim() == 3 and t.shape[2] == 3 if channels == 3 else t.dim() == 2)):
            raise _lib.SketchEditB200Error("images must be CUDA uint8 %s tensors" % shape)
        if (channels == 3 and t.stride(2) != 1) or (t.stride(1) != channels and t.shape[1] > 1) or t.stride(0) < channels * t.shape[1]:
            raise _lib.SketchEditB200Error("an image's pixels must be packed along its rows (got strides %r)" % (t.stride(),))
        if not (1 <= t.shape[0] <= 65535 and 1 <= t.shape[1] <= 65535):
            raise _lib.SketchEditB200Error("image sizes must be in [1, 65535], got %dx%d" % tuple(t.shape[:2]))
    dev = _device(*[(t, "image") for t in images])
    out, offs, out_bytes = _encode(codec, [t.data_ptr() for t in images], [t.stride(0) for t in images],
                                   [(int(t.shape[0]), int(t.shape[1])) for t in images], dev)
    return download_files(out, offs, out_bytes.cpu().tolist())


def _jpeg_codec(quality, subsampling, optimize, progressive=False):
    """``_encode``'s codec for JPEG at (quality, subsampling, optimize, progressive), checked. A progressive file has
    optimal tables whatever ``optimize`` is, as in libjpeg-turbo."""
    quality, subsampling = _check_jpeg_args(quality, subsampling, optimize, progressive)
    if progressive:
        return ("se_jpeg_encode_progressive_u8", JPEG_MAX_BATCH, (quality, subsampling),
                lambda h, w: jpeg_max_bytes(h, w, subsampling, progressive=True))
    return ("se_jpeg_encode_opt_u8", JPEG_MAX_BATCH, (quality, subsampling, int(bool(optimize))),
            lambda h, w: jpeg_max_bytes(h, w, subsampling))


def jpeg_encode_u8_packed(src, src_offsets, src_pitches, sizes, quality=75, subsampling=2, out=None, out_offsets=None,
                          optimize=False, progressive=False):
    """Baseline JPEG of RGB windows (``se_jpeg_encode_opt_u8``), byte for byte ``Image.save(buf, "JPEG", quality=quality,
    subsampling=subsampling, optimize=optimize)`` of each: image i is the ``sizes[i] = (h, w)`` window whose row r starts at byte ``src_offsets[i] +
    r * src_pitches[i]`` of its source, with ``src_pitches[i] >= 3 w``. ``src`` is one contiguous CUDA uint8 tensor, or a list
    of them with one per image; windows may overlap. ``out`` (optional, contiguous CUDA uint8) receives file i at
    ``out_offsets[i]`` and must hold ``jpeg_max_bytes(h, w, subsampling, progressive)`` bytes there. Returns ``(out,
    out_offsets, out_bytes)``: ``out_bytes`` is a CUDA int64 tensor of the files' lengths. Only enqueues work on the current
    stream. ``progressive=True`` writes ``save(..., progressive=True)``'s file instead (``se_jpeg_encode_progressive_u8``),
    the same whatever ``optimize`` is."""
    return _encode_packed(_jpeg_codec(quality, subsampling, optimize, progressive), 3, src, src_offsets, src_pitches, sizes,
                          out, out_offsets)


def jpeg_encode_u8(images, quality=75, subsampling=2, optimize=False, progressive=False):
    """JPEG files of CUDA uint8 [h, w, 3] RGB images, as ``bytes``: each is what ``Image.fromarray(img).save(buf, "JPEG",
    quality=quality, subsampling=subsampling, optimize=optimize)`` writes. An image may be a strided view (a box of a larger
    photo: pixels packed along a row, rows ``stride(0)`` bytes apart); it is encoded where it lies. One download of the
    lengths, then one of the bytes into pinned staging. quality and subsampling are Python or numpy integers, not bools;
    optimize is a bool. ``optimize=True`` builds Huffman tables for each image from its symbol counts, on the device: the
    pixels are the same and the file smaller. Pillow itself fails (OSError) to write an optimized file larger than its
    buffer of max(64 KiB, h w) bytes (2 h w from quality 95 on), such as noise; the device writes it.

    Device memory: the call allocates, through torch's caching allocator, ``out`` at ``jpeg_max_bytes`` per image and the
    scratch of ``se_jpeg_encode_opt_u8``, both sized for the worst-case file (26 bits per coefficient, every byte stuffed),
    and frees them on return. That is about 6.6 + 6.2 MB for a 1000x667 image at 4:2:0 and 104 + 98 MB for 4000x2667 (twice
    that at 4:4:4), some 50 times a typical file; concurrent calls hold their sum. ``optimize=True`` adds about 12 KB of
    scratch per image (its histograms and tables). Each call also zeroes the word stream in scratch (52 MB at 4000x2667,
    4:2:0).

    ``progressive=True`` (a bool) writes what ``save(..., progressive=True)`` writes, with either value of ``optimize``: the
    ten scans of libjpeg-turbo's jpeg_simple_progression, each with optimal tables from its own counts, coded on the device
    (``se_jpeg_encode_progressive_u8``). A page shows such a file coarse first and sharpens it as the rest arrives. Its
    ``out`` is ``jpeg_max_bytes(..., progressive=True)`` per image and its scratch about 2.2 times the baseline one: some
    229 + 219 MB at 4000x2667 with 4:2:0 (408 + 395 MB at 4:4:4), freed on return."""
    codec = _jpeg_codec(quality, subsampling, optimize, progressive)
    images = list(images)
    return _encode_list(codec, 3, images) if images else []


# ITU T.81 Annex K.1 quantisation bases, natural order: libjpeg's tables at a quality are these scaled (jpeg_quality_tables)
JPEG_LUMA_Q = (16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51,
               87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101,
               72, 92, 95, 98, 112, 100, 103, 99)
JPEG_CHROMA_Q = (17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66) + (99,) * 38
JPEG_MAX_MARKER = 65533       # most bytes after an APP marker's length field: Pillow's bound on its EXIF block and ICC chunks
JPEG_ICC_CHUNK = JPEG_MAX_MARKER - 14   # profile bytes per APP2 segment, after "ICC_PROFILE\0", its number and the count


def jpeg_quality_tables(quality):
    """The luma and chroma tables (natural order) libjpeg uses at ``quality`` in [1, 100] (jpeg_quality_scaling,
    jpeg_add_quant_table with force_baseline): ``save(quality=q)`` is byte for byte ``save(qtables=jpeg_quality_tables(q))``."""
    quality, _ = _check_jpeg_args(quality, 2)
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return [[min(255, max(1, (b * scale + 50) // 100)) for b in base] for base in (JPEG_LUMA_Q, JPEG_CHROMA_Q)]


def jpeg_app_segments(exif=b"", icc_profile=None):
    """The APP1 / APP2 segments Pillow 12.2 writes after APP0 for ``save(..., exif=exif, icc_profile=icc_profile)``, as
    ``bytes``: ``exif`` (bytes or a ``PIL.Image.Exif``, at most 65533 bytes, else ValueError("EXIF data is too long")) as one
    APP1 segment unless empty, then ``icc_profile`` (bytes or None) in chunks of 65519 bytes, each an APP2 segment
    ``ICC_PROFILE\\0`` + its number from 1 + the chunk count + the chunk. At most 255 chunks (a profile under 16 MB)."""
    from PIL import Image
    if isinstance(exif, Image.Exif):
        exif = exif.tobytes()
    if not isinstance(exif, (bytes, bytearray)):
        raise ValueError("exif must be bytes or a PIL.Image.Exif, got %r" % (type(exif).__name__,))
    if icc_profile is not None and not isinstance(icc_profile, (bytes, bytearray)):
        raise ValueError("icc_profile must be bytes or None, got %r" % (type(icc_profile).__name__,))
    if len(exif) > JPEG_MAX_MARKER:
        raise ValueError("EXIF data is too long")
    out = bytearray()
    if exif:
        out += b"\xff\xe1" + (2 + len(exif)).to_bytes(2, "big") + exif
    if icc_profile:
        chunks = [icc_profile[i:i + JPEG_ICC_CHUNK] for i in range(0, len(icc_profile), JPEG_ICC_CHUNK)]
        if len(chunks) > 255:
            raise ValueError("icc_profile is too long: %d bytes make more than 255 APP2 segments" % len(icc_profile))
        for i, c in enumerate(chunks, 1):
            out += b"\xff\xe2" + (2 + 14 + len(c)).to_bytes(2, "big") + b"ICC_PROFILE\0" + bytes([i, len(chunks)]) + c
    return bytes(out)


def _check_qtables(qtables):
    """Quantisation tables as a list of 1 to 4 lists of 64 ints in [0, 255], or ValueError. ``qtables`` is a dict (as
    ``Image.quantization`` gives it: keys 0, 1, ... taken in order, as Pillow takes them) or a list / tuple of tables in
    natural order. An entry above 255 would make Pillow write a 16-bit table and an extended-sequential (SOF1) file, which the
    device encoder does not; such tables are refused."""
    if isinstance(qtables, dict):
        qtables = [qtables[k] for k in range(len(qtables)) if k in qtables]
    if not isinstance(qtables, (list, tuple)) or not 1 <= len(qtables) <= 4:
        raise ValueError("qtables must be 1 to 4 tables of 64 entries")
    out = []
    for t in qtables:
        t = list(t) if isinstance(t, (list, tuple, np.ndarray, array.array)) else None
        if t is None or len(t) != 64 or not all(_is_int(v) for v in t):
            raise ValueError("qtables must be 1 to 4 tables of 64 integers")
        if not all(0 <= v <= 255 for v in t):
            raise ValueError("quantisation table entries must be in [0, 255]: larger ones need a 16-bit table (an "
                             "extended-sequential file), which the encoder does not write")
        out.append([int(v) for v in t])
    return out


def _check_tables_sampling(subsampling):
    """Pillow's subsampling for the tables entry: -1 (libjpeg's default, 4:2:0), 0, 1 or 2, as the entry's 0, 1 or 2."""
    if not _is_int(subsampling) or subsampling not in (-1, 0, 1, 2):
        raise ValueError("subsampling must be -1, 0 (4:4:4), 1 (4:2:2) or 2 (4:2:0), got %r" % (subsampling,))
    return 2 if subsampling == -1 else int(subsampling)


def jpeg_tables_max_bytes(h, w, subsampling, ntables, progressive=False, segments_len=0):
    """A true upper bound of the file ``jpeg_encode_tables_u8`` writes for an h x w image with ``ntables`` tables and
    ``segments_len`` bytes of APP segments (``se_jpeg_tables_max_bytes``)."""
    return _max_bytes(_lib.load().se_jpeg_tables_max_bytes, h, w, _check_tables_sampling(subsampling), ntables,
                      int(bool(progressive)), segments_len)


def jpeg_encode_tables_u8(images, qtables, subsampling, optimize=False, progressive=False, exif=b"", icc_profile=None):
    """JPEG files of CUDA uint8 [h, w, 3] RGB images with the given quantisation tables, as ``bytes``: each is what

        Image.fromarray(img).save(buf, "JPEG", qtables=qtables, subsampling=subsampling, optimize=optimize,
                                  progressive=progressive, exif=exif, icc_profile=icc_profile)

    writes (``se_jpeg_encode_tables_u8``), and so ``src.save(buf, "JPEG", quality="keep", ...)``'s file for
    ``qtables=src.quantization`` and ``subsampling=JpegImagePlugin.get_sampling(src)`` of a JPEG ``src``. ``qtables``: 1 to
    4 tables of 64 entries in [0, 255], natural order, as a list or as ``Image.quantization``'s dict (``_check_qtables``);
    ``subsampling`` -1 (libjpeg's default, 4:2:0), 0 (4:4:4), 1 (4:2:2) or 2 (4:2:0); ``exif`` and ``icc_profile`` as in
    ``jpeg_app_segments``. ``jpeg_quality_tables(q)`` gives the file of ``save(quality=q)``. Images, strides and device
    memory are as in ``jpeg_encode_u8``, plus the segments in each ``out`` slot."""
    qtables = _check_qtables(qtables)
    sub = _check_tables_sampling(subsampling)
    _check_jpeg_args(75, 2, optimize, progressive)
    segments = jpeg_app_segments(exif, icc_profile)
    images = list(images)
    if not images:
        return []
    tabs = (ctypes.c_ushort * (64 * len(qtables)))(*[v for t in qtables for v in t])
    seg = (ctypes.c_ubyte * len(segments)).from_buffer_copy(segments) if segments else None
    codec = ("se_jpeg_encode_tables_u8", JPEG_MAX_BATCH,
             (tabs, len(qtables), sub, int(bool(optimize)), int(bool(progressive)), seg, len(segments)),
             lambda h, w: jpeg_tables_max_bytes(h, w, sub, len(qtables), progressive, len(segments)))
    return _encode_list(codec, 3, images)


def download_files(out, offsets, lengths):
    """The files at ``offsets`` of the CUDA uint8 tensor ``out``, ``lengths[i]`` bytes each, as ``bytes``: one copy into
    pinned staging on the current stream of out's device, then a synchronise of that stream."""
    with torch.cuda.device(out.device):
        staging = torch.empty(max(1, sum(lengths)), dtype=torch.uint8, pin_memory=True)
        at = 0
        for o, k in zip(offsets, lengths):
            staging[at:at + k].copy_(out[o:o + k], non_blocking=True)
            at += k
        torch.cuda.current_stream().synchronize()
    host = staging.numpy()
    res, at = [], 0
    for k in lengths:
        res.append(host[at:at + k].tobytes())
        at += k
    return res


PNG_MAX_BATCH = 32       # images per se_png_encode_u8 call; the wrappers split longer lists into calls of this size


def png_max_bytes(h, w, channels=3):
    """A true upper bound of the PNG file of an h x w image of ``channels`` (1 or 3) bytes per pixel (``se_png_max_bytes``)."""
    return _max_bytes(_lib.load().se_png_max_bytes, h, w, channels)


def _png_codec(channels, swap_rb):
    """``_encode``'s codec for PNG of ``channels`` bytes per pixel (``swap_rb``: BGR pixels)."""
    return "se_png_encode_u8", PNG_MAX_BATCH, (channels, int(bool(swap_rb))), lambda h, w: png_max_bytes(h, w, channels)


def png_encode_u8_packed(src, src_offsets, src_pitches, sizes, channels, swap_rb=False, out=None, out_offsets=None):
    """PNG files of windows (``se_png_encode_u8``), byte for byte ``cv2.imencode(".png", img)[1]`` of each with img the window
    as BGR (``channels`` 3) or grey (1): image i is the ``sizes[i] = (h, w)`` window whose row r starts at byte ``src_offsets[i] +
    r * src_pitches[i]`` of its source, with ``src_pitches[i] >= channels * w``. ``swap_rb`` says the pixels are BGR (the
    forward's output); otherwise they are RGB. ``src`` is one contiguous CUDA uint8 tensor, or a list of them with one per image;
    windows may overlap. ``out`` (optional, contiguous CUDA uint8) receives file i at ``out_offsets[i]`` and must hold
    ``png_max_bytes(h, w, channels)`` bytes there. Returns ``(out, out_offsets, out_bytes)``: ``out_bytes`` is a CUDA int64
    tensor of the files' lengths. Only enqueues work on the current stream."""
    if channels not in (1, 3) or isinstance(channels, bool):
        raise ValueError("channels must be 1 or 3, got %r" % (channels,))
    return _encode_packed(_png_codec(channels, swap_rb), channels, src, src_offsets, src_pitches, sizes, out, out_offsets)


def png_encode_u8(images, swap_rb=False):
    """PNG files of CUDA uint8 images, as ``bytes``: [h, w, 3] RGB (``swap_rb``: BGR) or [h, w] grey, one channel count for the
    list. Each is ``cv2.imencode(".png", img)[1]`` of the image as BGR or grey. An image may be a strided view (a box of a larger
    photo: pixels packed along a row, rows ``stride(0)`` bytes apart); it is encoded where it lies. One download of the lengths,
    then one of the bytes into pinned staging.

    Device memory: the call allocates, through torch's caching allocator, ``out`` at ``png_max_bytes`` per image (the
    filtered data, h (1 + w c) bytes, stored) and the scratch of ``se_png_encode_u8`` (about 1.2 bytes per filtered byte, the
    word stream included), and frees them on return: about 2 + 2.4 MB for a 1000x667 RGB image and 32 + 38 MB for 4000x2667;
    concurrent calls hold their sum. Each call also zeroes the word stream in scratch (32 MB at 4000x2667)."""
    images = list(images)
    if not images:
        return []
    chans = {1 if isinstance(t, torch.Tensor) and t.dim() == 2 else 3 for t in images}
    if len(chans) > 1:
        raise _lib.SketchEditB200Error("images must all be [h, w] or all be [h, w, 3]")
    C = chans.pop()
    return _encode_list(_png_codec(C, swap_rb), C, images)


PNG_DECODE_MAX_BATCH = 256   # files per se_png_decode_u8 call; the wrappers split longer lists into calls of this size
# Files of at least this many raw bytes (filtered scanlines, h (1 + row bytes)) go to se_png_split_u8, one file per call,
# the rest to se_png_decode_u8's one warp per file. tools/png_split_bench.py measured the crossover (DESIGN.md 7b).
PNG_SPLIT_MIN_RAW = 4 << 20
PNG_SPLIT_MIN_CHUNK = 16 << 10   # compressed bytes per chunk of the split decoder: about one of zlib's default blocks
PNG_SPLIT_MAX_CHUNKS = 4096      # chunks per file; longer streams get longer chunks


def png_split_chunk_bytes(stream_bytes):
    """The chunk spacing of se_png_split_u8 for a zlib stream of ``stream_bytes`` bytes."""
    return max(PNG_SPLIT_MIN_CHUNK, -(-int(stream_bytes) // PNG_SPLIT_MAX_CHUNKS))


def png_raw_bytes(hd):
    """The raw filtered scanlines of the ``pngfile.PngHead`` hd: h (1 + row bytes)."""
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[hd.ctype]
    return hd.h * (1 + (hd.w * ch * hd.depth + 7) // 8)


def png_stage(heads):
    """The streams of the ``pngfile.PngHead`` list ``heads`` packed into one pinned uint8 tensor (``pngfile.stage``, the layout
    ``png_decode_u8_packed`` reads): ``(staging, offsets, lengths)`` of the streams."""
    return pngfile.stage(heads, lambda n: torch.empty(n, dtype=torch.uint8, pin_memory=True))


def png_decode_u8_packed(src, src_offsets, src_lengths, heads, modes, out=None, out_offsets=None):
    """Pixels of PNG files from their zlib streams (``se_png_decode_u8``), one launch per PNG_DECODE_MAX_BATCH files: file
    i's IDAT payloads, joined, are the ``src_lengths[i]`` bytes at ``src_offsets[i]`` of the contiguous CUDA uint8 tensor
    ``src``, followed there by its palette when it has one (``png_stage``'s layout); ``heads[i]`` is its
    ``pngfile.PngHead`` (size, depth, colour type, palette length; its ``stream`` is not read) and ``modes[i]`` (or one
    ``modes`` for all) is "RGB" or "L". ``out`` (optional) is one contiguous CUDA uint8 tensor or a list of them with one
    per file; file i's h x w x 3 or h x w bytes go to ``out_offsets[i]`` of its tensor. Returns ``(out, out_offsets,
    status)``: ``status`` is a CUDA int32 tensor, 0 where the pixels are ``np.asarray(Image.open(f).convert(mode))`` and
    nonzero where the file must go to Pillow. Only enqueues work on the current stream.

    A file of ``PNG_SPLIT_MIN_RAW`` raw bytes or more is decoded by ``se_png_split_u8`` across the whole GPU, with chunks of
    ``png_split_chunk_bytes`` of its stream; the others by one warp each. The split decoder's scratch is the file's raw
    scanlines plus 4 bytes per raw byte (about 160 MB for a 4000x2667 RGB file), held while the call runs."""
    n = len(heads)
    modes = [modes] * n if isinstance(modes, str) else list(modes)
    if len(modes) != n or len(src_offsets) != n or len(src_lengths) != n:
        raise _lib.SketchEditB200Error("src_offsets, src_lengths, heads and modes must have the same length")
    if any(m not in pngfile.MODES for m in modes):
        raise ValueError("modes must be 'RGB' or 'L', got %r" % (modes,))
    outs = list(out) if isinstance(out, (list, tuple)) else None
    if outs is not None and len(outs) != n:
        raise _lib.SketchEditB200Error("out (as a list) needs one tensor per file")
    named = [(src, "src")] + [(t, "out") for t in (outs if outs is not None else [out] if out is not None else [])]
    _chk_u8(*named)
    dev = _device(*named)
    src_offsets, src_lengths = [int(o) for o in src_offsets], [int(k) for k in src_lengths]
    plens = [len(hd.palette) for hd in heads]
    _check_windows("stream", src, src_offsets, [k + p for k, p in zip(src_lengths, plens)],
                   [(1, k + p) for k, p in zip(src_lengths, plens)], 1)
    plte_offs = [o + k for o, k in zip(src_offsets, src_lengths)]
    chans = [pngfile.MODES[m] for m in modes]
    nbytes = [hd.h * hd.w * c for hd, c in zip(heads, chans)]
    if outs is None:
        out, out_offsets = _out(out, out_offsets, nbytes, dev, "out_offsets")
        outs = [out] * n
    else:
        if out_offsets is None or len(out_offsets) != n:
            raise _lib.SketchEditB200Error("out needs one out_offsets entry per file")
        out_offsets = [int(o) for o in out_offsets]
        _check_windows("out", outs, out_offsets, nbytes, [(1, b) for b in nbytes], 1)
    status = torch.empty(n, device=dev, dtype=torch.int32)
    if n == 0:
        return out, out_offsets, status
    info = [(hd.h, hd.w, hd.depth, hd.ctype, len(hd.palette) // 3, c) for hd, c in zip(heads, chans)]
    dst = [t.data_ptr() + o for t, o in zip(outs, out_offsets)]
    lib = _lib.load()

    def call(sl, split):
        k = len(info[sl])
        a = (_ptr(src), _longs(src_offsets[sl]), _longs(src_lengths[sl]), _ints(info[sl]), _longs(plte_offs[sl]), k,
             (ctypes.c_void_p * k)(*dst[sl]), ctypes.c_void_p(status.data_ptr() + 4 * sl.start))
        if split:
            S = png_split_chunk_bytes(src_lengths[sl.start])
            return lambda scratch, size, stream: lib.se_png_split_u8(*a, S, scratch, size, stream)
        return lambda scratch, size, stream: lib.se_png_decode_u8(*a, scratch, size, stream)

    # runs of consecutive files of one decoder: one split file per call, up to PNG_DECODE_MAX_BATCH one-warp files
    split = [png_raw_bytes(hd) >= PNG_SPLIT_MIN_RAW for hd in heads]
    calls, k = [], 0
    while k < n:
        j = k + 1
        while j < n and not split[k] and not split[j] and j - k < PNG_DECODE_MAX_BATCH:
            j += 1
        calls.append(call(slice(k, j), split[k]))
        k = j
    _run_calls(calls, dev)
    return out, out_offsets, status


def png_decode_into(staged, heads, modes, files, dst, names, device):
    """Pixels of PNG files into place, always Pillow's: file k (``bytes``) is decoded to ``modes[k]`` ("RGB" or "L").
    ``heads[k]`` is its ``pngfile.PngHead``, or None when the parser sent it to Pillow; ``staged = (staging, offsets,
    lengths)`` holds the streams of the parsed files in order (``pngfile.stage``'s layout in a host tensor). ``dst[k] =
    (tensor, byte offset, (h, w))`` is where its pixels go in a CUDA uint8 tensor and the size its header gives, or None for
    a tensor of its own. The parsed files are decoded on ``device`` straight into place (one upload of the streams), the
    host waits once for the status words, then Pillow decodes the files the parser or the device refused, each checked
    against its size (a ``RuntimeError`` naming ``names[k]``) and uploaded. Runs on the current stream; returns
    ``{k: tensor}`` for the files without a ``dst``."""
    on_dev = [k for k, hd in enumerate(heads) if hd is not None]
    bad = [k for k, hd in enumerate(heads) if hd is None]
    if on_dev:
        staging, offsets, lengths = staged
        status = png_decode_u8_packed(staging.to(device, non_blocking=True), offsets, lengths, [heads[k] for k in on_dev],
                                      [modes[k] for k in on_dev], out=[dst[k][0] for k in on_dev],
                                      out_offsets=[dst[k][1] for k in on_dev])[2]
        status_h = torch.empty(len(on_dev), dtype=torch.int32, pin_memory=True)
        status_h.copy_(status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        ev.synchronize()
        bad += [k for k, s in zip(on_dev, status_h.tolist()) if s]
    own = {}
    for k in bad:
        px = np.array(pngfile.pillow_decode(files[k], modes[k]))   # a writable copy for torch
        if dst[k] is None:
            own[k] = torch.from_numpy(px).to(device)
            continue
        buf, o, hw = dst[k]
        if px.shape[:2] != tuple(hw):
            raise RuntimeError("%s decodes to %dx%d, its header says %dx%d" % ((names[k],) + px.shape[:2] + tuple(hw)))
        buf[o:o + px.size].copy_(torch.from_numpy(px).reshape(-1).pin_memory(), non_blocking=True)
    return own


def png_decode_u8(files, mode="RGB", device=None):
    """Pixels of PNG files (``bytes``) as CUDA uint8 tensors, [h, w, 3] for ``mode`` "RGB" and [h, w] for "L", each equal to
    ``np.asarray(Image.open(f).convert(mode))``, Pillow's exception included. Files ``pngfile.parse`` accepts are decoded on
    the device (one upload of their streams from pinned staging, then one download of the status words); the others, and
    any the device reports a nonzero status for, are decoded by Pillow and uploaded.

    Device memory: the pixels, the compressed streams and, while the call runs, each file's raw filtered scanlines
    (h (1 + w bytes per pixel) bytes)."""
    files = list(files)
    dev = torch.device("cuda") if device is None else torch.device(device)
    heads = []
    for f in files:
        try:
            heads.append(pngfile.parse(f))
        except pngfile.Host:
            heads.append(None)
    parsed = [hd for hd in heads if hd is not None]
    c = pngfile.MODES[mode]
    with torch.cuda.device(dev):
        offs, total = _aligned_offsets([hd.h * hd.w * c for hd in parsed])
        out = torch.empty(max(total, 1), device=dev, dtype=torch.uint8)
        at = iter(offs)
        dst = [None if hd is None else (out, next(at), (hd.h, hd.w)) for hd in heads]
        res = png_decode_into(png_stage(parsed) if parsed else None, heads, [mode] * len(files), files, dst,
                              ["file %d" % i for i in range(len(files))], dev)
    for i, (d, hd) in enumerate(zip(dst, heads)):
        if d is not None:
            res[i] = out[d[1]:d[1] + hd.h * hd.w * c].view((hd.h, hd.w, c) if c == 3 else (hd.h, hd.w))
    return [res[i] for i in range(len(files))]


def outputs_to_uint8(composed, mask):
    """test.py:25-27 on device -> (uint8 [B,H,W,3] BGR, uint8 [B,H,W])."""
    lib = _lib.load()
    composed, mask = _chk_in(composed), _chk_in(mask)
    B, _, H, W = composed.shape
    bgr = torch.empty(B, H, W, 3, device=composed.device, dtype=torch.uint8)
    mk = torch.empty(B, H, W, device=composed.device, dtype=torch.uint8)
    _lib.check(lib.se_outputs_to_uint8(_ptr(composed), _ptr(mask), B, H, W, _ptr(bgr), _ptr(mk), _stream()))
    return bgr, mk

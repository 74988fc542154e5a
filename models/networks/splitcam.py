"""Contextual attention modules with the reference's two-module surface
(reference models/networks/splitcam.py:17-174). On the GPU path similarity, masking, softmax and the
fold-sum paste run as ONE fused C-ABI call (``se_contextual_attention_forward``); P1 returns the
attention weights like the reference and hands the pasted features to P2 through the tensor it returns.
Only the configuration netG instantiates is implemented (editline_g.py:35-42)."""
import torch
import torch.nn as nn


class ReduceContextAttentionP1(nn.Module):
    def __init__(self, bkg_patch_size=4, stride=1, ufstride=1, softmax_scale=10., nn_hard=False, pd=1,
                 fuse_k=3, is_fuse=False, th=0.5, norm_type=1, is_th=False):
        super().__init__()
        cfg = (bkg_patch_size, stride, ufstride, softmax_scale, nn_hard, pd, is_fuse, th, norm_type, is_th)
        if cfg != (4, 2, 2, 10., False, 0, False, 0.1, 1, True):
            raise NotImplementedError("the CUDA contextual attention implements netG's configuration only "
                                      "(patch 4, stride 2, pd 0, scale 10, is_th th=0.1, norm_type 1); got %r" % (cfg,))
        self.precision = "bf16"

    def forward(self, f, b, mask=None):
        from sketchedit_b200.engine import contextual_attention
        if f.data_ptr() != b.data_ptr() or f.shape != b.shape:
            raise NotImplementedError("query and key maps must be the same tensor (netG calls cam_1(x, x, mask_s))")
        if mask is None:
            mask = torch.zeros(f.shape[0], 1, f.shape[2], f.shape[3], device=f.device)
        out, attn = contextual_attention(f.float(), mask.float(), precision=self.precision, want_attn=True)
        B, _, h, w = f.shape
        hs, ws = (h - 4) // 2 + 1, (w - 4) // 2 + 1
        attn = attn.view(B, hs * ws, hs, ws)
        attn._se_pasted = (b.data_ptr(), out)
        return attn


class ReduceContextAttentionP2(nn.Module):
    def __init__(self, bkg_patch_size=16, stride=8, ufstride=8, pd=4, mk=True):
        super().__init__()
        if (bkg_patch_size, stride, ufstride, pd, mk) != (4, 2, 2, 0, False):
            raise NotImplementedError("the CUDA contextual attention implements netG's paste configuration only")

    def forward(self, cos_similar, b, mask, dict_aux):
        if dict_aux:
            raise NotImplementedError("auxiliary reconstructions (dict_aux) are not on the inference path")
        tag = getattr(cos_similar, "_se_pasted", None)
        if tag is None or tag[0] != b.data_ptr():
            raise NotImplementedError("cam_2 must receive the attention returned by cam_1 for the same feature map")
        return tag[1], {}

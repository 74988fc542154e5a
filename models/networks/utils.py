"""Gated convolution modules with the reference's constructor signatures and parameter layout
(reference models/networks/utils.py:9-51). They own the fp32 OIHW ``weight`` / ``bias`` parameters
(state_dict source of truth); ``forward`` runs the layer on the CUDA kernels through the C ABI
(``se_gated_conv_forward``) -- the wgmma implicit-GEMM with the fused bias/ELU x sigmoid epilogue in
bf16 mode, the fp32 CUDA-core kernel in fp32 mode. No torch compute op is on this path."""
import torch
import torch.nn as nn


class gen_conv(nn.Conv2d):
    def __init__(self, cin, cout, ksize, stride=1, rate=1, activation=nn.ELU()):
        pad = int(rate * (ksize - 1) / 2)
        super().__init__(in_channels=cin, out_channels=cout, kernel_size=ksize, stride=stride, padding=pad,
                         dilation=rate, groups=1, bias=True)
        self.activation = activation
        self._se_owner = None      # (network module, layer name), set by the owning generator

    def _bound(self):
        if self._se_owner is None:
            raise RuntimeError("this gen_conv is not attached to a MDGenerator / DeepFillC2Generator; the CUDA path "
                               "packs weights per network (there is no stand-alone or CPU fallback)")
        return self._se_owner

    def forward(self, x):
        net, name = self._bound()
        return net.engine().gated_conv(net.NET_ID, name, x.float(), precision=net.precision)


class gen_deconv(gen_conv):
    """nearest x2 upsample followed by a 3x3 gated conv (reference utils.py:35-51); on the CUDA path the
    upsample is folded into four sub-pixel 2x2 convolutions and never materialised."""

    def __init__(self, cin, cout):
        super().__init__(cin, cout, ksize=3)


def bind_layers(net):
    """Give every gen_conv child of `net` a back-reference (without registering a module cycle)."""
    for name, mod in net.named_children():
        if isinstance(mod, gen_conv):
            object.__setattr__(mod, "_se_owner", (net, name))

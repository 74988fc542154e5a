"""GPU parity of the operators behind gen_conv / gen_deconv / contextual attention, through the C ABI.

fp32 mode  : "fp32" = fp32-parity arithmetic on the tensor cores (split-half fp16 operands, three wgmma products per tap),
             "fp32_direct" = the fp32 CUDA-core kernels (its cross-check); both vs the fp32 oracle, tolerance 1e-4 (abs,
             activations are O(1)).
bf16 mode  : wgmma kernels vs the oracle evaluated on the SAME bf16-rounded inputs and weights, so the
             only differences are fp32 accumulation order and the final bf16 rounding of the output:
             tolerance 2^-8 relative to max|y| (one bf16 ulp at the top of the range) + 1e-3.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import sketchedit_oracle as O
from tests.util_parity import bf16_round, engine, maxdiff, oracle_layer, rand_act
from sketchedit_b200.arch import layer_map

pytestmark = pytest.mark.gpu

# (net, layer, H, W): every distinct shape class of SURVEY.md section 8(d); odd tile remainders on purpose
LAYER_CASES = [
    ("M", "conv1", 24, 40),                     # 5x5 stem, 4 ch
    ("G", "conv1", 16, 16),                     # 5x5 stem, 5 ch
    ("G", "xconv1", 16, 32),                    # 5x5 stem, 3 ch
    ("M", "conv2_downsample", 32, 48),          # 24->96 s2
    ("G", "xconv2_downsample", 16, 32),         # 24->48 s2
    ("M", "conv3", 16, 24),                     # 48->96
    ("G", "xconv3", 16, 24),                    # 24->96
    ("M", "conv4_downsample", 32, 32),          # 48->192 s2
    ("G", "xconv4_downsample", 16, 48),         # 48->96 s2
    ("G", "xconv5", 8, 24),                     # 48->192
    ("M", "conv5", 16, 16),                     # 96->192
    ("M", "conv7_atrous", 16, 24),              # rate 2
    ("M", "conv8_atrous", 16, 16),              # rate 4
    ("M", "conv9_atrous", 24, 16),              # rate 8
    ("M", "conv10_atrous", 40, 24),             # rate 16
    ("G", "conv11", 16, 16),                    # 192->192
    ("G", "pmconv6", 8, 16),                    # ReLU gate
    ("M", "conv13_upsample_conv", 8, 24),       # deconv 96->96
    ("M", "conv15_upsample_conv", 16, 16),      # deconv 48->48
    ("M", "conv16", 16, 32),                    # 24->24
    ("M", "conv17", 16, 24),                    # head 12->3
    ("M", "conv_mask_17", 24, 16),              # head 12->1
]


@pytest.mark.parametrize("prec", ["fp32", "fp32_direct"])
@pytest.mark.parametrize("net,name,H,W", LAYER_CASES)
def test_gated_conv_fp32(net, name, H, W, prec):
    spec = layer_map(net)[name]
    x = rand_act((2, spec.cin, H, W), seed=hash((net, name)) % 1000)
    x = x + 1e-3 * rand_act((2, spec.cin, H, W), seed=hash((net, name)) % 1000 + 1)      # not bf16-representable: the lo halves matter
    y = engine().gated_conv(net, name, x.cuda(), precision=prec).cpu()
    ref = oracle_layer(net, name, x, bf16_weights=False)
    assert y.shape == ref.shape
    assert maxdiff(y, ref) <= 1e-4, (name, maxdiff(y, ref))


@pytest.mark.parametrize("net,name,H,W", LAYER_CASES)
def test_gated_conv_bf16_tensor_core(net, name, H, W):
    spec = layer_map(net)[name]
    x = rand_act((2, spec.cin, H, W), seed=hash((net, name)) % 1000 + 7)
    y = engine().gated_conv(net, name, x.cuda(), precision="bf16").cpu()
    head = spec.cin == 12
    ref = oracle_layer(net, name, x, bf16_weights=not head)   # heads keep fp32 weights on the CUDA-core path
    tol = float(ref.abs().max()) * 2.0 ** -8 + 1e-3
    if spec.kind == "deconv":
        tol *= 2     # sub-pixel taps are summed in fp32 and THEN rounded to bf16 (oracle rounds each tap)
    assert maxdiff(y, ref) <= tol, (name, maxdiff(y, ref), tol)


# (128, 128): Places config, L = 3969 keys; (128, 102): the reference's 408-wide input, L = 63 * 50 = 3150; (64, 64): CelebA, L = 961
CAM_CASES = [(16, 16, 2), (12, 20, 1), (32, 32, 1), (64, 64, 2), (128, 128, 1), (128, 102, 1)]


@pytest.mark.parametrize("h,w,B", CAM_CASES)
def test_contextual_attention_fp32(h, w, B):
    feat = F.relu(rand_act((B, 96, h, w), seed=h * w))          # pmconv6 output is ReLU-gated: non-negative
    mask = torch.zeros(B, 1, 4 * h, 4 * w)
    mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
    mask_s = F.avg_pool2d(mask, 4, 4)
    from sketchedit_b200.engine import contextual_attention
    out, attn = contextual_attention(feat.cuda(), mask_s.cuda(), precision="fp32", want_attn=True)
    ref, A = O.contextual_attention(feat, mask_s)
    assert maxdiff(attn.cpu(), A) <= 2e-4
    assert maxdiff(out.cpu(), ref) <= 2e-4 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("h,w,B", CAM_CASES)
def test_contextual_attention_fp32_split_gemm(h, w, B):
    """precision='fp32' without the attention-map output: the split-half fp16 wgmma GEMM attention (se_gemm_split.cu), which the
    fp32-on-tensor-cores forward uses; same tolerance as the CUDA-core fp32 attention above."""
    feat = F.relu(rand_act((B, 96, h, w), seed=h * w))
    mask = torch.zeros(B, 1, 4 * h, 4 * w)
    mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
    mask_s = F.avg_pool2d(mask, 4, 4)
    from sketchedit_b200.engine import contextual_attention
    out = contextual_attention(feat.cuda(), mask_s.cuda(), precision="fp32")
    ref, _ = O.contextual_attention(feat, mask_s)
    assert maxdiff(out.cpu(), ref) <= 2e-4 * max(1.0, float(ref.abs().max())), (maxdiff(out.cpu(), ref), float(ref.abs().max()))


@pytest.mark.parametrize("h,w,B", CAM_CASES)
def test_contextual_attention_bf16(h, w, B):
    # soft attention (small features) so bf16 logits cannot flip a hard arg-max
    feat = F.relu(rand_act((B, 96, h, w), seed=h * w + 1, scale=0.15))
    mask = torch.zeros(B, 1, 4 * h, 4 * w)
    mask[:, :, h:3 * h, w:2 * w + 8] = 1.0
    mask_s = F.avg_pool2d(mask, 4, 4)
    from sketchedit_b200.engine import contextual_attention
    out = contextual_attention(feat.cuda(), mask_s.cuda(), precision="bf16").cpu()
    ref, _ = O.contextual_attention(feat, mask_s)
    tol = 2e-2 * max(1.0, float(ref.abs().max()))
    assert maxdiff(out, ref) <= tol, (maxdiff(out, ref), tol)


def test_bad_arguments_fail_loudly():
    from sketchedit_b200._lib import SketchEditB200Error
    eng = engine()
    with pytest.raises(SketchEditB200Error):
        eng.gated_conv("M", "conv5", torch.zeros(1, 96, 8, 8), precision="bf16")        # CPU tensor
    with pytest.raises(SketchEditB200Error):
        eng.inference(torch.zeros(1, 3, 20, 20).cuda(), torch.zeros(1, 1, 20, 20).cuda())   # not a multiple of 8
    x, y = torch.zeros(1, 96, 8, 8).cuda(), torch.zeros(1, 96, 8, 8).cuda()
    rc = eng.lib.se_gated_conv_forward(eng.h, b"M", b"conv5", x.data_ptr(), 1, 8, 8, 2, y.data_ptr(), None)   # retired precision 2
    assert rc != 0 and b"precision 2" in eng.lib.se_last_error()

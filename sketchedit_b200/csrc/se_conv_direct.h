// CUDA-core direct convolution (se_conv_direct.cu).
#pragma once
#include "se_common.cuh"

namespace se {
// fp32 in and out; weights: fp32 [img][tap][Ci][CoutP]
int direct_launch(const ConvParams& c, int CoutP, cudaStream_t stream);
}  // namespace se

// Region-edit detail (se_detail.cu): the high frequencies a region edit's resize round trip removes, spread into the hole with
// netG's own attention weights (contextual residual aggregation), as an int16 plane the paste adds to the upsampled result.
#pragma once
#include "se_common.cuh"

namespace se {

// hole[i] = mbin[i] > 0.5 as 0 / 1 bytes: the mask netG inpaints, for se_forward_u8_export
int detail_hole_u8(const float* mbin, unsigned char* hole, long long n, cudaStream_t stream);

}  // namespace se

// Pillow-exact bicubic resampling of uint8 HWC images (se_resize.cu): the arithmetic of PIL.Image.resize(size) with the
// default filter (BICUBIC, no box, no reducing_gap) for 1- and 3-channel images, batched over images of different sizes.
#pragma once
#include "se_common.cuh"

namespace se {

constexpr int RESIZE_MAX_BATCH = 32;   // images per call: their descriptors travel as kernel parameters
constexpr int RESIZE_PREC_BITS = 22;   // fractional bits of the fixed-point coefficients (Pillow's PRECISION_BITS for 8 bpc)

// Pillow's coefficient table for one axis (in -> out samples): bounds[2*i] = first input sample of output i, bounds[2*i+1] =
// number of taps; coeffs[i*ksize + k] the fixed-point weights (zero beyond the taps). Host only. Returns ksize.
int resize_coeff_table(int in, int out, int* bounds, int* coeffs);
int resize_ksize(int in, int out);

}  // namespace se

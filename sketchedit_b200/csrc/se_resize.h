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

// The feather ramp of a box's paste mask (se_resize_composite_feather_u8, se_feather_u8), over one pair of opposite sides:
// a side of width f gives the pixel at distance d from its edge pixel (d = 0 on it) 255 * (d + 1) / (f + 1) when d < f and
// 255 otherwise; the ramp of a pixel is the least over its row's pair (top, bottom) and its column's pair (left, right).
// The division runs only inside a band and is exact integer division.
__device__ __forceinline__ int feather_pair(int d0, int d1, int f0, int f1) {
  int r = 255;
  if (d0 < f0) r = 255 * (d0 + 1) / (f0 + 1);
  if (d1 < f1) r = min(r, 255 * (d1 + 1) / (f1 + 1));
  return r;
}
// Pillow's paste rounding: DIV255(a) = (((a + 128) >> 8) + a + 128) >> 8; DIV255(255 * m) == m for every byte m
__device__ __forceinline__ int div255(int a) {
  const int t = a + 128;
  return ((t >> 8) + t) >> 8;
}

}  // namespace se

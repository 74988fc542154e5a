// Host-side interface of se_resize.cu for the other image entries of the library (se_thumbnail.cu).
#pragma once
#include <cuda_runtime.h>

#include "se_common.cuh"

namespace se {

constexpr int RESIZE_MAX_BATCH = 32;   // images per launch: their descriptors travel as kernel parameters

// One RGB image of resize_box_rgb: ih x iw pixels, row r at src + r * pitch, resampled to oh x ow (packed rows at dst) as
// Pillow's ImagingResample with the box (0, 0, in1_w, in1_h), box ends in C floats. An axis is resampled when its length
// changes or its box end is not its length (need_horizontal / need_vertical); v_first runs the vertical pass first. mid
// holds the pass intermediate when both axes are resampled: box_mid_bytes(b) bytes.
struct BoxResize {
  const unsigned char* src;
  long long pitch;
  int ih, iw;
  float in1_h, in1_w;
  unsigned char* dst;
  int oh, ow;
  unsigned char* mid;
  int v_first;
};
inline bool box_needs_h(const BoxResize& b) { return b.ow != b.iw || b.in1_w != (float)b.iw; }
inline bool box_needs_v(const BoxResize& b) { return b.oh != b.ih || b.in1_h != (float)b.ih; }
inline size_t box_mid_bytes(const BoxResize& b) {
  if (!box_needs_h(b) || !box_needs_v(b)) return 0;
  return scratch_round((size_t)(b.v_first ? b.oh * (size_t)b.iw : b.ih * (size_t)b.ow) * 3);
}

// Enqueues the passes of n <= RESIZE_MAX_BATCH images on st (an image needing neither pass is copied); the coefficient
// tables come from the device cache of se_resize.cu under its limit, keyed by (in, in1, out). Every table's ksize must fit
// the kernels' shared memory: a box scale in1 / out below 64 does.
int resize_box_rgb(const BoxResize* im, int n, cudaStream_t st);

}  // namespace se

// Pillow's reducing resize of RGB windows: Image.crop(box).resize(size, BICUBIC, reducing_gap=2.0), the resize of
// Image.thumbnail(size) (Pillow 12.2, PIL/Image.py resize and _get_safe_box), bit for bit.
//
// For a window of w x h pixels resized to ow x oh, Pillow takes the integer factors fx = int(w / ow / 2) or 1, fy likewise.
// If either is > 1 it first reduces the whole window (Image.reduce((fx, fy)); for a whole image _get_safe_box is the image
// itself): ceil(w / fx) x ceil(h / fy) cells, each averaged over the pixels it covers, so the right and bottom cells may be
// partial. Per channel, with s the cell's byte sum and n its pixel count, in uint32 arithmetic (libImaging/Reduce.c):
//     out = ((s + n / 2) * m) >> 24,   m = uint32(float(2^32) / float(256 n)).
// It then resamples the reduced image bicubically over the box (0, 0, w / fx, h / fy), box ends in C floats: the coefficient
// tables of se_resize.cu with scale = in1 / out. An axis is resampled when its length changes or its box end is not its
// length; a reduced image more than 100 times taller than wide whose height shrinks is resampled vertically first, any other
// horizontally first. Both passes are se_resize.cu's kernels (resize_box_rgb). The resample's scale stays below 4 (the
// reduce leaves less than twice reducing_gap), so its tables are at most 17 taps wide.
//
// reduce_kernel: a group of 2^lg threads per cell (lg chosen per image from the cell's size: one thread for the 3 x 3 cells
// of a 4000 x 2667 photo to 640 x 427, up to a block for the cells of a 1 x 1 thumbnail); the group's threads stride over
// the cell's columns and rows, and their uint32 sums meet through shuffles (and shared memory past a warp). uint32 sums
// wrap as Pillow's do; cells hold fewer than 2^24 pixels, so 256 n is exact in a float.
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_resize.h"

namespace se {

constexpr int R_THREADS = 256;
constexpr long long kMaxCell = (1LL << 24) - 1;   // pixels of a reduce cell

struct RImage {   // the reduce of one window: h x w pixels at src (rows pitch bytes apart) into oh x ow cells at dst (packed)
  const unsigned char* src;
  unsigned char* dst;
  long long pitch;
  int h, w, fx, fy, oh, ow;
  int lgx, lgy;   // 2^lgx x 2^lgy threads per cell, along its columns and its rows
  int block0;
};
struct ReduceList {
  RImage im[RESIZE_MAX_BATCH];
  int n;
};
static_assert(sizeof(ReduceList) <= 4096, "reduce descriptors must fit the kernel parameter space");

__global__ void __launch_bounds__(R_THREADS) reduce_kernel(const __grid_constant__ ReduceList L) {
  __shared__ uint32_t part[R_THREADS / 32][3];
  const RImage& d = L.im[image_of(L.im, L.n, &RImage::block0, (int)blockIdx.x)];
  const int lg = d.lgx + d.lgy;   // the same for every thread of the block
  const int j = threadIdx.x & ((1 << lg) - 1);
  const long long cell = (long long)(blockIdx.x - d.block0) * (R_THREADS >> lg) + (threadIdx.x >> lg);
  const bool valid = cell < (long long)d.oh * d.ow;
  uint32_t s0 = 0, s1 = 0, s2 = 0;
  int n = 0;
  if (valid) {
    const int cy = (int)(cell / d.ow), cx = (int)(cell - (long long)cy * d.ow);
    const int cw = min(d.fx, d.w - cx * d.fx), ch = min(d.fy, d.h - cy * d.fy);
    n = cw * ch;
    const unsigned char* p = d.src + (size_t)cy * d.fy * d.pitch + (size_t)cx * d.fx * 3;
    const int jx = j & ((1 << d.lgx) - 1), jy = j >> d.lgx;
    for (int r = jy; r < ch; r += 1 << d.lgy) {
      const unsigned char* q = p + (size_t)r * d.pitch;
      for (int c = jx; c < cw; c += 1 << d.lgx) {
        s0 += q[3 * c];
        s1 += q[3 * c + 1];
        s2 += q[3 * c + 2];
      }
    }
  }
  for (int o = 1; o < (1 << min(lg, 5)); o <<= 1) {   // groups are aligned runs of lanes
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lg > 5) {   // a group of several warps: lane 0 of the group's first warp adds the other warps' sums
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
      part[warp][0] = s0;
      part[warp][1] = s1;
      part[warp][2] = s2;
    }
    __syncthreads();
    if (j == 0)
      for (int k = 1; k < (1 << (lg - 5)); ++k) {
        s0 += part[warp + k][0];
        s1 += part[warp + k][1];
        s2 += part[warp + k][2];
      }
  }
  if (!valid || j != 0) return;
  const uint32_t m = (uint32_t)(4294967296.0f / (float)(256u * (uint32_t)n));
  const uint32_t a = (uint32_t)n / 2;
  unsigned char* o = d.dst + (size_t)cell * 3;
  o[0] = (unsigned char)(((s0 + a) * m) >> 24);
  o[1] = (unsigned char)(((s1 + a) * m) >> 24);
  o[2] = (unsigned char)(((s2 + a) * m) >> 24);
}

static int floor_log2(int v) {
  int k = 0;
  while ((2 << k) <= v) ++k;
  return k;
}

// Pillow's plan of one window: reduce factors, box ends, reduced size and pass order
struct Plan {
  int fx, fy, rh, rw;
  BoxResize b;
  size_t reduced_bytes, mid_bytes;
};

static Plan plan_of(int ih, int iw, int oh, int ow) {
  Plan p;
  p.fx = std::max((int)((double)iw / ow / 2.0), 1);
  p.fy = std::max((int)((double)ih / oh / 2.0), 1);
  const bool reduce = p.fx > 1 || p.fy > 1;
  p.rw = (iw + p.fx - 1) / p.fx;
  p.rh = (ih + p.fy - 1) / p.fy;
  memset(&p.b, 0, sizeof(p.b));
  p.b.ih = p.rh;
  p.b.iw = p.rw;
  p.b.in1_w = (float)((double)iw / p.fx);
  p.b.in1_h = (float)((double)ih / p.fy);
  p.b.oh = oh;
  p.b.ow = ow;
  p.b.v_first = (long long)p.rh > 100LL * p.rw && oh < p.rh;
  p.reduced_bytes = reduce ? scratch_round((size_t)p.rh * p.rw * 3) : 0;
  p.mid_bytes = box_mid_bytes(p.b);
  return p;
}

}  // namespace se

using namespace se;

extern "C" {

int se_resize_reducing_u8(const unsigned char* const* src, const long long* src_pitch, const int* src_hw, unsigned char* dst,
                          const long long* dst_off, const int* dst_hw, int n, void* scratch, long long* scratch_bytes,
                          void* stream) {
  SE_REQUIRE(n >= 0 && n <= RESIZE_MAX_BATCH, "n must be in [0, " + std::to_string(RESIZE_MAX_BATCH) + "] images per call");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_pitch && src_hw && dst_off && dst_hw), "null size / offset array");
  std::vector<Plan> plans(n);
  size_t need = 0;
  std::vector<size_t> at(n);
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    if (int rc = check_window(i, ih, iw, src_pitch[i], 3LL * iw, dst_off[i])) return rc;
    if (int rc = check_sides("image", i, oh, ow)) return rc;
    plans[i] = plan_of(ih, iw, oh, ow);
    SE_REQUIRE((long long)plans[i].fx * plans[i].fy <= kMaxCell,
               "image " + std::to_string(i) + ": reduce cells of " + std::to_string(plans[i].fx) + " x " + std::to_string(plans[i].fy) +
                   " pixels pass 2^24 - 1");
    at[i] = need;
    need += plans[i].reduced_bytes + plans[i].mid_bytes;
  }
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(dst && src && std::find(src, src + n, nullptr) == src + n, "null src / dst");
  ReduceList rl;
  memset(&rl, 0, sizeof(rl));
  long long blocks = 0;
  std::vector<BoxResize> boxes(n);
  for (int i = 0; i < n; ++i) {
    Plan& p = plans[i];
    BoxResize& b = boxes[i];
    b = p.b;
    unsigned char* s = (unsigned char*)scratch + at[i];
    b.dst = dst + dst_off[i];
    b.mid = p.mid_bytes ? s + p.reduced_bytes : nullptr;
    if (!p.reduced_bytes) {   // no reduce: the passes read the window
      b.src = src[i];
      b.pitch = src_pitch[i];
      continue;
    }
    b.src = s;
    b.pitch = 3LL * p.rw;
    RImage& r = rl.im[rl.n++];
    r.src = src[i];
    r.dst = s;
    r.pitch = src_pitch[i];
    r.h = src_hw[2 * i];
    r.w = src_hw[2 * i + 1];
    r.fx = p.fx;
    r.fy = p.fy;
    r.oh = p.rh;
    r.ow = p.rw;
    int lg = 0;   // about 16 pixels per thread, up to a block per cell
    while (lg < 8 && (32LL << lg) <= (long long)p.fx * p.fy) ++lg;
    r.lgx = std::min(lg, floor_log2(p.fx));
    r.lgy = std::min(lg - r.lgx, floor_log2(p.fy));
    r.block0 = (int)blocks;
    blocks += grid_of((long long)p.rh * p.rw, R_THREADS >> (r.lgx + r.lgy));
  }
  SE_REQUIRE(blocks < (1LL << 31), "batch too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  if (rl.n) {
    reduce_kernel<<<(unsigned)blocks, R_THREADS, 0, st>>>(rl);
    SE_CUDA_OK(cudaGetLastError());
  }
  return resize_box_rgb(boxes.data(), n, st);
}

}  // extern "C"

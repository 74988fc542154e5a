// Pillow-exact bicubic resampling of batches of uint8 HWC images (1 or 3 channels, every image its own source and target size).
//
// PIL.Image.resize(size) with the default filter (BICUBIC, no box, no reducing_gap) is separable: a horizontal pass writes a
// uint8 intermediate of the source's height, a vertical pass reads it. A pass runs only when its axis changes length; an image
// whose size does not change is copied. Each pass computes, in int32 fixed point,
//     acc = 2^21 + sum_k src[xmin + k] * coeff[k],   out = clamp(acc >> 22, 0, 255),
// with the coefficients Pillow builds in double (precompute_coeffs + normalize_coeffs_8bpc of libImaging/Resample.c). They are
// built here on the host in the same order, so the integer weights and therefore every output byte are Pillow's.
// Pillow computes only the intermediate rows the vertical pass reads; computing all of them gives the same values.
// se_resize_window_u8 resizes windows of larger images (rows a pitch apart, such as boxes of a photo kept on the device):
// Image.crop(box).resize(size) without the crop. se_resize_composite_feather_detail_u8 resizes results and their masks the same way
// and pastes boxes that may overlap into shared canvases in order, as sequential Image.paste(im, box, mask) calls do, with
// the blend fused into the vertical pass (paste_v_kernel); it fades each box's mask to 0 along the box edges it is given
// widths for. se_feather_u8 applies that fade to masks alone (feather_kernel). resize_box_rgb (se_resize.h) runs the same two
// passes with the fractional box of Image.resize(..., reducing_gap=...), in either order, for se_thumbnail.cu.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_resize.h"

namespace se {

constexpr int RESIZE_PREC_BITS = 22;   // fractional bits of the fixed-point coefficients (Pillow's PRECISION_BITS for 8 bpc)

// ------------------------------------------------------------------------------------------ coefficients (host, double)
static double bicubic_filter(double x) {   // Keys cubic, a = -0.5, support 2
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow: (in1 - in0) / outSize with the box in floats; in0 = 0 and, without a box, in1 = in
static double axis_scale(float in1, int out) { return (double)in1 / out; }

static int resize_ksize(float in1, int out) {
  const double scale = axis_scale(in1, out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(2.0 * fs) * 2 + 1;
}

// Pillow's coefficient table for one axis (in -> out samples over the box (0, in1); in1 = in without a box): bounds[2*i] =
// first input sample of output i, bounds[2*i+1] = number of taps; coeffs[i*ksize + k] the fixed-point weights (zero beyond
// the taps). Returns ksize.
static int resize_coeff_table(int in, float in1, int out, int* bounds, int* coeffs) {
  const double scale = axis_scale(in1, out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * fs, ss = 1.0 / fs;
  const int ksize = (int)ceil(support) * 2 + 1;
  std::vector<double> k(ksize);
  for (int i = 0; i < out; ++i) {
    const double center = (i + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      k[x] = bicubic_filter((x + xmin - center + 0.5) * ss);
      ww += k[x];
    }
    int* kk = coeffs + (size_t)i * ksize;
    for (int x = 0; x < ksize; ++x) {
      double w = 0.0;
      if (x < xmax) w = ww != 0.0 ? k[x] / ww : k[x];
      kk[x] = w < 0 ? (int)(-0.5 + w * (1 << RESIZE_PREC_BITS)) : (int)(0.5 + w * (1 << RESIZE_PREC_BITS));
    }
    bounds[2 * i] = xmin;
    bounds[2 * i + 1] = xmax;
  }
  return ksize;
}

// ------------------------------------------------------------------------------------------ device cache of the tables
// One table per (device, in, in1, out), in1 the box end's float bits (in itself without a box): a size seen before costs no
// host work and no copy. A new table is built and uploaded
// synchronously. Each device's tables are limited to g_table_cap bytes (se_resize_set_table_cache_limit). When a call's new
// tables would pass the limit, the device's cache is emptied after a device synchronise BEFORE the call looks up any table, so
// every table a call launches with stays allocated until its kernels have run. (A single call's own tables may exceed the limit.)
struct AxisTable {
  int* bounds = nullptr;   // [out][2], followed in the same allocation by coeffs [out][ksize]
  int* coeffs = nullptr;
  int ksize = 0;
  size_t bytes = 0;
};
static std::mutex g_resize_mu;   // guards the cache and its limit; held for the whole launch part of a call
struct TableKey {   // one axis: in samples, the box end in1 (in without a box), out samples
  int in;
  float in1;
  int out;
  bool operator==(const TableKey& o) const { return in == o.in && out == o.out && in1_bits() == o.in1_bits(); }
  uint32_t in1_bits() const {
    uint32_t u;
    memcpy(&u, &in1, 4);
    return u;
  }
};
static std::map<std::tuple<int, int, uint32_t, int>, AxisTable> g_tables;
constexpr size_t kDefaultTableCap = 256u << 20;
static size_t g_table_cap = kDefaultTableCap;

static std::tuple<int, int, uint32_t, int> cache_key(int dev, const TableKey& k) { return std::make_tuple(dev, k.in, k.in1_bits(), k.out); }
static TableKey plain_key(int in, int out) { return {in, (float)in, out}; }
static size_t table_bytes(const TableKey& k) { return (size_t)k.out * (2 + resize_ksize(k.in1, k.out)) * sizeof(int); }

static size_t held_bytes(int dev) {
  size_t held = 0;
  for (auto& kv : g_tables)
    if (std::get<0>(kv.first) == dev) held += kv.second.bytes;
  return held;
}

// the tables of one call: empties the device's cache first when the call's missing tables would pass the limit
static int reserve_tables(int dev, const std::vector<TableKey>& keys) {
  std::vector<TableKey> missing;
  size_t need = 0;
  for (auto& k : keys) {
    if (g_tables.count(cache_key(dev, k)) || std::find(missing.begin(), missing.end(), k) != missing.end()) continue;
    missing.push_back(k);
    need += table_bytes(k);
  }
  if (need == 0 || held_bytes(dev) + need <= g_table_cap) return 0;
  SE_CUDA_OK(cudaDeviceSynchronize());   // launches already enqueued may still read the tables
  for (auto i = g_tables.begin(); i != g_tables.end();) {
    if (std::get<0>(i->first) == dev) {
      SE_CUDA_OK(cudaFree(i->second.bounds));
      i = g_tables.erase(i);
    } else {
      ++i;
    }
  }
  return 0;
}

// the cached table of k, built and uploaded on a miss; never frees a table (reserve_tables does, before any lookup)
static int axis_table(int dev, const TableKey& k, const AxisTable** t) {
  const auto key = cache_key(dev, k);
  auto it = g_tables.find(key);
  if (it != g_tables.end()) {
    *t = &it->second;
    return 0;
  }
  AxisTable a;
  a.ksize = resize_ksize(k.in1, k.out);
  std::vector<int> host((size_t)k.out * (2 + a.ksize));
  resize_coeff_table(k.in, k.in1, k.out, host.data(), host.data() + 2 * (size_t)k.out);
  a.bytes = host.size() * sizeof(int);
  SE_CUDA_OK(cudaMalloc(&a.bounds, a.bytes));
  SE_CUDA_OK(cudaMemcpy(a.bounds, host.data(), a.bytes, cudaMemcpyHostToDevice));
  a.coeffs = a.bounds + 2 * (size_t)k.out;
  *t = &(g_tables[key] = a);
  return 0;
}

// ------------------------------------------------------------------------------------------ kernels
// Per-image descriptors travel as kernel parameters (RESIZE_MAX_BATCH of them, < 4 KB). A launch covers the tiles of all its
// images; tile0 is the first tile of an image, so a block finds its image by scanning the (at most 32) descriptors (image_of).
struct HPass {   // rows x in_w -> rows x out_w; source rows src_pitch bytes apart, destination rows packed
  const unsigned char* src;
  unsigned char* dst;
  const int* bounds;
  const int* coeffs;
  long long src_pitch;
  int ksize, rows, in_w, out_w, swap, tile0, tiles_x;
};
struct VPass {   // in_h x row_bytes -> out_h x row_bytes; source rows src_pitch bytes apart, destination rows packed;
                 // coeffs == nullptr: copy (one tap of weight 1 at the same row)
  const unsigned char* src;
  unsigned char* dst;
  const int* bounds;
  const int* coeffs;
  long long src_pitch;
  int ksize, in_h, out_h, row_bytes, groups, swap, vec, tile0, tiles_x;
};
template <typename P>
struct PassList {
  P p[RESIZE_MAX_BATCH];
  int n;
};

constexpr int H_TX = 32, H_TY = 8;    // horizontal tile: 32 output columns x 8 rows, one thread per output pixel
constexpr int V_TX = 64, V_TY = 4;    // vertical tile: 64 groups of 12 bytes x 4 output rows
constexpr int V_GROUP = 12;           // bytes per thread: 4 RGB pixels (R<->B swap stays inside a thread) or 12 L pixels

__device__ __forceinline__ int clip8(int acc) {
  const int v = acc >> RESIZE_PREC_BITS;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

template <int C>
__global__ void __launch_bounds__(H_TX * H_TY) resize_h_kernel(const __grid_constant__ PassList<HPass> L) {
  extern __shared__ int smem[];   // coeffs [H_TX][ksize], bounds [H_TX][2]
  const HPass& d = L.p[image_of(L.p, L.n, &HPass::tile0, (int)blockIdx.x)];
  const int t = blockIdx.x - d.tile0;
  const int x0 = (t % d.tiles_x) * H_TX, y = (t / d.tiles_x) * H_TY + threadIdx.y;
  const int ncol = min(H_TX, d.out_w - x0);
  const int tid = threadIdx.y * H_TX + threadIdx.x;
  int* sk = smem;
  int* sb = smem + H_TX * d.ksize;
  for (int j = tid; j < ncol * d.ksize; j += H_TX * H_TY) sk[j] = d.coeffs[(size_t)x0 * d.ksize + j];
  for (int j = tid; j < 2 * ncol; j += H_TX * H_TY) sb[j] = d.bounds[2 * x0 + j];
  __syncthreads();
  if ((int)threadIdx.x >= ncol || y >= d.rows) return;
  const int xmin = sb[2 * threadIdx.x], n = sb[2 * threadIdx.x + 1];
  const int* k = sk + threadIdx.x * d.ksize;   // ksize is odd: the 32 lanes hit 32 different banks
  const unsigned char* s = d.src + (size_t)y * d.src_pitch + (size_t)xmin * C;
  int acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) acc[c] = 1 << (RESIZE_PREC_BITS - 1);
  for (int x = 0; x < n; ++x) {
    const int w = k[x];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] += (int)s[x * C + c] * w;
  }
  unsigned char* o = d.dst + ((size_t)y * d.out_w + x0 + threadIdx.x) * C;
  if (C == 3) {
    const int r = clip8(acc[0]), b = clip8(acc[C - 1]);
    o[0] = (unsigned char)(d.swap ? b : r);
    o[1] = (unsigned char)clip8(acc[C > 1 ? 1 : 0]);
    o[2] = (unsigned char)(d.swap ? r : b);
  } else {
    o[0] = (unsigned char)clip8(acc[0]);
  }
}

// The vertical taps of output rows y0 .. y0 + nrow - 1 into shared memory (coeffs [V_TY][ksize], bounds [V_TY][2]); a pass
// without a table copies (one tap of weight 1 at the same row).
__device__ __forceinline__ void stage_v_taps(int* sk, int* sb, const int* bounds, const int* coeffs, int ksize, int y0, int nrow) {
  const int tid = threadIdx.y * V_TX + threadIdx.x;
  for (int j = tid; j < nrow * ksize; j += V_TX * V_TY) sk[j] = coeffs ? coeffs[(size_t)y0 * ksize + j] : (1 << RESIZE_PREC_BITS);
  for (int j = tid; j < 2 * nrow; j += V_TX * V_TY) sb[j] = bounds ? bounds[2 * y0 + j] : ((j & 1) ? 1 : y0 + j / 2);
}

// v[j] = clip8(2^21 + sum_x s[x * stride + j] * k[x]) for the bytes lo <= j < nb of NB: 32-bit loads when vec (then lo == 0,
// nb == NB and s, stride are 4-byte aligned), byte loads otherwise
template <int NB>
__device__ __forceinline__ void v_taps(const unsigned char* s, long long stride, const int* k, int n, int lo, int nb, bool vec,
                                       int (&v)[NB]) {
#pragma unroll
  for (int j = 0; j < NB; ++j) v[j] = 1 << (RESIZE_PREC_BITS - 1);
  if (vec) {
    for (int x = 0; x < n; ++x) {
      const uint32_t* q = reinterpret_cast<const uint32_t*>(s + (size_t)x * stride);
      uint32_t u[NB / 4];
#pragma unroll
      for (int w = 0; w < NB / 4; ++w) u[w] = __ldg(q + w);
      const int w = k[x];
#pragma unroll
      for (int j = 0; j < NB; ++j) v[j] += (int)((u[j >> 2] >> (8 * (j & 3))) & 0xffu) * w;
    }
  } else {
    for (int x = 0; x < n; ++x) {
      const unsigned char* r = s + (size_t)x * stride;
      const int w = k[x];
#pragma unroll
      for (int j = 0; j < NB; ++j)
        if (j >= lo && j < nb) v[j] += (int)r[j] * w;
    }
  }
#pragma unroll
  for (int j = 0; j < NB; ++j) v[j] = clip8(v[j]);
}

__device__ __forceinline__ void swap_rb12(int (&v)[V_GROUP]) {   // a group starts on a pixel boundary (12 = 4 x 3 bytes)
#pragma unroll
  for (int j = 0; j < V_GROUP; j += 3) {
    const int r = v[j];
    v[j] = v[j + 2];
    v[j + 2] = r;
  }
}

__device__ __forceinline__ void store12(unsigned char* o, const int (&v)[V_GROUP], int nb, bool vec) {
  if (vec) {
    uint32_t* q = reinterpret_cast<uint32_t*>(o);
#pragma unroll
    for (int w = 0; w < 3; ++w)
      q[w] = (uint32_t)v[4 * w] | ((uint32_t)v[4 * w + 1] << 8) | ((uint32_t)v[4 * w + 2] << 16) | ((uint32_t)v[4 * w + 3] << 24);
  } else {
#pragma unroll
    for (int j = 0; j < V_GROUP; ++j)
      if (j < nb) o[j] = (unsigned char)v[j];
  }
}

__global__ void __launch_bounds__(V_TX * V_TY) resize_v_kernel(const __grid_constant__ PassList<VPass> L) {
  extern __shared__ int smem[];   // coeffs [V_TY][ksize], bounds [V_TY][2]
  const VPass& d = L.p[image_of(L.p, L.n, &VPass::tile0, (int)blockIdx.x)];
  const int t = blockIdx.x - d.tile0;
  const int g = (t % d.tiles_x) * V_TX + threadIdx.x, y0 = (t / d.tiles_x) * V_TY;
  const int nrow = min(V_TY, d.out_h - y0);
  int* sk = smem;
  int* sb = smem + V_TY * d.ksize;
  stage_v_taps(sk, sb, d.bounds, d.coeffs, d.ksize, y0, nrow);
  __syncthreads();
  if ((int)threadIdx.y >= nrow || g >= d.groups) return;
  const int ymin = sb[2 * threadIdx.y], n = sb[2 * threadIdx.y + 1];
  const size_t p = (size_t)g * V_GROUP;
  const int nb = min(V_GROUP, d.row_bytes - (int)p);
  const bool vec = d.vec && nb == V_GROUP;
  int v[V_GROUP];
  v_taps(d.src + (size_t)ymin * d.src_pitch + p, d.src_pitch, sk + threadIdx.y * d.ksize, n, 0, nb, vec, v);
  if (d.swap) swap_rb12(v);
  store12(d.dst + (size_t)(y0 + threadIdx.y) * d.row_bytes + p, v, nb, vec);
}

// The feather ramp of a box's paste mask (paste_v_kernel, feather_kernel), over one pair of opposite sides: a side of width f
// gives the pixel at distance d from its edge pixel (d = 0 on it) 255 * (d + 1) / (f + 1) when d < f and 255 otherwise; the
// ramp of a pixel is the least over its row's pair (top, bottom) and its column's pair (left, right). The division runs only
// inside a band and is exact integer division.
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

// The paste of se_resize_composite_feather_detail_u8: boxes pasted in order into canvases (row pitch in bytes). For a box, the
// vertical pass of its result (3 channels) and of its mask, both in_h x out_w, to out_h, then Pillow's Image.paste blend of
// the result over the canvas with that mask, per channel:
//     dst = DIV255(base * (255 - m) + res * m),   DIV255(a) = ((t >> 8) + t) >> 8 with t = a + 128 (libImaging/Paste.c).
// A box with feather widths first takes m = DIV255(m * ramp) with the ramp of feather_pair at the pixel's place in the box;
// a box without them skips that step.
// A thread owns 4 pixels of one canvas row (x a multiple of 4). It reads the canvas bytes that some box of the launch covers,
// blends every covering box over them in the launch's order and writes them once; uncovered bytes are never touched. It reads
// before it writes the same bytes, so dst may be base. The 12 canvas bytes move as 32-bit words when every box that covers
// one of the 4 pixels covers all 4 and the canvas rows are 4-byte aligned, and a box's result and mask rows likewise.
struct PBox {   // a box at (oy, ox) of its canvas; rgb and mask are in_h x out_w (after the horizontal passes)
  const unsigned char* rgb;
  const unsigned char* mask;
  const int* bounds;   // the vertical table; nullptr: the height does not change (one tap of weight 1 at the same row)
  const int* coeffs;
  int oy, ox;
  unsigned short out_h, out_w, ksize, vec;   // sizes <= 65535 (check_resize); ksize <= 9685 (its shared-memory check)
  unsigned short feather[4];                 // ramp widths of the left, top, right, bottom sides; all 0: no ramp
};
static_assert(sizeof(PBox) == 56, "the feather widths fit PBox's former padding");
struct PCanvas {   // boxes box0 .. box0 + nbox - 1 of the launch, in order; tiles cover rows y0 .. y0 + h - 1 from column x0
  const unsigned char* base;
  unsigned char* dst;
  long long pitch;
  int y0, x0, h, groups, vec, box0, nbox, tile0, tiles_x;
};
struct PasteList {
  PBox b[RESIZE_MAX_BATCH];
  PCanvas p[RESIZE_MAX_BATCH];
  int n;   // canvases
};
static_assert(sizeof(PasteList) <= 4096, "paste descriptors must fit the kernel parameter space");
// se_resize_composite_feather_detail_u8: per box of the launch its int16 detail plane [out_h][out_w][3] (RGB) or nullptr.
// A separate parameter: PasteList fills the classic 4 KB of kernel parameters (sm_90 takes up to 32 KB).
struct PasteDetail {
  const short* d[RESIZE_MAX_BATCH];
};
constexpr int P_PIX = V_GROUP / 3;
static __device__ int g_unit_tap[1] = {1 << RESIZE_PREC_BITS};

// the pixels [lo, hi) of the 4 at canvas (y, x) that box b covers (lo >= hi: none)
__device__ __forceinline__ void box_span(const PBox& b, int y, int x, int& lo, int& hi) {
  const bool row = y >= b.oy && y < b.oy + b.out_h;
  lo = max(b.ox - x, 0);
  hi = row ? min(b.ox + b.out_w - x, P_PIX) : 0;
}

// A box with a detail plane adds it to the result after the vertical pass's clip8 and the channel swap, clamped to [0, 255]
// (one test per box and thread; a box without one runs the plain paste).
__global__ void __launch_bounds__(V_TX * V_TY) paste_v_kernel(const __grid_constant__ PasteList L, int swap,
                                                              const __grid_constant__ PasteDetail D) {
  const PCanvas& d = L.p[image_of(L.p, L.n, &PCanvas::tile0, (int)blockIdx.x)];
  const int t = blockIdx.x - d.tile0;
  const int g = (t % d.tiles_x) * V_TX + threadIdx.x, y = d.y0 + (t / d.tiles_x) * V_TY + threadIdx.y;
  if (g >= d.groups || y >= d.y0 + d.h) return;
  const int x = d.x0 + g * P_PIX;
  unsigned covered = 0;   // bit p: some box covers pixel x + p
  bool same = true;
  for (int i = d.box0; i < d.box0 + d.nbox; ++i) {
    int lo, hi;
    box_span(L.b[i], y, x, lo, hi);
    if (lo >= hi) continue;
    covered |= (1u << hi) - (1u << lo);
    same = same && lo == 0 && hi == P_PIX;
  }
  if (!covered) return;
  const bool vec = d.vec && same;
  const size_t at = (size_t)y * d.pitch + (size_t)x * 3;
  const unsigned char* ob = d.base + at;
  int c[V_GROUP];
  if (vec) {   // plain loads: base may be dst
    const uint32_t* q = reinterpret_cast<const uint32_t*>(ob);
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      const uint32_t u = q[w];
#pragma unroll
      for (int j = 0; j < 4; ++j) c[4 * w + j] = (int)((u >> (8 * j)) & 0xffu);
    }
  } else {
#pragma unroll
    for (int j = 0; j < V_GROUP; ++j) c[j] = (covered >> (j / 3)) & 1u ? (int)ob[j] : 0;
  }
  for (int i = d.box0; i < d.box0 + d.nbox; ++i) {
    const PBox& b = L.b[i];
    int lo, hi;
    box_span(b, y, x, lo, hi);
    if (lo >= hi) continue;
    const int r = y - b.oy;
    const int ymin = b.bounds ? __ldg(b.bounds + 2 * r) : r, n = b.bounds ? __ldg(b.bounds + 2 * r + 1) : 1;
    const int* k = b.bounds ? b.coeffs + (size_t)r * b.ksize : g_unit_tap;
    const bool bv = b.vec && lo == 0 && hi == P_PIX;
    const ptrdiff_t col = (ptrdiff_t)ymin * b.out_w + (x - b.ox);   // pixel 0 of the thread in the box's rows (may be < 0)
    int v[V_GROUP], m[P_PIX];
    v_taps(b.rgb + col * 3, b.out_w * 3, k, n, lo * 3, hi * 3, bv, v);
    v_taps(b.mask + col, b.out_w, k, n, lo, hi, bv, m);
    if (b.feather[0] | b.feather[1] | b.feather[2] | b.feather[3]) {
      const int rv = feather_pair(r, b.out_h - 1 - r, b.feather[1], b.feather[3]);
#pragma unroll
      for (int p = 0; p < P_PIX; ++p) {
        if (p < lo || p >= hi) continue;
        const int xb = x + p - b.ox;
        const int ramp = min(rv, feather_pair(xb, b.out_w - 1 - xb, b.feather[0], b.feather[2]));
        if (ramp < 255) m[p] = div255(m[p] * ramp);
      }
    }
    if (swap) swap_rb12(v);
    if (const short* dp = D.d[i]) {
      const short* dr = dp + ((ptrdiff_t)r * b.out_w + (x - b.ox)) * 3;   // pixel 0 of the thread (may lie left of the box)
#pragma unroll
      for (int j = 0; j < V_GROUP; ++j)
        if (j / 3 >= lo && j / 3 < hi) v[j] = min(max(v[j] + (int)dr[j], 0), 255);
    }
#pragma unroll
    for (int j = 0; j < V_GROUP; ++j) {
      if (j / 3 < lo || j / 3 >= hi) continue;
      const int a = c[j] * (255 - m[j / 3]) + v[j] * m[j / 3] + 128;
      c[j] = ((a >> 8) + a) >> 8;
    }
  }
  unsigned char* o = d.dst + at;
  if (vec) {
    store12(o, c, V_GROUP, true);
  } else {
#pragma unroll
    for (int j = 0; j < V_GROUP; ++j)
      if ((covered >> (j / 3)) & 1u) o[j] = (unsigned char)c[j];
  }
}

// se_feather_u8: m = DIV255(m * ramp) in place over box-sized 'L' images, with the ramp paste_v_kernel gives a feathered box.
// One thread per pixel; only the pixels inside a band are read and written.
struct FeatherImage {
  unsigned char* p;
  int h, w, tile0, tiles_x;
  unsigned short f[4];   // left, top, right, bottom
};
struct FeatherList {
  FeatherImage im[RESIZE_MAX_BATCH];
  int n;
};
constexpr int F_TX = 64, F_TY = 4;

__global__ void __launch_bounds__(F_TX * F_TY) feather_kernel(const __grid_constant__ FeatherList L) {
  const FeatherImage& d = L.im[image_of(L.im, L.n, &FeatherImage::tile0, (int)blockIdx.x)];
  const int t = blockIdx.x - d.tile0;
  const int x = (t % d.tiles_x) * F_TX + threadIdx.x, y = (t / d.tiles_x) * F_TY + threadIdx.y;
  if (x >= d.w || y >= d.h) return;
  const int ramp = min(feather_pair(y, d.h - 1 - y, d.f[1], d.f[3]), feather_pair(x, d.w - 1 - x, d.f[0], d.f[2]));
  if (ramp == 255) return;
  unsigned char* q = d.p + (size_t)y * d.w + x;
  *q = (unsigned char)div255(*q * ramp);
}

constexpr int kMaxSmem = 227 * 1024;

// the checks of image i that se_resize_window_u8 and se_resize_composite_feather_detail_u8 share besides its source's: the
// output's sides, and a filter that fits shared memory
static int check_resize(int i, int ih, int iw, int oh, int ow) {
  if (int rc = check_sides("image", i, oh, ow)) return rc;
  SE_REQUIRE(resize_ksize(iw, ow) * (H_TX + 2) * 4 <= kMaxSmem && resize_ksize(ih, oh) * (V_TY + 2) * 4 <= kMaxSmem,
             "image " + std::to_string(i) + ": downscale factor too large");
  return 0;
}

// appends the horizontal pass rows x iw -> rows x ow of src (rows src_pitch bytes apart) into dst (packed rows) to hl, over
// the box (0, in1) of the rows (in1 = iw: no box)
static int add_h_pass(int dev, PassList<HPass>& hl, long long& tiles, int& kmax, const unsigned char* src, long long src_pitch,
                      unsigned char* dst, int rows, int iw, float in1, int ow, int swap) {
  const AxisTable* t = nullptr;
  int rc = axis_table(dev, {iw, in1, ow}, &t);
  if (rc) return rc;
  HPass& h = hl.p[hl.n++];
  h.src = src;
  h.dst = dst;
  h.bounds = t->bounds;
  h.coeffs = t->coeffs;
  h.src_pitch = src_pitch;
  h.ksize = t->ksize;
  h.rows = rows;
  h.in_w = iw;
  h.out_w = ow;
  h.swap = swap;
  h.tile0 = (int)tiles;
  h.tiles_x = grid_of(ow, H_TX);
  tiles += (long long)h.tiles_x * grid_of(rows, H_TY);
  kmax = std::max(kmax, t->ksize);
  return 0;
}

template <int C>
static int launch_h(const PassList<HPass>& hl, long long tiles, int kmax, cudaStream_t st) {
  if (!hl.n) return 0;
  SE_CUDA_OK(cudaFuncSetAttribute(resize_h_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  resize_h_kernel<C><<<(unsigned)tiles, dim3(H_TX, H_TY), (H_TX * kmax + 2 * H_TX) * 4, st>>>(hl);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// the vertical table of ih -> oh over the box (0, in1) of the columns (in1 = ih: no box), or none (a copy) when the height
// does not change and there is no box
static int v_table(int dev, int ih, float in1, int oh, const int** bounds, const int** coeffs, int* ksize) {
  *bounds = *coeffs = nullptr;
  *ksize = 1;
  if (ih == oh && in1 == (float)ih) return 0;
  const AxisTable* t = nullptr;
  int rc = axis_table(dev, {ih, in1, oh}, &t);
  if (rc) return rc;
  *bounds = t->bounds;
  *coeffs = t->coeffs;
  *ksize = t->ksize;
  return 0;
}

// appends the vertical pass in_h x row_bytes -> oh x row_bytes of src (rows src_pitch bytes apart) into dst (packed rows) to
// vl, over the box (0, in1) of the columns (in1 = in_h: no box); without a box and a height change it copies
static int add_v_pass(int dev, PassList<VPass>& vl, long long& tiles, int& kmax, const unsigned char* src, long long src_pitch,
                      unsigned char* dst, int in_h, float in1, int oh, int row_bytes, int swap) {
  VPass& v = vl.p[vl.n++];
  v.src = src;
  v.dst = dst;
  v.src_pitch = src_pitch;
  int rc = v_table(dev, in_h, in1, oh, &v.bounds, &v.coeffs, &v.ksize);
  if (rc) return rc;
  v.in_h = in_h;
  v.out_h = oh;
  v.row_bytes = row_bytes;
  v.groups = grid_of(v.row_bytes, V_GROUP);
  v.swap = swap;
  v.vec = ((uintptr_t)v.src % 4 == 0) && ((uintptr_t)v.dst % 4 == 0) && v.row_bytes % 4 == 0 && src_pitch % 4 == 0;
  v.tile0 = (int)tiles;
  v.tiles_x = grid_of(v.groups, V_TX);
  tiles += (long long)v.tiles_x * grid_of(oh, V_TY);
  kmax = std::max(kmax, v.ksize);
  return 0;
}

static int launch_v(const PassList<VPass>& vl, long long tiles, int kmax, cudaStream_t st) {
  if (!vl.n) return 0;
  const int smem = (V_TY * kmax + 2 * V_TY) * 4;
  SE_CUDA_OK(cudaFuncSetAttribute(resize_v_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  resize_v_kernel<<<(unsigned)tiles, dim3(V_TX, V_TY), smem, st>>>(vl);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// The scratch query and the launches of se_resize_window_u8, after its checks: image i is read from src[i] (src may be
// nullptr in the query form), its rows pitch[i] bytes apart, and written packed at dst + dst_off[i].
static int resize_images(const unsigned char* const* src, const long long* pitch, const int* src_hw, unsigned char* dst,
                         const long long* dst_off, const int* dst_hw, int n, int C, int swap_rb, void* scratch,
                         long long* scratch_bytes, cudaStream_t st) {
  size_t need = 0;
  std::vector<size_t> mid(n);
  for (int i = 0; i < n; ++i) {
    mid[i] = need;
    if (src_hw[2 * i + 1] != dst_hw[2 * i + 1] && src_hw[2 * i] != dst_hw[2 * i]) need += scratch_round((size_t)src_hw[2 * i] * dst_hw[2 * i + 1] * C);
  }
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(dst && src && std::find(src, src + n, nullptr) == src + n, "null src / dst");
  std::lock_guard<std::mutex> lk(g_resize_mu);
  int dev = 0;
  SE_CUDA_OK(cudaGetDevice(&dev));
  {
    std::vector<TableKey> keys;
    for (int i = 0; i < n; ++i) {
      if (src_hw[2 * i + 1] != dst_hw[2 * i + 1]) keys.push_back(plain_key(src_hw[2 * i + 1], dst_hw[2 * i + 1]));
      if (src_hw[2 * i] != dst_hw[2 * i]) keys.push_back(plain_key(src_hw[2 * i], dst_hw[2 * i]));
    }
    int rc = reserve_tables(dev, keys);
    if (rc) return rc;
  }
  PassList<HPass> hl;
  PassList<VPass> vl;
  memset(&hl, 0, sizeof(hl));
  memset(&vl, 0, sizeof(vl));
  long long htiles = 0, vtiles = 0;
  int hk = 1, vk = 1;
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    const unsigned char* s = src[i];
    long long sp = pitch[i];
    unsigned char* o = dst + dst_off[i];
    if (iw != ow) {
      unsigned char* h_dst = ih != oh ? (unsigned char*)scratch + mid[i] : o;
      int rc = add_h_pass(dev, hl, htiles, hk, s, sp, h_dst, ih, iw, (float)iw, ow, ih == oh && swap_rb);
      if (rc) return rc;
      if (ih == oh) continue;
      s = h_dst;
      sp = (long long)ow * C;
    }
    // the vertical pass, or the copy of an image whose size does not change
    int rc = add_v_pass(dev, vl, vtiles, vk, s, sp, o, ih, (float)ih, oh, ow * C, swap_rb);
    if (rc) return rc;
  }
  SE_REQUIRE(htiles < (1LL << 31) && vtiles < (1LL << 31), "batch too large for one launch");
  int rc = C == 3 ? launch_h<3>(hl, htiles, hk, st) : launch_h<1>(hl, htiles, hk, st);
  if (rc) return rc;
  return launch_v(vl, vtiles, vk, st);
}

int resize_box_rgb(const BoxResize* im, int n, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_resize_mu);
  int dev = 0;
  SE_CUDA_OK(cudaGetDevice(&dev));
  {
    std::vector<TableKey> keys;
    for (int i = 0; i < n; ++i) {
      if (box_needs_h(im[i])) keys.push_back({im[i].iw, im[i].in1_w, im[i].ow});
      if (box_needs_v(im[i])) keys.push_back({im[i].ih, im[i].in1_h, im[i].oh});
    }
    int rc = reserve_tables(dev, keys);
    if (rc) return rc;
  }
  // three launches: the horizontal passes that come first, every vertical pass (or copy), the horizontal passes that come
  // after a vertical one
  PassList<HPass> h0, h1;
  PassList<VPass> vl;
  memset(&h0, 0, sizeof(h0));
  memset(&h1, 0, sizeof(h1));
  memset(&vl, 0, sizeof(vl));
  long long t0 = 0, t1 = 0, vt = 0;
  int k0 = 1, k1 = 1, vk = 1;
  for (int i = 0; i < n; ++i) {
    const BoxResize& b = im[i];
    const bool nh = box_needs_h(b), nv = box_needs_v(b);
    if (b.v_first && nh && nv) {
      int rc = add_v_pass(dev, vl, vt, vk, b.src, b.pitch, b.mid, b.ih, b.in1_h, b.oh, b.iw * 3, 0);
      if (rc) return rc;
      rc = add_h_pass(dev, h1, t1, k1, b.mid, 3LL * b.iw, b.dst, b.oh, b.iw, b.in1_w, b.ow, 0);
      if (rc) return rc;
      continue;
    }
    const unsigned char* s = b.src;
    long long sp = b.pitch;
    if (nh) {
      unsigned char* h_dst = nv ? b.mid : b.dst;
      int rc = add_h_pass(dev, h0, t0, k0, s, sp, h_dst, b.ih, b.iw, b.in1_w, b.ow, 0);
      if (rc) return rc;
      if (!nv) continue;
      s = h_dst;
      sp = 3LL * b.ow;
    }
    int rc = add_v_pass(dev, vl, vt, vk, s, sp, b.dst, b.ih, b.in1_h, b.oh, b.ow * 3, 0);
    if (rc) return rc;
  }
  SE_REQUIRE(t0 < (1LL << 31) && t1 < (1LL << 31) && vt < (1LL << 31), "batch too large for one launch");
  int rc = launch_h<3>(h0, t0, k0, st);
  if (rc) return rc;
  rc = launch_v(vl, vt, vk, st);
  if (rc) return rc;
  return launch_h<3>(h1, t1, k1, st);
}

// One box of se_resize_composite_feather_detail_u8: its result and mask (ih x iw), pasted at ow x oh into canvas `canvas` at (oy, ox).
struct PasteBox {
  const unsigned char* rgb;
  const unsigned char* mask;
  int ih, iw, oh, ow, canvas, oy, ox;
  int feather[4];   // left, top, right, bottom; zero when the call gives no widths
  const short* detail;   // int16 [oh][ow][3] added after the vertical pass, or nullptr
};
struct PasteCanvas {
  const unsigned char* base;
  unsigned char* dst;
  long long pitch;
};

// bytes of scratch box i needs (a width change: the result's and the mask's intermediates, ih x ow x 3 and ih x ow)
static size_t paste_scratch(int ih, int iw, int ow) {
  return iw != ow ? scratch_round((size_t)ih * ow * 3) + scratch_round((size_t)ih * ow) : 0;
}

// The boxes in order, RESIZE_MAX_BATCH per launch: the horizontal passes of a launch's boxes, then one paste_v_kernel in
// which each canvas's boxes keep their order; a later launch on the same stream continues the order. mid[i]: box i's scratch.
static int paste_boxes(const std::vector<PasteBox>& boxes, const std::vector<PasteCanvas>& canvases, const std::vector<size_t>& mid,
                       void* scratch, int swap_rb, cudaStream_t st) {
  std::lock_guard<std::mutex> lk(g_resize_mu);
  int dev = 0;
  SE_CUDA_OK(cudaGetDevice(&dev));
  {
    std::vector<TableKey> keys;
    for (auto& b : boxes) {
      if (b.iw != b.ow) keys.push_back(plain_key(b.iw, b.ow));
      if (b.ih != b.oh) keys.push_back(plain_key(b.ih, b.oh));
    }
    int rc = reserve_tables(dev, keys);
    if (rc) return rc;
  }
  const int n = (int)boxes.size();
  for (int c0 = 0; c0 < n; c0 += RESIZE_MAX_BATCH) {
    const int c1 = std::min(n, c0 + RESIZE_MAX_BATCH);
    PassList<HPass> h3, h1;
    PasteList pl;
    PasteDetail dl;
    memset(&h3, 0, sizeof(h3));
    memset(&h1, 0, sizeof(h1));
    memset(&pl, 0, sizeof(pl));
    memset(&dl, 0, sizeof(dl));
    long long t3 = 0, t1 = 0, ptiles = 0;
    int k3 = 1, k1 = 1;
    std::vector<int> order;   // the launch's boxes grouped by canvas (canvases in order of first appearance), in order
    for (int i = c0; i < c1; ++i) {
      if (std::find_if(order.begin(), order.end(), [&](int j) { return boxes[j].canvas == boxes[i].canvas; }) != order.end()) continue;
      for (int j = i; j < c1; ++j)
        if (boxes[j].canvas == boxes[i].canvas) order.push_back(j);
    }
    for (int j = 0; j < (int)order.size(); ++j) {
      const PasteBox& b = boxes[order[j]];
      PBox& p = pl.b[j];
      p.rgb = b.rgb;
      p.mask = b.mask;
      dl.d[j] = b.detail;
      if (b.iw != b.ow) {   // the paste reads the horizontal passes' output instead of the result itself
        unsigned char* s3 = (unsigned char*)scratch + mid[order[j]];
        unsigned char* s1 = s3 + scratch_round((size_t)b.ih * b.ow * 3);
        int rc = add_h_pass(dev, h3, t3, k3, b.rgb, 3LL * b.iw, s3, b.ih, b.iw, (float)b.iw, b.ow, 0);
        if (rc) return rc;
        rc = add_h_pass(dev, h1, t1, k1, b.mask, b.iw, s1, b.ih, b.iw, (float)b.iw, b.ow, 0);
        if (rc) return rc;
        p.rgb = s3;
        p.mask = s1;
      }
      int ksize = 1;
      int rc = v_table(dev, b.ih, (float)b.ih, b.oh, &p.bounds, &p.coeffs, &ksize);
      if (rc) return rc;
      p.ksize = (unsigned short)ksize;
      p.out_h = (unsigned short)b.oh;
      p.out_w = (unsigned short)b.ow;
      p.oy = b.oy;
      p.ox = b.ox;
      p.vec = b.ow % 4 == 0 && b.ox % 4 == 0 && ((uintptr_t)p.rgb | (uintptr_t)p.mask) % 4 == 0;
      for (int s = 0; s < 4; ++s) p.feather[s] = (unsigned short)b.feather[s];
      if (j == 0 || boxes[order[j - 1]].canvas != b.canvas) {
        const PasteCanvas& cv = canvases[b.canvas];
        PCanvas& c = pl.p[pl.n++];
        c.base = cv.base;
        c.dst = cv.dst;
        c.pitch = cv.pitch;
        c.vec = cv.pitch % 4 == 0 && ((uintptr_t)cv.base | (uintptr_t)cv.dst) % 4 == 0;
        c.box0 = j;
        c.y0 = c.x0 = INT_MAX;
        c.h = c.groups = 0;   // (y1, x1) until the canvas's last box
      }
      PCanvas& c = pl.p[pl.n - 1];
      ++c.nbox;
      c.y0 = std::min(c.y0, b.oy);
      c.x0 = std::min(c.x0, b.ox / P_PIX * P_PIX);
      c.h = std::max(c.h, b.oy + b.oh);
      c.groups = std::max(c.groups, b.ox + b.ow);
    }
    for (int i = 0; i < pl.n; ++i) {
      PCanvas& c = pl.p[i];
      c.h -= c.y0;
      c.groups = grid_of(c.groups - c.x0, P_PIX);
      c.tile0 = (int)ptiles;
      c.tiles_x = grid_of(c.groups, V_TX);
      ptiles += (long long)c.tiles_x * grid_of(c.h, V_TY);
    }
    SE_REQUIRE(t3 < (1LL << 31) && ptiles < (1LL << 31), "batch too large for one launch");
    int rc = launch_h<3>(h3, t3, k3, st);
    if (rc) return rc;
    rc = launch_h<1>(h1, t1, k1, st);
    if (rc) return rc;
    paste_v_kernel<<<(unsigned)ptiles, dim3(V_TX, V_TY), 0, st>>>(pl, swap_rb, dl);
    SE_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

}  // namespace se

using namespace se;

extern "C" {

int se_resize_coeffs(int in, int out, int* bounds, int* coeffs, long long cap) {
  if (in < 1 || out < 1 || in > kMaxDim || out > kMaxDim) {
    set_error("se_resize_coeffs: sizes must be in [1, 65535]");
    return -1;
  }
  const int ksize = resize_ksize(in, out);
  if (!bounds && !coeffs) return ksize;
  if (!bounds || !coeffs || cap < (long long)out * ksize) {
    set_error("se_resize_coeffs: bounds and coeffs must both be given, coeffs holding out * ksize = " + std::to_string((long long)out * ksize) +
              " ints (got cap " + std::to_string(cap) + ")");
    return -1;
  }
  return resize_coeff_table(in, (float)in, out, bounds, coeffs);
}

int se_resize_set_table_cache_limit(long long bytes) {
  SE_REQUIRE(bytes >= 0, "resize table cache limit must be >= 0 bytes (0 = the default)");
  std::lock_guard<std::mutex> lk(g_resize_mu);
  g_table_cap = bytes ? (size_t)bytes : kDefaultTableCap;
  return 0;
}

long long se_resize_table_cache_bytes(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  std::lock_guard<std::mutex> lk(g_resize_mu);
  return (long long)held_bytes(dev);
}

int se_resize_window_u8(const unsigned char* const* src, const long long* src_pitch, const int* src_hw, unsigned char* dst,
                        const long long* dst_off, const int* dst_hw, int n, int channels, int swap_rb, void* scratch,
                        long long* scratch_bytes, void* stream) {
  SE_REQUIRE(n >= 0 && n <= RESIZE_MAX_BATCH, "n must be in [0, " + std::to_string(RESIZE_MAX_BATCH) + "] images per call");
  SE_REQUIRE(channels == 1 || channels == 3, "channels must be 1 or 3");
  SE_REQUIRE(!swap_rb || channels == 3, "swap_rb needs 3 channels");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_pitch && src_hw && dst_off && dst_hw), "null size / offset array");
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1];
    if (int rc = check_window(i, ih, iw, src_pitch[i], (long long)iw * channels, dst_off[i])) return rc;
    if (int rc = check_resize(i, ih, iw, dst_hw[2 * i], dst_hw[2 * i + 1])) return rc;
  }
  return resize_images(src, src_pitch, src_hw, dst, dst_off, dst_hw, n, channels, swap_rb, scratch, scratch_bytes,
                       (cudaStream_t)stream);
}

int se_resize_composite_feather_detail_u8(const unsigned char* rgb, const long long* rgb_off, const unsigned char* mask,
                                          const long long* mask_off, const int* src_hw, unsigned char* canvas, const long long* canvas_off,
                                          const long long* canvas_pitch, const int* box_yx, const int* dst_hw, const int* feather,
                                          const short* detail, const long long* detail_off, int n, int swap_rb, void* scratch,
                                          long long* scratch_bytes, void* stream) {
  SE_REQUIRE(!detail || detail_off, "detail needs detail_off");
  SE_REQUIRE(n >= 0, "n must be >= 0 boxes");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (rgb_off && mask_off && src_hw && canvas_off && canvas_pitch && box_yx && dst_hw), "null size / offset array");
  size_t need = 0;
  std::vector<size_t> mid(n);
  std::map<long long, int> canvas_of;   // canvas offset -> canvas index
  std::vector<PasteCanvas> canvases;
  std::vector<PasteBox> boxes(n);
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    if (int rc = check_sides("image", i, ih, iw)) return rc;
    if (int rc = check_resize(i, ih, iw, oh, ow)) return rc;
    SE_REQUIRE(rgb_off[i] >= 0 && mask_off[i] >= 0 && canvas_off[i] >= 0 && box_yx[2 * i] >= 0 && box_yx[2 * i + 1] >= 0,
               "negative offset");
    SE_REQUIRE(canvas_pitch[i] >= 3LL * (box_yx[2 * i + 1] + ow),
               "box " + std::to_string(i) + ": the canvas pitch of " + std::to_string(canvas_pitch[i]) + " bytes is narrower than the box");
    auto it = canvas_of.emplace(canvas_off[i], (int)canvases.size()).first;
    if (it->second == (int)canvases.size()) canvases.push_back({canvas + canvas_off[i], canvas + canvas_off[i], canvas_pitch[i]});
    SE_REQUIRE(canvases[it->second].pitch == canvas_pitch[i], "box " + std::to_string(i) + ": boxes of one canvas must have one pitch");
    boxes[i] = {rgb + rgb_off[i], mask + mask_off[i], ih, iw, oh, ow, it->second, box_yx[2 * i], box_yx[2 * i + 1], {}, nullptr};
    if (detail && detail_off[i] >= 0) {
      SE_REQUIRE(detail_off[i] % 2 == 0, "box " + std::to_string(i) + ": detail_off must be a multiple of 2 bytes");
      boxes[i].detail = (const short*)((const char*)detail + detail_off[i]);
    }
    if (feather) {
      const int* f = feather + 4 * (size_t)i;
      SE_REQUIRE(f[0] >= 0 && f[0] <= ow && f[2] >= 0 && f[2] <= ow && f[1] >= 0 && f[1] <= oh && f[3] >= 0 && f[3] <= oh,
                 "box " + std::to_string(i) + ": feather widths (" + std::to_string(f[0]) + ", " + std::to_string(f[1]) + ", " +
                     std::to_string(f[2]) + ", " + std::to_string(f[3]) + ") must be in [0, the side's length]");
      for (int s = 0; s < 4; ++s) boxes[i].feather[s] = f[s];
    }
    mid[i] = need;
    need += paste_scratch(ih, iw, ow);
  }
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(rgb && mask && canvas, "null rgb / mask / canvas");
  return paste_boxes(boxes, canvases, mid, scratch, swap_rb, (cudaStream_t)stream);
}

int se_feather_u8(unsigned char* img, const long long* off, const int* hw, const int* feather, int n, void* stream) {
  SE_REQUIRE(n >= 0, "n must be >= 0 images");
  SE_REQUIRE(n == 0 || (off && hw && feather), "null offset / size / feather array");
  for (int i = 0; i < n; ++i) {
    const int h = hw[2 * i], w = hw[2 * i + 1];
    const int* f = feather + 4 * (size_t)i;
    if (int rc = check_sides("image", i, h, w)) return rc;
    SE_REQUIRE(off[i] >= 0, "negative offset");
    SE_REQUIRE(f[0] >= 0 && f[0] <= w && f[2] >= 0 && f[2] <= w && f[1] >= 0 && f[1] <= h && f[3] >= 0 && f[3] <= h,
               "image " + std::to_string(i) + ": feather widths (" + std::to_string(f[0]) + ", " + std::to_string(f[1]) + ", " +
                   std::to_string(f[2]) + ", " + std::to_string(f[3]) + ") must be in [0, the side's length]");
  }
  if (n == 0) return 0;
  SE_REQUIRE(img, "null img");
  FeatherList fl;
  memset(&fl, 0, sizeof(fl));
  long long tiles = 0;
  auto launch = [&]() -> int {
    if (fl.n) {
      SE_REQUIRE(tiles < (1LL << 31), "batch too large for one launch");
      feather_kernel<<<(unsigned)tiles, dim3(F_TX, F_TY), 0, (cudaStream_t)stream>>>(fl);
      SE_CUDA_OK(cudaGetLastError());
    }
    memset(&fl, 0, sizeof(fl));
    tiles = 0;
    return 0;
  };
  for (int i = 0; i < n; ++i) {
    const int* f = feather + 4 * (size_t)i;
    if (!(f[0] | f[1] | f[2] | f[3])) continue;   // no band: the image is left as it is
    FeatherImage& d = fl.im[fl.n++];
    d.p = img + off[i];
    d.h = hw[2 * i];
    d.w = hw[2 * i + 1];
    for (int s = 0; s < 4; ++s) d.f[s] = (unsigned short)f[s];
    d.tile0 = (int)tiles;
    d.tiles_x = grid_of(d.w, F_TX);
    tiles += (long long)d.tiles_x * grid_of(d.h, F_TY);
    if (fl.n == RESIZE_MAX_BATCH) {
      int rc = launch();
      if (rc) return rc;
    }
  }
  return launch();
}

}  // extern "C"

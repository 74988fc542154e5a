// Pillow-exact bicubic resampling of batches of uint8 HWC images (1 or 3 channels, every image its own source and target size).
//
// PIL.Image.resize(size) with the default filter (BICUBIC, no box, no reducing_gap) is separable: a horizontal pass writes a
// uint8 intermediate of the source's height, a vertical pass reads it. A pass runs only when its axis changes length; an image
// whose size does not change is copied. Each pass computes, in int32 fixed point,
//     acc = 2^21 + sum_k src[xmin + k] * coeff[k],   out = clamp(acc >> 22, 0, 255),
// with the coefficients Pillow builds in double (precompute_coeffs + normalize_coeffs_8bpc of libImaging/Resample.c). They are
// built here on the host in the same order, so the integer weights and therefore every output byte are Pillow's.
// Pillow computes only the intermediate rows the vertical pass reads; computing all of them gives the same values.
// se_resize_paste_u8 resizes a result and its mask the same way and pastes the result over a base image with Pillow's
// Image.paste(im, box, mask) blend, fused into the vertical pass (paste_v_kernel).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_resize.h"

namespace se {

// ------------------------------------------------------------------------------------------ coefficients (host, double)
static double bicubic_filter(double x) {   // Keys cubic, a = -0.5, support 2
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

static double axis_scale(int in, int out) { return (double)(float)in / out; }   // Pillow: (in1 - in0) / outSize, box in float

int resize_ksize(int in, int out) {
  const double scale = axis_scale(in, out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  return (int)ceil(2.0 * fs) * 2 + 1;
}

int resize_coeff_table(int in, int out, int* bounds, int* coeffs) {
  const double scale = axis_scale(in, out);
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
// One table per (device, in, out): a size seen before costs no host work and no copy. A new table is built and uploaded
// synchronously. Each device's tables are limited to g_table_cap bytes (se_resize_set_table_cache_limit). When a call's new
// tables would pass the limit, the device's cache is emptied after a device synchronise BEFORE the call looks up any table, so
// every table a call launches with stays allocated until its kernels have run. (A single call's own tables may exceed the limit.)
struct AxisTable {
  int* bounds = nullptr;   // [out][2], followed in the same allocation by coeffs [out][ksize]
  int* coeffs = nullptr;
  int ksize = 0;
  size_t bytes = 0;
};
static std::mutex g_resize_mu;   // guards the cache and its limit; held for a whole se_resize_u8 call
static std::map<std::tuple<int, int, int>, AxisTable> g_tables;
constexpr size_t kDefaultTableCap = 256u << 20;
static size_t g_table_cap = kDefaultTableCap;

static size_t table_bytes(int in, int out) { return (size_t)out * (2 + resize_ksize(in, out)) * sizeof(int); }

static size_t held_bytes(int dev) {
  size_t held = 0;
  for (auto& kv : g_tables)
    if (std::get<0>(kv.first) == dev) held += kv.second.bytes;
  return held;
}

// (in, out) pairs of one call: empties the device's cache first when the call's missing tables would pass the limit
static int reserve_tables(int dev, const std::vector<std::pair<int, int>>& pairs) {
  std::vector<std::pair<int, int>> missing;
  size_t need = 0;
  for (auto& p : pairs) {
    if (g_tables.count(std::make_tuple(dev, p.first, p.second)) || std::find(missing.begin(), missing.end(), p) != missing.end()) continue;
    missing.push_back(p);
    need += table_bytes(p.first, p.second);
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

// the cached table of (in, out), built and uploaded on a miss; never frees a table (reserve_tables does, before any lookup)
static int axis_table(int dev, int in, int out, const AxisTable** t) {
  const auto key = std::make_tuple(dev, in, out);
  auto it = g_tables.find(key);
  if (it != g_tables.end()) {
    *t = &it->second;
    return 0;
  }
  AxisTable a;
  a.ksize = resize_ksize(in, out);
  std::vector<int> host((size_t)out * (2 + a.ksize));
  resize_coeff_table(in, out, host.data(), host.data() + 2 * (size_t)out);
  a.bytes = host.size() * sizeof(int);
  SE_CUDA_OK(cudaMalloc(&a.bounds, a.bytes));
  SE_CUDA_OK(cudaMemcpy(a.bounds, host.data(), a.bytes, cudaMemcpyHostToDevice));
  a.coeffs = a.bounds + 2 * (size_t)out;
  *t = &(g_tables[key] = a);
  return 0;
}

// ------------------------------------------------------------------------------------------ kernels
// Per-image descriptors travel as kernel parameters (RESIZE_MAX_BATCH of them, < 4 KB). A launch covers the tiles of all its
// images; tile0 is the first tile of an image, so a block finds its image by scanning the (at most 32) descriptors.
struct HPass {   // rows x in_w -> rows x out_w
  const unsigned char* src;
  unsigned char* dst;
  const int* bounds;
  const int* coeffs;
  int ksize, rows, in_w, out_w, swap, tile0, tiles_x;
};
struct VPass {   // in_h x row_bytes -> out_h x row_bytes; coeffs == nullptr: copy (one tap of weight 1 at the same row)
  const unsigned char* src;
  unsigned char* dst;
  const int* bounds;
  const int* coeffs;
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

template <typename P>
__device__ __forceinline__ int find_image(const PassList<P>& L) {
  int i = 0;
  while (i + 1 < L.n && (int)blockIdx.x >= L.p[i + 1].tile0) ++i;
  return i;
}

template <int C>
__global__ void __launch_bounds__(H_TX * H_TY) resize_h_kernel(const __grid_constant__ PassList<HPass> L) {
  extern __shared__ int smem[];   // coeffs [H_TX][ksize], bounds [H_TX][2]
  const HPass& d = L.p[find_image(L)];
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
  const unsigned char* s = d.src + ((size_t)y * d.in_w + xmin) * C;
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

// v[j] = clip8(2^21 + sum_x s[x * stride + j] * k[x]) for the first nb of NB bytes: 32-bit loads when vec (then nb == NB and
// s, stride are 4-byte aligned), byte loads otherwise
template <int NB>
__device__ __forceinline__ void v_taps(const unsigned char* s, int stride, const int* k, int n, int nb, bool vec, int (&v)[NB]) {
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
        if (j < nb) v[j] += (int)r[j] * w;
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
  const VPass& d = L.p[find_image(L)];
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
  v_taps(d.src + (size_t)ymin * d.row_bytes + p, d.row_bytes, sk + threadIdx.y * d.ksize, n, nb, vec, v);
  if (d.swap) swap_rb12(v);
  store12(d.dst + (size_t)(y0 + threadIdx.y) * d.row_bytes + p, v, nb, vec);
}

// The paste of se_resize_paste_u8: the vertical pass of a result (3 channels) and of its mask, both in_h x out_w, to out_h,
// then Pillow's Image.paste blend of the result over base with that mask, per channel:
//     dst = DIV255(base * (255 - m) + res * m),   DIV255(a) = ((t >> 8) + t) >> 8 with t = a + 128 (libImaging/Paste.c).
// A thread owns 4 pixels of one output row: 12 result, 4 mask, 12 base and 12 dst bytes. It reads its base bytes before it
// writes the same dst bytes, so dst may be base.
struct PPass {
  const unsigned char* rgb;
  const unsigned char* mask;
  const unsigned char* base;
  unsigned char* dst;
  const int* bounds;
  const int* coeffs;
  int ksize, in_h, out_h, out_w, groups, swap, vec, tile0, tiles_x;
};
constexpr int P_PIX = V_GROUP / 3;

__global__ void __launch_bounds__(V_TX * V_TY) paste_v_kernel(const __grid_constant__ PassList<PPass> L) {
  extern __shared__ int smem[];   // coeffs [V_TY][ksize], bounds [V_TY][2]
  const PPass& d = L.p[find_image(L)];
  const int t = blockIdx.x - d.tile0;
  const int g = (t % d.tiles_x) * V_TX + threadIdx.x, y0 = (t / d.tiles_x) * V_TY;
  const int nrow = min(V_TY, d.out_h - y0);
  int* sk = smem;
  int* sb = smem + V_TY * d.ksize;
  stage_v_taps(sk, sb, d.bounds, d.coeffs, d.ksize, y0, nrow);
  __syncthreads();
  if ((int)threadIdx.y >= nrow || g >= d.groups) return;
  const int ymin = sb[2 * threadIdx.y], n = sb[2 * threadIdx.y + 1];
  const int* k = sk + threadIdx.y * d.ksize;
  const int x0 = g * P_PIX, np = min(P_PIX, d.out_w - x0);
  const bool vec = d.vec && np == P_PIX;
  int c[V_GROUP], m[P_PIX];
  v_taps(d.rgb + ((size_t)ymin * d.out_w + x0) * 3, d.out_w * 3, k, n, np * 3, vec, c);
  v_taps(d.mask + (size_t)ymin * d.out_w + x0, d.out_w, k, n, np, vec, m);
  if (d.swap) swap_rb12(c);
  const size_t o = ((size_t)(y0 + threadIdx.y) * d.out_w + x0) * 3;
  int b[V_GROUP];
  if (vec) {   // plain loads: base may be dst
    const uint32_t* q = reinterpret_cast<const uint32_t*>(d.base + o);
#pragma unroll
    for (int w = 0; w < 3; ++w) {
      const uint32_t u = q[w];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[4 * w + j] = (int)((u >> (8 * j)) & 0xffu);
    }
  } else {
#pragma unroll
    for (int j = 0; j < V_GROUP; ++j) b[j] = j < np * 3 ? (int)d.base[o + j] : 0;
  }
#pragma unroll
  for (int j = 0; j < V_GROUP; ++j) {
    const int a = b[j] * (255 - m[j / 3]) + c[j] * m[j / 3] + 128;
    c[j] = ((a >> 8) + a) >> 8;
  }
  store12(d.dst + o, c, np * 3, vec);
}

static int cdiv_i(long long a, long long b) { return (int)((a + b - 1) / b); }

constexpr int kMaxDim = 65535;
constexpr size_t kScratchAlign = 256;
constexpr int kMaxSmem = 227 * 1024;

static size_t scratch_round(size_t bytes) { return (bytes + kScratchAlign - 1) / kScratchAlign * kScratchAlign; }

// the checks of image i that se_resize_u8 and se_resize_paste_u8 share
static int check_image(int i, int ih, int iw, int oh, int ow) {
  SE_REQUIRE(ih >= 1 && iw >= 1 && oh >= 1 && ow >= 1 && ih <= kMaxDim && iw <= kMaxDim && oh <= kMaxDim && ow <= kMaxDim,
             "image " + std::to_string(i) + ": sizes must be in [1, 65535]");
  SE_REQUIRE(resize_ksize(iw, ow) * (H_TX + 2) * 4 <= kMaxSmem && resize_ksize(ih, oh) * (V_TY + 2) * 4 <= kMaxSmem,
             "image " + std::to_string(i) + ": downscale factor too large");
  return 0;
}

// appends the horizontal pass rows x iw -> rows x ow of src into dst (the table of iw -> ow must be cached) to hl
static int add_h_pass(int dev, PassList<HPass>& hl, long long& tiles, int& kmax, const unsigned char* src, unsigned char* dst,
                      int rows, int iw, int ow, int swap) {
  const AxisTable* t = nullptr;
  int rc = axis_table(dev, iw, ow, &t);
  if (rc) return rc;
  HPass& h = hl.p[hl.n++];
  h.src = src;
  h.dst = dst;
  h.bounds = t->bounds;
  h.coeffs = t->coeffs;
  h.ksize = t->ksize;
  h.rows = rows;
  h.in_w = iw;
  h.out_w = ow;
  h.swap = swap;
  h.tile0 = (int)tiles;
  h.tiles_x = cdiv_i(ow, H_TX);
  tiles += (long long)h.tiles_x * cdiv_i(rows, H_TY);
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

// the vertical table of ih -> oh, or none (a copy) when the height does not change
static int v_table(int dev, int ih, int oh, const int** bounds, const int** coeffs, int* ksize) {
  *bounds = *coeffs = nullptr;
  *ksize = 1;
  if (ih == oh) return 0;
  const AxisTable* t = nullptr;
  int rc = axis_table(dev, ih, oh, &t);
  if (rc) return rc;
  *bounds = t->bounds;
  *coeffs = t->coeffs;
  *ksize = t->ksize;
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
  return resize_coeff_table(in, out, bounds, coeffs);
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

int se_resize_u8(const unsigned char* src, const long long* src_off, const int* src_hw, unsigned char* dst, const long long* dst_off,
                 const int* dst_hw, int n, int channels, int swap_rb, void* scratch, long long* scratch_bytes, void* stream) {
  SE_REQUIRE(n >= 0 && n <= RESIZE_MAX_BATCH, "n must be in [0, " + std::to_string(RESIZE_MAX_BATCH) + "] images per call");
  SE_REQUIRE(channels == 1 || channels == 3, "channels must be 1 or 3");
  SE_REQUIRE(!swap_rb || channels == 3, "swap_rb needs 3 channels");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_off && src_hw && dst_off && dst_hw), "null size / offset array");
  const int C = channels;
  size_t need = 0;
  std::vector<size_t> mid(n);
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    int rc = check_image(i, ih, iw, oh, ow);
    if (rc) return rc;
    SE_REQUIRE(src_off[i] >= 0 && dst_off[i] >= 0, "negative offset");
    mid[i] = need;
    if (iw != ow && ih != oh) need += scratch_round((size_t)ih * ow * C);
  }
  if (!scratch) {
    *scratch_bytes = (long long)need;
    return 0;
  }
  SE_REQUIRE((size_t)*scratch_bytes >= need, "scratch holds " + std::to_string(*scratch_bytes) + " bytes, needs " + std::to_string(need));
  if (n == 0) return 0;
  SE_REQUIRE(src && dst, "null src / dst");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_resize_mu);
  int dev = 0;
  SE_CUDA_OK(cudaGetDevice(&dev));
  {
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < n; ++i) {
      if (src_hw[2 * i + 1] != dst_hw[2 * i + 1]) pairs.emplace_back(src_hw[2 * i + 1], dst_hw[2 * i + 1]);
      if (src_hw[2 * i] != dst_hw[2 * i]) pairs.emplace_back(src_hw[2 * i], dst_hw[2 * i]);
    }
    int rc = reserve_tables(dev, pairs);
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
    const unsigned char* s = src + src_off[i];
    unsigned char* o = dst + dst_off[i];
    if (iw != ow) {
      unsigned char* h_dst = ih != oh ? (unsigned char*)scratch + mid[i] : o;
      int rc = add_h_pass(dev, hl, htiles, hk, s, h_dst, ih, iw, ow, ih == oh && swap_rb);
      if (rc) return rc;
      if (ih == oh) continue;
      s = h_dst;
    }
    VPass& v = vl.p[vl.n++];   // the vertical pass, or the copy of an image whose size does not change
    v.src = s;
    v.dst = o;
    int rc = v_table(dev, ih, oh, &v.bounds, &v.coeffs, &v.ksize);
    if (rc) return rc;
    v.in_h = ih;
    v.out_h = oh;
    v.row_bytes = ow * C;
    v.groups = cdiv_i(v.row_bytes, V_GROUP);
    v.swap = swap_rb;
    v.vec = ((uintptr_t)v.src % 4 == 0) && ((uintptr_t)v.dst % 4 == 0) && v.row_bytes % 4 == 0;
    v.tile0 = (int)vtiles;
    v.tiles_x = cdiv_i(v.groups, V_TX);
    vtiles += (long long)v.tiles_x * cdiv_i(oh, V_TY);
    vk = std::max(vk, v.ksize);
  }
  SE_REQUIRE(htiles < (1LL << 31) && vtiles < (1LL << 31), "batch too large for one launch");
  int rc = C == 3 ? launch_h<3>(hl, htiles, hk, st) : launch_h<1>(hl, htiles, hk, st);
  if (rc) return rc;
  if (vl.n) {
    const int smem = (V_TY * vk + 2 * V_TY) * 4;
    SE_CUDA_OK(cudaFuncSetAttribute(resize_v_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    resize_v_kernel<<<(unsigned)vtiles, dim3(V_TX, V_TY), smem, st>>>(vl);
    SE_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

int se_resize_paste_u8(const unsigned char* rgb, const long long* rgb_off, const unsigned char* mask, const long long* mask_off,
                       const int* src_hw, const unsigned char* base, const long long* base_off, unsigned char* dst,
                       const long long* dst_off, const int* dst_hw, int n, int swap_rb, void* scratch, long long* scratch_bytes,
                       void* stream) {
  SE_REQUIRE(n >= 0 && n <= RESIZE_MAX_BATCH, "n must be in [0, " + std::to_string(RESIZE_MAX_BATCH) + "] images per call");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (rgb_off && mask_off && src_hw && base_off && dst_off && dst_hw), "null size / offset array");
  size_t need = 0;
  std::vector<size_t> mid(n);
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    int rc = check_image(i, ih, iw, oh, ow);
    if (rc) return rc;
    SE_REQUIRE(rgb_off[i] >= 0 && mask_off[i] >= 0 && base_off[i] >= 0 && dst_off[i] >= 0, "negative offset");
    mid[i] = need;   // a width change: the result's and the mask's intermediates, ih x ow x 3 and ih x ow
    if (iw != ow) need += scratch_round((size_t)ih * ow * 3) + scratch_round((size_t)ih * ow);
  }
  if (!scratch) {
    *scratch_bytes = (long long)need;
    return 0;
  }
  SE_REQUIRE((size_t)*scratch_bytes >= need, "scratch holds " + std::to_string(*scratch_bytes) + " bytes, needs " + std::to_string(need));
  if (n == 0) return 0;
  SE_REQUIRE(rgb && mask && base && dst, "null rgb / mask / base / dst");
  cudaStream_t st = (cudaStream_t)stream;
  std::lock_guard<std::mutex> lk(g_resize_mu);
  int dev = 0;
  SE_CUDA_OK(cudaGetDevice(&dev));
  {
    std::vector<std::pair<int, int>> pairs;
    for (int i = 0; i < n; ++i) {
      if (src_hw[2 * i + 1] != dst_hw[2 * i + 1]) pairs.emplace_back(src_hw[2 * i + 1], dst_hw[2 * i + 1]);
      if (src_hw[2 * i] != dst_hw[2 * i]) pairs.emplace_back(src_hw[2 * i], dst_hw[2 * i]);
    }
    int rc = reserve_tables(dev, pairs);
    if (rc) return rc;
  }
  PassList<HPass> h3, h1;
  PassList<PPass> pl;
  memset(&h3, 0, sizeof(h3));
  memset(&h1, 0, sizeof(h1));
  memset(&pl, 0, sizeof(pl));
  long long t3 = 0, t1 = 0, ptiles = 0;
  int k3 = 1, k1 = 1, pk = 1;
  for (int i = 0; i < n; ++i) {
    const int ih = src_hw[2 * i], iw = src_hw[2 * i + 1], oh = dst_hw[2 * i], ow = dst_hw[2 * i + 1];
    PPass& p = pl.p[pl.n++];
    p.rgb = rgb + rgb_off[i];
    p.mask = mask + mask_off[i];
    if (iw != ow) {   // the paste reads the horizontal passes' output instead of the result itself
      unsigned char* s3 = (unsigned char*)scratch + mid[i];
      unsigned char* s1 = s3 + scratch_round((size_t)ih * ow * 3);
      int rc = add_h_pass(dev, h3, t3, k3, p.rgb, s3, ih, iw, ow, 0);
      if (rc) return rc;
      rc = add_h_pass(dev, h1, t1, k1, p.mask, s1, ih, iw, ow, 0);
      if (rc) return rc;
      p.rgb = s3;
      p.mask = s1;
    }
    p.base = base + base_off[i];
    p.dst = dst + dst_off[i];
    int rc = v_table(dev, ih, oh, &p.bounds, &p.coeffs, &p.ksize);
    if (rc) return rc;
    p.in_h = ih;
    p.out_h = oh;
    p.out_w = ow;
    p.groups = cdiv_i(ow, P_PIX);
    p.swap = swap_rb;
    p.vec = ow % 4 == 0 && ((uintptr_t)p.rgb | (uintptr_t)p.mask | (uintptr_t)p.base | (uintptr_t)p.dst) % 4 == 0;
    p.tile0 = (int)ptiles;
    p.tiles_x = cdiv_i(p.groups, V_TX);
    ptiles += (long long)p.tiles_x * cdiv_i(oh, V_TY);
    pk = std::max(pk, p.ksize);
  }
  SE_REQUIRE(t3 < (1LL << 31) && ptiles < (1LL << 31), "batch too large for one launch");
  int rc = launch_h<3>(h3, t3, k3, st);
  if (rc) return rc;
  rc = launch_h<1>(h1, t1, k1, st);
  if (rc) return rc;
  SE_CUDA_OK(cudaFuncSetAttribute(paste_v_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  paste_v_kernel<<<(unsigned)ptiles, dim3(V_TX, V_TY), (V_TY * pk + 2 * V_TY) * 4, st>>>(pl);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

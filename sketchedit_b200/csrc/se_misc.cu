// Glue kernels of the generator forward: input packing, heads (12->3 / 12->1 conv + tanh/sigmoid + blends), global pooling,
// mask pooling, the fp32 attention operands and softmax, layout conversion. The kernels that touch activations are written once
// over the activation storage (F32 / Bf16 / Split below).
#include <type_traits>

#include "se_common.cuh"
#include "se_misc.h"

namespace se {

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------ activation storage
// Which words hold channel c of a pixel and how a value is encoded in them (DESIGN.md §4). Offsets count words of the storage;
// `lo` is the distance from a split-half hi word to its lo word (ignored by the other two). load8 / store8 move the 8 channels of
// one channel block of one pixel (16 B aligned in the channel-blocked storages; load8<N> reads only the first N of an fp32 row
// that ends there); get / put move one channel.
//   F32    fp32, NHWC in the forward                                         (fp32_direct)
//   Bf16   bf16, channel-blocked in the forward                              (bf16)
//   Split  fp16 hi + lo of 64 v (split_half), channel-blocked, the lo blocks after the hi blocks   (fp32)
struct F32 {
  static constexpr int kHalves = 1;
  static constexpr bool kBlocked = false;
  template <int N = 8>
  __device__ static void load8(const void* x, size_t o, size_t, float (&v)[8]) {
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = __ldg(static_cast<const float*>(x) + o + k);
  }
  __device__ static void store8(void* y, size_t o, size_t, const float (&v)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) static_cast<float*>(y)[o + k] = v[k];
  }
  __device__ static float get(const void* x, size_t o, size_t) { return __ldg(static_cast<const float*>(x) + o); }
  __device__ static void put(void* y, size_t o, size_t, float v) { static_cast<float*>(y)[o] = v; }
};

struct Bf16 {
  static constexpr int kHalves = 1;
  static constexpr bool kBlocked = true;
  template <int N = 8>
  __device__ static void load8(const void* x, size_t o, size_t, float (&v)[8]) {
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(x) + o));
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // a bf16x2 word is the (even, odd) channel pair
      v[2 * k] = __uint_as_float(w[k] << 16);
      v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u);
    }
  }
  __device__ static void store8(void* y, size_t o, size_t, const float (&v)[8]) {
    *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(y) + o) =
        make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
  }
  __device__ static float get(const void* x, size_t o, size_t) { return __bfloat162float(static_cast<const __nv_bfloat16*>(x)[o]); }
  __device__ static void put(void* y, size_t o, size_t, float v) { static_cast<__nv_bfloat16*>(y)[o] = __float2bfloat16(v); }
};

struct Split {
  static constexpr int kHalves = 2;
  static constexpr bool kBlocked = true;
  template <int N = 8>
  __device__ static void load8(const void* x, size_t o, size_t lo, float (&v)[8]) {
    const __half* p = static_cast<const __half*>(x) + o;
    const uint4 qh = __ldg(reinterpret_cast<const uint4*>(p)), ql = __ldg(reinterpret_cast<const uint4*>(p + lo));
    const __half* h = reinterpret_cast<const __half*>(&qh);
    const __half* l = reinterpret_cast<const __half*>(&ql);
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = join_half(h[k], l[k], kSplitActInv);
  }
  __device__ static void store8(void* y, size_t o, size_t lo, const float (&v)[8]) {
    __align__(16) __half h[8], l[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) split_half(v[k], kSplitActScale, h[k], l[k]);
    __half* p = static_cast<__half*>(y) + o;
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(p + lo) = *reinterpret_cast<const uint4*>(l);
  }
  __device__ static float get(const void* x, size_t o, size_t lo) {
    const __half* p = static_cast<const __half*>(x) + o;
    return join_half(p[0], p[lo], kSplitActInv);
  }
  __device__ static void put(void* y, size_t o, size_t lo, float v) {
    __half* p = static_cast<__half*>(y) + o;
    split_half(v, kSplitActScale, p[0], p[lo]);
  }
};

// runs f(St{}) for the storage of dtype dt
template <class F>
static int with_storage(int dt, F&& f) {
  if (dt == DT_F32) f(F32{});
  else if (dt == DT_BF16) f(Bf16{});
  else if (dt == DT_F16X2) f(Split{});
  else SE_REQUIRE(false, "activation storage " + std::to_string(dt));
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// word offset (and lo distance) of channel c of pixel (y, x) of image b in layout v of a storage with kHalves halves
template <int kHalves>
__device__ __forceinline__ size_t layout_offset(const Layout& v, long long b, int c, int y, int x, size_t& lo) {
  if (v.kind == LAYOUT_NHWC) {
    lo = 0;
    return (((size_t)b * v.H + y) * v.W + x) * v.ld + c;
  }
  if (v.kind == LAYOUT_C8) {
    lo = (size_t)(v.ld / kHalves) * v.H * v.W * 8;
    return ((((size_t)b * v.ld + (c >> 3)) * v.H + y) * v.W + x) * 8 + (c & 7);
  }
  if (v.kind == LAYOUT_S2D) {
    const int Hs = v.H / 2, Ws = v.W / 2, G = v.ld / 4;   // G: blocks of one parity group
    lo = (size_t)(G / kHalves) * Hs * Ws * 8;
    const int blk = ((y & 1) * 2 + (x & 1)) * G + (c >> 3);
    return ((((size_t)b * v.ld + blk) * Hs + (y >> 1)) * Ws + (x >> 1)) * 8 + (c & 7);
  }
  lo = (size_t)v.H * v.Wp * 8;   // LAYOUT_ROWS
  return (((size_t)b * kHalves * v.H + y) * v.Wp + x + v.padl) * 8 + c;
}

// ------------------------------------------------------------------------------------------ pack8
// reference editline2_g.py:62 (cat[image, sketch]) and editline_g.py:120-135 (mask-mul + cat), into packed rows
// [B][halves][H][Wp][8] (image at [padl, padl + W), pads written as zeros)
template <class St>
__global__ void pack8_kernel(const float* __restrict__ img, const float* __restrict__ sketch, const float* __restrict__ mask,
                             void* __restrict__ out, int B, int H, int W, int Wp, int padl, int img_mode, float sketch_scale,
                             int write_mask, int img2_mode) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // (b, y, xp)
  const long long HW = (long long)H * W;
  if (j >= (long long)B * H * Wp) return;
  const int xp = (int)(j % Wp);
  const long long by = j / Wp;
  const size_t o = (size_t)(j + (St::kHalves - 1) * (by / H) * H * Wp) * 8, lo = (size_t)H * Wp * 8;
  const int x = xp - padl;
  float v[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) v[c] = 0.0f;
  if (x >= 0 && x < W) {
    const long long b = by / H, pix = (by % H) * W + x;
    const long long i = b * HW + pix;
    const float m = mask ? mask[i] : 0.0f;
    const float a = img_mode == PACK_IMG_ONE ? 1.0f : (img_mode == PACK_IMG_ONE_MINUS_M ? 1.0f - m : m);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = img[(b * 3 + c) * HW + pix] * a;
    v[3] = (sketch ? sketch[i] : 1.0f) * sketch_scale;   // guide=None -> ones (reference editline_g.py:127-130)
    v[4] = write_mask ? m : 0.0f;
    if (img2_mode >= 0) {   // second masked copy of the image in channels 5..7 (the style encoder's input, stem pair conv1 + wconv1)
      const float a2 = img2_mode == PACK_IMG_ONE ? 1.0f : (img2_mode == PACK_IMG_ONE_MINUS_M ? 1.0f - m : m);
#pragma unroll
      for (int c = 0; c < 3; ++c) v[5 + c] = img[(b * 3 + c) * HW + pix] * a2;
    }
  }
  St::store8(out, o, lo, v);
}

int pack8(const float* img, const float* sketch, const float* mask, void* out, int dt, int B, int H, int W, int Wp, int padl,
          int img_mode, float sketch_scale, int write_mask, cudaStream_t s, int img2_mode) {
  const long long n = (long long)B * H * Wp;
  return with_storage(dt, [&](auto st) {
    pack8_kernel<decltype(st)><<<cdiv(n, 256), 256, 0, s>>>(img, sketch, mask, out, B, H, W, Wp, padl, img_mode, sketch_scale, write_mask,
                                                            img2_mode);
  });
}

// ------------------------------------------------------------------------------------------ heads
// 3x3 / pad 1 conv over a 12-channel map to COUT in {1,3} channels (reference conv17 / conv_mask_17 / allconv17: raw conv,
// utils.py:27) fused with the caller-side nonlinearity:
//   HEAD_MASK   sigmoid -> soft mask (NCHW) + binarised mask plane   (editline2_g.py:93, editline2_model.py:347)
//   HEAD_TANH   tanh -> NCHW                                         (editline2_g.py:84)
//   HEAD_COARSE tanh -> [optional NCHW], xnow = t*m + img*(1-m)*(1-m) into packed rows   (editline_g.py:176-181)
//   HEAD_FINE   tanh -> [optional NCHW], composed = t*soft + img*(1-soft) (NCHW)       (editline_g.py:220, editline2_model.py:132)
// The input is fp32 NHWC [B][H][W][12] or two channel blocks [B][2 * halves][H][W][8]. The weights are a by-value kernel
// parameter: they sit in the constant bank and feed the FMAs directly.
template <int COUT>
struct HeadWeights {
  float2 w[9][6][COUT];   // [tap][channel pair][out] = (w[tap][2p][o], w[tap][2p+1][o])
  float b[COUT];
};
template <class St, int COUT>
__global__ void __launch_bounds__(128) head_kernel(const __grid_constant__ HeadWeights<COUT> hw, const __grid_constant__ HeadIO io) {
  // the *_bs strides are set (head_launch); mask_bs and composed_bs are 4*HW when the output is a view into a packed [B,4,H,W] output
  // bf16 sums each output as an (even, odd) pair of partial sums over the channel pairs of its bf16x2 words, the bias added last;
  // the fp32 storages keep one FMA chain from the bias in channel order (the order tests/util_stages.py bounds)
  constexpr bool kPairs = std::is_same<St, Bf16>::value;
  const int H = io.H, W = io.W;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long HW = (long long)H * W;
  if (i >= io.B * HW) return;
  const long long b = i / HW, pix = i % HW;
  const int yy = (int)(pix / W), xx = (int)(pix % W);
  float2 acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = make_float2(kPairs ? 0.0f : hw.b[o], 0.0f);
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int iy = yy + t / 3 - 1, ix = xx + t % 3 - 1;
    if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
    const long long q = (long long)iy * W + ix;
    float v[2][8];   // channels 0..7, 8..11 (12..15: padding of the second block)
    if constexpr (St::kBlocked) {
      const size_t o = ((size_t)b * 2 * St::kHalves * HW + q) * 8, blk = (size_t)HW * 8;
      St::load8(io.x, o, 2 * blk, v[0]);
      St::load8(io.x, o + blk, 2 * blk, v[1]);
    } else {
      St::load8(io.x, (size_t)(b * HW + q) * 12, 0, v[0]);
      St::template load8<4>(io.x, (size_t)(b * HW + q) * 12 + 8, 0, v[1]);
    }
#pragma unroll
    for (int p = 0; p < 6; ++p) {
      const float xe = v[p / 4][(2 * p) % 8], xo = v[p / 4][(2 * p + 1) % 8];
#pragma unroll
      for (int o = 0; o < COUT; ++o) {
        const float2 wv = hw.w[t][p][o];
        if (kPairs) {
          acc[o].x = fmaf(xe, wv.x, acc[o].x);
          acc[o].y = fmaf(xo, wv.y, acc[o].y);
        } else {
          acc[o].x = fmaf(xo, wv.y, fmaf(xe, wv.x, acc[o].x));
        }
      }
    }
  }
  float r[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) r[o] = kPairs ? hw.b[o] + (acc[o].x + acc[o].y) : acc[o].x;
  if (io.mode == HEAD_MASK) {
    const float sg = 1.0f / (1.0f + expf(-r[0]));
    io.mask[b * io.mask_bs + pix] = sg;
    io.mask_bin[i] = sg > 0.5f ? 1.0f : 0.0f;
    if (io.mask_u8) io.mask_u8[i] = (unsigned char)(int)(sg * 255.0f);   // test.py:25: (mask * 255).astype(uint8)
    return;
  }
  float t3[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) t3[o] = tanhf(r[o]);
  if (io.mode == HEAD_TANH) {
#pragma unroll
    for (int o = 0; o < COUT; ++o) io.stage[(b * COUT + o) * HW + pix] = t3[o];
  } else if (io.mode == HEAD_COARSE) {
    const float m = io.blend[i];
    float pk[8];
#pragma unroll
    for (int o = 0; o < 8; ++o) pk[o] = 0.0f;
#pragma unroll
    for (int o = 0; o < COUT; ++o) {
      if (io.stage) io.stage[(b * COUT + o) * HW + pix] = t3[o];
      const float xin = io.img[(b * 3 + o) * HW + pix] * (1.0f - m);
      pk[o] = io.no_mask_coarse ? t3[o] : (t3[o] * m + xin * (1.0f - m));
    }
    const size_t o = (((size_t)b * St::kHalves * H + yy) * io.Wp + xx + io.padl) * 8;   // packed rows, as pack8 writes them
    St::store8(io.packed, o, (size_t)H * io.Wp * 8, pk);
  } else {  // HEAD_FINE
    const float m = io.blend[b * io.blend_bs + pix];
#pragma unroll
    for (int o = 0; o < COUT; ++o) {
      if (io.stage) io.stage[(b * COUT + o) * HW + pix] = t3[o];
      const float cv = t3[o] * m + io.img[(b * 3 + o) * HW + pix] * (1.0f - m);
      if (io.composed) io.composed[b * io.composed_bs + o * HW + pix] = cv;
      if (io.bgr_u8) io.bgr_u8[i * 3 + (2 - o)] = (unsigned char)(int)((cv + 1.0f) / 2.0f * 255.0f);   // test.py:26-35: truncate, HWC, RGB -> BGR
    }
  }
}

template <int COUT>
static int head_launch(HeadIO io, int dt, const float* w_host, const float* b_host, cudaStream_t s) {
  HeadWeights<COUT> hw;
  for (int t = 0; t < 9; ++t)
    for (int p = 0; p < 6; ++p)
      for (int o = 0; o < COUT; ++o) hw.w[t][p][o] = make_float2(w_host[(t * 12 + 2 * p) * COUT + o], w_host[(t * 12 + 2 * p + 1) * COUT + o]);
  for (int o = 0; o < COUT; ++o) hw.b[o] = b_host[o];
  const long long HW = (long long)io.H * io.W;
  if (!io.blend_bs) io.blend_bs = HW;
  if (!io.mask_bs) io.mask_bs = HW;
  if (!io.composed_bs) io.composed_bs = 3 * HW;
  return with_storage(dt, [&](auto st) { head_kernel<decltype(st), COUT><<<cdiv(io.B * HW, 128), 128, 0, s>>>(hw, io); });
}
int head(HeadIO io, int dt, const float* w_host, const float* b_host, int cout, cudaStream_t s) {
  SE_REQUIRE(cout == 1 || cout == 3, "head cout");
  return cout == 1 ? head_launch<1>(io, dt, w_host, b_host, s) : head_launch<3>(io, dt, w_host, b_host, s);
}

// ------------------------------------------------------------------------------------------ plane reductions
// per (image, channel) reduction over the h x w plane:
//   RED_MAX / RED_AVG      global pooling            (editline_g.py:160-165)
//   RED_RNORM              1/sqrt(sum x^2 + 1e-8)    (splitcam.py:40; fp32 NHWC only: the fp32 attention key norm)
// fp32 NHWC: one thread column per channel
__global__ void plane_reduce_kernel(const float* __restrict__ x, int ldx, int C, int HW, int mode, float* __restrict__ out) {
  __shared__ float red[8][33];
  const int b = blockIdx.y;
  const int c = blockIdx.x * 32 + threadIdx.x;
  float acc = (mode == RED_MAX) ? -INFINITY : 0.0f;
  if (c < C) {
    const float* xp = x + (size_t)b * HW * ldx + c;   // pixel pitch ldx
#pragma unroll 4   // left to itself nvcc unrolls further and needs 32 registers instead of 22-24
    for (int p = threadIdx.y; p < HW; p += 8) {
      const float v = xp[(size_t)p * ldx];
      if (mode == RED_MAX) acc = fmaxf(acc, v);
      else if (mode == RED_AVG) acc += v;
      else acc = fmaf(v, v, acc);
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int j = 1; j < 8; ++j) {
      const float v = red[j][threadIdx.x];
      acc = (mode == RED_MAX) ? fmaxf(acc, v) : acc + v;
    }
    if (mode == RED_AVG) acc /= (float)HW;
    if (mode == RED_RNORM) acc = 1.0f / sqrtf(acc + 1e-8f);
    out[(size_t)b * C + c] = acc;
  }
}

// channel-blocked (bf16, split-half): one block per (image, channel block), the plane is HW contiguous pixels of 8 channels
template <class St>
__global__ void plane_reduce_c8_kernel(const void* __restrict__ x, int ld, int C, int HW, int mode, float* __restrict__ out) {
  __shared__ float red[8][8];
  const int b = blockIdx.y, cb = blockIdx.x;
  const size_t o = ((size_t)b * ld + cb) * HW * 8, lo = (size_t)(ld / St::kHalves) * HW * 8;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = (mode == RED_MAX) ? -INFINITY : 0.0f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    float v[8];
    St::load8(x, o + (size_t)p * 8, lo, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = (mode == RED_MAX) ? fmaxf(acc[i], v[i]) : acc[i] + v[i];
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
    for (int o = 16; o; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, acc[i], o);
      acc[i] = (mode == RED_MAX) ? fmaxf(acc[i], t) : acc[i] + t;
    }
  const int wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 8; ++i) red[wid][i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 8) {
    float r = red[0][threadIdx.x];
    for (int j = 1; j < nw; ++j) r = (mode == RED_MAX) ? fmaxf(r, red[j][threadIdx.x]) : r + red[j][threadIdx.x];
    if (mode == RED_AVG) r /= (float)HW;
    const int c = cb * 8 + threadIdx.x;
    if (c < C) out[(size_t)b * C + c] = r;
  }
}

int plane_reduce(const void* x, int dt, int B, int HW, int C, int ld, int mode, float* out, cudaStream_t s) {
  if (dt == DT_F32) {
    plane_reduce_kernel<<<dim3(cdiv(C, 32), B), dim3(32, 8), 0, s>>>((const float*)x, ld, C, HW, mode, out);
    SE_CUDA_OK(cudaGetLastError());
    return 0;
  }
  SE_REQUIRE(mode == RED_MAX || mode == RED_AVG, "channel-blocked reductions: max / avg");
  SE_REQUIRE(dt == DT_BF16 || dt == DT_F16X2, "channel-blocked storage");
  const dim3 grid((C + 7) / 8, B);
  if (dt == DT_BF16) plane_reduce_c8_kernel<Bf16><<<grid, 256, 0, s>>>(x, ld, C, HW, mode, out);
  else plane_reduce_c8_kernel<Split><<<grid, 256, 0, s>>>(x, ld, C, HW, mode, out);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// nearest 1x1 -> h x w broadcast of the pooled vector v [B][C] into channels [choff, choff + C) (editline_g.py:166-167:
// interpolate + cat); one thread per (image, channel block, pixel)
template <class St>
__global__ void broadcast_kernel(const float* __restrict__ v, void* __restrict__ y, int C, int HW, int ld, int choff, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long p = i % HW;
  long long r = i / HW;
  const int cb = (int)(r % (C >> 3));
  const long long b = r / (C >> 3);
  float f[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) f[k] = v[b * C + cb * 8 + k];
  if constexpr (St::kBlocked) St::store8(y, (((size_t)b * ld + (choff >> 3) + cb) * HW + p) * 8, (size_t)(ld / St::kHalves) * HW * 8, f);
  else St::store8(y, ((size_t)b * HW + p) * ld + choff + cb * 8, 0, f);
}

int broadcast_channels(const float* v, void* y, int dt, int B, int HW, int C, int ld, int choff, cudaStream_t s) {
  SE_REQUIRE(C % 8 == 0 && choff % 8 == 0, "the broadcast writes whole channel blocks");
  const long long n = (long long)B * (C >> 3) * HW;
  return with_storage(dt, [&](auto st) { broadcast_kernel<decltype(st)><<<cdiv(n, 256), 256, 0, s>>>(v, y, C, HW, ld, choff, n); });
}

// ------------------------------------------------------------------------------------------ mask pooling
// avg_pool2d(mask, 4, 4) (editline_g.py:204) and the per-key valid flag of cam_1
// (splitcam.py:49-53,89-90: mean over the 4x4 patch of (1 - mask_s) > th).
__global__ void avgpool4_kernel(const float* __restrict__ m, float* __restrict__ out, int B, int H, int W) {
  const int h = H / 4, w = W / 4;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * h * w) return;
  const int x = (int)(i % w), y = (int)((i / w) % h);
  const long long b = i / ((long long)h * w);
  float a = 0.0f;
  for (int u = 0; u < 4; ++u)
    for (int v = 0; v < 4; ++v) a += m[(b * H + 4 * y + u) * W + 4 * x + v];
  out[i] = a * (1.0f / 16.0f);
}

int avgpool4(const float* m, float* out, int B, int H, int W, cudaStream_t s) {
  avgpool4_kernel<<<cdiv((long long)B * (H / 4) * (W / 4), 256), 256, 0, s>>>(m, out, B, H, W);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void cam_colmask_kernel(const float* __restrict__ mask_s, float* __restrict__ out, int B, int h, int w, int hs, int ws,
                                   int patch, int stride, float th) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * hs * ws) return;
  const int lx = (int)(i % ws), ly = (int)((i / ws) % hs);
  const long long b = i / ((long long)hs * ws);
  float a = 0.0f;
  for (int u = 0; u < patch; ++u)
    for (int v = 0; v < patch; ++v) a += 1.0f - mask_s[(b * h + ly * stride + u) * w + lx * stride + v];
  // the reference takes mean over v then over u of exact multiples of 1/16: the order does not matter
  out[i] = (a / (float)(patch * patch) > th) ? 1.0f : 0.0f;
}

int cam_colmask(const float* mask_s, float* out, int B, int h, int w, int hs, int ws, float th, cudaStream_t s) {
  cam_colmask_kernel<<<cdiv((long long)B * hs * ws, 256), 256, 0, s>>>(mask_s, out, B, h, w, hs, ws, 4, 2, th);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------ attention operands (fp32)
// Keys  K[l][(u,v,c)] = f[2ly+u, 2lx+v, c] * rnorm[c]        (splitcam.py:39-44, norm_type 1, 4x4 / stride 2)
// direct layout: fp32 [b][tap][c][CoutP]
__global__ void cam_pack_k_direct_kernel(const float* __restrict__ f, const float* __restrict__ rnorm, float* __restrict__ out,
                                         int B, int h, int w, int C, int ws, int L, int CoutP, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int l = (int)(i % CoutP);
  long long r = i / CoutP;
  const int c = (int)(r % C); r /= C;
  const int tap = (int)(r % 16);
  const long long b = r / 16;
  float v = 0.0f;
  if (l < L) {
    const int ly = l / ws, lx = l % ws, u = tap / 4, vv = tap % 4;
    v = f[((b * h + 2 * ly + u) * w + 2 * lx + vv) * C + c] * rnorm[b * C + c];
  }
  out[i] = v;
}

int cam_pack_k(const float* f, const float* rnorm, float* out, int B, int h, int w, int C, int ws, int L, int Lpad, cudaStream_t s) {
  const long long total = (long long)B * 16 * C * Lpad;
  cam_pack_k_direct_kernel<<<cdiv(total, 256), 256, 0, s>>>(f, rnorm, out, B, h, w, C, ws, L, Lpad, total);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// Values for the fold-sum written as 4 sub-pixel (parity) 2x2 "convolutions" over the token image
// P[b, ny, nx, l] (splitcam.py:152, utils.py:102-128):
//   out[2yy+py, 2xx+px, c] = sum_{a,b in {0,1}} sum_l P[yy-a, xx-b, l] * f[2ly+py+2a, 2lx+px+2b, c]
// direct layout: fp32 [pc][b][tap][l (Ci = Lpad)][CoutP = C]
__global__ void cam_pack_v_direct_kernel(const float* __restrict__ f, float* __restrict__ out, int B, int h, int w, int C, int ws, int L,
                                         int Lpad, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  long long r = i / C;
  const int l = (int)(r % Lpad); r /= Lpad;
  const int tap = (int)(r % 4); r /= 4;
  const long long b = r % B;
  const int pc = (int)(r / B);
  float v = 0.0f;
  if (l < L) {
    const int ly = l / ws, lx = l % ws, py = pc / 2, px = pc % 2, a = tap / 2, bb = tap % 2;
    v = f[((b * h + 2 * ly + py + 2 * a) * w + 2 * lx + px + 2 * bb) * C + c];
  }
  out[i] = v;
}

int cam_pack_v(const float* f, float* out, int B, int h, int w, int C, int ws, int L, int Lpad, cudaStream_t s) {
  const long long total = 4LL * B * 4 * Lpad * C;
  cam_pack_v_direct_kernel<<<cdiv(total, 256), 256, 0, s>>>(f, out, B, h, w, C, ws, L, Lpad, total);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// softmax over the key axis of the logits S[row][0..L) (fp32, row pitch lds) -> P[row][0..Lpad) with
// zero padding (splitcam.py:105; the scale 10 and the key mask are already applied by the GEMM epilogue).
__global__ void softmax_rows_kernel(const float* __restrict__ S, int lds, float* __restrict__ P, int ldp, int L) {
  // one 256-thread block per row; up to SM_MAXV values per thread stay in registers (rows <= 256*SM_MAXV keys),
  // longer rows fall back to re-reading
  constexpr int SM_MAXV = 16;
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* s = S + row * lds;
  float* p = P + row * ldp;
  const bool fits = L <= 256 * SM_MAXV;
  float v[SM_MAXV];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < SM_MAXV; ++k) {
    const int i = threadIdx.x + k * 256;
    v[k] = (fits && i < L) ? s[i] : -INFINITY;
    mx = fmaxf(mx, v[k]);
  }
  if (!fits)
    for (int i = threadIdx.x; i < L; i += 256) mx = fmaxf(mx, s[i]);
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.0f;
  if (fits) {
#pragma unroll
    for (int k = 0; k < SM_MAXV; ++k) {
      v[k] = expf(v[k] - mx);      // exp(-inf) = 0 for the padding lanes
      sum += v[k];
    }
  } else {
    for (int i = threadIdx.x; i < L; i += 256) sum += expf(s[i] - mx);
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.0f;
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  if (fits) {
#pragma unroll
    for (int k = 0; k < SM_MAXV; ++k) {
      const int i = threadIdx.x + k * 256;
      if (i < ldp) p[i] = i < L ? v[k] * inv : 0.0f;
    }
  } else {
    for (int i = threadIdx.x; i < ldp; i += 256) p[i] = i < L ? expf(s[i] - mx) * inv : 0.0f;
  }
}

int softmax_rows(const float* S, int lds, float* P, int ldp, long long rows, int L, cudaStream_t s) {
  softmax_rows_kernel<<<(unsigned)rows, 256, 0, s>>>(S, lds, P, ldp, L);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------ layout conversion
// between an fp32 tensor (NCHW, or NHWC when nhwc) of B x C x v.H x v.W and an activation in layout v; one thread per element of
// the fp32 tensor. Channels and pixels of the activation outside the fp32 tensor are not written.
__device__ __forceinline__ void f32_coords(long long i, int nhwc, int C, int H, int W, long long& b, int& c, int& y, int& x) {
  if (nhwc) { c = (int)(i % C); i /= C; }
  x = (int)(i % W); i /= W;
  y = (int)(i % H); i /= H;
  if (!nhwc) { c = (int)(i % C); i /= C; }
  b = i;
}
template <class St>
__global__ void f32_to_act_kernel(const float* __restrict__ x, int nhwc, void* __restrict__ y, const Layout v, int C, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long b;
  int c, py, px;
  f32_coords(i, nhwc, C, v.H, v.W, b, c, py, px);
  size_t lo;
  const size_t o = layout_offset<St::kHalves>(v, b, c, py, px, lo);
  St::put(y, o, lo, x[i]);
}
template <class St>
__global__ void act_to_f32_kernel(const void* __restrict__ x, const Layout v, float* __restrict__ y, int nhwc, int C, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long b;
  int c, py, px;
  f32_coords(i, nhwc, C, v.H, v.W, b, c, py, px);
  size_t lo;
  const size_t o = layout_offset<St::kHalves>(v, b, c, py, px, lo);
  y[i] = St::get(x, o, lo);
}

static int check_layout(const Layout& v, int C) {
  SE_REQUIRE(v.kind != LAYOUT_S2D || (C % 8 == 0 && v.H % 2 == 0 && v.W % 2 == 0), "space-to-depth needs C % 8 == 0 and even H, W");
  SE_REQUIRE(v.kind != LAYOUT_ROWS || C <= 8, "packed rows hold 8 channels");
  return 0;
}
int f32_to_act(const float* x, int nhwc, void* y, int dt, const Layout& v, int B, int C, cudaStream_t s) {
  int rc = check_layout(v, C);
  if (rc) return rc;
  const long long total = (long long)B * C * v.H * v.W;
  return with_storage(dt, [&](auto st) { f32_to_act_kernel<decltype(st)><<<cdiv(total, 256), 256, 0, s>>>(x, nhwc, y, v, C, total); });
}
int act_to_f32(const void* x, int dt, const Layout& v, float* y, int nhwc, int B, int C, cudaStream_t s) {
  int rc = check_layout(v, C);
  if (rc) return rc;
  const long long total = (long long)B * C * v.H * v.W;
  return with_storage(dt, [&](auto st) { act_to_f32_kernel<decltype(st)><<<cdiv(total, 256), 256, 0, s>>>(x, v, y, nhwc, C, total); });
}

// reference data/testimage_dataset.py:89-103 on device: image uint8 HWC RGB -> fp32 NCHW (ToTensor: /255; Normalize(0.5, 0.5)),
// sketch uint8 (already resized to the image) -> {0, 1} fp32 (ToTensor then > 0). A caller-supplied edit mask (mask_u8, optional)
// -> its soft plane v/255 (ToTensor; the inverse of the (int)(m * 255) output codec: trunc((v/255)*255) == v for every byte) and
// its binarised plane (soft > 0.5, the comparison of head_kernel's HEAD_MASK branch: 1 exactly for v >= 128)
__global__ void u8_to_inputs_kernel(const unsigned char* __restrict__ img_u8, const unsigned char* __restrict__ sk_u8, float* __restrict__ img,
                                    float* __restrict__ sk, int B, long long HW, const unsigned char* __restrict__ mask_u8,
                                    float* __restrict__ mask_soft, float* __restrict__ mask_bin) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const long long b = i / HW, pix = i % HW;
#pragma unroll
  for (int c = 0; c < 3; ++c) img[(b * 3 + c) * HW + pix] = (__fdiv_rn((float)img_u8[i * 3 + c], 255.0f) - 0.5f) / 0.5f;
  sk[i] = sk_u8[i] > 0 ? 1.0f : 0.0f;
  if (mask_u8) {
    const float m = __fdiv_rn((float)mask_u8[i], 255.0f);
    mask_soft[i] = m;
    mask_bin[i] = m > 0.5f ? 1.0f : 0.0f;
  }
}
int u8_to_inputs(const unsigned char* img_u8, const unsigned char* sk_u8, const unsigned char* mask_u8, float* img, float* sk, float* mask_soft,
                 float* mask_bin, int B, int H, int W, cudaStream_t s) {
  SE_REQUIRE(!mask_u8 || (mask_soft && mask_bin), "an edit mask needs its soft and binarised planes");
  const long long HW = (long long)H * W;
  u8_to_inputs_kernel<<<cdiv(B * HW, 256), 256, 0, s>>>(img_u8, sk_u8, img, sk, B, HW, mask_u8, mask_soft, mask_bin);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// a caller-supplied fp32 edit mask -> the binarised plane netG inpaints: m > 0.5 (editline2_model.py:347), the comparison of
// head_kernel's HEAD_MASK branch, so netM's own soft mask binarises to the bytes the plain forward uses
__global__ void binarise_kernel(const float* __restrict__ m, float* __restrict__ out, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) out[i] = m[i] > 0.5f ? 1.0f : 0.0f;
}
int binarise(const float* m, float* out, long long n, cudaStream_t s) {
  binarise_kernel<<<cdiv(n, 256), 256, 0, s>>>(m, out, n);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// test.py:25-27,33-35: (mask*255).astype(uint8); ((x+1)/2*255).astype(uint8) (truncation), CHW->HWC, RGB->BGR
__global__ void to_uint8_kernel(const float* __restrict__ comp, const float* __restrict__ mask, unsigned char* __restrict__ bgr,
                                unsigned char* __restrict__ mk, int B, long long HW) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const long long b = i / HW, pix = i % HW;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = (comp[(b * 3 + c) * HW + pix] + 1.0f) / 2.0f * 255.0f;
    bgr[i * 3 + (2 - c)] = (unsigned char)(int)v;
  }
  if (mk) mk[i] = (unsigned char)(int)(mask[i] * 255.0f);
}

int to_uint8(const float* comp, const float* mask, unsigned char* bgr, unsigned char* mk, int B, int H, int W, cudaStream_t s) {
  const long long HW = (long long)H * W;
  to_uint8_kernel<<<cdiv(B * HW, 256), 256, 0, s>>>(comp, mask, bgr, mk, B, HW);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// zero-fill helper for padded channel tails
int fill_zero(void* p, size_t bytes, cudaStream_t s) {
  SE_CUDA_OK(cudaMemsetAsync(p, 0, bytes, s));
  return 0;
}

}  // namespace se

// Region-edit detail: contextual residual aggregation (Yi et al., CVPR 2020) on netG's own attention weights. A region edit
// runs the network on its box resampled to the working size Wn x Hn and resizes the result back; the detail the round trip
// removed (the photo minus its down-and-up resample, zero inside the hole) is gathered for each hole patch from the known
// patches with the softmax weights the forward's contextual attention computed, and the paste adds it to the upsampled result.
//
// Geometry (exact integers; DESIGN.md section 7b): box bw x bh, patch grid ws x hs = (Wn/8 - 1) x (Hn/8 - 1), patch (py, px)
// covers working pixels [8py, 8py + 16) x [8px, 8px + 16).
//   u(x)   = ((2x + 1) Wn) / (2 bw)                  working column of box column x's centre; v(y) likewise
//   ax(px) = min { x : u(x) >= 8 px }                box-column anchor of patch column px; ay likewise
//   R(x,y) = hole(u(x), v(y)) ? 0 : photo - low      low = resize(resize(photo, (Wn, Hn)), (bw, bh)), Pillow bicubic
//   A(x,y) = (1/nq) sum_{q covering (u, v)} sum_k P[k,q] R(min(ax(k) + x - ax(q), bw - 1), min(ay(k) + y - ay(q), bh - 1))
//   D(x,y) = hole(u(x), v(y)) ? round_half_away(A) : 0          (int16, per RGB channel)
//
// Per box three launches and one GEMM: the inner sum is a GEMM over the keys, C[q][(dy, dx, c)] = sum_k P[k,q] Rp[k][(dy, dx, c)]
// with Rp[k][(dy, dx, c)] = R(min(ay(k) + dy, bh - 1), min(ax(k) + dx, bw - 1), c) over the footprint 0 <= dx < fw,
// 0 <= dy < fh (fw = ceil(16 bw / Wn) + 2 holds x - ax(q) for every pixel of patch q). It runs on se_gemm_split.cu's split-half
// fp16 wgmma GEMM: P as hi + lo (about 22 bits), R exact in fp16 (integers of magnitude <= 255, lo = 0).
#include <cuda_fp16.h>
#include <stdint.h>

#include <algorithm>
#include <string>

#include "../../include/sketchedit_b200.h"
#include "se_detail.h"
#include "se_gemm_split.h"

namespace se {

constexpr float kDetailScaleP = 16384.0f;   // P <= 1 stored times 2^14 (fp16 range); the GEMM's scale undoes it exactly

struct DetailBox {
  int bh, bw, Hn, Wn, hs, ws, L;
  int Mp;       // L rounded up to 256: queries (M) and keys (K) of the GEMM
  int fw, fh;   // footprint
  int N, Np;    // fw * fh * 3, rounded up to 256
};

static DetailBox detail_box(int bh, int bw, int Hn, int Wn) {
  DetailBox d;
  d.bh = bh; d.bw = bw; d.Hn = Hn; d.Wn = Wn;
  d.hs = Hn / 8 - 1; d.ws = Wn / 8 - 1; d.L = d.hs * d.ws;
  d.Mp = (d.L + 255) / 256 * 256;
  d.fw = (int)((16LL * bw + Wn - 1) / Wn) + 2;
  d.fh = (int)((16LL * bh + Hn - 1) / Hn) + 2;
  d.N = d.fw * d.fh * 3;
  d.Np = (d.N + 255) / 256 * 256;
  return d;
}

// scratch of one box: the P operand, the residual operand, the GEMM's output
static size_t detail_a_bytes(const DetailBox& d) { return scratch_round((size_t)2 * d.Mp * d.Mp * 2); }
static size_t detail_b_bytes(const DetailBox& d) { return scratch_round((size_t)2 * d.Np * d.Mp * 2); }
static size_t detail_scratch(const DetailBox& d) { return detail_a_bytes(d) + detail_b_bytes(d) + scratch_round((size_t)d.Mp * d.Np * 4); }

__device__ __forceinline__ int work_of(int x, int b, int n) { return (int)(((2LL * x + 1) * n) / (2LL * b)); }
// min { x >= 0 : work_of(x, b, n) >= 8 p }: (2x + 1) n >= 16 p b
__device__ __forceinline__ int anchor(int p, int b, int n) {
  const long long num = 16LL * p * b - n;
  return num <= 0 ? 0 : (int)((num + 2LL * n - 1) / (2LL * n));
}

__global__ void detail_hole_kernel(const float* __restrict__ mbin, unsigned char* __restrict__ hole, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) hole[i] = mbin[i] > 0.5f ? 1 : 0;
}

// A (K-blocked, K-major): fp16 [hi | lo][Mp / 8][Mp][8], element (row q, column k) = P[k][q] * kDetailScaleP
__global__ void detail_pack_p_kernel(const float* __restrict__ attn, uint4* __restrict__ A, int L, int Mp) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)Mp / 8 * Mp) return;
  const int q = (int)(i % Mp), kb = (int)(i / Mp);
  uint32_t hi[4], lo[4];
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    const int k = kb * 8 + j;
    const float p0 = k < L && q < L ? __ldg(attn + (size_t)k * L + q) : 0.0f;
    const float p1 = k + 1 < L && q < L ? __ldg(attn + (size_t)(k + 1) * L + q) : 0.0f;
    __half h0, l0, h1, l1;
    split_half(p0, kDetailScaleP, h0, l0);
    split_half(p1, kDetailScaleP, h1, l1);
    hi[j >> 1] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
    lo[j >> 1] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
  }
  A[(size_t)kb * Mp + q] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  A[((size_t)Mp / 8 + kb) * Mp + q] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// Rp (MN-major): fp16 [hi | lo][Np / 8][Mp][8], element (row k, column n = (dy fw + dx) 3 + c); lo = 0 (R is exact in fp16)
__global__ void detail_pack_r_kernel(const unsigned char* __restrict__ photo, long long pitch, const unsigned char* __restrict__ low,
                                     const unsigned char* __restrict__ hole, const DetailBox d, uint4* __restrict__ Rp) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)d.Np / 8 * d.Mp) return;
  const int k = (int)(i % d.Mp), nb = (int)(i / d.Mp);
  uint32_t hi[4] = {0, 0, 0, 0};
  if (k < d.L) {
    const int ax = anchor(k % d.ws, d.bw, d.Wn), ay = anchor(k / d.ws, d.bh, d.Hn);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = nb * 8 + j;
      int r = 0;
      if (n < d.N) {
        const int c = n % 3, t = n / 3;
        const int sx = min(ax + t % d.fw, d.bw - 1), sy = min(ay + t / d.fw, d.bh - 1);
        if (!hole[(size_t)work_of(sy, d.bh, d.Hn) * d.Wn + work_of(sx, d.bw, d.Wn)])
          r = (int)photo[sy * pitch + sx * 3 + c] - (int)low[((size_t)sy * d.bw + sx) * 3 + c];
      }
      hi[j >> 1] |= (uint32_t)__half_as_ushort(__int2half_rn(r)) << (16 * (j & 1));
    }
  }
  Rp[(size_t)nb * d.Mp + k] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
  Rp[((size_t)d.Np / 8 + nb) * d.Mp + k] = make_uint4(0, 0, 0, 0);
}

// D and (optional) A per box pixel from the GEMM's C [Mp][Np]: the up to 4 patches covering the pixel, in (py, px) order
__global__ void detail_fold_kernel(const float* __restrict__ C, const unsigned char* __restrict__ hole, const DetailBox d, short* __restrict__ D,
                                   float* __restrict__ agg) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)d.bh * d.bw) return;
  const int y = (int)(i / d.bw), x = (int)(i % d.bw);
  const int u = work_of(x, d.bw, d.Wn), v = work_of(y, d.bh, d.Hn);
  float a[3] = {0.0f, 0.0f, 0.0f};
  const bool in = hole[(size_t)v * d.Wn + u] != 0;
  if (in) {
    int nq = 0;
    for (int py = v / 8 - 1; py <= v / 8; ++py) {
      if (py < 0 || py >= d.hs) continue;
      const int ay = anchor(py, d.bh, d.Hn);
      for (int px = u / 8 - 1; px <= u / 8; ++px) {
        if (px < 0 || px >= d.ws) continue;
        const float* row = C + (size_t)(py * d.ws + px) * d.Np + ((size_t)(y - ay) * d.fw + (x - anchor(px, d.bw, d.Wn))) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) a[c] += row[c];
        ++nq;
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) a[c] /= (float)nq;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    D[i * 3 + c] = in ? (short)roundf(a[c]) : (short)0;   // roundf: half away from zero; |A| <= 255
    if (agg) agg[i * 3 + c] = a[c];
  }
}

int detail_hole_u8(const float* mbin, unsigned char* hole, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  detail_hole_kernel<<<grid_of(n, 256), 256, 0, stream>>>(mbin, hole, n);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

static int detail_one(const unsigned char* photo, long long pitch, const unsigned char* low, const unsigned char* hole, const float* attn,
                      const DetailBox& d, short* D, float* agg, void* scratch, cudaStream_t st) {
  void* A = scratch;
  void* Rp = (char*)scratch + detail_a_bytes(d);
  float* C = (float*)((char*)Rp + detail_b_bytes(d));
  {
    const long long n = (long long)d.Mp / 8 * d.Mp;
    detail_pack_p_kernel<<<grid_of(n, 256), 256, 0, st>>>(attn, (uint4*)A, d.L, d.Mp);
    SE_CUDA_OK(cudaGetLastError());
  }
  {
    const long long n = (long long)d.Np / 8 * d.Mp;
    detail_pack_r_kernel<<<grid_of(n, 256), 256, 0, st>>>(photo, pitch, low, hole, d, (uint4*)Rp);
    SE_CUDA_OK(cudaGetLastError());
  }
  int rc = gemm_split_mn(A, Rp, C, d.Mp, d.Mp, d.Np, 1.0f / kDetailScaleP, st);
  if (rc) return rc;
  const long long n = (long long)d.bh * d.bw;
  detail_fold_kernel<<<grid_of(n, 256), 256, 0, st>>>(C, hole, d, D, agg);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

using namespace se;

extern "C" {

int se_detail_u8(const unsigned char* const* photo, const long long* photo_pitch, const int* box_hw, int n, int Hn, int Wn,
                 const unsigned char* low, const long long* low_off, const unsigned char* hole, const long long* hole_off, const float* attn,
                 const long long* attn_off, short* D, const long long* d_off, float* agg, const long long* agg_off, void* scratch,
                 long long* scratch_bytes, void* stream) {
  SE_REQUIRE(n >= 0, "n must be >= 0 boxes");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(Hn % 8 == 0 && Wn % 8 == 0 && Hn >= 16 && Wn >= 16, "the working size must be multiples of 8 and >= 16");
  SE_REQUIRE(n == 0 || (photo_pitch && box_hw && low_off && hole_off && attn_off && d_off), "null size / offset array");
  SE_REQUIRE(!agg || agg_off, "agg needs agg_off");
  size_t need = 0;
  for (int i = 0; i < n; ++i) {
    const int bh = box_hw[2 * i], bw = box_hw[2 * i + 1];
    if (int rc = check_sides("box", i, bh, bw)) return rc;
    SE_REQUIRE(photo_pitch[i] >= 3LL * bw, "box " + std::to_string(i) + ": the photo pitch is narrower than the box's row");
    // every patch position needs a box-pixel anchor: u(bw - 1) >= Wn - 16 (bw >= Wn / 32), likewise rows
    SE_REQUIRE((2LL * bw - 1) * Wn / (2LL * bw) >= Wn - 16 && (2LL * bh - 1) * Hn / (2LL * bh) >= Hn - 16,
               "box " + std::to_string(i) + ": " + std::to_string(bh) + " x " + std::to_string(bw) +
                   " is below 1/32 of the working size on a side: some patches have no anchor in it");
    SE_REQUIRE(low_off[i] >= 0 && hole_off[i] >= 0 && attn_off[i] >= 0 && attn_off[i] % 4 == 0 && d_off[i] >= 0 && d_off[i] % 2 == 0 &&
                   (!agg || (agg_off[i] >= 0 && agg_off[i] % 4 == 0)),
               "box " + std::to_string(i) + ": offsets must be >= 0 and aligned to their element size");
    need = std::max(need, detail_scratch(detail_box(bh, bw, Hn, Wn)));
  }
  SE_REQUIRE(((uintptr_t)scratch & 255) == 0, "scratch must be 256 B aligned");
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(photo && low && hole && attn && D, "null photo / low / hole / attn / D");
  for (int i = 0; i < n; ++i) {   // in order on one stream: every box reuses the scratch
    SE_REQUIRE(photo[i] != nullptr, "null photo window");
    const DetailBox d = detail_box(box_hw[2 * i], box_hw[2 * i + 1], Hn, Wn);
    int rc = detail_one(photo[i], photo_pitch[i], low + low_off[i], hole + hole_off[i], (const float*)((const char*)attn + attn_off[i]), d,
                        (short*)((char*)D + d_off[i]), agg ? (float*)((char*)agg + agg_off[i]) : nullptr, scratch, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return 0;
}

}  // extern "C"

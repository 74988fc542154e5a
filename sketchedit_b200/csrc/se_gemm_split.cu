// Contextual attention of the fp32-on-tensor-cores mode (SE_PREC_FP32_TC): the two attention GEMMs as split-half fp16
// wgmma GEMMs (three products per K step: hi*hi + hi*lo + lo*hi, fp32 accumulation in registers: ~22 significant bits), with the
// same semantics as the CUDA-core path in se_engine.cu run_cam (reference models/networks/splitcam.py:37-108,132-174 with
// netG's configuration, editline_g.py:35-42: 4x4 patches at stride 2, keys normalised per (image, channel) plane, logits x10,
// masked keys -> logit 0, softmax over the keys, paste = fold-SUM of the weighted raw patches):
//
//   pack     Q[n][(u,v,c)] = f[2ny+u, 2nx+v, c]          K[l][(u,v,c)] = Q[l][(u,v,c)] * rnorm[c]
//   S GEMM   S[n][l] = 10 * m_l * sum_k Q[n][k] K[l][k]                      (A = Q, B = K, both K-major)
//   softmax  P[n][l] = softmax_l S[n][l]                                      (fp32; padding keys excluded)
//   PV GEMM  O[n][(u,v,c)] = sum_l P[n][l] Q[l][(u,v,c)]                      (A = P K-major, B = Q MN-major: the SAME buffer)
//   fold     out[y, x, c] = sum over (n, u, v) with 2ny+u = y, 2nx+v = x of O[n][(u,v,c)]
//
// Operand layout ("K-blocked", the channel-blocked layout of se_conv_c8.cu with GEMM rows as pixels): fp16
// [image][hi | lo][K / 8][rows][8]. A TMA box {8, rows, 4 K-blocks} lands in shared memory as the canonical no-swizzle
// K-major wgmma layout (core matrix = 8 rows x 16 B contiguous; SBO = 128 B, LBO = rows x 16 B); read along its rows instead
// ({8, 32 rows, 32 blocks}) the same buffer is an MN-major operand (LBO = 128 B = next 8 K, SBO = 512 B = next 8 N).
// Values are stored times a power of two per operand (fp16 exponent range, see se_common.cuh kSplitActScale); the epilogue
// undoes it exactly.
//
// Bands: S and P are Mp x Mp per image, so large maps run S GEMM -> softmax -> PV GEMM per band of query rows [n0, n0 + band)
// (M rows of both GEMMs) through band-sized S and P buffers; O stays whole and is folded once. Each row's arithmetic does not
// depend on the band split.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "se_gemm_split.h"
#include "se_tc_device.cuh"

namespace se {

constexpr int GS_BM = 128, GS_BN = 256, GS_BK = 32;           // CTA tile; K per pipeline stage
constexpr int GS_A_BYTES = GS_BM * GS_BK * 2;                 // 8 KB  (one half: hi or lo)
constexpr int GS_B_BYTES = GS_BN * GS_BK * 2;                 // 16 KB
constexpr int GS_STAGE = 2 * GS_A_BYTES + 2 * GS_B_BYTES;     // 48 KB: A_hi | A_lo | B_hi | B_lo
constexpr int GS_STAGES = 4;
constexpr int GS_THREADS = 288;                               // warps 0-7: two consumer warpgroups (rows 0-63 / 64-127), warp 8: TMA producer
constexpr int GS_SMEM = 1024 + GS_STAGES * GS_STAGE;

constexpr float kScaleQ = kSplitActScale;       // raw feature patches (queries / values)
constexpr float kScaleK = 32768.0f;             // normalised keys: |k| <= 1
constexpr float kScaleP = 16384.0f;             // probabilities: p <= 1

struct GemmSplitParams {
  int K;                       // multiple of GS_BK
  int a_row0;                  // first A row (M tile 0 starts here)
  float* C;                    // fp32 [image][Mp][ldc]
  long long c_img_stride;
  int ldc;
  float scale;                 // accumulator -> value (includes 1 / (operand scales))
  const float* colscale;       // optional [image][ncs]: multiplies column n (0 beyond ncs)
  int ncs;
};

// ------------------------------------------------------------------------------------------ pack: Q and K patch matrices
// f: fp32 NHWC [B][h][w][C] (C = 8 * CB). Q, Kn: fp16 [B][2][16 * CB][Mp][8]. One thread = one (patch n, tap, channel block).
__global__ void cam_split_pack_kernel(const float* __restrict__ f, const float* __restrict__ rnorm, uint4* __restrict__ Q, uint4* __restrict__ Kn,
                                      int h, int w, int CB, int ws, int L, int Mp, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int n = (int)(i % Mp);
  long long r = i / Mp;
  const int kb = (int)(r % (16 * CB));
  const long long b = r / (16 * CB);
  const int tap = kb / CB, cb = kb % CB;
  uint32_t qh[4] = {0, 0, 0, 0}, ql[4] = {0, 0, 0, 0}, kh[4] = {0, 0, 0, 0}, kl[4] = {0, 0, 0, 0};
  if (n < L) {
    const int ny = n / ws, nx = n % ws, u = tap >> 2, v = tap & 3;
    const float4* src = reinterpret_cast<const float4*>(f + (((size_t)b * h + 2 * ny + u) * w + 2 * nx + v) * (CB * 8) + cb * 8);
    const float4* rn = reinterpret_cast<const float4*>(rnorm + (size_t)b * CB * 8 + cb * 8);
    const float4 a0 = src[0], a1 = src[1], r0 = rn[0], r1 = rn[1];
    const float x[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    const float rr[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
    for (int k = 0; k < 8; k += 2) {
      __half h0, l0, h1, l1;
      split_half(x[k], kScaleQ, h0, l0);
      split_half(x[k + 1], kScaleQ, h1, l1);
      qh[k >> 1] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
      ql[k >> 1] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
      split_half(x[k] * rr[k], kScaleK, h0, l0);
      split_half(x[k + 1] * rr[k + 1], kScaleK, h1, l1);
      kh[k >> 1] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
      kl[k >> 1] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
  }
  const size_t KB = (size_t)16 * CB;
  const size_t oh = ((size_t)(b * 2) * KB + kb) * Mp + n, ol = ((size_t)(b * 2 + 1) * KB + kb) * Mp + n;
  Q[oh] = make_uint4(qh[0], qh[1], qh[2], qh[3]);
  Q[ol] = make_uint4(ql[0], ql[1], ql[2], ql[3]);
  Kn[oh] = make_uint4(kh[0], kh[1], kh[2], kh[3]);
  Kn[ol] = make_uint4(kl[0], kl[1], kl[2], kl[3]);
}

// ------------------------------------------------------------------------------------------ the GEMM
// C[img][m][n] = scale * colscale[img][n] * sum_k (A_hi B_hi + A_hi B_lo + A_lo B_hi)[m][n];   grid (N tiles, M tiles, images)
template <bool kBMN>
__global__ void __launch_bounds__(GS_THREADS, 1)
gemm_split_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmSplitParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* const smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t full_bar[GS_STAGES], empty_bar[GS_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, mt = blockIdx.y, img = blockIdx.z;
  const int ksteps = p.K / GS_BK;

  if (threadIdx.x == 0) {
    for (int i = 0; i < GS_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }   // one arrival per consumer warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ==================================================================== TMA producer
    if (elect_one()) {
      for (int ks = 0; ks < ksteps; ++ks) {
        const int s = ks % GS_STAGES;
        const uint32_t ph = (uint32_t)(ks / GS_STAGES) & 1u;
        mbar_wait(&empty_bar[s], ph ^ 1u, 1);
        mbar_expect_tx(&full_bar[s], GS_STAGE);
        uint8_t* st = smem + (size_t)s * GS_STAGE;
        tma_load_4d(st, &tmA, &full_bar[s], 0, p.a_row0 + mt * GS_BM, ks * (GS_BK / 8), img * 2);
        tma_load_4d(st + GS_A_BYTES, &tmA, &full_bar[s], 0, p.a_row0 + mt * GS_BM, ks * (GS_BK / 8), img * 2 + 1);
        if (kBMN) {   // rows of the buffer are the K dimension here: box {8, 32 K rows, 32 N blocks}
          tma_load_4d(st + 2 * GS_A_BYTES, &tmB, &full_bar[s], 0, ks * GS_BK, nt * (GS_BN / 8), img * 2);
          tma_load_4d(st + 2 * GS_A_BYTES + GS_B_BYTES, &tmB, &full_bar[s], 0, ks * GS_BK, nt * (GS_BN / 8), img * 2 + 1);
        } else {
          tma_load_4d(st + 2 * GS_A_BYTES, &tmB, &full_bar[s], 0, nt * GS_BN, ks * (GS_BK / 8), img * 2);
          tma_load_4d(st + 2 * GS_A_BYTES + GS_B_BYTES, &tmB, &full_bar[s], 0, nt * GS_BN, ks * (GS_BK / 8), img * 2 + 1);
        }
      }
    }
  } else {
    // ==================================================================== consumers: M = 64 rows each, N = 256, fp16 x fp16 -> fp32
    const int wg = warp >> 2, wq = warp & 3;
    // A, K-major no-swizzle: LBO = next K block (128 rows x 16 B), SBO = next 8 rows; this warpgroup's rows start 64 rows in
    // B, K-major: LBO = 256 rows x 16 B, SBO = 128 B.  MN-major: LBO = next 8 K rows (128 B), SBO = next N block (32 rows x 16 B)
    const uint32_t a_lbo = GS_BM * 16, a_sbo = 128, a_m = (uint32_t)wg * 64u * 16u;
    const uint32_t b_lbo = kBMN ? 128u : (uint32_t)GS_BN * 16u, b_sbo = kBMN ? (uint32_t)GS_BK * 16u : 128u;
    const uint32_t a_k16 = 2u * GS_BM * 16;                         // two K blocks further
    const uint32_t b_k16 = kBMN ? 256u : 2u * GS_BN * 16;
    const uint32_t base = smem_u32(smem);
    float acc[GS_BN / 2];
#pragma unroll
    for (int i = 0; i < GS_BN / 2; ++i) acc[i] = 0.0f;
    int prev = -1;
    for (int ks = 0; ks < ksteps; ++ks) {
      const int s = ks % GS_STAGES;
      const uint32_t ph = (uint32_t)(ks / GS_STAGES) & 1u;
      mbar_wait(&full_bar[s], ph, 2);
      const uint32_t st = base + (uint32_t)s * GS_STAGE;
      const uint32_t aH = st + a_m, aL = st + GS_A_BYTES + a_m, bH = st + 2 * GS_A_BYTES, bL = st + 2 * GS_A_BYTES + GS_B_BYTES;
      wg_fence();
      wg_fence_acc(acc);
#pragma unroll
      for (int k = 0; k < GS_BK / 16; ++k) {
        const uint64_t dAH = wg_desc(aH + k * a_k16, a_lbo, a_sbo, WG_SW_NONE), dAL = wg_desc(aL + k * a_k16, a_lbo, a_sbo, WG_SW_NONE);
        const uint64_t dBH = wg_desc(bH + k * b_k16, b_lbo, b_sbo, WG_SW_NONE), dBL = wg_desc(bL + k * b_k16, b_lbo, b_sbo, WG_SW_NONE);
        Wgmma<GS_BN, true, kBMN ? 1 : 0>::mma(acc, dAH, dBH, (ks | k) ? 1u : 0u);
        Wgmma<GS_BN, true, kBMN ? 1 : 0>::mma(acc, dAH, dBL, 1u);
        Wgmma<GS_BN, true, kBMN ? 1 : 0>::mma(acc, dAL, dBH, 1u);
      }
      wg_commit();
      if (prev >= 0) {
        wg_wait<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
    }
    wg_wait<0>();
    wg_fence_acc(acc);
    // epilogue straight from the fragment: row 64 wg + 16 wq + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
    const float* cs = p.colscale ? p.colscale + (size_t)img * p.ncs : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float* crow = p.C + (size_t)img * p.c_img_stride + (size_t)(mt * GS_BM + 64 * wg + frag_row(wq, lane, h)) * p.ldc + nt * GS_BN;
#pragma unroll
      for (int j = 0; j < GS_BN / 8; ++j) {
        const int c = frag_col(lane, j), n0 = nt * GS_BN + c;
        float v0 = acc[4 * j + 2 * h] * p.scale, v1 = acc[4 * j + 2 * h + 1] * p.scale;
        if (cs) {
          v0 *= n0 < p.ncs ? __ldg(cs + n0) : 0.0f;
          v1 *= n0 + 1 < p.ncs ? __ldg(cs + n0 + 1) : 0.0f;
        }
        *reinterpret_cast<float2*>(crow + c) = make_float2(v0, v1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ softmax -> P (split-half, K-blocked)
// S: fp32 [B][rows][Np] (query rows n_base + r); P: fp16 [B][2][Np / 8][rows][8] (times kScaleP). Rows of any length, read
// from global memory. Block = 8 rows (one warp each computes its row's statistics); query rows >= L and keys >= L are 0.
// attn (optional): the fp32 weights before the split, [B][L keys][L queries] (the layout of cam_1's return value).
__global__ void __launch_bounds__(256) cam_split_softmax_kernel(const float* __restrict__ S, uint4* __restrict__ P, int L, int rows, int n_base, int Np,
                                                                float* __restrict__ attn) {
  __shared__ float s_inv[8], s_max[8];
  const int b = blockIdx.y, r0 = blockIdx.x * 8, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* src = S + ((size_t)b * rows + r0) * Np;
  {
    const float* row = src + (size_t)warp * Np;
    float mx = -INFINITY;
    for (int l = lane; l < L; l += 32) mx = fmaxf(mx, row[l]);
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.0f;
    for (int l = lane; l < L; l += 32) sum += expf(row[l] - mx);
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) { s_max[warp] = mx; s_inv[warp] = 1.0f / sum; }
  }
  __syncthreads();
  const size_t LB = (size_t)Np / 8;
  for (int i = threadIdx.x; i < (int)LB * 8; i += 256) {
    const int lb = i >> 3, r = i & 7;
    const int n = n_base + r0 + r;
    uint32_t hi[4] = {0, 0, 0, 0}, lo[4] = {0, 0, 0, 0};
    if (n < L) {
      const float4* row4 = reinterpret_cast<const float4*>(src + (size_t)r * Np + lb * 8);   // Np % 256 == 0: 32 B aligned
      const float4 a0 = row4[0], a1 = row4[1];
      const float row[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float mx = s_max[r], inv = s_inv[r];
#pragma unroll
      for (int k = 0; k < 8; k += 2) {
        const float p0 = (lb * 8 + k < L) ? expf(row[k] - mx) * inv : 0.0f;
        const float p1 = (lb * 8 + k + 1 < L) ? expf(row[k + 1] - mx) * inv : 0.0f;
        if (attn) {
          if (lb * 8 + k < L) attn[((size_t)b * L + lb * 8 + k) * L + n] = p0;
          if (lb * 8 + k + 1 < L) attn[((size_t)b * L + lb * 8 + k + 1) * L + n] = p1;
        }
        __half h0, l0, h1, l1;
        split_half(p0, kScaleP, h0, l0);
        split_half(p1, kScaleP, h1, l1);
        hi[k >> 1] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        lo[k >> 1] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
      }
    }
    P[((size_t)(b * 2) * LB + lb) * rows + r0 + r] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    P[((size_t)(b * 2 + 1) * LB + lb) * rows + r0 + r] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// ------------------------------------------------------------------------------------------ fold-sum
// O: fp32 [B][Mp][16 * C] (column (u*4+v)*C + c); out: fp32 NHWC [B][h][w][C]. Fixed summation order (u, v ascending).
__global__ void cam_split_fold_kernel(const float* __restrict__ O, float* __restrict__ out, int h, int w, int C, int hs, int ws, int Mp, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % (C / 4));
  long long r = i / (C / 4);
  const int x = (int)(r % w); r /= w;
  const int y = (int)(r % h);
  const long long b = r / h;
  float4 acc = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  for (int u = y & 1; u < 4; u += 2) {
    const int ny = (y - u) >> 1;
    if (y - u < 0 || ny >= hs) continue;
    for (int v = x & 1; v < 4; v += 2) {
      const int nx = (x - v) >> 1;
      if (x - v < 0 || nx >= ws) continue;
      const float4 t = *reinterpret_cast<const float4*>(O + ((size_t)b * Mp + (size_t)ny * ws + nx) * (16 * C) + (u * 4 + v) * C + c4 * 4);
      acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
  }
  *reinterpret_cast<float4*>(out + i * 4) = acc;
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn gs_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
// fp16 [images2 = 2 * B][blocks][rows][8] viewed as (8, rows, blocks, images2); box (8, box_rows, box_blocks, 1)
static int gs_map(CUtensorMap* tm, const void* base, int rows, int blocks, int images2, int box_rows, int box_blocks) {
  EncodeTiledFn enc = gs_encode_fn();
  SE_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[4] = {8, (cuuint64_t)rows, (cuuint64_t)blocks, (cuuint64_t)images2};
  cuuint64_t strides[3] = {16, (cuuint64_t)rows * 16, (cuuint64_t)blocks * rows * 16};
  cuuint32_t box[4] = {8, (cuuint32_t)box_rows, (cuuint32_t)box_blocks, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SE_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(split GEMM) failed, CUresult=" + std::to_string((int)r));
  return 0;
}

int cam_split_plan(int B, int h, int w, int C, long long limit, CamSplitPlan* out) {
  SE_REQUIRE(h % 2 == 0 && w % 2 == 0 && h >= 4 && w >= 4 && C % 8 == 0, "attention map must be even-sized, >= 4, channels a multiple of 8");
  CamSplitPlan p;
  p.B = B; p.h = h; p.w = w; p.C = C;
  p.hs = (h - 4) / 2 + 1; p.ws = (w - 4) / 2 + 1; p.L = p.hs * p.ws;
  p.Mp = (p.L + GS_BN - 1) / GS_BN * GS_BN;        // patches padded to the N tile (they are rows of A and of both B operands)
  p.KQ = 16 * C;
  SE_REQUIRE(p.KQ % GS_BN == 0, "16 * channels must be a multiple of 256");   // N of the PV GEMM
  p.q_bytes = (size_t)B * 2 * (p.KQ / 8) * p.Mp * 16;
  // the tallest band (a multiple of the 128-row M tile) whose S and P fit the limit
  const size_t row_bytes = (size_t)B * p.Mp * (4 + 4);   // one query row: S fp32 + P as fp16 hi and lo
  p.band = p.Mp;
  if (row_bytes * p.Mp > (size_t)limit) {
    p.band = (int)((size_t)limit / row_bytes / GS_BM * GS_BM);
    SE_REQUIRE(p.band >= GS_BM, "attention workspace limit of " + std::to_string(limit) + " bytes is below the " +
                                     std::to_string(row_bytes * GS_BM) + " bytes one band of " + std::to_string(GS_BM) +
                                     " query rows needs at this size and batch");
  }
  p.n_bands = (p.Mp + p.band - 1) / p.band;
  p.s_bytes = (size_t)B * p.band * p.Mp * 4;
  p.p_bytes = (size_t)B * 2 * (p.Mp / 8) * p.band * 16;
  p.o_bytes = (size_t)B * p.Mp * p.KQ * 4;
  *out = p;
  return 0;
}

static int gs_launch(bool bmn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmSplitParams& p, int n_tiles, int m_tiles, int B, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    SE_CUDA_OK(cudaFuncSetAttribute(gemm_split_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GS_SMEM));
    SE_CUDA_OK(cudaFuncSetAttribute(gemm_split_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GS_SMEM));
    attr_done = true;
  }
  SE_REQUIRE(p.K % GS_BK == 0 && p.ldc % 4 == 0, "split GEMM shape");
  dim3 grid(n_tiles, m_tiles, B);
  if (bmn) gemm_split_kernel<true><<<grid, GS_THREADS, GS_SMEM, stream>>>(tmA, tmB, p);
  else gemm_split_kernel<false><<<grid, GS_THREADS, GS_SMEM, stream>>>(tmA, tmB, p);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

int cam_forward_split(const float* f, const float* rnorm, const float* colmask, float* out, const CamSplitPlan& pl, void* Q, void* Kn, float* S, void* P,
                      float* O, float* attn, cudaStream_t stream) {
  const int B = pl.B, C = pl.C, CB = C / 8, L = pl.L, Mp = pl.Mp;
  SE_REQUIRE(((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(Kn) | reinterpret_cast<uintptr_t>(P)) & 127) == 0 &&
                 ((reinterpret_cast<uintptr_t>(S) | reinterpret_cast<uintptr_t>(O) | reinterpret_cast<uintptr_t>(f) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             "attention buffers must be 128 B aligned");
  {
    const long long total = (long long)B * 16 * CB * Mp;
    cam_split_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(f, rnorm, (uint4*)Q, (uint4*)Kn, pl.h, pl.w, CB, pl.ws, L, Mp, total);
    SE_CUDA_OK(cudaGetLastError());
  }
  CUtensorMap tmQ, tmK, tmV;
  int rc = gs_map(&tmQ, Q, Mp, pl.KQ / 8, 2 * B, GS_BM, GS_BK / 8);
  if (rc) return rc;
  rc = gs_map(&tmK, Kn, Mp, pl.KQ / 8, 2 * B, GS_BN, GS_BK / 8);
  if (rc) return rc;
  rc = gs_map(&tmV, Q, Mp, pl.KQ / 8, 2 * B, GS_BK, GS_BN / 8);
  if (rc) return rc;
  for (int n0 = 0; n0 < Mp; n0 += pl.band) {
    const int rows = n0 + pl.band < Mp ? pl.band : Mp - n0;   // a multiple of GS_BM (Mp is one of GS_BN)
    {   // S[n0 + r] = 10 * m_l * Q K^T
      GemmSplitParams p;
      p.K = pl.KQ; p.a_row0 = n0; p.C = S; p.c_img_stride = (long long)rows * Mp; p.ldc = Mp;
      p.scale = 10.0f / (kScaleQ * kScaleK); p.colscale = colmask; p.ncs = L;
      rc = gs_launch(false, tmQ, tmK, p, Mp / GS_BN, rows / GS_BM, B, stream);
      if (rc) return rc;
    }
    cam_split_softmax_kernel<<<dim3(rows / 8, B), 256, 0, stream>>>(S, (uint4*)P, L, rows, n0, Mp, attn);
    SE_CUDA_OK(cudaGetLastError());
    {   // O[n0 + r] = P Q  (B operand = the query patches again, read MN-major)
      CUtensorMap tmP;
      rc = gs_map(&tmP, P, rows, Mp / 8, 2 * B, GS_BM, GS_BK / 8);
      if (rc) return rc;
      GemmSplitParams p;
      p.K = Mp; p.a_row0 = 0; p.C = O + (size_t)n0 * pl.KQ; p.c_img_stride = (long long)Mp * pl.KQ; p.ldc = pl.KQ;
      p.scale = 1.0f / (kScaleP * kScaleQ); p.colscale = nullptr; p.ncs = 0;
      rc = gs_launch(true, tmP, tmV, p, pl.KQ / GS_BN, rows / GS_BM, B, stream);
      if (rc) return rc;
    }
  }
  {
    const long long total = (long long)B * pl.h * pl.w * (C / 4);
    cam_split_fold_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(O, out, pl.h, pl.w, C, pl.hs, pl.ws, Mp, total);
    SE_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

int gemm_split_mn(const void* A, const void* B, float* C, int M, int K, int N, float scale, cudaStream_t stream) {
  SE_REQUIRE(M % GS_BM == 0 && K % GS_BK == 0 && N % GS_BN == 0 && M > 0 && K > 0 && N > 0, "split GEMM: M, K, N multiples of 128, 32, 256");
  SE_REQUIRE(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 127) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0,
             "split GEMM operands must be 128 B aligned");
  CUtensorMap tmA, tmB;
  int rc = gs_map(&tmA, A, M, K / 8, 2, GS_BM, GS_BK / 8);
  if (rc) return rc;
  rc = gs_map(&tmB, B, K, N / 8, 2, GS_BK, GS_BN / 8);
  if (rc) return rc;
  GemmSplitParams p;
  p.K = K; p.a_row0 = 0; p.C = C; p.c_img_stride = (long long)M * N; p.ldc = N;
  p.scale = scale; p.colscale = nullptr; p.ncs = 0;
  return gs_launch(true, tmA, tmB, p, N / GS_BN, M / GS_BM, 1, stream);
}

}  // namespace se

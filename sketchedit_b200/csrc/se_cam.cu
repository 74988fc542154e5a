// Contextual attention (reference models/networks/splitcam.py:37-108,132-174 with netG's configuration, editline_g.py:35-42:
// 4x4 patches at stride 2, keys normalised per (image, channel) plane, logits x10, masked keys -> logit 0, soft attention,
// paste = fold-SUM of the weighted raw patches) with wgmma on the tensor cores of sm_90a, in three steps:
//
//   prep   rnorm[c] = 1 / sqrt(sum_plane f^2 + 1e-8);  fn = f * rnorm  (same layout as f);  per-key logit scale
//   S      P[n, l]  = softmax_l(10 * m_l * <Q_n, K_l>)        cam_s_kernel   (QK^T twice: statistics sweep + output sweep)
//   PV     out[2y+py, 2x+px, c] = sum_{a,b} sum_l P[(y-a, x-b), l] * f[2l + (py+2a, px+2b), c]          cam_pv_kernel
//
// Nothing is packed or unfolded: the feature map arrives SPACE-TO-DEPTH channel-blocked, [B][4 parities x 12 blocks][h/2][w/2][8]
// bf16 (written that way by pmconv6's epilogue). A 4x4 / stride-2 patch tap (u, v) of patch n is then pixel n + (u>>1, v>>1) of
// parity plane (u&1, v&1): a stride-1 window, so ONE TMA box (17 x 9 positions of the planes) holds all 16 taps of a tile of
// 16 x 8 patches, and eight horizontally adjacent patches x eight channels are one no-swizzle wgmma core matrix (the trick of
// se_conv_c8.cu). Queries (A), keys (B, K-major) and values (B, MN-major) are all such boxes; tap / channel selection is
// descriptor start-address arithmetic.
//
// Both GEMM kernels run 288 threads: two consumer warpgroups (wgmma, accumulators in registers, epilogue on the fragments) and a
// TMA producer warp.
//
// Probabilities are the only attention-sized tensor that touches HBM: bf16 P[B][key block][hs][ws][8] ("channel-blocked with
// keys as channels"), written once by the S kernel and read once (per output tile) by the PV kernel. The logits never
// leave the registers: the S kernel sweeps the key tiles twice per query tile - sweep 0 keeps the running row maximum and sum
// (fp32, per lane, combined over the row's quad of lanes at the end), sweep 1 recomputes the logits and writes
// exp(t - max) / sum. Key order inside P is the S kernel's tile order, which is also the order the PV kernel walks the keys.
//
// Bands: P is L x L per image, so large maps run in bands of query rows [q0, q1) (q0 a multiple of 16: the S tiles keep their
// alignment) through one band-sized P buffer. Output class row y reads query rows y - 1 and y, so band [q0, q1) writes class
// rows [q0, q1) (the last band also row hs) and needs query row q0 - 1 as well: it is carried over from the previous band
// (buffer row 0) by one strided copy instead of being recomputed. Every row's S and PV arithmetic is the same as in a single
// band, so the output does not depend on the band split.
#include "se_cam.h"

#include <stdlib.h>

#include <vector>

#include "se_tc_device.cuh"

namespace se {

constexpr int CAM_CB = 12;                 // channel blocks of the 96-channel map
constexpr int CAM_TH = 16, CAM_TW = 8;     // query tile: 128 positions = two wgmma M = 64 halves
constexpr int CAM_HR = CAM_TH + 1, CAM_WR = CAM_TW + 1;   // its window in a parity plane (taps reach +1 row / column)
constexpr int CAM_PLANE = CAM_HR * CAM_WR * 16;           // bytes of one channel block of a 17 x 9 window = LBO of the K-major operands
constexpr int CAM_ROW = CAM_WR * 16;                      // bytes of one window row = SBO
constexpr int CAM_Q_TX = 4 * CAM_CB * CAM_PLANE;          // query window, all four parities: 117,504 B
constexpr int CAM_Q_BYTES = (CAM_Q_TX + 1023) / 1024 * 1024;
constexpr int CAM_K_TX = CAM_CB * CAM_PLANE;              // key window of one parity (one 16 x 8 half of a 32 x 8 key tile)
constexpr int CAM_K_STAGE = (CAM_K_TX + 1023) / 1024 * 1024;
constexpr int CAM_S_STAGES = 3;
constexpr int CAM_KEYS = 256;              // keys per key tile (two 128-key accumulator tiles)
// PV: output tile = 8 x 8 positions (wgmma M = 64); a stage = 64 keys: P window (8 key blocks x 9 x 9) + value windows of
// all four parities (12 blocks x 9 x 9 each)
constexpr int CAM_PV_TH = 8;
constexpr int CAM_PPLANE = 9 * 9 * 16;                    // one key block of the 9 x 9 P window = LBO of the K-major A operand
constexpr int CAM_PW_TX = 8 * CAM_PPLANE;                 // 10,368 B
constexpr int CAM_VPLANE = 9 * 9 * 16;                    // one channel block of a 9 x 9 value window = SBO of the MN-major operand
constexpr int CAM_V_TX = CAM_CB * CAM_VPLANE;             // 15,552 B
constexpr int CAM_V_PITCH = (CAM_V_TX + 127) / 128 * 128;
__host__ __device__ constexpr int CAM_V_OFF(int par) { return CAM_PW_TX + par * CAM_V_PITCH; }   // 128 B aligned
constexpr int CAM_PV_STAGE = (CAM_V_OFF(4) + 1023) / 1024 * 1024;
constexpr int CAM_PV_STAGES = 3;
constexpr int CAM_CONSUMER_WARPS = 8;
constexpr int CAM_THREADS = 32 * CAM_CONSUMER_WARPS + 32;

// ------------------------------------------------------------------------------------------ prep kernels
// one block per (channel block, image): sum of squares over the four parity planes in a fixed order (deterministic: the
// attention must not depend on the batch an image is in), then fn = f * rnorm for the same planes
__global__ void __launch_bounds__(256) cam_norm_kernel(const __nv_bfloat16* __restrict__ f, __nv_bfloat16* __restrict__ fn, int plane_px) {
  __shared__ float red[8][8];
  __shared__ float rn[8];
  const int cb = blockIdx.x, b = blockIdx.y;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.0f;
  for (int par = 0; par < 4; ++par) {
    const uint4* src = reinterpret_cast<const uint4*>(f) + ((size_t)b * 48 + par * CAM_CB + cb) * plane_px;
    for (int px = threadIdx.x; px < plane_px; px += 256) {
      const uint4 q = src[px];
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&q);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 v = __bfloat1622float2(h2[i]);
        acc[2 * i] = fmaf(v.x, v.x, acc[2 * i]);
        acc[2 * i + 1] = fmaf(v.y, v.y, acc[2 * i + 1]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
    for (int o = 16; o; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
  if ((threadIdx.x & 31) == 0)
    for (int i = 0; i < 8; ++i) red[threadIdx.x >> 5][i] = acc[i];
  __syncthreads();
  if (threadIdx.x < 8) {
    float s = 0.0f;
    for (int j = 0; j < 8; ++j) s += red[j][threadIdx.x];
    rn[threadIdx.x] = 1.0f / sqrtf(s + 1e-8f);   // splitcam.py:40
  }
  __syncthreads();
  float r[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = rn[i];
  for (int par = 0; par < 4; ++par) {
    const size_t base = ((size_t)b * 48 + par * CAM_CB + cb) * plane_px;
    const uint4* src = reinterpret_cast<const uint4*>(f) + base;
    uint4* dst = reinterpret_cast<uint4*>(fn) + base;
    for (int px = threadIdx.x; px < plane_px; px += 256) {
      const uint4 q = src[px];
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&q);
      float2 v0 = __bfloat1622float2(h2[0]), v1 = __bfloat1622float2(h2[1]), v2 = __bfloat1622float2(h2[2]), v3 = __bfloat1622float2(h2[3]);
      dst[px] = make_uint4(pack_bf16x2(v0.x * r[0], v0.y * r[1]), pack_bf16x2(v1.x * r[2], v1.y * r[3]), pack_bf16x2(v2.x * r[4], v2.y * r[5]),
                           pack_bf16x2(v3.x * r[6], v3.y * r[7]));
    }
  }
}

// per key, in the S kernel's tile order: 10 * log2(e) * [mean over the 4x4 patch of (1 - mask_s) > 0.1]  (splitcam.py:49-53,89-90,
// 104-105: masked keys keep logit 0), -1 for the padding keys of a tile (they must not take part in the softmax at all)
__global__ void cam_colscale_kernel(const float* __restrict__ mask_s, float* __restrict__ cs, int B, int h, int w, int hs, int ws, int tk_x, int KT) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)B * KT * CAM_KEYS) return;
  const int c = (int)(i % CAM_KEYS);
  const int j = (int)((i / CAM_KEYS) % KT);
  const long long b = i / ((long long)CAM_KEYS * KT);
  const int ky = (j / tk_x) * 32 + c / 8, kx = (j % tk_x) * 8 + c % 8;
  float v = -1.0f;
  if (ky < hs && kx < ws) {
    float a = 0.0f;
    for (int u = 0; u < 4; ++u)
      for (int t = 0; t < 4; ++t) a += 1.0f - mask_s[(b * h + 2 * ky + u) * w + 2 * kx + t];
    v = (a / 16.0f > 0.1f) ? 10.0f * 1.4426950408889634f : 0.0f;
  }
  cs[i] = v;
}

// P -> the reference's cam_1 return layout [B][L keys (row-major patch index)][hs*ws queries], fp32 (module surface / tests)
__global__ void cam_attn_export_kernel(const __nv_bfloat16* __restrict__ P, float* __restrict__ attn, int B, int hs, int ws, int tk_x, int KB) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long L = (long long)hs * ws;
  if (i >= (long long)B * L * L) return;
  const int n = (int)(i % L);
  const int l = (int)((i / L) % L);
  const long long b = i / (L * L);
  const int ky = l / ws, kx = l % ws;
  const int j = (ky / 32) * tk_x + kx / 8;
  const int kb = j * 32 + (ky % 32);
  attn[i] = __bfloat162float(P[(((b * KB + kb) * hs + n / ws) * ws + n % ws) * 8 + (kx % 8)]);
}

// ------------------------------------------------------------------------------------------ S kernel
// One CTA per query tile (16 x 8 queries, persistent over the tiles of the batch): warps 0-7 = two consumer warpgroups
// (queries 0-63 / 64-127 of the tile: wgmma M = 64, N = 128 keys = one 16 x 8 half of a 32 x 8 key tile), warp 8 = TMA
// producer. A query row's logits live in one quad of lanes (accumulator fragment), so the softmax statistics need
// only two shuffles per row.
struct CamSParams {
  int hs, ws;
  int q0, q1, qa, prows;   // band query rows [q0, q1); P buffer row r holds query row qa + r, prows rows per key block
  int tq_x, tq_n, n_tiles;
  int tk_x, KT, KB;
  const float* colscale;
  __nv_bfloat16* P;
};

__global__ void __launch_bounds__(CAM_THREADS, 1)
cam_s_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const CamSParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + CAM_Q_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sK + CAM_S_STAGES * CAM_K_STAGE);
  uint64_t* q_full = bars;
  uint64_t* q_empty = bars + 1;
  uint64_t* k_full = bars + 2;
  uint64_t* k_empty = k_full + CAM_S_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(q_empty, CAM_CONSUMER_WARPS);
    for (int i = 0; i < CAM_S_STAGES; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], CAM_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int n_kt = 4 * p.KT;   // accumulator tiles per query tile: two sweeps over the key tiles, two 128-key halves each

  if (warp == CAM_CONSUMER_WARPS) {
    // ==================================================================== producer
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmQ)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmK)) : "memory");
    }
    int stage = 0;
    uint32_t phase = 0, qphase = 0;
    for (int qt = blockIdx.x; qt < p.n_tiles; qt += gridDim.x) {
      const int img = qt / p.tq_n, t = qt - img * p.tq_n;
      const int qy0 = p.q0 + (t / p.tq_x) * CAM_TH, qx0 = (t % p.tq_x) * CAM_TW;
      mbar_wait(q_empty, qphase ^ 1, 10);
      if (elect_one()) {
        mbar_expect_tx(q_full, CAM_Q_TX);
        tma_load_4d(sQ, &tmQ, q_full, qx0 * 8, qy0, 0, img);
      }
      __syncwarp();
      qphase ^= 1;
      for (int it = 0; it < n_kt; ++it) {
        const int jj = it % (2 * p.KT), j = jj >> 1, hh = jj & 1;
        const int ky0 = (j / p.tk_x) * 32 + 16 * hh, kx0 = (j % p.tk_x) * 8;
        for (int par = 0; par < 4; ++par) {
          mbar_wait(&k_empty[stage], phase ^ 1, 11);
          if (elect_one()) {
            mbar_expect_tx(&k_full[stage], CAM_K_TX);
            tma_load_4d(sK + stage * CAM_K_STAGE, &tmK, &k_full[stage], kx0 * 8, ky0, par * CAM_CB, img);
          }
          __syncwarp();
          if (++stage == CAM_S_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ==================================================================== consumers: logits, softmax statistics, probabilities
    const int wg = warp >> 2, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    const uint32_t a_m = (uint32_t)wg * 8u * CAM_ROW;   // queries 64..127 = tile rows 8..15
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
    int stage = 0;
    uint32_t phase = 0, qphase = 0;
    for (int qt = blockIdx.x; qt < p.n_tiles; qt += gridDim.x) {
      const int img = qt / p.tq_n, t = qt - img * p.tq_n;
      int qy[2], qx[2];
      bool valid[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        qy[h] = p.q0 + (t / p.tq_x) * CAM_TH + 8 * wg + 2 * wq + h;
        qx[h] = (t % p.tq_x) * CAM_TW + (lane >> 2);
        valid[h] = qy[h] < p.q1 && qx[h] < p.ws;
      }
      float m_run[2] = {-INFINITY, -INFINITY}, s_run[2] = {0.0f, 0.0f}, inv[2] = {0.0f, 0.0f};
      mbar_wait(q_full, qphase, 12);
      qphase ^= 1;
      for (int it = 0; it < n_kt; ++it) {
        const bool second = it >= 2 * p.KT;
        const int jj = it % (2 * p.KT), j = jj >> 1, hh = jj & 1;
        if (it == 2 * p.KT) {
          // combine the four lanes' partial statistics of each row
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float M = m_run[h];
            M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 1));
            M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 2));
            float S = m_run[h] > -INFINITY ? s_run[h] * ex2_approx(m_run[h] - M) : 0.0f;
            S += __shfl_xor_sync(0xffffffffu, S, 1);
            S += __shfl_xor_sync(0xffffffffu, S, 2);
            m_run[h] = M;
            inv[h] = 1.0f / S;
          }
        }
        int prev = -1;
        for (int par = 0; par < 4; ++par) {
          mbar_wait(&k_full[stage], phase, 14);
          const uint32_t aQ = base + (uint32_t)(par * CAM_CB) * CAM_PLANE + a_m;
          const uint32_t aK = base + CAM_Q_BYTES + (uint32_t)stage * CAM_K_STAGE;
          wg_fence();
          wg_fence_acc(acc);
#pragma unroll
          for (int tap = 0; tap < 4; ++tap) {
            const uint32_t toff = (uint32_t)((tap >> 1) * CAM_WR + (tap & 1)) * 16u;   // (a, b) = tap offsets inside the window
#pragma unroll
            for (int k2 = 0; k2 < 6; ++k2) {
              const uint32_t koff = (uint32_t)(2 * k2) * CAM_PLANE + toff;
              Wgmma<128, false, 0>::mma(acc, wg_desc(aQ + koff, CAM_PLANE, CAM_ROW, WG_SW_NONE), wg_desc(aK + koff, CAM_PLANE, CAM_ROW, WG_SW_NONE),
                                        (par | tap | k2) ? 1u : 0u);
            }
          }
          wg_commit();
          if (prev >= 0) {
            wg_wait<1>();
            release(&k_empty[prev]);
          }
          prev = stage;
          if (++stage == CAM_S_STAGES) { stage = 0; phase ^= 1; }
        }
        wg_wait<0>();
        wg_fence_acc(acc);
        release(&k_empty[prev]);
        if (it == n_kt - 1) release(q_empty);   // the query window is free once every MMA of this tile has retired
        // logits in log2 units; padding keys (scale < 0) are excluded, masked keys (scale 0) keep logit 0
        const float* cs = p.colscale + ((size_t)img * p.KT + j) * CAM_KEYS + hh * 128;
#pragma unroll
        for (int b = 0; b < 16; ++b) {
          const float2 c2 = __ldg(reinterpret_cast<const float2*>(cs + frag_col(lane, b)));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float& v0 = acc[4 * b + 2 * h];
            float& v1 = acc[4 * b + 2 * h + 1];
            v0 = c2.x < 0.0f ? -INFINITY : v0 * c2.x;
            v1 = c2.y < 0.0f ? -INFINITY : v1 * c2.y;
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!second) {
            float mx = -INFINITY;
#pragma unroll
            for (int b = 0; b < 16; ++b) mx = fmaxf(mx, fmaxf(acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]));
            if (mx > -INFINITY) {
              const float mn = fmaxf(m_run[h], mx);
              float s = 0.0f;
#pragma unroll
              for (int b = 0; b < 16; ++b) s += ex2_approx(acc[4 * b + 2 * h] - mn) + ex2_approx(acc[4 * b + 2 * h + 1] - mn);
              s_run[h] = s_run[h] * ex2_approx(m_run[h] - mn) + s;   // m_run = -inf: s_run is 0 and ex2(-inf) = 0
              m_run[h] = mn;
            }
          } else if (valid[h]) {
            // key column c of this half = key (row hh * 16 + c / 8, column c % 8) of tile j: P block j * 32 + hh * 16 + c / 8
            uint32_t* prow = reinterpret_cast<uint32_t*>(p.P) +
                             ((((size_t)img * p.KB + (size_t)j * 32 + hh * 16) * p.prows + (qy[h] - p.qa)) * p.ws + qx[h]) * 4 + (lane & 3);
            const size_t pstep = (size_t)p.prows * p.ws * 4;   // next key block
#pragma unroll
            for (int b = 0; b < 16; ++b)
              prow[b * pstep] = pack_bf16x2(ex2_approx(acc[4 * b + 2 * h] - m_run[h]) * inv[h], ex2_approx(acc[4 * b + 2 * h + 1] - m_run[h]) * inv[h]);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ PV kernel
// One CTA per output tile (8 x 8 positions of the sub-pixel class grid, persistent): both consumer warpgroups take all 64
// positions (wgmma M = 64, A = probabilities); warpgroup g produces sub-pixel classes 2g and 2g + 1 (N = 96 channels each,
// B = values of that parity, MN-major). Warp 8 = TMA producer.
struct CamPVParams {
  int h, w, Hs, Ws;
  int y0, y1, qa;       // band: class rows [y0, y1); row 0 of the P tensor map is query row qa
  int to_x, to_n, n_tiles;
  int tk_x, n_chunks;   // 64-key chunks = KB / 8
  __nv_bfloat16* out;   // [B][12][h][w][8]
};

__global__ void __launch_bounds__(CAM_THREADS, 1)
cam_pv_kernel(const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmV, const CamPVParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CAM_PV_STAGES * CAM_PV_STAGE);
  uint64_t* full = bars;
  uint64_t* empty = bars + CAM_PV_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < CAM_PV_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CAM_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == CAM_CONSUMER_WARPS) {
    // ==================================================================== producer
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmP)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmV)) : "memory");
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int ot = blockIdx.x; ot < p.n_tiles; ot += gridDim.x) {
      const int img = ot / p.to_n, t = ot - img * p.to_n;
      const int yy0 = p.y0 + (t / p.to_x) * CAM_PV_TH, xx0 = (t % p.to_x) * CAM_TW;
      for (int c = 0; c < p.n_chunks; ++c) {
        const int j = c >> 2;
        const int kyc = (j / p.tk_x) * 32 + (c & 3) * 8, kx0 = (j % p.tk_x) * 8;
        mbar_wait(&empty[stage], phase ^ 1, 20);
        if (elect_one()) {
          uint8_t* st = smem + stage * CAM_PV_STAGE;
          mbar_expect_tx(&full[stage], CAM_PW_TX + 4 * CAM_V_TX);
          // probabilities of the queries (yy - a, xx - b), a, b in {0, 1}: window starts one row / column before the tile
          tma_load_4d(st, &tmP, &full[stage], (xx0 - 1) * 8, yy0 - 1 - p.qa, c * 8, img);
          for (int par = 0; par < 4; ++par) tma_load_4d(st + CAM_V_OFF(par), &tmV, &full[stage], kx0 * 8, kyc, par * CAM_CB, img);
        }
        __syncwarp();
        if (++stage == CAM_PV_STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ==================================================================== consumers
    const int wg = warp >> 2, wq = warp & 3;
    const uint32_t base = smem_u32(smem);
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    float acc0[48], acc1[48];
#pragma unroll
    for (int i = 0; i < 48; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
    int stage = 0;
    uint32_t phase = 0;
    for (int ot = blockIdx.x; ot < p.n_tiles; ot += gridDim.x) {
      const int img = ot / p.to_n, t = ot - img * p.to_n;
      int prev = -1;
      for (int c = 0; c < p.n_chunks; ++c) {
        mbar_wait(&full[stage], phase, 22);
        const uint32_t st = base + (uint32_t)stage * CAM_PV_STAGE;
        const uint32_t aV0 = st + CAM_V_OFF(2 * wg), aV1 = st + CAM_V_OFF(2 * wg + 1);
        wg_fence();
        wg_fence_acc(acc0);
        wg_fence_acc(acc1);
#pragma unroll
        for (int tap = 0; tap < 4; ++tap) {
          const int a = tap >> 1, b = tap & 1;
          const uint32_t poff = (uint32_t)((1 - a) * CAM_WR + (1 - b)) * 16u;   // query (yy - a, xx - b) inside the 9 x 9 window
          const uint32_t voff = (uint32_t)(a * 9 + b) * 16u;                    // value pixel (ky + a, kx + b) inside the 9 x 9 window
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const uint64_t da = wg_desc(st + (uint32_t)(2 * k2) * CAM_PPLANE + poff, CAM_PPLANE, CAM_ROW, WG_SW_NONE);
            const uint32_t vb = (uint32_t)(2 * k2) * 9u * 16u + voff;
            const uint32_t accum = (c | tap | k2) ? 1u : 0u;
            Wgmma<96, false, 1>::mma(acc0, da, wg_desc(aV0 + vb, 9 * 16, CAM_VPLANE, WG_SW_NONE), accum);
            Wgmma<96, false, 1>::mma(acc1, da, wg_desc(aV1 + vb, 9 * 16, CAM_VPLANE, WG_SW_NONE), accum);
          }
        }
        wg_commit();
        if (prev >= 0) {
          wg_wait<1>();
          release(&empty[prev]);
        }
        prev = stage;
        if (++stage == CAM_PV_STAGES) { stage = 0; phase ^= 1; }
      }
      wg_wait<0>();
      wg_fence_acc(acc0);
      wg_fence_acc(acc1);
      if (prev >= 0) release(&empty[prev]);
      // epilogue: class g = (py, px) = parity of the values, output pixel (2 yy + py, 2 xx + px)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int yy = p.y0 + (t / p.to_x) * CAM_PV_TH + 2 * wq + h, xx = (t % p.to_x) * CAM_TW + (lane >> 2);
        if (yy >= p.y1 || xx >= p.Ws) continue;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int g = 2 * wg + q;
          const int oy = 2 * yy + (g >> 1), ox = 2 * xx + (g & 1);
          uint32_t* o = reinterpret_cast<uint32_t*>(p.out) + ((((size_t)img * CAM_CB) * p.h + oy) * p.w + ox) * 4 + (lane & 3);
          const size_t ostep = (size_t)p.h * p.w * 4;   // next channel block
#pragma unroll
          for (int b = 0; b < 12; ++b) {
            const float v0 = q ? acc1[4 * b + 2 * h] : acc0[4 * b + 2 * h], v1 = q ? acc1[4 * b + 2 * h + 1] : acc0[4 * b + 2 * h + 1];
            o[b * ostep] = pack_bf16x2(v0, v1);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn cam_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// channel-blocked 4-D view (8*W, H, blocks, N) of a bf16 tensor [N][blocks][Hp][W][8] (H <= Hp rows of each plane are in
// the view); box = (cols x 8, rows, nblk, 1)
static int cam_map(CUtensorMap* tm, const void* base, int W, int H, int Hp, int blocks, int N, int cols, int rows, int nblk) {
  EncodeTiledFn enc = cam_encode_fn();
  SE_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[4] = {(cuuint64_t)W * 8, (cuuint64_t)H, (cuuint64_t)blocks, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)W * 16, (cuuint64_t)Hp * W * 16, (cuuint64_t)blocks * Hp * W * 16};
  cuuint32_t box[4] = {(cuuint32_t)(cols * 8), (cuuint32_t)rows, (cuuint32_t)nblk, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SE_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(attention) failed, CUresult=" + std::to_string((int)r));
  return 0;
}

int cam_plan(int B, int h, int w, long long limit, bool single_band, CamPlan* out) {
  SE_REQUIRE(h % 2 == 0 && w % 2 == 0 && h >= 4 && w >= 4, "attention map must be even-sized and >= 4");
  CamPlan p;
  p.B = B; p.h = h; p.w = w;
  p.Hs = h / 2; p.Ws = w / 2;
  p.hs = p.Hs - 1; p.ws = p.Ws - 1;
  p.tq_x = (p.ws + CAM_TW - 1) / CAM_TW;
  p.tk_x = (p.ws + 7) / 8;
  p.KT = p.tk_x * ((p.hs + 31) / 32);
  p.KB = p.KT * 32;
  p.to_x = (p.Ws + CAM_TW - 1) / CAM_TW;
  p.fn_bytes = (size_t)B * 48 * p.Hs * p.Ws * 16;
  p.cs_bytes = (size_t)B * p.KT * CAM_KEYS * 4;
  // the tallest band whose P fits the limit; several bands take 16-row multiples plus the carried row
  const size_t row_bytes = (size_t)B * p.KB * p.ws * 16;   // one query row of P, every key block and image
  p.band = p.prows = p.hs;
  if (!single_band && row_bytes * p.hs > (size_t)limit) {
    const long long fit = (long long)((size_t)limit / row_bytes) - 1;
    const int band = (int)(fit < p.hs ? fit : p.hs) / CAM_TH * CAM_TH;
    const size_t min_bytes = row_bytes * (p.hs < CAM_TH + 1 ? p.hs : CAM_TH + 1);
    SE_REQUIRE(band >= CAM_TH, "attention workspace limit of " + std::to_string(limit) + " bytes is below the " + std::to_string(min_bytes) +
                                   " bytes one band of " + std::to_string(CAM_TH) + " query rows needs at this size and batch");
    p.band = band;
    p.prows = band + 1;
  }
  p.n_bands = (p.hs + p.band - 1) / p.band;
  p.p_bytes = row_bytes * p.prows;
  *out = p;
  return 0;
}

static int g_cam_sms = 0, g_cam_optin = 0;
static const int kCamSSmem = 1024 + CAM_Q_BYTES + CAM_S_STAGES * CAM_K_STAGE + 64 * 8;
static const int kCamPVSmem = 1024 + CAM_PV_STAGES * CAM_PV_STAGE + 64 * 8;

// persistent launch: one CTA per SM at most, each walks tiles blockIdx.x, + gridDim.x, ...
static int cam_launch(const void* kernel, int n_tiles, int smem, cudaStream_t stream, void** args) {
  const int grid = n_tiles < g_cam_sms ? n_tiles : g_cam_sms;
  SE_CUDA_OK(cudaLaunchKernel(kernel, dim3(grid), dim3(CAM_THREADS), args, (size_t)smem, stream));
  return 0;
}

int cam_forward_tc(const void* f_s2d, const float* mask_s, void* out_c8, const CamPlan& pl, void* fn, float* colscale, void* P, float* attn,
                   cudaStream_t stream) {
  SE_REQUIRE((reinterpret_cast<uintptr_t>(f_s2d) & 127) == 0 && (reinterpret_cast<uintptr_t>(fn) & 127) == 0 && (reinterpret_cast<uintptr_t>(P) & 127) == 0 &&
                 (reinterpret_cast<uintptr_t>(out_c8) & 15) == 0 && (reinterpret_cast<uintptr_t>(colscale) & 15) == 0,
             "attention buffers must be 128 B aligned");
  if (!g_cam_sms) {
    int dev = 0;
    SE_CUDA_OK(cudaGetDevice(&dev));
    SE_CUDA_OK(cudaDeviceGetAttribute(&g_cam_sms, cudaDevAttrMultiProcessorCount, dev));
    SE_CUDA_OK(cudaDeviceGetAttribute(&g_cam_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    SE_CUDA_OK(cudaFuncSetAttribute(cam_s_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_cam_optin));
    SE_CUDA_OK(cudaFuncSetAttribute(cam_pv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_cam_optin));
  }
  SE_REQUIRE(kCamSSmem <= g_cam_optin && kCamPVSmem <= g_cam_optin, "attention shared-memory plan exceeds the opt-in limit");
  const int B = pl.B;
  cam_norm_kernel<<<dim3(CAM_CB, B), 256, 0, stream>>>((const __nv_bfloat16*)f_s2d, (__nv_bfloat16*)fn, pl.Hs * pl.Ws);
  {
    const long long n = (long long)B * pl.KT * CAM_KEYS;
    cam_colscale_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(mask_s, colscale, B, pl.h, pl.w, pl.hs, pl.ws, pl.tk_x, pl.KT);
  }
  SE_CUDA_OK(cudaGetLastError());
  SE_REQUIRE(!attn || pl.n_bands == 1, "the attention-map output needs a single band");
  CUtensorMap tmQ, tmK, tmV;
  int rc = cam_map(&tmQ, f_s2d, pl.Ws, pl.Hs, pl.Hs, 48, B, CAM_WR, CAM_HR, 48);
  if (rc) return rc;
  rc = cam_map(&tmK, fn, pl.Ws, pl.Hs, pl.Hs, 48, B, CAM_WR, CAM_HR, CAM_CB);
  if (rc) return rc;
  rc = cam_map(&tmV, f_s2d, pl.Ws, pl.Hs, pl.Hs, 48, B, 9, 9, CAM_CB);
  if (rc) return rc;
  const size_t prow_bytes = (size_t)pl.ws * 16;   // one query row of one key block of P
  for (int q0 = 0, prev_qa = 0; q0 < pl.hs; q0 += pl.band) {
    const int q1 = q0 + pl.band < pl.hs ? q0 + pl.band : pl.hs;
    const int qa = q0 ? q0 - 1 : 0;   // query row held in buffer row 0
    if (q0) {
      // carry query row q0 - 1 (the previous band's last row) into buffer row 0 of every key block and image
      char* Pb = (char*)P;
      SE_CUDA_OK(cudaMemcpy2DAsync(Pb, (size_t)pl.prows * prow_bytes, Pb + (size_t)(q0 - 1 - prev_qa) * prow_bytes, (size_t)pl.prows * prow_bytes,
                                   prow_bytes, (size_t)B * pl.KB, cudaMemcpyDeviceToDevice, stream));
    }
    prev_qa = qa;
    {
      CamSParams sp;
      sp.hs = pl.hs; sp.ws = pl.ws;
      sp.q0 = q0; sp.q1 = q1; sp.qa = qa; sp.prows = pl.prows;
      sp.tq_x = pl.tq_x; sp.tq_n = pl.tq_x * ((q1 - q0 + CAM_TH - 1) / CAM_TH); sp.n_tiles = B * sp.tq_n;
      sp.tk_x = pl.tk_x; sp.KT = pl.KT; sp.KB = pl.KB;
      sp.colscale = colscale; sp.P = (__nv_bfloat16*)P;
      void* args[3] = {&tmQ, &tmK, &sp};
      rc = cam_launch((const void*)cam_s_kernel, sp.n_tiles, kCamSSmem, stream, args);
      if (rc) return rc;
    }
    if (attn) {
      const long long n = (long long)B * pl.hs * pl.ws * pl.hs * pl.ws;
      cam_attn_export_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>((const __nv_bfloat16*)P, attn, B, pl.hs, pl.ws, pl.tk_x, pl.KB);
      SE_CUDA_OK(cudaGetLastError());
    }
    {
      // class rows [q0, q1) (the last band also row hs) read query rows [q0 - 1, q1): rows outside [qa, q1) are out of the
      // map's bounds and load as zeros, as query rows -1 and hs must
      const int y1 = q1 == pl.hs ? pl.Hs : q1;
      CUtensorMap tmP;
      rc = cam_map(&tmP, P, pl.ws, q1 - qa, pl.prows, pl.KB, B, CAM_WR, CAM_PV_TH + 1, 8);
      if (rc) return rc;
      CamPVParams pp;
      pp.h = pl.h; pp.w = pl.w; pp.Hs = pl.Hs; pp.Ws = pl.Ws;
      pp.y0 = q0; pp.y1 = y1; pp.qa = qa;
      pp.to_x = pl.to_x; pp.to_n = pl.to_x * ((y1 - q0 + CAM_PV_TH - 1) / CAM_PV_TH); pp.n_tiles = B * pp.to_n;
      pp.tk_x = pl.tk_x; pp.n_chunks = pl.KB / 8;
      pp.out = (__nv_bfloat16*)out_c8;
      void* args[3] = {&tmP, &tmV, &pp};
      rc = cam_launch((const void*)cam_pv_kernel, pp.n_tiles, kCamPVSmem, stream, args);
      if (rc) return rc;
    }
  }
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

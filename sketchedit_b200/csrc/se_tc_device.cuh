// Device-side building blocks shared by the wgmma kernels (se_conv_c8.cu, se_cam.cu, se_gemm_split.cu): mbarrier / TMA
// PTX wrappers, wgmma matrix descriptors and synchronisation, and the fused convolution epilogue on register fragments.
#pragma once
#include <cuda_fp16.h>

#include "se_common.cuh"
#include "se_wgmma.cuh"

namespace se {

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug traps after ~2 s of wall time (%globaltimer) instead of hanging the GPU. The timer is read only
// after 256 failed attempts, so it stays off the wake-up path. (`tag` names the wait site; kept for debugging builds.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag) {
  (void)tag;
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b64 t0, t1;\n\t.reg .b32 n;\n\t"
      "mov.u64 t0, 0;\n\t"
      "OUTER_%=:\n\t"
      "mov.u32 n, 0;\n\t"
      "INNER_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 256;\n\t"
      "@p bra INNER_%=;\n\t"
      "mov.u64 t1, %%globaltimer;\n\t"
      "setp.eq.u64 p, t0, 0;\n\t"
      "@p mov.u64 t0, t1;\n\t"
      "sub.u64 t1, t1, t0;\n\t"
      "setp.lt.u64 p, t1, 2000000000;\n\t"
      "@p bra OUTER_%=;\n\t"
      "trap;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// linear global -> shared bulk copy (bytes % 16 == 0), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// the same copy multicast to every CTA of the cluster in cta_mask: lands at dst's offset in each, completes on each CTA's own
// mbarrier at bar's offset
__device__ __forceinline__ void bulk_load_1d_multicast(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t cta_mask) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
               : "memory");
}

// ------------------------------------------------------------------------------------------ thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster: orders shared-memory writes and mbarrier inits before it, across the cluster
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at bar's offset in the shared memory of cluster CTA `cta`. Release at CTA scope: a consumer
// releases a stage its retired wgmma no longer reads, and that needs no fence. (.release.cluster puts a GPU-scope
// MEMBAR before the arrive, which waits for every global store the thread has in flight, e.g. the previous epilogue's.)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\tmbarrier.arrive.release.cta.shared::cluster.b64 _, [ra];\n\t}"
               ::"r"(smem_u32(bar)), "r"(cta) : "memory");
}

// one lane of a fully converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------ wgmma
// Matrix descriptor (sm_90): start address, leading / stride byte offsets (16 B units), layout type in bits 62-63.
// No-swizzle K-major operand: core matrices of 8 rows x 16 B; LBO = next core matrix along K, SBO = next 8 rows.
// No-swizzle MN-major operand: LBO = next 8 K rows, SBO = next 8 M/N elements.
enum : uint32_t { WG_SW_NONE = 0, WG_SW128 = 1, WG_SW64 = 2 };
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | ((uint64_t)layout << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// named barrier `id` (not 0: __syncthreads) over n threads: bar.arrive signals without waiting, bar.sync waits
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Accumulator fragment of m64nNk16 (thread = lane of warp w of the warpgroup): d[4j + 2h + e] holds
// row 16w + lane/4 + 8h, column 8j + 2(lane%4) + e.
__device__ __forceinline__ int frag_row(int w, int lane, int h) { return 16 * w + (lane >> 2) + 8 * h; }
__device__ __forceinline__ int frag_col(int lane, int j) { return 8 * j + 2 * (lane & 3); }

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ------------------------------------------------------------------------------------------ epilogue
// Epilogue constants in shared memory, three float arrays of `n` entries each, indexed by ACCUMULATOR COLUMN:
//   [0,n)  bias b    [n,2n)  b * log2(e) (ELU exponent)    [2n,3n)  0.5 * b (sigmoid-as-tanh argument)
// (gated layers: column c = feature c, column goff + c = its gate; see gated_column)
__device__ __forceinline__ void epi_fill_constants(float* cst, int n, const float* bias, const EpiParams& e, int tid, int nthreads) {
  const int half = e.Cout >> 1;
  for (int i = tid; i < n; i += nthreads) {
    const int ch = i < half ? i : (i >= e.goff && i < e.goff + half ? half + i - e.goff : -1);   // -1: padding column
    const float b = (bias != nullptr && ch >= 0 && ch < e.Cout) ? bias[ch] : 0.0f;
    cst[i] = b;
    cst[n + i] = b * 1.4426950408889634f;
    cst[2 * n + i] = 0.5f * b;
  }
}

// one gated output: act(f + b) * sigmoid(g + b')  (reference utils.py:29-32)
//   sigmoid(x) = 0.5 * tanh(0.5 x) + 0.5 (one MUFU); the accumulator column of a gate already holds 0.5 * g (the gate
//   weights are packed pre-multiplied by 0.5), hb = 0.5 * b'. ELU's exp as ex2 with the bias folded into the FMA (bl = b * log2 e).
template <bool kElu>
__device__ __forceinline__ float gate_one(float f, float ghalf, float b, float bl, float hb) {
  const float fv = f + b;
  float a;
  if (kElu) {
    const float ex = ex2_approx(fmaf(f, 1.4426950408889634f, bl)) - 1.0f;
    a = fv > 0.0f ? fv : ex;
  } else {
    a = fmaxf(fv, 0.0f);
  }
  const float h = 0.5f * a;
  return fmaf(h, tanh_approx(ghalf + hb), h);
}

// Split-half mode (DT_F16X2, the fp32-on-tensor-cores path): same gate, fp32-accurate math (ex2 / rcp approximations are good
// to ~2^-22; no tanh.approx). `s` = 1 / (activation scale * weight scale) of the split-half operands (se_common.cuh:
// kSplitActScale, ClassW::s_wscale). ELU's exp(x) - 1 cancels near 0 (ex2.approx is good to 2^-22 of exp(x), i.e. 2.4e-7
// ABSOLUTE, 2.4e-4 of x = -1e-3): above -1/16 the degree-5 Taylor polynomial of expm1 is used instead (remainder < 1e-10).
template <bool kElu>
__device__ __forceinline__ float gate_one_exact(float f, float ghalf, float b, float hb, float s) {
  const float fv = fmaf(f, s, b);
  float a;
  if (kElu) {
    const float big = ex2_approx(fv * 1.4426950408889634f) - 1.0f;
    const float small = fv * fmaf(fv, fmaf(fv, fmaf(fv, fmaf(fv, 1.0f / 120.0f, 1.0f / 24.0f), 1.0f / 6.0f), 0.5f), 1.0f);
    a = fv > 0.0f ? fv : (fv > -0.0625f ? small : big);
  } else {
    a = fmaxf(fv, 0.0f);
  }
  const float gx = 2.0f * fmaf(ghalf, s, hb);
  return a * rcp_approx(1.0f + ex2_approx(-gx * 1.4426950408889634f));
}

// Element offset of channel (c & 7) of block 0 of pixel (img, oy, ox) in the launch's output tensor; block b of the pixel
// is e.blk_stride elements further on (plus e.blk_jump * 8 from block blk_split on).
//   out_c8 == 0: NHWC, pixel pitch ldo, channel offset choff                          (blk_stride = 8)
//   out_c8 == 1: channel-blocked [N][ldo blocks][Hout][Wout][8]                      (blk_stride = Hout * Wout * 8)
//   out_c8 == 2: channel-blocked space-to-depth for a stride-2 consumer: [N][4 * ldo/4 blocks][Hout/2][Wout/2][8], parity
//                (oy&1, ox&1) selects the block group (par_stride blocks apart)     (blk_stride = Hout/2 * Wout/2 * 8)
// Fused layer pairs: channel blocks >= blk_split belong to the second layer's tensor, blk_jump 16 B units further on.
__device__ __forceinline__ size_t epi_pixel_offset(const EpiParams& e, int img, int oy, int ox, int c) {
  if (e.out_c8 == 0) return (((size_t)img * e.Hout + oy) * e.Wout + ox) * e.ldo + e.choff + c;
  size_t unit;
  if (e.out_c8 == 2) {
    const size_t Hs = e.Hout >> 1, Ws = e.Wout >> 1, par = ((oy & 1) << 1) | (ox & 1);
    unit = (((size_t)img * e.ldo + par * e.par_stride + (e.choff >> 3)) * Hs + (oy >> 1)) * Ws + (ox >> 1);
  } else {
    unit = (((size_t)img * e.ldo + (e.choff >> 3)) * e.Hout + oy) * e.Wout + ox;
  }
  return unit * 8 + (c & 7);
}

__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}

// Fused gated epilogue of one 64 x NT accumulator fragment (one warpgroup's half of a 128-position tile):
//   out[c] = act(acc[c] + b[c]) * sigmoid(acc[goff + c] + b[Cout/2 + c])   (goff = NT / 2, act = ELU or ReLU: kElu)
// kF16: split-half output (exact-class math, hi and lo stores). kPaired: every column pair of the fragment is one aligned
// 4 B store (channel-blocked outputs, or NHWC with even pitch / offset and Cout / 2 = goff); otherwise NHWC stores are per
// channel and stop at Cout / 2. Channel-blocked outputs also get the padding channels of their last block written (as 0:
// padding columns hold zero weights and zero bias), because the next layer's tensor-core MMAs read whole blocks.
// Everything that depends on the launch only (mode, layout, block strides) is resolved outside the unrolled loop: row half h of
// the fragment writes pixel offset base[h] (if ok[h]), block j at base[h] + j * blk_stride. `cst` = shared-memory address
// of the constants (epi_fill_constants, n = NT + 32).
template <int NT, bool kF16, bool kElu, bool kPaired>
__device__ __forceinline__ void conv_epilogue(const EpiParams& e, uint32_t cst, const float (&acc)[NT / 2], const size_t (&base)[2],
                                              const bool (&ok)[2], int lane) {
  static_assert(!kF16 || kPaired, "split-half outputs are channel-blocked");
  constexpr int n = NT + 32, goff = NT / 2, G = NT / 16;   // G: fragment block of the gate column goff + c
  const int c0 = 2 * (lane & 3);
  const uint32_t cq = cst + 4u * (uint32_t)c0;
  const int lim = e.Cout >> 1;   // NHWC (not paired): channels written
  const uint32_t jump = (uint32_t)e.blk_jump * 8u;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!ok[h]) continue;
    if constexpr (kF16) {
      __half* y = reinterpret_cast<__half*>(e.y) + base[h];
      __half* ylo = y + (size_t)e.split_stride * 8;   // the lo part of a block, split_stride 16 B units further on
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const float2 b = lds_f2(cq + 32u * j), hb = lds_f2(cq + 4u * (2 * n + goff) + 32u * j);
        float v0 = gate_one_exact<kElu>(acc[4 * j + 2 * h], acc[4 * (j + G) + 2 * h], b.x, hb.x, e.scale);
        float v1 = gate_one_exact<kElu>(acc[4 * j + 2 * h + 1], acc[4 * (j + G) + 2 * h + 1], b.y, hb.y, e.scale);
        // split-half output: hi = fp16(64 v), lo = fp16(64 v - hi)
        v0 = fminf(fmaxf(v0 * kSplitActScale, -kSplitActMax), kSplitActMax);
        v1 = fminf(fmaxf(v1 * kSplitActScale, -kSplitActMax), kSplitActMax);
        const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
        const uint32_t off = (uint32_t)j * (uint32_t)e.blk_stride + (j >= e.blk_split ? jump : 0u);
        *reinterpret_cast<uint32_t*>(y + off) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        *reinterpret_cast<uint32_t*>(ylo + off) = pack_f16x2(v0 - __half2float(h0), v1 - __half2float(h1));
      }
    } else {
      __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(e.y) + base[h];
#pragma unroll
      for (int j = 0; j < G; ++j) {
        const float2 b = lds_f2(cq + 32u * j), hb = lds_f2(cq + 4u * (2 * n + goff) + 32u * j);
        float2 bl = make_float2(0.0f, 0.0f);
        if constexpr (kElu) bl = lds_f2(cq + 4u * n + 32u * j);
        const float v0 = gate_one<kElu>(acc[4 * j + 2 * h], acc[4 * (j + G) + 2 * h], b.x, bl.x, hb.x);
        const float v1 = gate_one<kElu>(acc[4 * j + 2 * h + 1], acc[4 * (j + G) + 2 * h + 1], b.y, bl.y, hb.y);
        const uint32_t off = (uint32_t)j * (uint32_t)e.blk_stride + (j >= e.blk_split ? jump : 0u);
        if constexpr (kPaired) {
          *reinterpret_cast<uint32_t*>(y + off) = pack_bf16x2(v0, v1);
        } else {
          const int c = 8 * j + c0;
          if (c < lim) y[off] = __float2bfloat16(v0);
          if (c + 1 < lim) y[off + 1] = __float2bfloat16(v1);
        }
      }
    }
  }
}

}  // namespace se

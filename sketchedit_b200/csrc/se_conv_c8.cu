// wgmma implicit-GEMM convolution over CHANNEL-BLOCKED activations ("C8": [N][C/8][H][W][8] bf16) for sm_90a.
//
// Why this layout: 8 horizontally adjacent pixels of one channel block are 128 contiguous bytes = exactly one wgmma
// "core matrix" (8 rows x 16 B) of the no-swizzle K-major operand layout. So a spatial region of the input landed
// in shared memory by ONE TMA box [blocks][rows][cols*8] is directly usable as the A operand of EVERY tap of the
// convolution: the tap only changes the descriptor's start address (LBO = block plane size, SBO = row pitch).
//   * stride-1 convs with dilation <= 2 and the four sub-pixel classes of the x2 deconvs: the (16+2p) x (8+2p) halo
//     of a 16 x 8 output tile is loaded once per tile (ring of buffers) and re-used by all taps  ("HALO" mode;
//     A traffic drops from taps x tile to ~1.4 x tile, TMA row requests by >10x)
//   * dilation >= 4: one box per tap                                                           ("PERTAP" mode)
//   * 5x5 stems over the 8-channel packed input: GEMM-K runs over the pixel window (LBO = 16 B): 5 taps x 3 MMAs.
// The B operand (weights) is the pre-swizzled stage image of se_conv_tc.h, either streamed per k-step with
// cp.async.bulk or, when the whole layer fits (<= ~112 KB), loaded once and kept resident in shared memory.
//   * stride-2 3x3 layers read a SPACE-TO-DEPTH C8 tensor (written that way by the producer's epilogue): every tap is a
//     stride-1 read of one parity group, selected by a per-tap channel-block offset (C8Layer::tap_cb).
// 288 threads: warps 0-7 are two consumer warpgroups (rows 0-63 / 64-127 of every 128-position tile: wgmma M = 64 each,
// accumulators in registers, fused epilogue straight from the fragments, se_tc_device.cuh), warp 8 is the TMA producer.
// Two-team launches (TEAMS = 2, resident weights): 544 threads, a second pair of consumer warpgroups in warps 8-15 runs
// every other tile of the CTA from the same weight image and halo ring; the producer is warp 16.
#include "se_conv_c8.h"

#include <stdlib.h>

#include <atomic>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_tc_device.cuh"

namespace se {

constexpr int C8_TH = 16, C8_TW = 8;   // output tile: 16 rows x 8 columns = 128 positions
constexpr int C8_CONSUMER_WARPS = 8;   // of one team: two warpgroups
__host__ __device__ constexpr int c8_threads(int teams) { return 32 * C8_CONSUMER_WARPS * teams + 32; }   // the producer is the last warp
constexpr int C8_MAX_STAGES = 8;

// slot / phase parity of iteration i in a ring of n slots (shift = log2 n, or < 0: n is not a power of two)
__device__ __forceinline__ void ring_of(int i, int n, int shift, int& slot, uint32_t& phase) {
  if (shift >= 0) { slot = i & (n - 1); phase = (uint32_t)(i >> shift) & 1u; }
  else { const int qd = i / n; slot = i - qd * n; phase = (uint32_t)qd & 1u; }
}

// NT: GEMM N (accumulator columns) of the layer; kF16: operands are fp16 (split-half mode) instead of bf16.
// k-step shape: R64 64-wide K units of M64 K16 MMAs each, then R32 32-wide units of two. A k-step is one fully unrolled
// wgmma chain between one fence and one commit: with a run-time shape ptxas keeps the accumulators live across a loop and
// inserts a warpgroup.arrive before every wgmma, so each one closed its own group.
// p.ncls > 1: fused sub-pixel classes of a x2 deconv (C8Group): the consumers run over VIRTUAL tiles v = tile * ncls + class;
// the producer loads one (union) halo per real tile, a class selects its resident weight image (cls_bytes apart), its
// A-offset row aoff[class * C8_CLS_UNITS + unit] and its output sub-pixel offset; the halo buffer is released after the
// tile's last class.
// TEAMS: teams of two consumer warpgroups (warps 8t .. 8t + 7). Team t runs the CTA's tiles riter = t, t + TEAMS, ...: the
// tile sequence, the producer and the ring slot of a tile are those of one team, and a halo buffer is read by one team only
// (a_empty counts that team's 8 warps). The teams share the resident weights, the constants and aoff, and are not ordered
// against each other: each ping-pongs on its own pair of named barriers. Two teams need resident weights and one k-step.
template <int NT, bool kF16, int R64, int M64, int R32, int TEAMS>
__global__ void __launch_bounds__(c8_threads(TEAMS), 1)
conv_c8_kernel(const __grid_constant__ CUtensorMap tmA, const C8Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // carve: [halo A buffers][resident weights][stages: (tap A box) + (B image)] [barriers][bias]
  // the two-team form runs ping-pong launches only (c8_launch): resident weights, one halo per tile, one k-step, no cluster;
  // what serves the streamed and per-tap plans compiles away in it
  constexpr bool kTeams = TEAMS > 1;
  const bool halo = kTeams || p.mode == C8_HALO;
  constexpr int b64_bytes = NT * 128, b32_bytes = NT * 64;
  constexpr int b_bytes = R64 * b64_bytes + R32 * b32_bytes;
  const int stage_a = halo ? 0 : p.a_bytes;
  const int stage_b = p.resident ? 0 : b_bytes;
  const int stage_bytes = stage_a + stage_b;
  const bool staged = !kTeams && stage_bytes > 0;
  uint8_t* sHalo = smem;
  uint8_t* sWres = sHalo + (halo ? p.a_bufs * p.a_bytes : 0);
  uint8_t* sStages = sWres + (p.resident ? p.wres_bytes : 0);
  uint8_t* tail = sStages + (size_t)p.num_stages * stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty_bar = full_bar + C8_MAX_STAGES;
  uint64_t* a_full = empty_bar + C8_MAX_STAGES;
  uint64_t* a_empty = a_full + C8_MAX_ABUFS;
  uint64_t* wres_bar = a_empty + C8_MAX_ABUFS;
  float* bias_s = reinterpret_cast<float*>(wres_bar + 2);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // 2-CTA cluster (streamed weights): both CTAs run the same number of tiles in lockstep and share every B stage, rank r
  // multicasting part r of it; a stage slot is free when the consumers of BOTH CTAs have released it
  const bool clustered = !kTeams && p.cluster > 1;
  const uint32_t rank = clustered ? cluster_ctarank() : 0u;
  if (threadIdx.x == 0) {
    for (int i = 0; i < C8_MAX_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], C8_CONSUMER_WARPS * p.cluster);   // one arrival per consumer warp of each CTA
    }
    for (int i = 0; i < C8_MAX_ABUFS; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], C8_CONSUMER_WARPS);
    }
    mbar_init(wres_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int cst_n = NT + 32;
  epi_fill_constants(bias_s, cst_n, p.bias, p.e, threadIdx.x, c8_threads(TEAMS));
  // a cluster's barriers are initialised before any multicast or remote arrive reaches them
  if (clustered) cluster_sync();
  else __syncthreads();

  const int total_tiles = p.N * p.tiles_x * p.tiles_y;
  const int ksteps = kTeams ? 1 : p.ksteps;
  // CTA b runs tiles b, b + gridDim.x, ... (gridDim.x = 2 x clusters: rank r of cluster q runs tiles 2 (q + k G) + r) for as
  // long as its cluster's rank-0 tile exists; when that one is the last tile, rank 1 is a PHANTOM for the pair: it loads no
  // A, issues its B parts and releases the stages unread, so that its partner's stages complete
  const int first_tile = (int)blockIdx.x - (int)rank;

  if (warp == C8_CONSUMER_WARPS * TEAMS) {
    // ==================================================================== producer
    if (lane == 0) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    if (p.resident && elect_one()) {
      // whole layer's weights, once: bulk copies of <= 64 KB
      mbar_expect_tx(wres_bar, (uint32_t)p.wres_bytes);
      for (int off = 0; off < p.wres_bytes; off += 65536) {
        const int n = min(65536, p.wres_bytes - off);
        bulk_load_1d(sWres + off, p.w + off, (uint32_t)n, wres_bar);
      }
    }
    __syncwarp();
    // B stage part of this CTA: all of it, or (cluster) part `rank` of a split at whole 1024 B swizzle atoms
    const int b_split = (b_bytes >> 11) << 10;
    const int b_off = rank ? b_split : 0, b_len = clustered ? (rank ? b_bytes - b_split : b_split) : b_bytes;
    int stage = 0, iter = 0;
    uint32_t phase = 0;
    // tile coordinates advance incrementally by gridDim.x tiles (mixed radix step), no per-tile integer division
    int tx = blockIdx.x % p.tiles_x, ty = (blockIdx.x / p.tiles_x) % p.tiles_y, img = blockIdx.x / (p.tiles_x * p.tiles_y);
    for (int tile = blockIdx.x; tile - (int)rank < total_tiles; tile += gridDim.x, ++iter) {
      if (tile != (int)blockIdx.x) {
        tx += p.step_x;
        if (tx >= p.tiles_x) { tx -= p.tiles_x; ++ty; }
        ty += p.step_y;
        if (ty >= p.tiles_y) { ty -= p.tiles_y; ++img; }
        img += p.step_img;
      }
      const int x0 = tx * C8_TW, y0 = ty * C8_TH;
      const bool load_a = tile < total_tiles;   // false: phantom
      if (halo && load_a) {
        int ab;
        uint32_t aphase;
        ring_of(iter, p.a_bufs, p.a_shift, ab, aphase);
        mbar_wait(&a_empty[ab], aphase ^ 1, 5);
        if (elect_one()) {
          mbar_expect_tx(&a_full[ab], (uint32_t)p.a_tx_bytes);
          tma_load_4d(sHalo + (size_t)ab * p.a_bytes, &tmA, &a_full[ab], (x0 - p.pad_x0) * 8, y0 - p.pad_y0, p.x_cb_off, img);
        }
        __syncwarp();
      }
      if (staged) {
        for (int ks = 0; ks < ksteps; ++ks) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 1);
          uint8_t* st = sStages + (size_t)stage * stage_bytes;
          if (elect_one()) {
            // (cluster: the whole B stage lands here, the partner's part possibly before this expect_tx)
            mbar_expect_tx(&full_bar[stage], (uint32_t)((halo || !load_a ? 0 : p.a_tx_bytes) + stage_b));
            if (!p.resident) {
              const uint8_t* src = p.w + (size_t)ks * b_bytes + b_off;
              if (clustered) bulk_load_1d_multicast(st + stage_a + b_off, src, (uint32_t)b_len, &full_bar[stage], 0x3);
              else bulk_load_1d(st + stage_a, src, (uint32_t)b_len, &full_bar[stage]);
            }
            if (!halo && load_a) {   // PERTAP: a stage is one tap, or one 64-channel chunk of a tap (cpt > 1)
              const int t = ks / p.cpt, ch = ks - t * p.cpt;
              tma_load_4d(st, &tmA, &full_bar[stage], (x0 + p.dx[t]) * 8, y0 + p.dy[t], p.x_cb_off + p.tap_cb[t] + 8 * ch, img);
            }
          }
          __syncwarp();
          if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ==================================================================== consumers: MMA + epilogue
    const int team = TEAMS > 1 ? warp / C8_CONSUMER_WARPS : 0;
    const int wg = (warp >> 2) & 1, wq = warp & 3;
    const uint32_t smem_base = smem_u32(smem);
    const uint32_t off_wres = halo ? (uint32_t)(p.a_bufs * p.a_bytes) : 0u;
    const uint32_t off_stages = off_wres + (p.resident ? (uint32_t)p.wres_bytes : 0u);
    const uint32_t a_m = (uint32_t)wg * 8u * (uint32_t)p.sbo_bytes;   // rows 64..127 of the tile = tile rows 8..15
    const uint32_t n_u64 = p.ntaps * p.n64;
    const int ncls = p.ncls;
    const uint32_t cst_s = smem_u32(bias_s);
    const bool elu = p.e.epi == EPI_GATE_ELU, paired = p.e.paired != 0;
    if (p.resident) mbar_wait(wres_bar, 0, 6);
    auto release = [&](uint64_t* bar) {
      __syncwarp();
      if (lane == 0) mbar_arrive(bar);
    };
    // a weight stage is released on this CTA's barrier and (cluster) on the partner's
    auto release_stage = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if (clustered) mbar_arrive_cluster(&empty_bar[s], rank ^ 1u);
      }
    };
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.0f;
    int stage = 0;
    uint32_t phase = 0;
    const int my_tiles = (first_tile < total_tiles) ? (total_tiles - first_tile + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const int nv = (my_tiles > team ? (my_tiles - team + TEAMS - 1) / TEAMS : 0) * ncls;   // this team's virtual tiles
    // Ping-pong (resident weights, one k-step per tile: plain layers, stems, stem pairs, fused classes): the two warpgroups'
    // MMA phases alternate on named barriers 1 + 2 team and 2 + 2 team (the team's 256 threads). Warpgroup 1 issues its MMAs of virtual
    // tile v after warpgroup 0 has issued its own of v, warpgroup 0 those of v + 1 after warpgroup 1 has issued its own of v.
    // The tensor cores run them in issue order, so each warpgroup's epilogue overlaps the other's MMAs: a tile takes
    // max(2m, m + E) instead of 2m + E (m: one half tile's MMAs, E: its epilogue).
    //  * resident plans have >= 2 halo buffers (c8_configure, checked in c8_launch): the producer loads tile v + 1 while
    //    warpgroup 1 still reads tile v;
    //  * every bar.arrive meets its bar.sync: warpgroup 0 arrives on 1 for every v, where warpgroup 1 syncs; warpgroup 1
    //    arrives on 2 for every v but the last, warpgroup 0 syncs on it for every v but the first. No barrier is left
    //    half-arrived at exit, whatever the team's tile count (0 and 1 included).
    // Streamed launches keep both warpgroups in lockstep: their stage ring cannot cover one that lags a whole MMA phase.
    const bool pingpong = kTeams || (p.resident && ksteps == 1);
    const int bar_wg0 = 2 + 2 * team, bar_wg1 = 1 + 2 * team;   // where warpgroup 0 / 1 waits for the other's issue
    // the team's tile coordinates advance by TEAMS x gridDim.x tiles (mixed radix step, as the producer's by gridDim.x)
    int riter = team, cls = 0;
    int tx, ty, img;
    {
      const int t0 = (int)blockIdx.x + team * (int)gridDim.x;
      tx = t0 % p.tiles_x; ty = (t0 / p.tiles_x) % p.tiles_y; img = t0 / (p.tiles_x * p.tiles_y);
    }
    for (int v = 0; v < nv; ++v) {
      if (v > 0 && ++cls == ncls) {
        cls = 0;
        riter += TEAMS;
        tx += p.cstep_x;
        if (tx >= p.tiles_x) { tx -= p.tiles_x; ++ty; }
        ty += p.cstep_y;
        if (ty >= p.tiles_y) { ty -= p.tiles_y; ++img; }
        img += p.cstep_img;
      }
      const int tile = (int)blockIdx.x + riter * (int)gridDim.x;
      if (tile >= total_tiles) {   // phantom (clusters stream their weights: ncls == 1)
        for (int ks = 0; ks < ksteps; ++ks) {
          mbar_wait(&full_bar[stage], phase, 3);
          release_stage(stage);
          if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
        }
        continue;
      }
      int ab = 0;
      if (halo) {
        uint32_t aph;
        ring_of(riter, p.a_bufs, p.a_shift, ab, aph);
        mbar_wait(&a_full[ab], aph, 7);
      }
      if (pingpong && (wg == 1 || v > 0)) named_bar_sync(wg == 0 ? bar_wg0 : bar_wg1, 256);
      int prev = -1;
      for (int ks = 0; ks < ksteps; ++ks) {
        if (staged) mbar_wait(&full_bar[stage], phase, 3);
        const uint32_t st = smem_base + off_stages + (uint32_t)stage * stage_bytes;
        const uint32_t sB = p.resident ? smem_base + off_wres + (uint32_t)cls * (uint32_t)p.cls_bytes + (uint32_t)ks * b_bytes : st + stage_a;
        const uint32_t sA = (halo ? smem_base + (uint32_t)ab * p.a_bytes : st) + a_m;
        const int ub = cls * C8_CLS_UNITS;
        const int u0 = ub + ks * R64, v0 = ub + (int)n_u64 + ks * R32;
        const uint32_t acc0 = ks ? 1u : 0u;   // the tile's first MMA overwrites the accumulators
        wg_fence();
        wg_fence_acc(acc);
#pragma unroll
        for (int j = 0; j < R64; ++j) {
          const uint32_t a0 = sA + p.aoff[u0 + j];
          const uint32_t b0 = sB + (uint32_t)(j * b64_bytes);
#pragma unroll
          for (int k = 0; k < M64; ++k)
            Wgmma<NT, kF16, 0>::mma(acc, wg_desc(a0 + k * p.kstep_bytes, p.lbo_bytes, p.sbo_bytes, WG_SW_NONE),
                                    wg_desc(b0 + 32u * k, 16u, 1024u, WG_SW128), j + k ? 1u : acc0);
        }
#pragma unroll
        for (int j = 0; j < R32; ++j) {
          const uint32_t a0 = sA + p.aoff[v0 + j];
          const uint32_t b0 = sB + (uint32_t)(R64 * b64_bytes + j * b32_bytes);
#pragma unroll
          for (int k = 0; k < 2; ++k)
            Wgmma<NT, kF16, 0>::mma(acc, wg_desc(a0 + k * p.kstep_bytes, p.lbo_bytes, p.sbo_bytes, WG_SW_NONE),
                                    wg_desc(b0 + 32u * k, 16u, 512u, WG_SW64), R64 + j + k ? 1u : acc0);
        }
        wg_commit();
        if (staged) {
          // keep one k-step in flight: the previous k-step's stage is free once its group has completed
          if (prev >= 0) {
            wg_wait<1>();
            release_stage(prev);
          }
          prev = stage;
          if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
        }
      }
      if (pingpong && (wg == 0 || v + 1 < nv)) named_bar_arrive(wg == 0 ? bar_wg1 : bar_wg0, 256);
      wg_wait<0>();
      wg_fence_acc(acc);
      if (prev >= 0) release_stage(prev);
      if (halo && cls == ncls - 1) release(&a_empty[ab]);
      // output pixel of fragment row half h (sub-pixel classes: osy = osx = 2 and a per-class offset)
      const int ooy = ncls > 1 ? p.cls_ooy[cls] : p.e.ooy, oox = ncls > 1 ? p.cls_oox[cls] : p.e.oox;
      size_t base[2];
      bool ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ry = 8 * wg + 2 * wq + h, rx = lane >> 2;   // tile row / column of fragment row 64 wg + frag_row(wq, lane, h)
        const int py = ty * C8_TH + ry, px = tx * C8_TW + rx;
        ok[h] = py < p.Ho && px < p.Wo;
        base[h] = epi_pixel_offset(p.e, img, py * p.e.osy + ooy, px * p.e.osx + oox, 2 * (lane & 3));
      }
      if (elu) {
        if (kF16 || paired) conv_epilogue<NT, kF16, true, true>(p.e, cst_s, acc, base, ok, lane);
        else conv_epilogue<NT, false, true, false>(p.e, cst_s, acc, base, ok, lane);
      } else {
        if (kF16 || paired) conv_epilogue<NT, kF16, false, true>(p.e, cst_s, acc, base, ok, lane);
        else conv_epilogue<NT, false, false, false>(p.e, cst_s, acc, base, ok, lane);
      }
    }
  }
  // no CTA of a cluster exits while its partner may still multicast into its shared memory or arrive on its barriers
  if (clustered) cluster_sync();
}

// ------------------------------------------------------------------------------------------ host
void fill_epi(const ConvParams& c, int NT, EpiParams* e) {
  e->y = c.y; e->out_c8 = c.out_c8;
  e->Hout = c.Hout; e->Wout = c.Wout; e->ldo = c.ldo; e->choff = c.choff;
  e->osy = c.osy; e->ooy = c.ooy; e->osx = c.osx; e->oox = c.oox;
  e->epi = c.epi; e->scale = c.scale;
  e->Cout = c.Cout; e->NT = NT;
  e->blk_split = c.out_blk_split > 0 ? c.out_blk_split : (1 << 20);
  e->blk_jump = c.out_blk_split > 0 ? c.out_blk_jump : 0;
  e->par_stride = c.out_par_stride > 0 ? c.out_par_stride : (c.ldo >> 2);
  const long long plane = c.out_c8 == 2 ? (long long)(c.Hout / 2) * (c.Wout / 2) : (long long)c.Hout * c.Wout;
  e->blk_stride = (int)(c.out_c8 ? plane * 8 : 8);
  e->goff = gated_goff(c.Cout);
  e->paired = (c.out_c8 != 0 || (((c.ldo | c.choff) & 1) == 0 && c.Cout / 2 == e->goff)) ? 1 : 0;
  e->split_stride = (int)c.out_split_stride;
}
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn c8_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int g_sms = 0, g_optin = 0;
static const int kSmemBudget = 200 * 1024;
static const int kResidentMax = 112 * 1024;

// geometry shared by the weight packer (stage grouping) and the launcher
int c8_configure(C8Layer* L, int ntaps, const int8_t* dy, const int8_t* dx, int Ci, int Cout, bool stem, const int8_t* tap_cb) {
  L->stem = stem;
  int cb_max = 0;
  for (int t = 0; t < ntaps; ++t) {
    L->tap_cb[t] = tap_cb ? tap_cb[t] : 0;
    cb_max = L->tap_cb[t] > cb_max ? L->tap_cb[t] : cb_max;
  }
  int mn_y = 0, mx_y = 0, mn_x = 0, mx_x = 0;
  for (int t = 0; t < ntaps; ++t) {
    mn_y = dy[t] < mn_y ? dy[t] : mn_y; mx_y = dy[t] > mx_y ? dy[t] : mx_y;
    mn_x = dx[t] < mn_x ? dx[t] : mn_x; mx_x = dx[t] > mx_x ? dx[t] : mx_x;
  }
  const int extra_x = stem ? 5 : 0;   // the stem's GEMM-K walks 6 pixels to the right of the tap origin
  const int HR = C8_TH + (mx_y - mn_y), WR = C8_TW + (mx_x - mn_x) + extra_x;
  TcWeights& w = L->w;
  w.ntaps = ntaps;
  L->mmas64 = (stem || Ci == 48) ? 3 : 4;   // 48 channels = three K16 slices of the one 64-wide unit: the fourth would multiply padding
  if (stem) { w.n64 = 1; w.n32 = 0; }
  else {
    w.n64 = Ci / 64;
    int rem = Ci - 64 * w.n64;
    if (rem > 32) { ++w.n64; rem = 0; }
    w.n32 = rem > 0 ? 1 : 0;
  }
  // the box covers the zero-padded GEMM K (whole 64 / 32 channel chunks): blocks past the tensor are TMA zero fill,
  // so the MMAs never multiply stale shared memory (possibly NaN bit patterns) by the zero weight columns
  // (space-to-depth layers: a tap starts at its own channel block; the zero weight columns of its last chunk may then
  //  multiply the next parity's finite activations instead of TMA zeros, which is just as harmless)
  L->cb_in = stem ? 1 + cb_max : cb_max + (w.n64 * 64 + w.n32 * 32) / 8;   // (split-half stem input: hi block + lo block)
  const long long halo_bytes = (long long)L->cb_in * HR * WR * 16;
  w.NT = (gated_goff(Cout) + Cout / 2 + 15) / 16 * 16;   // every layer on this path is gated: gate columns start at goff
  w.n_tiles = 1;
  w.img_bytes = 0;
  const long long wbytes = (long long)ntaps * w.NT * (w.n64 * 128 + w.n32 * 64);
  // halo re-use while the region stays small enough to sit next to the weight stages (one or two buffers,
  // decided at launch); larger dilations fetch one box per tap
  L->mode = (halo_bytes <= 72 * 1024) ? C8_HALO : C8_PERTAP;
  if (L->mode == C8_HALO) {
    L->HR = HR; L->WR = WR; L->pad_y0 = -mn_y; L->pad_x0 = -mn_x;
  } else {
    L->HR = C8_TH; L->WR = C8_TW; L->pad_y0 = 0; L->pad_x0 = 0;
    L->cb_in = (w.n64 * 64 + w.n32 * 32) / 8;   // a box per tap, starting at the tap's own channel block (C8Params::tap_cb)
  }
  L->a_tx_bytes = L->cb_in * L->HR * L->WR * 16;
  L->a_bytes = (L->a_tx_bytes + 1023) / 1024 * 1024;
  L->resident = (wbytes <= kResidentMax) && (2 * L->a_bytes + wbytes <= kSmemBudget);
  // stage grouping: PERTAP -> one tap per stage; otherwise B-only stages of <= 48 KB (whole taps for mixed chunking)
  if (L->resident && L->mode == C8_HALO) {
    // nothing is streamed per k-step: one k-step issues every MMA of the tile back to back
    w.r64 = ntaps * w.n64;
    w.r32 = ntaps * w.n32;
  } else if (L->mode == C8_PERTAP || (w.n64 > 0 && w.n32 > 0)) { w.r64 = w.n64; w.r32 = w.n32; }
  else {
    const int unit = w.n64 ? w.NT * 128 : w.NT * 64, total = ntaps * (w.n64 ? w.n64 : w.n32);
    int best = 1;
    for (int k = 1; k <= 8 && k <= total; ++k)
      if (total % k == 0 && k * unit <= 48 * 1024) best = k;
    if (w.n64) { w.r64 = best; w.r32 = 0; } else { w.r64 = 0; w.r32 = best; }
  }
  if (L->mode == C8_PERTAP && w.n32 == 0 && w.n64 > 1 && 2 * (L->a_bytes + w.NT * w.n64 * 128) > kSmemBudget) {
    // two stages of a whole tap do not fit (the 192-channel split-half layers): one 64-channel chunk per stage
    L->chunks_per_tap = w.n64;
    L->cb_in = 8;
    L->a_tx_bytes = L->cb_in * L->HR * L->WR * 16;
    L->a_bytes = (L->a_tx_bytes + 1023) / 1024 * 1024;
    w.r64 = 1;
  }
  if (L->mode == C8_PERTAP) SE_REQUIRE(tc_ksteps(w) == ntaps * L->chunks_per_tap, "per-tap stages must be whole taps or whole chunks");
  return 0;
}

// The instantiations: every (N, split-half, k-step shape) that c8_configure / c8_configure_group plan for a layer, fused
// class group or stem pair of the two generators, in both precisions (split-half layers count three product taps per tap).
// This one table selects the kernel of a launch, gets the shared-memory opt-in and keys the cluster-occupancy cache;
// se_model_finalize checks every packed layer against it (c8_instantiated).
// teams = 2: the instantiation also has a two-team form (fn2), which c8_launch runs where its plan allows (c8_teams).
typedef void (*C8Kernel)(CUtensorMap, C8Params);
struct C8Inst { int nt; bool f16; int r64, m64, r32, teams; C8Kernel fn, fn2; };
#define C8_INST(nt, f16, r64, m64, r32) {nt, f16, r64, m64, r32, 1, conv_c8_kernel<nt, f16, r64, m64, r32, 1>, nullptr}
#define C8_INST2(nt, f16, r64, m64, r32) \
  {nt, f16, r64, m64, r32, 2, conv_c8_kernel<nt, f16, r64, m64, r32, 1>, conv_c8_kernel<nt, f16, r64, m64, r32, 2>}
static const C8Inst kC8Insts[] = {
    // bf16 (resident weights: the whole tile is one k-step)
    C8_INST2(32, false, 0, 0, 9),   // 24->24
    C8_INST2(48, false, 0, 0, 9),   // 24->48 stride 2
    C8_INST2(48, false, 4, 3, 0),   // deconv 48->48 class
    C8_INST2(48, false, 5, 3, 0),   // 5x5 stem
    C8_INST2(96, false, 0, 0, 9),   // 24->96 stride 1 and 2
    C8_INST(96, false, 4, 4, 4),    // deconv 96->96 class
    C8_INST2(96, false, 5, 3, 0),   // stem pair
    C8_INST2(96, false, 9, 3, 0),   // 48->96
    // bf16, streamed weights
    C8_INST(96, false, 3, 3, 0),    // 48->96 stride 2
    C8_INST(192, false, 1, 3, 0),   // 48->192 (stride 1 and 2)
    C8_INST(192, false, 1, 4, 0),   // 192->192
    C8_INST(192, false, 1, 4, 1),   // 96->192 (all rates)
    // split-half
    C8_INST2(32, true, 0, 0, 27),   // 24->24 (resident)
    C8_INST(48, true, 0, 0, 3),     // 24->48 stride 2
    C8_INST(48, true, 12, 3, 0),    // deconv 48->48 class (resident; split-half halos leave a ring of two)
    C8_INST2(48, true, 15, 3, 0),   // 5x5 stem (resident)
    C8_INST(96, true, 0, 0, 3),     // 24->96 stride 1 and 2
    C8_INST(96, true, 1, 3, 0),     // 48->96 stride 2 (one box per tap)
    C8_INST(96, true, 1, 4, 1),     // deconv 96->96 class
    C8_INST(96, true, 3, 3, 0),     // 48->96, stem pair
    C8_INST(192, true, 1, 3, 0),    // 48->192 (stride 1 and 2)
    C8_INST(192, true, 1, 4, 0),    // 192->192 (one 64-channel chunk per stage)
    C8_INST(192, true, 1, 4, 1),    // 96->192 (all rates)
};
#undef C8_INST
#undef C8_INST2
static const C8Inst* c8_inst(const C8Layer& L, bool f16) {
  const TcWeights& w = L.w;
  const int r64 = w.n64 ? w.r64 : 0, r32 = w.n32 ? w.r32 : 0, m64 = r64 ? L.mmas64 : 0;
  for (const C8Inst& k : kC8Insts)
    if (k.nt == w.NT && k.f16 == f16 && k.r64 == r64 && k.m64 == m64 && k.r32 == r32) return &k;
  return nullptr;
}
static int c8_set_smem_attr(int bytes) {
  for (const C8Inst& k : kC8Insts) {
    SE_CUDA_OK(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (k.fn2) SE_CUDA_OK(cudaFuncSetAttribute(k.fn2, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  }
  return 0;
}
int c8_instantiated(const C8Layer& L, bool f16, const std::string& name) {
  const TcWeights& w = L.w;
  SE_REQUIRE(c8_inst(L, f16) != nullptr,
             "layer " + name + (f16 ? " (split-half)" : "") + ": no conv_c8_kernel instantiation for N = " + std::to_string(w.NT) +
                 ", k-step of " + std::to_string(w.n64 ? w.r64 : 0) + " x " + std::to_string(L.mmas64) + " + " +
                 std::to_string(w.n32 ? w.r32 : 0) + " x 2 MMAs (se_conv_c8.cu: kC8Insts)");
  return 0;
}
static void c8_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int grid, int teams, int smem_bytes, int cluster, cudaStream_t stream) {
  *cfg = cudaLaunchConfig_t();
  cfg->gridDim = dim3(grid);
  cfg->blockDim = dim3(c8_threads(teams));
  cfg->dynamicSmemBytes = smem_bytes;
  cfg->stream = stream;
  if (cluster > 1) {
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cluster;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg->attrs = attr;
    cfg->numAttrs = 1;
  }
}
// clusters of 2 CTAs that can be resident at once, per (instantiation, shared memory size); asked once, outside graph capture
// (the engine runs a launch sequence eagerly before it captures it)
static int c8_max_clusters(C8Kernel k, int smem_bytes, int* out) {
  static std::mutex mu;
  static std::map<std::pair<C8Kernel, int>, int> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find({k, smem_bytes});
  if (it == cache.end()) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attr;
    c8_launch_config(&cfg, &attr, 2 * g_sms, 1, smem_bytes, 2, 0);
    int n = 0;
    SE_CUDA_OK(cudaOccupancyMaxActiveClusters(&n, k, &cfg));
    SE_REQUIRE(n > 0, "no 2-CTA cluster of conv_c8_kernel fits on the device");
    it = cache.emplace(std::make_pair(k, smem_bytes), n).first;
  }
  *out = it->second;
  return 0;
}

// launch record (se_c8_log_enable): one branch per launch while it is off
struct C8LogEntry { std::string name; int rec[SE_C8_REC_LEN]; };
static std::atomic<bool> g_c8_log{false};
static std::mutex g_c8_log_mu;
static std::vector<C8LogEntry> g_c8_log_recs;
static std::string g_c8_log_label;
bool c8_log_on() { return g_c8_log.load(std::memory_order_relaxed); }
void c8_log_label(const std::string& name) {
  std::lock_guard<std::mutex> lk(g_c8_log_mu);
  g_c8_log_label = name;
}
static void c8_log_append(const C8Params& p, const ConvParams& c, int inst, int teams, int grid, int total_tiles) {
  C8LogEntry e;
  int* r = e.rec;
  r[SE_C8_INST] = inst; r[SE_C8_TEAMS] = teams; r[SE_C8_CLUSTER] = p.cluster; r[SE_C8_GRID] = grid;
  r[SE_C8_TOTAL_TILES] = total_tiles; r[SE_C8_N] = p.N; r[SE_C8_TILES_X] = p.tiles_x; r[SE_C8_TILES_Y] = p.tiles_y;
  r[SE_C8_HO] = p.Ho; r[SE_C8_WO] = p.Wo;
  r[SE_C8_STEP_X] = p.step_x; r[SE_C8_STEP_Y] = p.step_y; r[SE_C8_STEP_IMG] = p.step_img;
  r[SE_C8_CSTEP_X] = p.cstep_x; r[SE_C8_CSTEP_Y] = p.cstep_y; r[SE_C8_CSTEP_IMG] = p.cstep_img;
  r[SE_C8_MODE] = p.mode; r[SE_C8_CPT] = p.cpt; r[SE_C8_NCLS] = p.ncls; r[SE_C8_A_BUFS] = p.a_bufs;
  r[SE_C8_NUM_STAGES] = p.num_stages;
  r[SE_C8_OUT_C8] = c.out_c8; r[SE_C8_CHOFF] = c.choff; r[SE_C8_LDO] = c.ldo;
  r[SE_C8_PHANTOM] = p.cluster > 1 && total_tiles % 2 == 1;
  r[SE_C8_BLK_SPLIT] = c.out_blk_split > 0 ? c.out_blk_split : 0;
  std::lock_guard<std::mutex> lk(g_c8_log_mu);
  e.name = g_c8_log_label;
  g_c8_log_recs.push_back(e);
}

static const int kGroupSmemMax = 222 * 1024;   // fused classes may use (almost) the whole opt-in window: weights of all classes + 2 halos

int c8_configure_group(C8Group* G, int ncls, int ntaps, const int8_t (*dy)[8], const int8_t (*dx)[8], const int* ooy, const int* oox, int Ci, int Cout) {
  if (ncls < 2 || ncls > C8_MAX_CLS || ntaps > 8) return 1;
  int mn_y = 0, mx_y = 0, mn_x = 0, mx_x = 0;
  for (int c = 0; c < ncls; ++c)
    for (int t = 0; t < ntaps; ++t) {
      mn_y = dy[c][t] < mn_y ? dy[c][t] : mn_y; mx_y = dy[c][t] > mx_y ? dy[c][t] : mx_y;
      mn_x = dx[c][t] < mn_x ? dx[c][t] : mn_x; mx_x = dx[c][t] > mx_x ? dx[c][t] : mx_x;
    }
  C8Layer& L = G->geo;
  L = C8Layer();
  TcWeights& w = L.w;
  w.ntaps = ntaps;
  w.n64 = Ci / 64;
  int rem = Ci - 64 * w.n64;
  if (rem > 32) { ++w.n64; rem = 0; }
  w.n32 = rem > 0 ? 1 : 0;
  w.NT = (gated_goff(Cout) + Cout / 2 + 15) / 16 * 16;
  w.n_tiles = 1;
  w.img_bytes = 0;
  w.r64 = ntaps * w.n64;      // resident weights + halo: one k-step issues every MMA of a (tile, class)
  w.r32 = ntaps * w.n32;
  L.mmas64 = Ci == 48 ? 3 : 4;
  if (w.r64 + w.r32 > C8_CLS_UNITS) return 1;
  L.mode = C8_HALO;
  L.resident = true;
  L.stem = false;
  L.cb_in = (w.n64 * 64 + w.n32 * 32) / 8;
  L.HR = C8_TH + (mx_y - mn_y); L.WR = C8_TW + (mx_x - mn_x);
  L.pad_y0 = -mn_y; L.pad_x0 = -mn_x;
  L.a_tx_bytes = L.cb_in * L.HR * L.WR * 16;
  L.a_bytes = (L.a_tx_bytes + 1023) / 1024 * 1024;
  G->ncls = ncls;
  G->ntaps = ntaps;
  G->cls_bytes = ntaps * w.NT * (w.n64 * 128 + w.n32 * 64);
  for (int c = 0; c < ncls; ++c) {
    for (int t = 0; t < ntaps; ++t) { G->dy[c][t] = dy[c][t]; G->dx[c][t] = dx[c][t]; }
    G->ooy[c] = ooy[c]; G->oox[c] = oox[c];
  }
  // weights of all classes + two halo buffers + barriers / constants must fit the opt-in window
  if (1024 + ncls * G->cls_bytes + 2 * L.a_bytes + 4096 > kGroupSmemMax) return 1;
  return 0;
}

int c8_launch(const ConvParams& c, const C8Layer& L_in, cudaStream_t stream, const C8Group* grp) {
  const C8Layer& L = grp ? grp->geo : L_in;
  const TcWeights& w = L.w;
  SE_REQUIRE((c.in_dt == DT_BF16 || c.in_dt == DT_F16X2) && c.in_c8 == 1, "conv_c8 reads 16-bit channel-blocked activations");
  SE_REQUIRE((c.in_dt == DT_F16X2) == (c.f16x2 != 0) && (c.out_dt == DT_F16X2) == (c.f16x2 != 0), "split-half mode: both sides");
  SE_REQUIRE(c.stride == 1, "conv_c8 handles stride-1 convolutions");
  SE_REQUIRE((reinterpret_cast<uintptr_t>(c.x) & 127) == 0, "input base must be 128 B aligned");
  SE_REQUIRE(c.ntaps == w.ntaps && c.ntaps <= MAX_TAPS, "tap count mismatch");
  for (int t = 0; t < c.ntaps && !grp; ++t) SE_REQUIRE(c.tap_cb[t] == L.tap_cb[t], "per-tap channel blocks differ from the packed layer");
  SE_REQUIRE(c.Wi * 8 <= (1 << 30) && L.WR * 8 <= 256 && L.HR <= 256 && L.cb_in <= 256, "TMA box limits");
  SE_REQUIRE(c.epi == EPI_GATE_ELU || c.epi == EPI_GATE_RELU, "conv_c8 runs gated epilogues only");
  SE_REQUIRE(w.NT == 2 * gated_goff(c.Cout), "gated layers keep the gate columns in the upper half of the tile");
  C8Params p;
  memset(&p, 0, sizeof(p));
  p.f16 = c.f16x2 ? 1 : 0;
  for (int t = 0; t < c.ntaps; ++t) p.tap_cb[t] = L.tap_cb[t];
  p.N = c.N; p.Ho = c.Ho; p.Wo = c.Wo;
  p.tiles_x = (c.Wo + C8_TW - 1) / C8_TW;
  p.tiles_y = (c.Ho + C8_TH - 1) / C8_TH;
  p.ntaps = c.ntaps;
  memcpy(p.dy, c.dy, sizeof(p.dy));
  memcpy(p.dx, c.dx, sizeof(p.dx));
  p.n64 = w.n64; p.n32 = w.n32; p.NT = w.NT;
  p.ksteps = tc_ksteps(w);
  p.w = reinterpret_cast<const uint8_t*>(grp ? grp->w_all : w.data);
  p.mode = L.mode; p.HR = L.HR; p.WR = L.WR; p.pad_y0 = L.pad_y0; p.pad_x0 = L.pad_x0;
  p.cb_in = L.cb_in; p.x_cb_off = c.x_cb_off; p.cpt = L.chunks_per_tap;
  p.a_bytes = L.a_bytes; p.a_tx_bytes = L.a_tx_bytes;
  p.resident = L.resident ? 1 : 0;
  p.wres_bytes = grp ? grp->ncls * grp->cls_bytes : (int)tc_weight_bytes_per_image(w);
  p.ncls = grp ? grp->ncls : 1;
  p.cls_bytes = grp ? grp->cls_bytes : 0;
  for (int k = 0; k < C8_MAX_CLS; ++k) { p.cls_ooy[k] = grp && k < grp->ncls ? grp->ooy[k] : 0; p.cls_oox[k] = grp && k < grp->ncls ? grp->oox[k] : 0; }
  if (L.stem) { p.lbo_bytes = 16; p.kstep_bytes = 32; }
  else { p.lbo_bytes = L.HR * L.WR * 16; p.kstep_bytes = 2 * p.lbo_bytes; }
  p.sbo_bytes = L.WR * 16;
  p.bias = c.bias;
  fill_epi(c, w.NT, &p.e);
  {
    // A-operand byte offsets inside the shared-memory region, per K unit (tile independent):
    // 64-wide units first (u = tap*n64 + chunk), then the 32-wide unit of each tap
    const bool halo = (L.mode == C8_HALO);
    const int n_u64 = c.ntaps * w.n64, n_u32 = c.ntaps * w.n32;
    SE_REQUIRE(n_u64 + n_u32 < C8_MAX_UNITS, "too many K units");
    SE_REQUIRE(!grp || n_u64 + n_u32 <= C8_CLS_UNITS, "too many K units per class");
    for (int k = 0; k < (grp ? grp->ncls : 1); ++k)
      for (int u = 0; u < n_u64 + n_u32; ++u) {
        const bool is64 = u < n_u64;
        const int t = is64 ? u / w.n64 : u - n_u64;
        // PERTAP: the box starts at the tap's block (at the unit's own chunk when cpt > 1)
        const int cb0 = L.chunks_per_tap > 1 ? 0 : (halo ? L.tap_cb[t] : 0) + (is64 ? (u - t * w.n64) * 8 : w.n64 * 8);
        const int tdy = grp ? grp->dy[k][t] : c.dy[t], tdx = grp ? grp->dx[k][t] : c.dx[t];
        const int oy = halo ? tdy + L.pad_y0 : 0, ox = halo ? tdx + L.pad_x0 : 0;
        p.aoff[k * C8_CLS_UNITS + u] = (uint32_t)((cb0 * L.HR + oy) * L.WR + ox) * 16u;
      }
  }
  SE_REQUIRE(c.Cout % 2 == 0 && (c.out_dt == DT_BF16 || c.out_dt == DT_F16X2), "gated epilogue needs even Cout, 16-bit out");
  SE_REQUIRE(!c.out_c8 || c.choff % 8 == 0, "C8 output needs a channel offset multiple of 8");
  SE_REQUIRE(!c.f16x2 || c.out_c8 != 0, "split-half output is channel-blocked");
  SE_REQUIRE(c.out_c8 != 2 || (c.Hout % 2 == 0 && c.Wout % 2 == 0 && c.ldo % 4 == 0 && (c.Cout / 2) % 8 == 0),
             "space-to-depth output: even size, whole channel blocks");
  {
    const long long plane = c.out_c8 == 2 ? (long long)(c.Hout / 2) * (c.Wout / 2) : (long long)c.Hout * c.Wout;
    SE_REQUIRE((long long)(w.NT / 16) * (c.out_c8 ? 8 * plane : 8) + 8LL * p.e.blk_jump < (1LL << 31), "output block offsets must fit in 31 bits");
  }

  const int total_tiles = p.N * p.tiles_x * p.tiles_y;
  const int smem_budget = grp ? kGroupSmemMax - 4096 : kSmemBudget;
  const int b_bytes = tc_stage_b_bytes(w);
  const int stage_bytes = (L.mode == C8_HALO ? 0 : L.a_bytes) + (L.resident ? 0 : b_bytes);
  int fixed = (L.resident ? p.wres_bytes : 0);
  // halo ring: two buffers (one if they do not fit next to three weight stages); with nothing streamed per k-step a tile is
  // short against a TMA round trip, so the ring is as deep as shared memory allows
  p.a_bufs = 2;
  if (L.mode == C8_HALO) {
    if (fixed + 2 * L.a_bytes + 3 * stage_bytes > smem_budget) p.a_bufs = 1;
    if (stage_bytes == 0)
      while (p.a_bufs < C8_MAX_ABUFS && fixed + 2 * p.a_bufs * L.a_bytes <= smem_budget) p.a_bufs *= 2;
    fixed += p.a_bufs * L.a_bytes;
  }
  p.a_shift = -1;
  for (int sh = 0; sh < 4; ++sh) if ((1 << sh) == p.a_bufs) p.a_shift = sh;
  SE_REQUIRE(p.a_bufs <= C8_MAX_ABUFS, "halo ring plan");
  SE_REQUIRE(!grp || (p.a_bufs >= 2 && p.ksteps == 1), "fused classes need two halo buffers and a single k-step");
  SE_REQUIRE(!(L.resident && p.ksteps == 1) || p.a_bufs >= 2, "ping-pong warpgroups need two halo buffers");
  int stages = stage_bytes ? (smem_budget - fixed) / stage_bytes : 1;
  if (stages > C8_MAX_STAGES) stages = C8_MAX_STAGES;
  SE_REQUIRE(stages >= (stage_bytes ? 2 : 1), "shared memory plan does not fit");
  p.num_stages = stages;
  const int smem_bytes = 1024 + fixed + stages * stage_bytes + (2 * C8_MAX_STAGES + 2 * C8_MAX_ABUFS + 2) * 8 + 3 * (p.NT + 32) * 4 + 64;

  EncodeTiledFn enc = c8_encode_fn();
  SE_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
  if (!g_sms) {
    int dev = 0;
    SE_CUDA_OK(cudaGetDevice(&dev));
    SE_CUDA_OK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev));
    SE_CUDA_OK(cudaDeviceGetAttribute(&g_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    { int rc_attr = c8_set_smem_attr(g_optin); if (rc_attr) return rc_attr; }
  }
  SE_REQUIRE(smem_bytes <= g_optin, "shared memory plan exceeds the opt-in limit");

  CUtensorMap tmA;
  {
    // C8 activations viewed as (8*W, H, CB, N): a row of the box is WR pixels x 16 B, contiguous in memory
    cuuint64_t dims[4] = {(cuuint64_t)c.Wi * 8, (cuuint64_t)c.Hi, (cuuint64_t)c.ldx, (cuuint64_t)c.N};
    cuuint64_t strides[3] = {(cuuint64_t)c.Wi * 16, (cuuint64_t)c.Hi * c.Wi * 16, (cuuint64_t)c.ldx * c.Hi * c.Wi * 16};
    cuuint32_t box[4] = {(cuuint32_t)(L.WR * 8), (cuuint32_t)L.HR, (cuuint32_t)L.cb_in, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(c.x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    SE_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(C8) failed, CUresult=" + std::to_string((int)r));
  }
  const C8Inst* inst = c8_inst(L, p.f16 != 0);
  SE_REQUIRE(inst != nullptr, "no conv_c8_kernel instantiation for the layer's plan (N = " + std::to_string(p.NT) + ")");
  // streamed weights: 2-CTA clusters read each weight stage from L2 once per pair of neighbouring tiles (TMA multicast)
  p.cluster = L.resident ? 1 : 2;
  int grid = total_tiles < g_sms ? total_tiles : g_sms;
  // Two teams: a ping-pong launch (resident weights, one k-step) whose instantiation has the two-team form, whose CTAs run
  // at least two tiles, and whose halo ring holds a buffer per team and two more to load ahead into
  const int teams = (inst->teams == 2 && L.resident && p.ksteps == 1 && p.a_bufs >= 4 && total_tiles > grid) ? 2 : 1;
  const C8Kernel kernel = teams == 2 ? inst->fn2 : inst->fn;
  if (p.cluster > 1) {
    int max_clusters = 0;
    { int rc_occ = c8_max_clusters(kernel, smem_bytes, &max_clusters); if (rc_occ) return rc_occ; }
    const int pairs = (total_tiles + 1) / 2;
    grid = 2 * (pairs < max_clusters ? pairs : max_clusters);
  }
  p.step_x = grid % p.tiles_x;
  p.step_y = (grid / p.tiles_x) % p.tiles_y;
  p.step_img = grid / (p.tiles_x * p.tiles_y);
  p.cstep_x = (teams * grid) % p.tiles_x;
  p.cstep_y = (teams * grid / p.tiles_x) % p.tiles_y;
  p.cstep_img = teams * grid / (p.tiles_x * p.tiles_y);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr;
  c8_launch_config(&cfg, &attr, grid, teams, smem_bytes, p.cluster, stream);
  SE_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, tmA, p));
  if (c8_log_on()) c8_log_append(p, c, (int)(inst - kC8Insts), teams, grid, total_tiles);
  return 0;
}

}  // namespace se

// ============================================================================================ C ABI: launch record
extern "C" {

int se_c8_log_enable(int on) {
  std::lock_guard<std::mutex> lk(se::g_c8_log_mu);
  se::g_c8_log = on != 0;
  se::g_c8_log_recs.clear();
  se::g_c8_log_label.clear();
  return 0;
}

int se_c8_log_count(void) {
  std::lock_guard<std::mutex> lk(se::g_c8_log_mu);
  return (int)se::g_c8_log_recs.size();
}

int se_c8_log_get(int i, char* name, int name_cap, int* rec) {
  std::lock_guard<std::mutex> lk(se::g_c8_log_mu);
  SE_REQUIRE(i >= 0 && i < (int)se::g_c8_log_recs.size(),
             "launch record index " + std::to_string(i) + " of " + std::to_string(se::g_c8_log_recs.size()));
  const se::C8LogEntry& e = se::g_c8_log_recs[i];
  if (name && name_cap > 0) {
    const size_t n = std::min(e.name.size(), (size_t)name_cap - 1);
    memcpy(name, e.name.data(), n);
    name[n] = 0;
  }
  if (rec) memcpy(rec, e.rec, sizeof(e.rec));
  return 0;
}

int se_c8_inst_count(void) { return (int)(sizeof(se::kC8Insts) / sizeof(se::kC8Insts[0])); }

int se_c8_inst_info(int i, int* info) {
  SE_REQUIRE(i >= 0 && i < se_c8_inst_count() && info, "instantiation index " + std::to_string(i) + " of " + std::to_string(se_c8_inst_count()));
  const se::C8Inst& k = se::kC8Insts[i];
  info[SE_C8_INST_NT] = k.nt; info[SE_C8_INST_F16] = k.f16 ? 1 : 0; info[SE_C8_INST_R64] = k.r64;
  info[SE_C8_INST_M64] = k.m64; info[SE_C8_INST_R32] = k.r32; info[SE_C8_INST_TEAMS] = k.teams;
  return 0;
}

}  // extern "C"

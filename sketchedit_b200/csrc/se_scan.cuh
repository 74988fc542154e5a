// Exclusive scan of unsigned counts into 64-bit offsets over a whole device array, shared by the entropy coders
// (se_jpeg.cu, se_png.cu): per tile of SCAN_TILE counts a block scan, one block scans the tile sums, then the sums are added.
#pragma once
#include "se_common.cuh"

namespace se {

constexpr int SCAN_T = 256, SCAN_V = 8, SCAN_TILE = SCAN_T * SCAN_V;

template <int NT>
__device__ __forceinline__ unsigned long long block_exclusive_scan(unsigned long long v, unsigned long long* total) {
  __shared__ unsigned long long warp_sum[NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    unsigned long long s = lane < NT / 32 ? warp_sum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < NT / 32) warp_sum[lane] = s;
  }
  __syncthreads();
  const unsigned long long before = (wid ? warp_sum[wid - 1] : 0) + x - v;
  *total = warp_sum[NT / 32 - 1];
  __syncthreads();   // warp_sum is reused by the next call
  return before;
}

static __global__ void __launch_bounds__(SCAN_T) scan_tiles(const unsigned* in, unsigned long long* out, unsigned long long* sums,
                                                      long long n) {
  const long long base = (long long)blockIdx.x * SCAN_TILE + (long long)threadIdx.x * SCAN_V;
  unsigned v[SCAN_V];
  unsigned long long s = 0;
#pragma unroll
  for (int j = 0; j < SCAN_V; ++j) {
    v[j] = base + j < n ? in[base + j] : 0u;
    s += v[j];
  }
  unsigned long long total;
  unsigned long long run = block_exclusive_scan<SCAN_T>(s, &total);
#pragma unroll
  for (int j = 0; j < SCAN_V; ++j) {
    if (base + j < n) out[base + j] = run;
    run += v[j];
  }
  if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

static __global__ void __launch_bounds__(1024) scan_sums(unsigned long long* sums, long long n) {
  unsigned long long carry = 0;
  for (long long c = 0; c < n; c += 1024) {
    const long long i = c + threadIdx.x;
    const unsigned long long v = i < n ? sums[i] : 0;
    unsigned long long total;
    const unsigned long long before = block_exclusive_scan<1024>(v, &total);
    if (i < n) sums[i] = carry + before;
    carry += total;
  }
}

static __global__ void __launch_bounds__(SCAN_T) scan_add(unsigned long long* out, const unsigned long long* sums, long long n) {
  const long long i = (long long)blockIdx.x * SCAN_T + threadIdx.x;
  if (i < n) out[i] += sums[i / SCAN_TILE];
}

static int exclusive_scan(const unsigned* in, unsigned long long* out, unsigned long long* sums, long long n, cudaStream_t st) {
  const long long tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  scan_tiles<<<(unsigned)tiles, SCAN_T, 0, st>>>(in, out, sums, n);
  scan_sums<<<1, 1024, 0, st>>>(sums, tiles);
  scan_add<<<(unsigned)((n + SCAN_T - 1) / SCAN_T), SCAN_T, 0, st>>>(out, sums, n);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

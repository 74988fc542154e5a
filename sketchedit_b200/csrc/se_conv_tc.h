// Weight stage images of the wgmma convolution (se_conv_c8.cu): the swizzled shared-memory layout shared by the packer
// (se_engine.cu) and the kernel.
#pragma once
#include "se_common.cuh"

namespace se {

// The GEMM K axis of one tap is cut into `n64` chunks of 64 channels (128 B rows, SWIZZLE_128B) followed by
// `n32` (0 or 1) chunk of 32 channels (64 B rows, SWIZZLE_64B); channels beyond Ci are zero (TMA OOB fill).
// One pipeline stage holds r64 consecutive 64-wide units and r32 consecutive 32-wide units.
//
// Weights are stored in global memory as the exact shared-memory image of each stage (already swizzled),
// so a stage's B operand is ONE linear cp.async.bulk:
//   image(img, n_tile, kstep) at  data + img*img_bytes + (n_tile*ksteps + kstep) * stage_b_bytes
//   = r64 x [NT rows x 128 B] followed by r32 x [NT rows x 64 B]
struct TcWeights {
  const void* data = nullptr;   // device, bf16, pre-swizzled stage images
  int ntaps = 0;
  int n64 = 0, n32 = 0;         // chunks per tap
  int r64 = 0, r32 = 0;         // units per pipeline stage
  int NT = 0;                   // GEMM N per tile (Cout padded to 16), <= 256
  int n_tiles = 1;
  long long img_bytes = 0;      // bytes between images for per-image weights (attention), 0 = shared
};

inline int tc_ksteps(const TcWeights& w) { return w.n64 ? w.ntaps * w.n64 / w.r64 : w.ntaps * w.n32 / w.r32; }
inline int tc_stage_b_bytes(const TcWeights& w) { return w.NT * (w.r64 * 128 + w.r32 * 64); }
inline long long tc_weight_bytes_per_image(const TcWeights& w) { return (long long)w.n_tiles * tc_ksteps(w) * tc_stage_b_bytes(w); }

// byte offset of (row r, byte kb within the row) inside a K-major operand tile with RB-byte rows whose base is
// 1024 B aligned: the 128B / 64B TMA + wgmma swizzle (cute Swizzle<3,4,3> / Swizzle<2,4,3>).
__host__ __device__ inline uint32_t tc_swizzle_offset(int r, int kb, int RB) {
  uint32_t off = (uint32_t)r * RB + kb;
  return off ^ (((off >> 7) & (RB == 128 ? 7u : 3u)) << 4);
}

// where element (unit kind/index, n, k) of a stage lands inside the stage's B image
__host__ __device__ inline uint32_t tc_b_image_offset(int NT, int r64, bool is64, int j, int n, int k) {
  if (is64) return (uint32_t)j * NT * 128 + tc_swizzle_offset(n, k * 2, 128);
  return (uint32_t)r64 * NT * 128 + (uint32_t)j * NT * 64 + tc_swizzle_offset(n, k * 2, 64);
}

void fill_epi(const ConvParams& c, int NT, EpiParams* e);

}  // namespace se

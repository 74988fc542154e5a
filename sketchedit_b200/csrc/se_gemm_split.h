// Contextual attention of the fp32-on-tensor-cores mode: split-half fp16 wgmma GEMMs over explicit patch matrices (se_gemm_split.cu).
#pragma once
#include "se_common.cuh"

namespace se {

struct CamSplitPlan {
  int B, h, w, C;
  int hs, ws, L;     // patch grid (4x4 patches, stride 2) and its size
  int Mp;            // L rounded up to 256: rows of every patch matrix, pitch of S
  int KQ;            // 16 * C: K of the S GEMM, N of the PV GEMM
  int band;          // query rows (M rows of both GEMMs) per band: Mp (one band) or a multiple of 128
  int n_bands;
  size_t q_bytes;    // query (= value) patches and normalised key patches, each
  size_t s_bytes, p_bytes, o_bytes;   // S and P: one band
};
// limit: bytes S and P may take together (the quadratic buffers)
int cam_split_plan(int B, int h, int w, int C, long long limit, CamSplitPlan* out);

// f: fp32 NHWC [B][h][w][C]; rnorm: fp32 [B][C] (1 / plane norm); colmask: fp32 [B][L] (0 / 1 per key); out: fp32 NHWC [B][h][w][C].
// Q, Kn (q_bytes each), S (s_bytes), P (p_bytes), O (o_bytes): workspace, 128 B aligned. attn (optional): fp32 [B][L][L], the
// softmax weights as computed before their split, in cam_1's layout [key][query].
int cam_forward_split(const float* f, const float* rnorm, const float* colmask, float* out, const CamSplitPlan& pl, void* Q, void* Kn, float* S, void* P,
                      float* O, float* attn, cudaStream_t stream);

// One split-half GEMM C = scale * (A_hi B_hi + A_hi B_lo + A_lo B_hi), C fp32 [M][N] row-major. A: fp16 [hi | lo][K / 8][M][8]
// (K-major, K-blocked), B: fp16 [hi | lo][N / 8][K][8] (MN-major: rows are K). M, K, N multiples of 128, 32 and 256; A and B
// 128 B aligned. Operands stored times a power of two come back through scale.
int gemm_split_mn(const void* A, const void* B, float* C, int M, int K, int N, float scale, cudaStream_t stream);

}  // namespace se

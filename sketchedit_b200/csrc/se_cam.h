// Contextual attention on the tensor cores, straight from the space-to-depth channel-blocked feature map (se_cam.cu).
#pragma once
#include "se_common.cuh"

namespace se {

// workspace sizes for a batch of B maps of h x w (C = 96): normalised copy of the map, per-key logit scale, probabilities
struct CamPlan {
  int B, h, w;
  int Hs, Ws;       // space-to-depth planes (h/2 x w/2) = grid of one sub-pixel output class
  int hs, ws;       // patch grid (4x4 patches, stride 2): Hs - 1, Ws - 1
  int tq_x;         // query tiles (16 x 8 patches) per row
  int tk_x, KT;     // key tiles (32 x 8 patches = 256 keys) per row / per image
  int KB;           // 8-key blocks of P per image = KT * 32
  int to_x;         // output tiles (8 x 8 positions of the class grid) per row
  int band;         // query rows per band: hs (one band) or a multiple of 16
  int n_bands;
  int prows;        // rows of the P buffer: hs for one band, band + 1 (the carried row q0 - 1) otherwise
  size_t fn_bytes, cs_bytes, p_bytes;
};
// limit: bytes P may take (the only quadratic buffer); single_band ignores it (the caller keeps the whole P, e.g. for attn)
int cam_plan(int B, int h, int w, long long limit, bool single_band, CamPlan* out);

// f_s2d: bf16 [B][4*12][h/2][w/2][8] (space-to-depth channel-blocked, 96 channels); mask_s: fp32 [B][h][w];
// out_c8: bf16 [B][12][h][w][8]. fn / colscale / P: workspace of the sizes cam_plan reports.
// attn (optional, one band only): fp32 [B][L][hs*ws] softmax weights in the reference's cam_1 layout (tests / module surface only).
int cam_forward_tc(const void* f_s2d, const float* mask_s, void* out_c8, const CamPlan& pl, void* fn, float* colscale, void* P, float* attn,
                   cudaStream_t stream);

}  // namespace se

// Contextual attention on the tensor cores, straight from the space-to-depth channel-blocked feature map (se_cam.cu).
#pragma once
#include "se_common.cuh"

namespace se {

// workspace sizes for a batch of B maps of h x w (C = 96): normalised copy of the map, per-key logit scale, probabilities
struct CamPlan {
  int B, h, w;
  int Hs, Ws;       // space-to-depth planes (h/2 x w/2) = grid of one sub-pixel output class
  int hs, ws;       // patch grid (4x4 patches, stride 2): Hs - 1, Ws - 1
  int tq_x, tq_n;   // query tiles (16 x 8 patches) per row / per image
  int tk_x, KT;     // key tiles (32 x 8 patches = 256 keys) per row / per image
  int KB;           // 8-key blocks of P per image = KT * 32
  int to_x, to_n;   // output tiles (8 x 8 positions of the class grid) per row / per image
  size_t fn_bytes, cs_bytes, p_bytes;
};
int cam_plan(int B, int h, int w, CamPlan* out);

// f_s2d: bf16 [B][4*12][h/2][w/2][8] (space-to-depth channel-blocked, 96 channels); mask_s: fp32 [B][h][w];
// out_c8: bf16 [B][12][h][w][8]. fn / colscale / P: workspace of the sizes cam_plan reports.
// attn (optional): fp32 [B][L][hs*ws] softmax weights in the reference's cam_1 layout (tests / module surface only).
int cam_forward_tc(const void* f_s2d, const float* mask_s, void* out_c8, const CamPlan& pl, void* fn, float* colscale, void* P, float* attn,
                   cudaStream_t stream);

}  // namespace se

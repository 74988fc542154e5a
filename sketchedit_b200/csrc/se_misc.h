// Glue kernels (se_misc.cu). dt = activation storage (DT_F32 / DT_BF16 / DT_F16X2, se_common.cuh).
#pragma once
#include "se_common.cuh"

namespace se {

enum { PACK_IMG_ONE = 0, PACK_IMG_ONE_MINUS_M = 1, PACK_IMG_M = 2 };
enum { HEAD_MASK = 0, HEAD_TANH = 1, HEAD_COARSE = 2, HEAD_FINE = 3 };
enum { RED_MAX = 0, RED_AVG = 1, RED_RNORM = 2 };

// Where an activation of B images lives (the numbering of SE_TAP_LAYOUT). ld: NHWC pixel pitch in elements, else channel blocks
// per image, both halves of a split-half tensor counted.
//   LAYOUT_NHWC  [B][H][W][ld]
//   LAYOUT_C8    channel-blocked [B][ld][H][W][8]; split-half: the lo blocks ld / 2 blocks after the hi blocks
//   LAYOUT_S2D   channel-blocked space-to-depth [B][ld][H/2][W/2][8]: pixel (y, x) in parity group (y&1)*2 + (x&1) of ld / 4
//                blocks (split-half: hi, then lo blocks, per group); H, W: the full-resolution size
//   LAYOUT_ROWS  packed 8-channel rows [B][halves][H][Wp][8], the image at x + padl
enum { LAYOUT_NHWC = 0, LAYOUT_C8 = 1, LAYOUT_S2D = 2, LAYOUT_ROWS = 3 };
struct Layout { int kind, H, W, ld, Wp, padl; };

int pack8(const float* img, const float* sketch, const float* mask, void* out, int dt, int B, int H, int W, int Wp, int padl,
          int img_mode, float sketch_scale, int write_mask, cudaStream_t s, int img2_mode = -1);   // img2_mode >= 0: channels 5..7 = img * f(mask)
// One head launch, passed by value. Outputs are written where set; *_bs: elements between images, 0 = dense. x: fp32 NHWC
// [B][H][W][12] or two channel blocks. blend: the mask blended with, [B,H,W] (HEAD_COARSE: the binarised one, dense; HEAD_FINE:
// the soft one). stage: the tanh result [B,cout,H,W]. packed: HEAD_COARSE's blend in packed rows as pack8 writes them.
struct HeadIO {
  const void* x;
  int B, H, W, mode;
  const float *img, *blend;
  long long blend_bs;
  float* mask;                       // HEAD_MASK: sigmoid, with its binarised plane and bytes
  long long mask_bs;
  float* mask_bin;
  unsigned char* mask_u8;
  float *stage, *composed;           // HEAD_FINE: composed, with its BGR HWC bytes
  long long composed_bs;
  unsigned char* bgr_u8;
  void* packed;
  int Wp, padl, no_mask_coarse;
};
// w_host / b_host: host copies of the [9][12][cout] weights and the bias (the kernel parameters are built from them)
int head(HeadIO io, int dt, const float* w_host, const float* b_host, int cout, cudaStream_t s);
// fp32: NHWC with pixel pitch ld; bf16 / split-half: channel-blocked with ld blocks per image (max / avg only)
int plane_reduce(const void* x, int dt, int B, int HW, int C, int ld, int mode, float* out, cudaStream_t s);
// v [B][C] into channels [choff, choff + C) of every pixel: fp32 NHWC (pitch ld), else channel-blocked (ld blocks per image)
int broadcast_channels(const float* v, void* y, int dt, int B, int HW, int C, int ld, int choff, cudaStream_t s);
int avgpool4(const float* m, float* out, int B, int H, int W, cudaStream_t s);
int cam_colmask(const float* mask_s, float* out, int B, int h, int w, int hs, int ws, float th, cudaStream_t s);
int cam_pack_k(const float* f, const float* rnorm, float* out, int B, int h, int w, int C, int ws, int L, int Lpad, cudaStream_t s);
int cam_pack_v(const float* f, float* out, int B, int h, int w, int C, int ws, int L, int Lpad, cudaStream_t s);
int softmax_rows(const float* S, int lds, float* P, int ldp, long long rows, int L, cudaStream_t s);
// fp32 [B][C][v.H][v.W] (nhwc: [B][v.H][v.W][C]) -> channels [0, C) of the activation y in layout v, and back
int f32_to_act(const float* x, int nhwc, void* y, int dt, const Layout& v, int B, int C, cudaStream_t s);
int act_to_f32(const void* x, int dt, const Layout& v, float* y, int nhwc, int B, int C, cudaStream_t s);
// mask_u8: an edit mask's bytes [B,H,W] or null; decoded into its soft plane v/255 and binarised plane (v/255 > 0.5), fp32 [B,H,W]
int u8_to_inputs(const unsigned char* img_u8, const unsigned char* sk_u8, const unsigned char* mask_u8, float* img, float* sk, float* mask_soft,
                 float* mask_bin, int B, int H, int W, cudaStream_t s);
// out[i] = m[i] > 0.5 ? 1 : 0 over n floats
int binarise(const float* m, float* out, long long n, cudaStream_t s);
int to_uint8(const float* comp, const float* mask, unsigned char* bgr, unsigned char* mk, int B, int H, int W, cudaStream_t s);
int fill_zero(void* p, size_t bytes, cudaStream_t s);

}  // namespace se

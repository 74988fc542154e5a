// Shared device/host helpers for the sketchedit_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

namespace se {

// ------------------------------------------------------------------------------------------
// error plumbing: every C-ABI entry point returns 0 on success, non-zero on failure and leaves
// a message retrievable through se_last_error().
void set_error(const std::string& msg);
const char* last_error();

#define SE_CUDA_OK(expr)                                                                      \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      se::set_error(std::string(#expr) + " -> " + cudaGetErrorString(_e) + " at " + __FILE__ + \
                    ":" + std::to_string(__LINE__));                                          \
      return 1;                                                                               \
    }                                                                                         \
  } while (0)

#define SE_REQUIRE(cond, msg)                                                                 \
  do {                                                                                        \
    if (!(cond)) {                                                                            \
      se::set_error(std::string("requirement failed: ") + #cond + " : " + (msg) + " at " +    \
                    __FILE__ + ":" + std::to_string(__LINE__));                               \
      return 2;                                                                               \
    }                                                                                         \
  } while (0)

// ------------------------------------------------------------------------------------------
// batch entries of the image I/O (resize, composite, detail, JPEG and PNG codecs)
constexpr int kMaxDim = 65535;   // largest image side they take: the JPEG header's 16-bit size fields

// scratch arrays start at multiples of 256 bytes
inline size_t scratch_round(size_t bytes) { return (bytes + 255) / 256 * 256; }
// blocks of per_block threads covering `threads` threads; also tiles of per_block covering a length
inline unsigned grid_of(long long threads, int per_block) { return (unsigned)((threads + per_block - 1) / per_block); }

// The scratch protocol of a batch entry that takes (void* scratch, long long* scratch_bytes): without scratch the call is a
// query and stores the bytes it needs; with it, the scratch must hold them. Either way a call of no images ends here.
#define SE_SCRATCH(scratch, scratch_bytes, need, n)                                                                  \
  do {                                                                                                               \
    const long long _need = (long long)(need);                                                                       \
    if (!(scratch)) {                                                                                                \
      *(scratch_bytes) = _need;                                                                                      \
      return 0;                                                                                                      \
    }                                                                                                                \
    SE_REQUIRE(*(scratch_bytes) >= _need,                                                                            \
               "scratch holds " + std::to_string(*(scratch_bytes)) + " bytes, needs " + std::to_string(_need));     \
    if ((n) == 0) return 0;                                                                                          \
  } while (0)

// the sides of item i ("image", "box", "file") of a batch
inline int check_sides(const char* item, int i, int h, int w) {
  SE_REQUIRE(h >= 1 && w >= 1 && h <= kMaxDim && w <= kMaxDim, std::string(item) + " " + std::to_string(i) + ": sizes must be in [1, 65535]");
  return 0;
}

// window i of the encoders and the resize: its sides, its output offset and a source pitch of at least its row of `row` bytes
inline int check_window(int i, int h, int w, long long pitch, long long row, long long out_off) {
  if (int rc = check_sides("image", i, h, w)) return rc;
  SE_REQUIRE(out_off >= 0, "negative offset");
  SE_REQUIRE(pitch >= row, "image " + std::to_string(i) + ": the source pitch of " + std::to_string(pitch) +
                               " bytes is narrower than its row of " + std::to_string(row) + " bytes");
  return 0;
}

#ifdef __CUDACC__
// The image of a batch that unit g (a tile, block or chunk of the launch) belongs to: images hold consecutive units from
// their member `first` on, so it is the last image whose first unit is at or before g.
template <typename D, typename T>
__device__ __forceinline__ int image_of(const D* im, int n, T D::*first, T g) {
  int i = 0;
  while (i + 1 < n && g >= im[i + 1].*first) ++i;
  return i;
}
#endif

// ------------------------------------------------------------------------------------------
// tile geometry shared by every convolution kernel: one CTA tile = 8 x 16 output positions
constexpr int TILE_H = 8;
constexpr int TILE_W = 16;
constexpr int TILE_M = TILE_H * TILE_W;  // 128 = two wgmma M = 64 halves
constexpr int MAX_TAPS = 64;              // 9 taps x 3 operand-split products (+ space-to-depth / deconv variants)
constexpr int KCHUNK = 32;               // bf16 elements per K chunk = 64 B = SWIZZLE_64B span

enum Epilogue : int {
  EPI_GATE_ELU = 0,   // ELU(y[c]) * sigmoid(y[c + Cout/2])              (reference utils.py:29-32)
  EPI_GATE_RELU = 1,  // ReLU(y[c]) * sigmoid(y[c + Cout/2])             (pmconv6, editline_g.py:89-90)
  EPI_LINEAR = 2,     // (y[c] + bias[c]) * scale * colscale[n][c]       (raw conv / attention GEMMs)
};

enum DType : int { DT_BF16 = 0, DT_F32 = 1, DT_F16X2 = 2 };
// DT_F16X2: "split half" storage of an fp32 tensor for the fp32-on-tensor-cores mode: value = hi + lo with hi = fp16(v),
// lo = fp16(v - hi) (22 significant bits). A channel-blocked tensor keeps the hi blocks first and the lo blocks `CB` blocks
// further on ([N][2*CB][H][W][8]; space-to-depth: per parity group). A convolution then is three wgmma products per tap,
// x_hi*w_hi + x_hi*w_lo + x_lo*w_hi (the dropped lo*lo term is 2^-22 relative), accumulated in fp32.

// One generalised convolution launch. Positions p=(py,px) on an Ho x Wo grid; input pixel for tap t
// is (py*stride + dy[t], px*stride + dx[t]) (zero outside the image); output pixel is
// (py*osy + ooy, px*osx + oox) inside an Hout x Wout image with pixel pitch ldo and channel
// offset choff. Weights may differ per image (attention), w_img_stride = 0 otherwise.
struct ConvParams {
  // input
  const void* x;        // NHWC, dtype in_dt, pixel pitch ldx elements (or C8, see in_c8)
  int in_dt;
  int in_c8;            // 1: input is C8 = [N][ldx blocks][Hi][Wi][8] starting at channel block x_cb_off (se_conv_c8.cu only)
  int x_cb_off;
  int N, Hi, Wi, Ci, ldx;
  long long x_row_pitch, x_img_pitch;   // elements; 0 = dense (Wi*ldx, Hi*Wi*ldx). ldx may be < Ci (overlapping windows)
  // position grid + taps
  int Ho, Wo, stride;
  int ntaps;
  int8_t dy[MAX_TAPS], dx[MAX_TAPS];
  int8_t tap_cb[MAX_TAPS];   // C8 input only: first channel block read by tap t (space-to-depth layers), else 0
  // weights / bias
  const void* w;        // layout depends on the kernel (see se_conv_direct.cu / se_conv_tc.cu)
  long long w_img_stride;   // elements between images (0 = shared)
  const float* bias;    // [Cout] or nullptr
  const float* bias_host;   // optional host copy of bias: lets the tensor-core kernels pass the epilogue constants as kernel parameters
  int Cout;             // pre-gate output channels (GEMM N, real)
  // output
  void* y;
  int out_dt;
  int out_c8;           // 0: NHWC (pitch ldo, channel offset choff); 1: C8 = [N][ldo blocks][H][W][8], choff % 8 == 0 (bf16 only)
  int Hout, Wout, ldo, choff;
  int osy, ooy, osx, oox;
  int out_blk_split, out_blk_jump, out_par_stride;   // fused layer pairs (EpiParams::blk_split ..); 0 = plain layer
  int f16x2;                    // split-half mode (DT_F16X2): fp16 operands, split-half output, exact-math epilogue
  long long out_split_stride;   // f16x2: 16 B units between the hi and the lo part of an output block
  // epilogue
  int epi;
  float scale;                  // EPI_LINEAR
  const float* colscale;        // EPI_LINEAR: [N][Cout] or nullptr
};

// Output side of one gated conv_c8 launch. Layouts: NHWC (pixel pitch ldo elements, channel offset choff) or
// C8 = [N][CBtot][H][W][8] (ldo = CBtot channel blocks, choff multiple of 8).
struct EpiParams {
  void* y;
  int out_c8;   // 0 NHWC, 1 channel-blocked, 2 channel-blocked space-to-depth (see epilogue)
  int Hout, Wout, ldo, choff;
  int osy, ooy, osx, oox;
  int epi;       // EPI_GATE_ELU or EPI_GATE_RELU
  float scale;   // split-half: accumulator -> pre-activation
  int Cout, NT;
  // two gated layers fused along N (stem pairs that read the same packed input): output blocks >= blk_split belong to the second
  // layer's tensor, blk_jump (16 B units) further on; par_stride = channel blocks between the parity groups of a
  // space-to-depth output (ldo / 4 unless two such tensors share the buffer). blk_split = 1 << 20: off.
  int blk_split, blk_jump, par_stride;
  int blk_stride;     // elements between channel block b and b + 1 of one output pixel
  int paired;         // every column pair of the fragment is one aligned 4 B store (see conv_epilogue)
  int split_stride;   // split-half output (DT_F16X2): the lo part of every block is stored split_stride (16 B units) further on
  int goff;   // accumulator column of gate channel 0 (= Cout/2 rounded up to 8; the weight image places feature c at column c
              // and its gate at goff + c, columns in between are zero weights)
};
// Split-half tensors (DT_F16X2) store value * kSplitActScale: fp16's narrow exponent would otherwise push the lo half of every
// activation below ~0.25 into the subnormals (quantum 2^-24: ~1e-6 relative at 0.03). Times 64 the pair keeps ~22 bits down to
// |v| = 2^-9 and stays finite up to |v| = 1000 (saturating beyond). Weights are scaled per class by a power of two of their own
// (ClassW::s_wscale); the epilogue multiplies the accumulator by 1 / (kSplitActScale * s_wscale) inside the bias FMA.
constexpr float kSplitActScale = 64.0f, kSplitActInv = 1.0f / 64.0f, kSplitActMax = 65000.0f;

#ifdef __CUDACC__
// the split-half encoding of v times `scale` (kSplitActScale for activations) and its inverse (inv = 1 / scale)
__device__ __forceinline__ void split_half(float v, float scale, __half& hi, __half& lo) {
  const float s = fminf(fmaxf(v * scale, -kSplitActMax), kSplitActMax);
  hi = __float2half_rn(s);
  lo = __float2half_rn(s - __half2float(hi));
}
__device__ __forceinline__ float join_half(__half hi, __half lo, float inv) { return (__half2float(hi) + __half2float(lo)) * inv; }
#endif
// column of output channel n in the B (weight) image / accumulator of a gated layer
inline int gated_goff(int Cout) { return ((Cout / 2) + 7) / 8 * 8; }
inline int gated_column(int Cout, int n) { const int half = Cout / 2; return n < half ? n : gated_goff(Cout) + (n - half); }

// ------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
#endif

}  // namespace se

// CUDA-core direct convolution with the same op descriptor as the wgmma kernel.
//
// Roles: (1) every convolution of the fp32_direct mode, the cross-check of the tensor-core modes (activations and weights in
// fp32, fp32 FMA accumulation, expf / expm1f), including its attention GEMMs, (2) the heads (12 -> 3 / 12 -> 1) of the
// per-operator API in every mode.
// Weights: fp32 [img][tap][Ci][CoutP] with CoutP = Cout rounded up to 4.
#include "se_common.cuh"
#include "se_conv_direct.h"

namespace se {

constexpr int DC_THREADS = TILE_M;   // one thread per output position of the 8 x 16 tile
constexpr int DC_CK = 32;            // input channels staged per step
constexpr int DC_CO = 32;            // accumulators per thread (16 feature + 16 gate, or 32 linear)

__global__ void __launch_bounds__(DC_THREADS)
conv_direct_kernel(const ConvParams p, const int CoutP) {
  __shared__ float ws[DC_CK][DC_CO];
  __shared__ int col_of[DC_CO];        // accumulator slot -> pre-gate output channel (-1 = unused)

  const int tiles_x = (p.Wo + TILE_W - 1) / TILE_W;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  const int img = blockIdx.z;
  const int grp = blockIdx.y;
  const int tid = threadIdx.x;
  const int ry = tid / TILE_W, rx = tid % TILE_W;
  const int py = ty * TILE_H + ry, px = tx * TILE_W + rx;
  const bool valid = (py < p.Ho) && (px < p.Wo);
  const bool gated = (p.epi != EPI_LINEAR);
  const int half = p.Cout >> 1;

  if (tid < DC_CO) {
    int c;
    if (gated) {
      const int f = grp * (DC_CO / 2) + (tid % (DC_CO / 2));
      c = (f < half) ? (tid < DC_CO / 2 ? f : half + f) : -1;
    } else {
      const int f = grp * DC_CO + tid;
      c = (f < p.Cout) ? f : -1;
    }
    col_of[tid] = c;
  }
  __syncthreads();

  float acc[DC_CO];
#pragma unroll
  for (int i = 0; i < DC_CO; ++i) acc[i] = 0.0f;

  const float* xin = reinterpret_cast<const float*>(p.x);
  const float* wbase = reinterpret_cast<const float*>(p.w) + (size_t)img * p.w_img_stride;

  for (int t = 0; t < p.ntaps; ++t) {
    const int iy = py * p.stride + p.dy[t], ix = px * p.stride + p.dx[t];
    const bool inb = valid && iy >= 0 && iy < p.Hi && ix >= 0 && ix < p.Wi;
    const long long row_pitch = p.x_row_pitch ? p.x_row_pitch : (long long)p.Wi * p.ldx;
    const long long img_pitch = p.x_img_pitch ? p.x_img_pitch : (long long)p.Hi * row_pitch;
    const float* xp = xin + (size_t)img * img_pitch + (size_t)(inb ? iy : 0) * row_pitch + (size_t)(inb ? ix : 0) * p.ldx;
    for (int c0 = 0; c0 < p.Ci; c0 += DC_CK) {
      const int cc = min(DC_CK, p.Ci - c0);
      __syncthreads();
      for (int i = tid; i < DC_CK * DC_CO; i += DC_THREADS) {
        const int ci = i / DC_CO, s = i % DC_CO;
        const int col = col_of[s];
        ws[ci][s] = (ci < cc && col >= 0) ? wbase[((size_t)t * p.Ci + c0 + ci) * CoutP + col] : 0.0f;
      }
      __syncthreads();
      if (inb) {
        for (int ci = 0; ci < cc; ++ci) {
          const float xv = xp[c0 + ci];
          const float4* wr = reinterpret_cast<const float4*>(&ws[ci][0]);
#pragma unroll
          for (int s4 = 0; s4 < DC_CO / 4; ++s4) {
            const float4 w4 = wr[s4];
            acc[s4 * 4 + 0] = fmaf(xv, w4.x, acc[s4 * 4 + 0]);
            acc[s4 * 4 + 1] = fmaf(xv, w4.y, acc[s4 * 4 + 1]);
            acc[s4 * 4 + 2] = fmaf(xv, w4.z, acc[s4 * 4 + 2]);
            acc[s4 * 4 + 3] = fmaf(xv, w4.w, acc[s4 * 4 + 3]);
          }
        }
      }
    }
  }
  if (!valid) return;

  const int oy = py * p.osy + p.ooy, ox = px * p.osx + p.oox;
  const size_t opix = ((size_t)img * p.Hout + oy) * p.Wout + ox;
  if (gated) {
#pragma unroll
    for (int s = 0; s < DC_CO / 2; ++s) {
      const int f = grp * (DC_CO / 2) + s;
      if (f < half) {
        const float fv = acc[s] + (p.bias ? p.bias[f] : 0.0f);
        const float gv = acc[s + DC_CO / 2] + (p.bias ? p.bias[half + f] : 0.0f);
        const float a = (p.epi == EPI_GATE_ELU) ? (fv > 0.0f ? fv : expm1f(fv)) : fmaxf(fv, 0.0f);
        reinterpret_cast<float*>(p.y)[opix * p.ldo + p.choff + f] = a * (1.0f / (1.0f + expf(-gv)));
      }
    }
  } else {
#pragma unroll
    for (int s = 0; s < DC_CO; ++s) {
      const int c = grp * DC_CO + s;
      if (c < p.Cout) {
        float r = acc[s] + (p.bias ? p.bias[c] : 0.0f);
        r *= p.scale * (p.colscale ? p.colscale[(size_t)img * p.Cout + c] : 1.0f);
        reinterpret_cast<float*>(p.y)[opix * p.ldo + p.choff + c] = r;
      }
    }
  }
}

int direct_launch(const ConvParams& c, int CoutP, cudaStream_t stream) {
  SE_REQUIRE(c.in_dt == DT_F32 && c.out_dt == DT_F32, "the direct kernel reads and writes fp32");
  SE_REQUIRE(c.ntaps <= MAX_TAPS, "too many taps");
  SE_REQUIRE(CoutP >= c.Cout, "CoutP");
  const bool gated = c.epi != EPI_LINEAR;
  SE_REQUIRE(!gated || c.Cout % 2 == 0, "gated epilogue needs even Cout");
  const int tiles = ((c.Wo + TILE_W - 1) / TILE_W) * ((c.Ho + TILE_H - 1) / TILE_H);
  const int units = gated ? c.Cout / 2 : c.Cout;
  const int per = gated ? DC_CO / 2 : DC_CO;
  dim3 grid(tiles, (units + per - 1) / per, c.N);
  conv_direct_kernel<<<grid, DC_THREADS, 0, stream>>>(c, CoutP);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

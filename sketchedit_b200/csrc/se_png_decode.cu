// PNG decoding into uint8 pixels, pixel for pixel what np.asarray(Image.open(f).convert(mode)) gives for mode "RGB" or "L"
// (Pillow 12), for non-interlaced files of colour types 0 (depths 1/2/4/8), 2 (8), 3 (1/2/4/8), 4 (8) and 6 (8). The host
// parses the container (sketchedit_b200/pngfile.py) and passes each file's IDAT payloads as one zlib stream; tests/
// util_png_decode.py restates the stages below in numpy.
//
// One warp per file, one launch:
//   inflate: se_inflate.cuh into the file's raw filtered scanlines (scratch), then Adler-32 over them;
//   rows:    a wavefront over 32 rows at a time: lane j reconstructs row r0 + j one pixel (one byte below depth 8) behind
//            lane j - 1, so the pixel above comes from lane j - 1 by a shuffle and the one to the left from the lane's own
//            registers; lane 0 reads the row above from memory, where lane 31 of the previous 32 rows wrote it back. Each
//            reconstructed pixel is unpacked, looked up in the palette, converted to the requested mode and stored.
// The file's status word is 0 only when every stage succeeded; any other value sends the file to Pillow.
#include <string.h>

#include <string>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_inflate.cuh"

namespace se {

constexpr int PNG_DECODE_MAX_BATCH = 256;   // files per call: their descriptors travel as kernel parameters

struct PDec {
  long long src_off, src_len, plte_off, raw_off;
  unsigned char* out;
  int h, w, depth, ctype, npal, mode;   // mode: output bytes per pixel, 1 ("L") or 3 ("RGB")
};
struct PDecList {
  const unsigned char* src;
  unsigned char* raw;
  int* status;
  int n;
  PDec f[PNG_DECODE_MAX_BATCH];
};

__host__ __device__ inline int channels_of(int ctype) { return ctype == 2 ? 3 : ctype == 4 ? 2 : ctype == 6 ? 4 : 1; }
static inline long long row_bytes(int w, int depth, int ctype) { return ((long long)w * channels_of(ctype) * depth + 7) / 8; }
static inline long long raw_bytes(int h, int w, int depth, int ctype) { return (long long)h * (1 + row_bytes(w, depth, ctype)); }

__device__ __forceinline__ unsigned char paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (unsigned char)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

// Pillow's L24 >> 16 (Convert.c): the "L" of an RGB pixel
__device__ __forceinline__ unsigned char luma(unsigned r, unsigned g, unsigned b) {
  return (unsigned char)((r * 19595u + g * 38470u + b * 7471u + 0x8000u) >> 16);
}

__device__ __forceinline__ void put(unsigned char* o, int mode, unsigned r, unsigned g, unsigned b) {
  if (mode == 1) {
    o[0] = luma(r, g, b);
  } else {
    o[0] = (unsigned char)r;
    o[1] = (unsigned char)g;
    o[2] = (unsigned char)b;
  }
}

__global__ void __launch_bounds__(32) png_decode_kernel(const __grid_constant__ PDecList L) {
  __shared__ InflateTabs tabs;
  __shared__ unsigned char pal[768];
  const int lane = threadIdx.x;
  const PDec& F = L.f[blockIdx.x];
  if (F.ctype == 3)
    for (int k = lane; k < 3 * F.npal; k += 32) pal[k] = L.src[F.plte_off + k];
  unsigned char* raw = L.raw + F.raw_off;
  const int bpp_bits = channels_of(F.ctype) * F.depth;
  const long long rowb = ((long long)F.w * bpp_bits + 7) / 8, stride = rowb + 1;
  int st = inflate_zlib(L.src + F.src_off, F.src_len, raw, (long long)F.h * stride, tabs, lane, 32);
  __syncwarp();
  if (st == INF_OK) {
    const int bpp = bpp_bits < 8 ? 1 : bpp_bits / 8;   // bytes per filter unit
    const long long npx = rowb / bpp;
    const int per = 8 / (F.depth < 8 ? F.depth : 8);   // pixels per byte below depth 8
    const unsigned vmask = (1u << (F.depth < 8 ? F.depth : 8)) - 1;
    const unsigned scale = F.depth == 1 ? 255 : F.depth == 2 ? 85 : F.depth == 4 ? 17 : 1;
    unsigned char* out = F.out;
    int err = 0;
    for (int r0 = 0; r0 < F.h; r0 += 32) {
      const int r = r0 + lane;
      const bool active = r < F.h;
      unsigned char* row = raw + (long long)r * stride;
      const int ft = active ? row[0] : 0;
      if (ft > 4) err = PNG_FILTER;
      const bool keep = lane == 31;   // the last row of a full group is the row above the next group
      unsigned left = 0, upleft = 0, last = 0;
      for (long long t = 0; t < npx + 31; ++t) {
        const long long p = t - lane;
        unsigned up = __shfl_up_sync(0xFFFFFFFFu, last, 1);
        if (lane == 0) {
          up = 0;
          if (r0 > 0 && p >= 0 && p < npx) {
            const unsigned char* a = raw + (long long)(r0 - 1) * stride + 1 + p * bpp;
            for (int c = 0; c < bpp; ++c) up |= (unsigned)a[c] << (8 * c);
          }
        }
        if (active && p >= 0 && p < npx) {
          unsigned char* x = row + 1 + p * bpp;
          unsigned cur = 0;
          for (int c = 0; c < bpp; ++c) {
            const int a = (left >> (8 * c)) & 0xFF, b = (up >> (8 * c)) & 0xFF, cc = (upleft >> (8 * c)) & 0xFF;
            int v = x[c];
            switch (ft) {
              case 1: v += a; break;
              case 2: v += b; break;
              case 3: v += (a + b) >> 1; break;
              case 4: v += paeth(a, b, cc); break;
              default: break;
            }
            cur |= (unsigned)(v & 0xFF) << (8 * c);
          }
          if (keep) for (int c = 0; c < bpp; ++c) x[c] = (unsigned char)(cur >> (8 * c));
          unsigned char* o = out + ((long long)r * F.w) * F.mode;
          if (F.depth < 8) {
            for (int k = 0; k < per; ++k) {
              const long long xpix = p * per + k;
              if (xpix >= F.w) break;
              const unsigned v = (cur >> (8 - F.depth * (k + 1))) & vmask;
              unsigned char* q = o + xpix * F.mode;
              if (F.ctype == 3) {
                if ((int)v >= F.npal) err = PNG_PALETTE;
                else put(q, F.mode, pal[3 * v], pal[3 * v + 1], pal[3 * v + 2]);
              } else {
                put(q, F.mode, v * scale, v * scale, v * scale);
              }
            }
          } else {
            unsigned char* q = o + p * F.mode;
            const unsigned b0 = cur & 0xFF, b1 = (cur >> 8) & 0xFF, b2 = (cur >> 16) & 0xFF;
            if (F.ctype == 2 || F.ctype == 6) {
              put(q, F.mode, b0, b1, b2);
            } else if (F.ctype == 3) {
              if ((int)b0 >= F.npal) err = PNG_PALETTE;
              else put(q, F.mode, pal[3 * b0], pal[3 * b0 + 1], pal[3 * b0 + 2]);
            } else {   // grey, grey + alpha
              put(q, F.mode, b0, b0, b0);
            }
          }
          left = cur;
          last = cur;
        }
        upleft = (p >= 0) ? up : 0;
      }
      __syncwarp();
    }
    // the first of the lanes' errors in lane order
    const unsigned any = __ballot_sync(0xFFFFFFFFu, err != 0);
    if (any) st = __shfl_sync(0xFFFFFFFFu, err, __ffs(any) - 1);
  }
  if (lane == 0) L.status[blockIdx.x] = st;
}

}  // namespace se

using namespace se;

extern "C" {

int se_png_decode_u8(const unsigned char* src, const long long* src_off, const long long* src_len, const int* info,
                     const long long* plte_off, int n, unsigned char* const* out, int* status_dev,
                     void* scratch, long long* scratch_bytes, void* stream) {
  SE_REQUIRE(n >= 0 && n <= PNG_DECODE_MAX_BATCH, "n must be in [0, " + std::to_string(PNG_DECODE_MAX_BATCH) + "] files per call");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_off && src_len && info), "null length / offset / info array");
  long long need = 0;
  for (int i = 0; i < n; ++i) {
    const int* f = info + 6 * i;
    const int h = f[0], w = f[1], depth = f[2], ctype = f[3], npal = f[4], mode = f[5];
    const std::string at = "file " + std::to_string(i) + ": ";
    if (int rc = check_sides("file", i, h, w)) return rc;
    const bool ok = (ctype == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                    (ctype == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                    ((ctype == 2 || ctype == 4 || ctype == 6) && depth == 8);
    SE_REQUIRE(ok, at + "colour type " + std::to_string(ctype) + " at depth " + std::to_string(depth) + " is not decoded here");
    SE_REQUIRE(ctype == 3 ? (npal >= 1 && npal <= 256 && plte_off != nullptr && plte_off[i] >= 0) : npal == 0,
               at + "a palette of 1 to 256 entries goes with colour type 3 only");
    SE_REQUIRE(mode == 1 || mode == 3, at + "mode must be 1 (L) or 3 (RGB)");
    SE_REQUIRE(src_off[i] >= 0 && src_len[i] >= 0, at + "negative offset or length");
    need += (raw_bytes(h, w, depth, ctype) + 15) / 16 * 16;
  }
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(src && out && status_dev, "null src / out / status");
  for (int i = 0; i < n; ++i) SE_REQUIRE(out[i] != nullptr, "null out");
  PDecList L;
  memset(&L, 0, sizeof(L));
  L.src = src;
  L.raw = (unsigned char*)scratch;
  L.status = status_dev;
  L.n = n;
  long long at = 0;
  for (int i = 0; i < n; ++i) {
    const int* f = info + 6 * i;
    PDec& d = L.f[i];
    d.src_off = src_off[i];
    d.src_len = src_len[i];
    d.raw_off = at;
    d.out = out[i];
    d.h = f[0];
    d.w = f[1];
    d.depth = f[2];
    d.ctype = f[3];
    d.npal = f[4];
    d.mode = f[5];
    d.plte_off = d.ctype == 3 ? plte_off[i] : 0;
    at += (raw_bytes(d.h, d.w, d.depth, d.ctype) + 15) / 16 * 16;
  }
  png_decode_kernel<<<n, 32, 0, (cudaStream_t)stream>>>(L);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

// What the two PNG decoders (se_png_decode.cu, se_png_split.cu) share: the checks of their file arguments, and the row
// stage (unfilter, unpack, palette and conversion to "RGB" or "L" of a file's raw filtered scanlines, 32 rows per warp).
#pragma once

#include <string>

#include "se_common.cuh"
#include "se_inflate.cuh"

namespace se {

constexpr int PNG_DECODE_MAX_BATCH = 256;   // files per call: their descriptors travel as kernel parameters

// What the row stage needs of a file; mode is the output bytes per pixel, 1 ("L") or 3 ("RGB").
struct PRows {
  unsigned char* out;
  int h, w, depth, ctype, npal, mode;
};

__host__ __device__ inline int channels_of(int ctype) { return ctype == 2 ? 3 : ctype == 4 ? 2 : ctype == 6 ? 4 : 1; }
__host__ __device__ inline long long row_bytes(int w, int depth, int ctype) { return ((long long)w * channels_of(ctype) * depth + 7) / 8; }
__host__ __device__ inline long long raw_bytes(int h, int w, int depth, int ctype) { return (long long)h * (1 + row_bytes(w, depth, ctype)); }

// The checks of the arguments both decoders take (their header comment, sketchedit_b200.h), up to the scratch query.
inline int png_check_files(const long long* src_off, const long long* src_len, const int* info, const long long* plte_off,
                           int n, long long* scratch_bytes) {
  SE_REQUIRE(n >= 0 && n <= PNG_DECODE_MAX_BATCH, "n must be in [0, " + std::to_string(PNG_DECODE_MAX_BATCH) + "] files per call");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_off && src_len && info), "null length / offset / info array");
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
  }
  return 0;
}

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

// A row group with no other warp to wait for or to tell: the one-warp decoder's.
struct RowsAlone {
  __device__ void before(long long) {}
  __device__ void after(long long, long long) {}
};

// Rows r0 .. r0 + 31 of the file F, whose raw filtered scanlines are `raw` (pal: its palette in shared memory). A wavefront:
// lane j reconstructs row r0 + j one pixel (one byte below depth 8) behind lane j - 1, so the pixel above comes from lane
// j - 1 by a shuffle and the one to the left from the lane's own registers; lane 0 reads the row above from memory, where
// lane 31 of the previous group wrote it back. Each reconstructed pixel is unpacked, looked up in the palette, converted
// and stored. sync.before(t) runs on all lanes before step t (lane 0 reads pixel t of the row above in it) and
// sync.after(t, d) after it, d being the pixels of row r0 + 31 written back so far. A filter type past 4 or a palette index
// past the palette sets err.
template <class Sync>
__device__ __forceinline__ void png_row_group(const PRows& F, unsigned char* raw, const unsigned char* pal, int r0, int lane,
                                              int& err, Sync& sync) {
  const int bpp_bits = channels_of(F.ctype) * F.depth;
  const long long rowb = ((long long)F.w * bpp_bits + 7) / 8, stride = rowb + 1;
  const int bpp = bpp_bits < 8 ? 1 : bpp_bits / 8;   // bytes per filter unit
  const long long npx = rowb / bpp;
  const int per = 8 / (F.depth < 8 ? F.depth : 8);   // pixels per byte below depth 8
  const unsigned vmask = (1u << (F.depth < 8 ? F.depth : 8)) - 1;
  const unsigned scale = F.depth == 1 ? 255 : F.depth == 2 ? 85 : F.depth == 4 ? 17 : 1;
  unsigned char* out = F.out;
  const int r = r0 + lane;
  const bool active = r < F.h;
  unsigned char* row = raw + (long long)r * stride;
  const int ft = active ? row[0] : 0;
  if (ft > 4) err = PNG_FILTER;
  const bool keep = lane == 31;   // the last row of a full group is the row above the next group
  unsigned left = 0, upleft = 0, last = 0;
  for (long long t = 0; t < npx + 31; ++t) {
    sync.before(t);
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
    sync.after(t, t - 30 < 0 ? 0 : t - 30 < npx ? t - 30 : npx);
  }
  __syncwarp();
}

}  // namespace se

// Baseline JPEG encoding of uint8 RGB windows, byte for byte what PIL.Image.save(buf, "JPEG", quality=q, subsampling=s) writes
// for an RGB image without info, s = 0 (4:4:4) or 2 (4:2:0), with libjpeg-turbo's defaults (islow DCT, no smoothing, Annex K
// Huffman tables, no restart markers). The encoder is integer arithmetic from start to finish, so every byte is libjpeg-turbo's.
// tests/util_jpeg.py restates each stage in numpy; the comments below name the libjpeg-turbo source a stage follows.
// se_jpeg_encode_tables_u8 runs the same kernels with the caller's quantisation tables, 4:2:2 besides (h2v1 downsampling,
// 16x8 MCUs: tests/util_jpeg_keep.py), and APP1 / APP2 segments after APP0, which the host copies into each file.
//
// One call encodes up to JPEG_MAX_BATCH windows (rows a pitch apart) in these launches on one stream:
//   dct:    one thread per 8x8 block: the window's samples with the last row and column repeated, RGB -> YCbCr (jccolor.c),
//           h2v2 or h2v1 downsampling (jcsample.c), level shift, islow FDCT (jfdctint.c), quantisation by libjpeg-turbo's reciprocals
//           (jcdctmgr.c); writes the zigzag coefficients, the quantised DC and the block's AC bit count.
//   bits:   one thread per block: the DC difference and the block's total bit count (a dummy luma block of a 4:2:0 or 4:2:2
//           MCU, wholly outside the image, codes DC difference 0 and EOB, as jccoefct.c makes it).
//   scan:   exclusive scan of the bit counts (three launches, scan_tiles / scan_sums / scan_add).
//   pack:   one thread per block writes its Huffman codes at its bit offset into a zeroed 32-bit word stream, merging the words
//           it shares with its neighbours by atomicOr.
//   stuff:  per 64-byte chunk of the stream: count its 0xFF bytes, scan the counts, then write the chunk after the header with
//           0x00 after each 0xFF (the last byte padded with 1-bits); the last chunk writes EOI and the image's byte count.
//   header: one block per image writes the header, a function of (h, w, tables, subsampling) built on the host, around the
//           APP1 / APP2 segments the host has copied after APP0.
// With optimize = 1 (Pillow's optimize=True) se_jpeg_opt.cu counts each image's symbols after the bits kernel, builds its
// Huffman tables, writes its header and recounts the block bits; pack then codes with the image's tables from scratch and
// stuff writes the data after the image's header, whose length is on the device.
#include <string.h>

#include <algorithm>
#include <mutex>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/sketchedit_b200.h"
#include "se_jpeg.h"
#include "se_scan.cuh"

namespace se {

// ------------------------------------------------------------------------------------------ tables (ITU T.81 Annex K)
static const unsigned char kLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                         14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                         18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                         49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const unsigned char kChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                           99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                           99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
constexpr unsigned char kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                       41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                       30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct HuffSpec {   // code counts per length 1..16, then the symbols
  unsigned char counts[16];
  unsigned char syms[162];
  int nsym;
};
constexpr HuffSpec kDcLuma = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
constexpr HuffSpec kDcChroma = {{0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11}, 12};
constexpr HuffSpec kAcLuma = {
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
     0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
     0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
     0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
     0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
     0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
     0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
     0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    162};
constexpr HuffSpec kAcChroma = {
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08,
     0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25,
     0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47,
     0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74,
     0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97,
     0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
     0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4,
     0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    162};

constexpr HuffCodes huff_codes(const HuffSpec& s) {   // Annex C
  HuffCodes h{};
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < s.counts[len - 1]; ++i, ++k, ++code) {
      h.code[s.syms[k]] = (unsigned short)code;
      h.size[s.syms[k]] = (unsigned char)len;
    }
    code <<= 1;
  }
  return h;
}
// [0] DC luma, [1] DC chroma, [2] AC luma, [3] AC chroma
__constant__ HuffCodes c_huff[4] = {huff_codes(kDcLuma), huff_codes(kDcChroma), huff_codes(kAcLuma), huff_codes(kAcChroma)};

// ------------------------------------------------------------------------------------------ quantisation (host)
struct QuantTab {   // per natural index: q = ((|x| + corr) * recip) >> shift, the sign restored (jcdctmgr.c, 16-bit DCTELEM)
  unsigned short recip[64], corr[64];
  unsigned char shift[64];
  unsigned char q[64];   // the quantiser itself, for the DQT segment
};

static int quality_scale(int quality) { return quality < 50 ? 5000 / quality : 200 - 2 * quality; }   // jpeg_quality_scaling

// the quantiser q[i] (natural order, 1..255) and its reciprocal, correction and shift
static QuantTab quant_tab(const unsigned short* q) {
  QuantTab t{};
  for (int i = 0; i < 64; ++i) {
    const unsigned divisor = 8u * q[i];   // the FDCT output is scaled by 8
    int b = 31 - __builtin_clz(divisor);
    int r = 16 + b;
    unsigned fq = (1u << r) / divisor, fr = (1u << r) % divisor, c = divisor / 2;
    if (fr == 0) {
      fq >>= 1;
      --r;
    } else if (fr <= divisor / 2) {
      ++c;
    } else {
      ++fq;
    }
    t.q[i] = (unsigned char)q[i];
    t.recip[i] = (unsigned short)fq;
    t.corr[i] = (unsigned short)c;
    t.shift[i] = (unsigned char)r;
  }
  return t;
}

static QuantTab quant_tab(const unsigned char* base, int quality) {
  const int scale = quality_scale(quality);
  unsigned short q[64];
  for (int i = 0; i < 64; ++i) q[i] = (unsigned short)std::min(255, std::max(1, (base[i] * scale + 50) / 100));   // force_baseline
  return quant_tab(q);
}

// the luma and chroma tables of one quality, built once per quality
static const QuantTab* quant_tabs(int quality) {
  static std::mutex mu;
  static QuantTab tabs[101][2];
  static bool built[101] = {};
  std::lock_guard<std::mutex> lk(mu);
  if (!built[quality]) {
    tabs[quality][0] = quant_tab(kLumaQ, quality);
    tabs[quality][1] = quant_tab(kChromaQ, quality);
    built[quality] = true;
  }
  return tabs[quality];
}

static void put16(std::vector<unsigned char>& v, int x) {
  v.push_back((unsigned char)(x >> 8));
  v.push_back((unsigned char)x);
}

static void put_dht(std::vector<unsigned char>& v, int cls_id, const HuffSpec& s) {
  v.insert(v.end(), {0xFF, 0xC4});
  put16(v, 2 + 1 + 16 + s.nsym);
  v.push_back((unsigned char)cls_id);
  v.insert(v.end(), s.counts, s.counts + 16);
  v.insert(v.end(), s.syms, s.syms + s.nsym);
}

// Pillow's table of component c when the call has nq DQT segments (JpegEncode.c): one table serves all, two split luma and
// chroma, three give each component its own
static int comp_table(int nq, int c) { return std::min(c, nq - 1); }

// SOI, JFIF APP0 1.01 (density 1:1, units 0), DQT 0 .. nq - 1 (zigzag order), SOF0, DHT DC0 AC0 DC1 AC1, SOS (jcmarker.c)
static std::vector<unsigned char> jpeg_header(int h, int w, const QuantTab* qt, int nq, int subsampling) {
  std::vector<unsigned char> v = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  for (int t = 0; t < nq; ++t) {
    v.insert(v.end(), {0xFF, 0xDB, 0, 67, (unsigned char)t});
    for (int k = 0; k < 64; ++k) v.push_back(qt[t].q[kZigzag[k]]);
  }
  v.insert(v.end(), {0xFF, 0xC0, 0, 17, 8});
  put16(v, h);
  put16(v, w);
  const unsigned char y = subsampling == 2 ? 0x22 : subsampling == 1 ? 0x21 : 0x11;
  v.insert(v.end(), {3, 1, y, (unsigned char)comp_table(nq, 0), 2, 0x11, (unsigned char)comp_table(nq, 1), 3, 0x11,
                     (unsigned char)comp_table(nq, 2)});
  put_dht(v, 0x00, kDcLuma);
  put_dht(v, 0x10, kAcLuma);
  put_dht(v, 0x01, kDcChroma);
  put_dht(v, 0x11, kAcChroma);
  v.insert(v.end(), {0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  return v;
}

static long long image_blocks(int h, int w, int sub) {
  const int mh = mcu_h(sub), mw = mcu_w(sub);
  return (long long)((h + mh - 1) / mh) * ((w + mw - 1) / mw) * mcu_blocks(sub);
}

long long jpeg_max_bytes(int h, int w, int subsampling, long long header_bytes) {
  return header_bytes + 2 * (image_blocks(h, w, subsampling) * (JPEG_MAX_BLOCK_BITS / 8)) + 2;
}

// ------------------------------------------------------------------------------------------ kernels
constexpr int kWordsPerBlock = JPEG_MAX_BLOCK_BITS / 32;
constexpr int kChunkBytes = 64;   // bytes of the stream per stuffing thread
constexpr int kThreads = 128;

struct JpegQuant {   // the call's tables, and each component's table: components sharing a table read the same words
  unsigned short recip[3][64], corr[3][64];
  unsigned char shift[3][64];
  unsigned char tq[3];
};
static_assert(sizeof(JpegList) + sizeof(JpegQuant) <= 4096, "descriptors must fit the kernel parameter space");

__device__ __forceinline__ int color(int comp, int r, int g, int b) {   // jccolor.c, 16-bit fixed point
  if (comp == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (comp == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// one pass of jfdctint.c over the 8 values d[o], d[o + s], ..., d[o + 7 s]
__device__ __forceinline__ void fdct8(int (&d)[64], int o, int s, bool first) {
  constexpr int C = 13, P = 2;
  const int sh = first ? C - P : C + P;
  int t0 = d[o] + d[o + 7 * s], t7 = d[o] - d[o + 7 * s];
  int t1 = d[o + s] + d[o + 6 * s], t6 = d[o + s] - d[o + 6 * s];
  int t2 = d[o + 2 * s] + d[o + 5 * s], t5 = d[o + 2 * s] - d[o + 5 * s];
  int t3 = d[o + 3 * s] + d[o + 4 * s], t4 = d[o + 3 * s] - d[o + 4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  d[o] = first ? (t10 + t11) * (1 << P) : descale(t10 + t11, P);
  d[o + 4 * s] = first ? (t10 - t11) * (1 << P) : descale(t10 - t11, P);
  int z1 = (t12 + t13) * 4433;
  d[o + 2 * s] = descale(z1 + t13 * 6270, sh);
  d[o + 6 * s] = descale(z1 - t12 * 15137, sh);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * 9633;
  t4 *= 2446;
  t5 *= 16819;
  t6 *= 25172;
  t7 *= 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[o + 7 * s] = descale(t4 + z1 + z3, sh);
  d[o + 5 * s] = descale(t5 + z2 + z4, sh);
  d[o + 3 * s] = descale(t6 + z2 + z3, sh);
  d[o + s] = descale(t7 + z1 + z4, sh);
}

// the code tables in shared memory: a warp's blocks look up different symbols, which constant memory would serialise
__device__ __forceinline__ void stage_huff(HuffCodes* sh, int first, int count) {
  const unsigned* s = reinterpret_cast<const unsigned*>(c_huff + first);
  unsigned* d = reinterpret_cast<unsigned*>(sh);
  for (int j = threadIdx.x; j < count * (int)(sizeof(HuffCodes) / 4); j += blockDim.x) d[j] = s[j];
  __syncthreads();
}

// f(std::integral_constant<int, k>) for k = 0 .. 63 in order: zigzag(k) is then a constant and v[zigzag(k)] a register
__host__ __device__ constexpr int zigzag(int k) { return kZigzag[k]; }
template <class F, int... K>
__device__ __forceinline__ void for_each_zigzag(F&& f, std::integer_sequence<int, K...>) {
  (f(std::integral_constant<int, K>{}), ...);
}

__global__ void __launch_bounds__(kThreads) jpeg_dct_kernel(const __grid_constant__ JpegList L, const __grid_constant__ JpegQuant Q,
                                                            JpegScratch S) {
  __shared__ HuffCodes sh_ac[2];
  stage_huff(sh_ac, 2, 2);
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= L.blocks) return;
  const JImg& d = L.im[image_of(L.im, L.n, &JImg::blk0, g)];
  const BlockAt b = block_at(d, L.sub, g - d.blk0);
  if (b.dummy) return;   // its DC and bits come from the block before it (jpeg_bits_kernel, jpeg_pack_kernel)
  int v[64];
  if (L.sub == 2 && b.comp) {   // h2v2: rows repeated to an even count, columns to the MCU width, chroma rows to the block grid
    const int ch = (d.h + 1) / 2;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int cy = min(b.by * 8 + r, ch - 1);
      const unsigned char* r0 = d.src + (size_t)min(2 * cy, d.h - 1) * d.pitch;
      const unsigned char* r1 = d.src + (size_t)min(2 * cy + 1, d.h - 1) * d.pitch;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int x0 = min(b.bx * 16 + 2 * c, d.w - 1) * 3, x1 = min(b.bx * 16 + 2 * c + 1, d.w - 1) * 3;
        const int s = color(b.comp, r0[x0], r0[x0 + 1], r0[x0 + 2]) + color(b.comp, r0[x1], r0[x1 + 1], r0[x1 + 2]) +
                      color(b.comp, r1[x0], r1[x0 + 1], r1[x0 + 2]) + color(b.comp, r1[x1], r1[x1 + 1], r1[x1 + 2]);
        v[r * 8 + c] = ((s + 1 + (c & 1)) >> 2) - 128;
      }
    }
  } else if (L.sub == 1 && b.comp) {   // h2v1: columns repeated to the MCU width, rows to the block grid
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const unsigned char* row = d.src + (size_t)min(b.by * 8 + r, d.h - 1) * d.pitch;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int x0 = min(b.bx * 16 + 2 * c, d.w - 1) * 3, x1 = min(b.bx * 16 + 2 * c + 1, d.w - 1) * 3;
        const int s = color(b.comp, row[x0], row[x0 + 1], row[x0 + 2]) + color(b.comp, row[x1], row[x1 + 1], row[x1 + 2]);
        v[r * 8 + c] = ((s + (c & 1)) >> 1) - 128;
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const unsigned char* row = d.src + (size_t)min(b.by * 8 + r, d.h - 1) * d.pitch;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const int x = min(b.bx * 8 + c, d.w - 1) * 3;
        v[r * 8 + c] = color(b.comp, row[x], row[x + 1], row[x + 2]) - 128;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct8(v, r * 8, 1, true);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct8(v, c, 8, false);
  const int t = Q.tq[b.comp];
  const HuffCodes& ac = sh_ac[b.comp ? 1 : 0];
  unsigned bits = 0;
  int run = 0;
  for_each_zigzag(
      [&](auto kc) {
        constexpr int k = decltype(kc)::value, n = zigzag(k);
        const int x = v[n], a = x < 0 ? -x : x;
        const int q = (int)(((unsigned)(a + Q.corr[t][n]) * Q.recip[t][n]) >> Q.shift[t][n]);
        const int y = x < 0 ? -q : q;
        S.coef[(size_t)k * L.blocks + g] = (short)y;
        if (k == 0) return;
        if (y == 0) {
          ++run;
          return;
        }
        const int nb = nbits(y);
        bits += (run >> 4) * ac.size[0xF0] + ac.size[((run & 15) << 4) | nb] + nb;
        run = 0;
      },
      std::make_integer_sequence<int, 64>{});
  if (run) bits += ac.size[0x00];
  S.bits[g] = bits;
}

__global__ void __launch_bounds__(kThreads) jpeg_bits_kernel(const __grid_constant__ JpegList L, JpegScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= L.blocks) return;
  const JImg& d = L.im[image_of(L.im, L.n, &JImg::blk0, g)];
  const long long e = g - d.blk0;
  const BlockAt b = block_at(d, L.sub, e);
  const HuffCodes& dch = c_huff[b.comp ? 1 : 0];
  if (b.dummy) {
    S.bits[g] = dch.size[0] + c_huff[2].size[0x00];
    S.dcdiff[g] = 0;
    return;
  }
  const long long p = prev_same_comp(L.sub, e);
  const int diff = S.coef[g] - (p < 0 ? 0 : dc_of(d, L.sub, S.coef, p));
  const int nb = nbits(diff);
  S.bits[g] += dch.size[nb] + nb;
  S.dcdiff[g] = diff;
}

__device__ __forceinline__ void put_value(unsigned long long& acc, int& n, unsigned* w, long long& wi, const HuffCodes& h,
                                          int sym, int v, int nb) {
  const unsigned bits = (unsigned)(v < 0 ? v - 1 : v) & ((1u << nb) - 1);
  put_bits(acc, n, w, wi, ((unsigned)h.code[sym] << nb) | bits, h.size[sym] + nb);
}

__global__ void __launch_bounds__(kThreads) jpeg_pack_kernel(const __grid_constant__ JpegList L, JpegScratch S) {
  __shared__ HuffCodes sh[4];
  stage_huff(sh, 0, 4);
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= L.blocks) return;
  const int i = image_of(L.im, L.n, &JImg::blk0, g);
  const JImg& d = L.im[i];
  const BlockAt b = block_at(d, L.sub, g - d.blk0);
  const unsigned long long at = S.bitoff[g] - S.bitoff[d.blk0];
  unsigned* w = S.words + d.word0;
  long long wi = (long long)(at >> 5);
  int n = (int)(at & 31);
  unsigned long long acc = 0;
  const HuffCodes* T = S.tabs ? S.tabs[i].codes : sh;   // the image's optimal tables, or Annex K's
  const HuffCodes& dch = T[b.comp ? 1 : 0];
  const HuffCodes& ach = T[b.comp ? 3 : 2];
  const int diff = S.dcdiff[g];
  put_value(acc, n, w, wi, dch, nbits(diff), diff, nbits(diff));
  int run = 0;
  if (!b.dummy) {
    for (int k = 1; k < 64; ++k) {
      const int y = S.coef[(size_t)k * L.blocks + g];
      if (y == 0) {
        ++run;
        continue;
      }
      for (; run > 15; run -= 16) put_bits(acc, n, w, wi, ach.code[0xF0], ach.size[0xF0]);
      const int nb = nbits(y);
      put_value(acc, n, w, wi, ach, (run << 4) | nb, y, nb);
      run = 0;
    }
  }
  if (run || b.dummy) put_bits(acc, n, w, wi, ach.code[0x00], ach.size[0x00]);
  if (n) atomicOr(w + wi, (unsigned)(acc << (32 - n)));
}

// ---- stuffing
__device__ __forceinline__ unsigned long long image_bits(const JImg& d, const JImg* next, const JpegList& L, const JpegScratch& S) {
  const long long last = (next ? next->blk0 : L.blocks) - 1;
  return S.bitoff[last] + S.bits[last] - S.bitoff[d.blk0];
}

template <bool WRITE>
__global__ void __launch_bounds__(kThreads) jpeg_stuff_kernel(const __grid_constant__ JpegList L, JpegScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= L.chunks) return;
  const int i = image_of(L.im, L.n, &JImg::chunk0, g);
  const JImg& d = L.im[i];
  const unsigned long long nbits = image_bits(d, i + 1 < L.n ? &L.im[i + 1] : nullptr, L, S);
  const long long nbytes = (long long)((nbits + 7) >> 3);
  const long long c = g - d.chunk0, j0 = c * kChunkBytes, j1 = min(j0 + kChunkBytes, nbytes);
  const unsigned* w = S.words + d.word0;
  if (!WRITE) {
    unsigned ff = 0;
    for (long long j = j0; j < j1; ++j) ff += stream_byte(w, j, nbits) == 0xFFu;
    S.ffcnt[g] = ff;
    return;
  }
  if (j0 >= nbytes) return;
  unsigned char* o = d.out + (S.hdr_len ? S.hdr_len[i] : L.hdr) + j0 + (S.ffoff[g] - S.ffoff[d.chunk0]);
  for (long long j = j0; j < j1; ++j) {
    const unsigned v = stream_byte(w, j, nbits);
    *o++ = (unsigned char)v;
    if (v == 0xFFu) *o++ = 0;
  }
  if (j1 == nbytes) {   // the image's last chunk
    o[0] = 0xFF;
    o[1] = 0xD9;
    *d.out_bytes = (long long)(o + 2 - d.out);
  }
}

__global__ void __launch_bounds__(kThreads) jpeg_header_kernel(const __grid_constant__ HeaderList H) {
  unsigned char* o = H.out[blockIdx.x];
  for (int j = threadIdx.x; j < H.len; j += kThreads) o[header_at(H, j)] = header_byte(H, blockIdx.x, j);
}

// ------------------------------------------------------------------------------------------ host
struct JpegLayout {   // the call's block, word and chunk counts and where its arrays lie in scratch
  long long blocks = 0, words = 0, chunks = 0;
  size_t coef = 0, bits = 0, dcdiff = 0, bitoff = 0, words_at = 0, ffcnt = 0, ffoff = 0, sums = 0, hist = 0, tabs = 0,
         hdr_len = 0, prog = 0, total = 0;
};

static long long chunks_of(long long blocks) { return (blocks * kWordsPerBlock * 4 + kChunkBytes - 1) / kChunkBytes; }

// progressive: the coefficients and the dct kernel's bit counts, then se_jpeg_prog.cu's arrays of `prog` bytes
static JpegLayout jpeg_layout(const int* hw, int n, int sub, bool optimize, bool progressive, size_t prog) {
  JpegLayout l;
  for (int i = 0; i < n; ++i) {
    const long long b = image_blocks(hw[2 * i], hw[2 * i + 1], sub);
    l.blocks += b;
    if (progressive) continue;
    l.words += b * kWordsPerBlock;
    l.chunks += chunks_of(b);
  }
  const long long tiles = (std::max(l.blocks, l.chunks) + SCAN_TILE - 1) / SCAN_TILE;
  size_t at = 0;
  auto take = [&](size_t bytes) {
    const size_t p = at;
    at += scratch_round(bytes);
    return p;
  };
  l.coef = take((size_t)l.blocks * 64 * sizeof(short));
  l.bits = take((size_t)l.blocks * sizeof(unsigned));
  if (progressive) {
    l.prog = take(prog);
    l.total = at;
    return l;
  }
  l.dcdiff = take((size_t)l.blocks * sizeof(int));
  l.bitoff = take((size_t)l.blocks * sizeof(unsigned long long));
  l.words_at = take((size_t)l.words * sizeof(unsigned));
  l.ffcnt = take((size_t)l.chunks * sizeof(unsigned));
  l.ffoff = take((size_t)l.chunks * sizeof(unsigned long long));
  l.sums = take((size_t)std::max(tiles, 1LL) * sizeof(unsigned long long));
  l.hist = take(optimize ? (size_t)n * 4 * 256 * sizeof(unsigned long long) : 0);
  l.tabs = take(optimize ? (size_t)n * sizeof(JpegTables) : 0);
  l.hdr_len = take(optimize ? (size_t)n * sizeof(int) : 0);
  l.total = at;
  return l;
}

// What a call writes besides the pixels: its DQT tables, subsampling and APP1 / APP2 segments
struct JpegFormat {
  QuantTab qt[3];                        // DQT tables 0 .. nq - 1
  int nq = 2, sub = 2;
  const unsigned char* meta = nullptr;   // host bytes of the segments, written after APP0
  long long meta_len = 0;
};

// the format of the quality entries: the Annex K tables at `quality`, no segments
static JpegFormat quality_format(int quality, int subsampling) {
  JpegFormat F;
  const QuantTab* qt = quant_tabs(quality);
  F.qt[0] = qt[0];
  F.qt[1] = qt[1];
  F.sub = subsampling;
  return F;
}

constexpr long long kMaxMeta = 1LL << 30;   // APP1 / APP2 bytes a call takes

// se_jpeg_encode_tables_u8's check of its segments: each one FF E1 or FF E2 with a length that matches, back to back
static int check_segments(const unsigned char* seg, long long len) {
  SE_REQUIRE(len >= 0 && len <= kMaxMeta, "segments_len must be in [0, 2^30]");
  SE_REQUIRE(len == 0 || seg != nullptr, "null segments");
  for (long long at = 0; at < len;) {
    SE_REQUIRE(len - at >= 4, "segment at byte " + std::to_string(at) + " is cut short");
    SE_REQUIRE(seg[at] == 0xFF && (seg[at + 1] == 0xE1 || seg[at + 1] == 0xE2),
               "segment at byte " + std::to_string(at) + " is not an APP1 (FF E1) or APP2 (FF E2) marker");
    const int n = seg[at + 2] << 8 | seg[at + 3];
    SE_REQUIRE(n >= 2 && n <= len - at - 2, "segment at byte " + std::to_string(at) + " has length " + std::to_string(n) +
                                                " and " + std::to_string(len - at - 2) + " bytes after its marker");
    at += 2 + n;
  }
  return 0;
}

// the table count, entries and subsampling of se_jpeg_encode_tables_u8 and its bound
static int check_tables_format(int ntables, int subsampling) {
  SE_REQUIRE(ntables >= 1 && ntables <= 4, "ntables must be in [1, 4]");
  SE_REQUIRE(subsampling >= 0 && subsampling <= 2, "subsampling must be 0 (4:4:4), 1 (4:2:2) or 2 (4:2:0)");
  return 0;
}

}  // namespace se

using namespace se;

extern "C" {

long long se_jpeg_max_bytes(int h, int w, int subsampling) {
  if (h < 1 || w < 1 || h > kMaxDim || w > kMaxDim || (subsampling != 0 && subsampling != 2)) {
    set_error("se_jpeg_max_bytes: sizes must be in [1, 65535] and subsampling 0 (4:4:4) or 2 (4:2:0)");
    return -1;
  }
  return jpeg_max_bytes(h, w, subsampling);
}

long long se_jpeg_progressive_max_bytes(int h, int w, int subsampling) {
  if (h < 1 || w < 1 || h > kMaxDim || w > kMaxDim || (subsampling != 0 && subsampling != 2)) {
    set_error("se_jpeg_progressive_max_bytes: sizes must be in [1, 65535] and subsampling 0 (4:4:4) or 2 (4:2:0)");
    return -1;
  }
  return jpeg_prog_max_bytes(h, w, subsampling);
}

long long se_jpeg_tables_max_bytes(int h, int w, int subsampling, int ntables, int progressive, long long segments_len) {
  if (h < 1 || w < 1 || h > kMaxDim || w > kMaxDim || subsampling < 0 || subsampling > 2 || ntables < 1 || ntables > 4 ||
      (progressive != 0 && progressive != 1) || segments_len < 0 || segments_len > kMaxMeta) {
    set_error("se_jpeg_tables_max_bytes: sizes must be in [1, 65535], subsampling 0, 1 or 2, ntables in [1, 4], progressive 0 "
              "or 1 and segments_len in [0, 2^30]");
    return -1;
  }
  const int nq = std::min(ntables, 3);
  return progressive ? jpeg_prog_max_bytes(h, w, subsampling, jpeg_sof_end(nq, segments_len))
                     : jpeg_max_bytes(h, w, subsampling, jpeg_header_bytes(nq, segments_len));
}

}  // extern "C"

namespace se {

// every entry: the quality entries (progressive = false, or true with optimize = 0) and se_jpeg_encode_tables_u8, whose
// format F is checked by the caller
static int jpeg_encode(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, const JpegFormat& F,
                       int optimize, bool progressive, unsigned char* out, const long long* out_off, long long* out_bytes_dev,
                       void* scratch, long long* scratch_bytes, void* stream) {
  SE_REQUIRE(n >= 0 && n <= JPEG_MAX_BATCH, "n must be in [0, " + std::to_string(JPEG_MAX_BATCH) + "] images per call");
  SE_REQUIRE(optimize == 0 || optimize == 1, "optimize must be 0 or 1");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_pitch && hw && out_off), "null size / offset array");
  for (int i = 0; i < n; ++i)
    if (int rc = check_window(i, hw[2 * i], hw[2 * i + 1], src_pitch[i], 3LL * hw[2 * i + 1], out_off[i])) return rc;
  const int subsampling = F.sub;
  JpegList L;
  ProgList P;
  ProgScratch PS;
  memset(&L, 0, sizeof(L));
  memset(&P, 0, sizeof(P));
  memset(&PS, 0, sizeof(PS));
  L.n = n;
  L.sub = subsampling;
  for (int i = 0; i < n; ++i) {
    L.im[i].h = hw[2 * i];
    L.im[i].w = hw[2 * i + 1];
  }
  const JpegLayout lay = jpeg_layout(hw, n, subsampling, optimize, progressive,
                                     progressive ? jpeg_prog_layout(L, nullptr, &P, &PS) : 0);
  SE_SCRATCH(scratch, scratch_bytes, lay.total, n);
  SE_REQUIRE(src && out && out_bytes_dev, "null src / out / out_bytes");
  for (int i = 0; i < n; ++i) SE_REQUIRE(src[i] != nullptr, "null src");
  SE_REQUIRE(lay.blocks < (1LL << 31) * kThreads && lay.chunks < (1LL << 31) * kThreads, "batch too large for one launch");
  SE_REQUIRE(P.slots < (1LL << 31) * kThreads && P.chunks < (1LL << 31) * kThreads, "batch too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;

  JpegQuant Q;
  memset(&Q, 0, sizeof(Q));
  for (int t = 0; t < F.nq; ++t) {
    memcpy(Q.recip[t], F.qt[t].recip, sizeof(Q.recip[t]));
    memcpy(Q.corr[t], F.qt[t].corr, sizeof(Q.corr[t]));
    memcpy(Q.shift[t], F.qt[t].shift, sizeof(Q.shift[t]));
  }
  for (int c = 0; c < 3; ++c) Q.tq[c] = (unsigned char)comp_table(F.nq, c);
  HeaderList H;
  memset(&H, 0, sizeof(H));
  const std::vector<unsigned char> hdr = jpeg_header(1, 1, F.qt, F.nq, subsampling);
  memcpy(H.bytes, hdr.data(), hdr.size());
  H.len = (int)hdr.size();
  H.sof_end = jpeg_sof_end(F.nq, 0);
  H.meta = (int)F.meta_len;
  L.hdr = H.len + H.meta;
  long long blk = 0, word = 0, chunk = 0;
  for (int i = 0; i < n; ++i) {
    const int h = hw[2 * i], w = hw[2 * i + 1], m = mcu_w(subsampling);
    JImg& d = L.im[i];
    d.src = src[i];
    d.out = out + out_off[i];
    d.out_bytes = out_bytes_dev + i;
    d.pitch = src_pitch[i];
    d.h = h;
    d.w = w;
    d.mcu_x = (w + m - 1) / m;
    d.blk0 = blk;
    d.word0 = word;
    d.chunk0 = chunk;
    const long long b = image_blocks(h, w, subsampling);
    blk += b;
    word += b * kWordsPerBlock;
    chunk += chunks_of(b);
    H.out[i] = d.out;
    H.hw[i][0] = (unsigned short)h;
    H.hw[i][1] = (unsigned short)w;
    // the segments go straight into each file after APP0; the header kernels write around them
    if (F.meta_len)
      SE_CUDA_OK(cudaMemcpyAsync(d.out + JPEG_APP0_END, F.meta, (size_t)F.meta_len, cudaMemcpyHostToDevice, st));
  }
  L.blocks = blk;
  L.chunks = chunk;
  unsigned char* s = (unsigned char*)scratch;
  JpegScratch S;
  S.coef = (short*)(s + lay.coef);
  S.bits = (unsigned*)(s + lay.bits);
  S.dcdiff = (int*)(s + lay.dcdiff);
  S.bitoff = (unsigned long long*)(s + lay.bitoff);
  S.words = (unsigned*)(s + lay.words_at);
  S.ffcnt = (unsigned*)(s + lay.ffcnt);
  S.ffoff = (unsigned long long*)(s + lay.ffoff);
  S.sums = (unsigned long long*)(s + lay.sums);
  S.hist = optimize ? (unsigned long long*)(s + lay.hist) : nullptr;
  S.tabs = optimize ? (JpegTables*)(s + lay.tabs) : nullptr;
  S.hdr_len = optimize ? (int*)(s + lay.hdr_len) : nullptr;

  if (progressive) {
    jpeg_prog_layout(L, s + lay.prog, &P, &PS);
    PS.coef = S.coef;
    jpeg_dct_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, Q, S);
    SE_CUDA_OK(cudaGetLastError());
    return jpeg_progressive(L, H, P, PS, st);
  }
  SE_CUDA_OK(cudaMemsetAsync(S.words, 0, (size_t)lay.words * sizeof(unsigned), st));
  if (!optimize) jpeg_header_kernel<<<n, kThreads, 0, st>>>(H);
  jpeg_dct_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, Q, S);
  jpeg_bits_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  int rc;
  if (optimize) {   // the DC differences are in place; the bit counts so far are Annex K's and are rewritten
    SE_CUDA_OK(cudaMemsetAsync(S.hist, 0, lay.tabs - lay.hist, st));
    if ((rc = jpeg_optimize_tables(L, S, st))) return rc;
    if ((rc = jpeg_optimize_header(L, H, S, st))) return rc;
  }
  rc = exclusive_scan(S.bits, S.bitoff, S.sums, L.blocks, st);
  if (rc) return rc;
  jpeg_pack_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, S);
  jpeg_stuff_kernel<false><<<grid_of(L.chunks, kThreads), kThreads, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  rc = exclusive_scan(S.ffcnt, S.ffoff, S.sums, L.chunks, st);
  if (rc) return rc;
  jpeg_stuff_kernel<true><<<grid_of(L.chunks, kThreads), kThreads, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

// the quality entries' checks of quality and subsampling
static int check_quality(int quality, int subsampling) {
  SE_REQUIRE(quality >= 1 && quality <= 100, "quality must be in [1, 100]");
  SE_REQUIRE(subsampling == 0 || subsampling == 2, "subsampling must be 0 (4:4:4) or 2 (4:2:0)");
  return 0;
}

}  // namespace se

extern "C" {

int se_jpeg_encode_opt_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int quality,
                          int subsampling, int optimize, unsigned char* out, const long long* out_off, long long* out_bytes_dev,
                          void* scratch, long long* scratch_bytes, void* stream) {
  if (int rc = check_quality(quality, subsampling)) return rc;
  return jpeg_encode(src, src_pitch, hw, n, quality_format(quality, subsampling), optimize, false, out, out_off, out_bytes_dev,
                     scratch, scratch_bytes, stream);
}

int se_jpeg_encode_progressive_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n,
                                  int quality, int subsampling, unsigned char* out, const long long* out_off,
                                  long long* out_bytes_dev, void* scratch, long long* scratch_bytes, void* stream) {
  if (int rc = check_quality(quality, subsampling)) return rc;
  return jpeg_encode(src, src_pitch, hw, n, quality_format(quality, subsampling), 0, true, out, out_off, out_bytes_dev,
                     scratch, scratch_bytes, stream);
}

int se_jpeg_encode_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int quality, int subsampling,
                      unsigned char* out, const long long* out_off, long long* out_bytes_dev, void* scratch, long long* scratch_bytes,
                      void* stream) {
  return se_jpeg_encode_opt_u8(src, src_pitch, hw, n, quality, subsampling, 0, out, out_off, out_bytes_dev, scratch, scratch_bytes,
                               stream);
}

int se_jpeg_encode_tables_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n,
                             const unsigned short* qtables, int ntables, int subsampling, int optimize, int progressive,
                             const unsigned char* segments, long long segments_len, unsigned char* out, const long long* out_off,
                             long long* out_bytes_dev, void* scratch, long long* scratch_bytes, void* stream) {
  if (int rc = check_tables_format(ntables, subsampling)) return rc;
  SE_REQUIRE(qtables != nullptr, "null qtables");
  SE_REQUIRE(progressive == 0 || progressive == 1, "progressive must be 0 or 1");
  SE_REQUIRE(optimize == 0 || optimize == 1, "optimize must be 0 or 1");
  for (int k = 0; k < 64 * ntables; ++k)
    SE_REQUIRE(qtables[k] <= 255, "table " + std::to_string(k / 64) + " entry " + std::to_string(k % 64) + " is " +
                                      std::to_string(qtables[k]) + ": entries must be in [0, 255] (8-bit baseline tables)");
  if (int rc = check_segments(segments, segments_len)) return rc;
  JpegFormat F;
  F.nq = std::min(ntables, 3);
  for (int t = 0; t < F.nq; ++t) {
    unsigned short q[64];
    for (int k = 0; k < 64; ++k) q[k] = std::max<unsigned short>(1, qtables[64 * t + k]);   // jpeg_add_quant_table at scale 100
    F.qt[t] = quant_tab(q);
  }
  F.sub = subsampling;
  F.meta = segments;
  F.meta_len = segments_len;
  return jpeg_encode(src, src_pitch, hw, n, F, progressive ? 0 : optimize, progressive, out, out_off, out_bytes_dev, scratch,
                     scratch_bytes, stream);
}

}  // extern "C"

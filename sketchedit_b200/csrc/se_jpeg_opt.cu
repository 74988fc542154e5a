// Optimal Huffman tables for se_jpeg_encode_opt_u8 with optimize = 1: byte for byte what PIL.Image.save(buf, "JPEG",
// quality=q, subsampling=s, optimize=True) writes, libjpeg-turbo's two-pass encode. tests/util_jpeg_optimize.py restates
// each step in numpy. After se_jpeg.cu's dct and bits kernels have left the quantised coefficients and DC differences in
// scratch, per call:
//   hist:   one thread per 8x8 block counts the symbols the block codes (DC category, AC run/size, ZRL, EOB; a dummy luma
//           block of a 4:2:0 or 4:2:2 MCU codes DC 0 and EOB) into its image's four 256-bin histograms: a CTA counts its first image's
//           blocks in shared memory and adds them to global memory once, and any other image's straight to global memory.
//   tables: one warp per (image, table), or per (image, scan, table) for se_jpeg_prog.cu, runs ITU T.81 Annex K.2 with
//           libjpeg's tie rule, limits the lengths to 16 bits (Annex K.3), drops the reserved code and lists the symbols;
//           writes the codes and the DHT contents.
//   header: one CTA per image writes SOI..SOF0 around the APP1 / APP2 segments the host copied there, the four DHT segments
//           of its tables and SOS, and the header's length.
//   bits:   one thread per block, its bit count with the image's tables (replacing the Annex K count).
// se_jpeg.cu's scan, pack and stuff kernels then read the tables and the header length from scratch. The counts are
// integers, so every launch order gives the same tables.
#include "../../include/sketchedit_b200.h"
#include "se_jpeg.h"

namespace se {

namespace {

constexpr int kThreads = 128;
constexpr int kMaxCandidate = 1000000000;   // libjpeg never picks a count above this for a merge (its starting minimum)
constexpr int kMaxLen = 64;                 // unlimited code lengths: merged counts stay <= 2e9, so a path has < 47 merges

// the symbols block g codes, in coding order: f(table, symbol) with table 0 DC luma, 1 DC chroma, 2 AC luma, 3 AC chroma
template <class F>
__device__ __forceinline__ void block_symbols(const JpegList& L, const JpegScratch& S, const JImg& d, long long g, F&& f) {
  const BlockAt b = block_at(d, L.sub, g - d.blk0);
  const int c = b.comp ? 1 : 0;
  f(c, nbits(S.dcdiff[g]));   // a dummy's difference is 0
  int run = 0;
  if (!b.dummy) {
    for (int k = 1; k < 64; ++k) {
      const int y = S.coef[(size_t)k * L.blocks + g];
      if (y == 0) {
        ++run;
        continue;
      }
      for (; run > 15; run -= 16) f(2 + c, 0xF0);
      f(2 + c, (run << 4) | nbits(y));
      run = 0;
    }
  }
  if (run || b.dummy) f(2 + c, 0x00);
}

__global__ void __launch_bounds__(kThreads) jpeg_hist_kernel(const __grid_constant__ JpegList L, JpegScratch S) {
  __shared__ unsigned sh[4 * 256];
  for (int j = threadIdx.x; j < 4 * 256; j += kThreads) sh[j] = 0;
  __syncthreads();
  const long long g0 = (long long)blockIdx.x * kThreads, g = g0 + threadIdx.x;
  const int i0 = image_of(L.im, L.n, &JImg::blk0, g0);
  if (g < L.blocks) {
    const int i = image_of(L.im, L.n, &JImg::blk0, g);
    unsigned long long* gh = S.hist + (size_t)i * 4 * 256;
    block_symbols(L, S, L.im[i], g, [&](int t, int sym) {
      if (i == i0)
        atomicAdd(sh + t * 256 + sym, 1u);
      else
        atomicAdd(gh + t * 256 + sym, 1ull);
    });
  }
  __syncthreads();
  unsigned long long* gh = S.hist + (size_t)i0 * 4 * 256;
  for (int j = threadIdx.x; j < 4 * 256; j += kThreads)
    if (sh[j]) atomicAdd(gh + j, (unsigned long long)sh[j]);
}

// the lowest key over the warp
__device__ __forceinline__ unsigned long long warp_min(unsigned long long k) {
#pragma unroll
  for (int o = 16; o; o >>= 1) k = min(k, __shfl_xor_sync(0xFFFFFFFFu, k, o));
  return k;
}

constexpr int kPer = (257 + 31) / 32;   // symbols per lane: lane l holds symbols l, l + 32, ..., symbol 256 on lane 0

struct TableShared {
  unsigned char size[257];       // unlimited code length per symbol
  int bits[kMaxLen + 1];         // symbols per length
  int at[kMaxLen + 1];           // the first list position of each unlimited length
};

// One warp per table: blockIdx.x is the slot (an image, or one scan of an image), warp t its table t of ntab, counted in
// hist[slot][t][256].
__global__ void __launch_bounds__(kThreads) jpeg_table_kernel(const unsigned long long* hist_all, JpegTables* tabs, int ntab) {
  __shared__ TableShared shared[4];
  const int t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  TableShared& W = shared[t];
  const unsigned long long* hist = hist_all + ((size_t)blockIdx.x * ntab + t) * 256;
  JpegTables& out = tabs[blockIdx.x];
  HuffCodes& hc = out.codes[t];

  // Annex K.2: merge the least frequent entry c1 with the next least frequent c2; among equal counts the higher symbol
  // goes first. Every symbol of both trees gets one bit longer; c1 then names the merged tree and holds its count.
  unsigned long long freq[kPer];
  int root[kPer], size[kPer];
#pragma unroll
  for (int s = 0; s < kPer; ++s) {
    const int j = lane + 32 * s;
    freq[s] = j < 256 ? hist[j] : j == 256 ? 1 : 0;
    root[s] = j;
    size[s] = 0;
  }
  constexpr unsigned long long kNone = ~0ull;
  for (;;) {
    unsigned long long k1 = kNone;
#pragma unroll
    for (int s = 0; s < kPer; ++s)
      if (freq[s] && freq[s] <= kMaxCandidate) k1 = min(k1, freq[s] << 9 | (511 - (lane + 32 * s)));
    k1 = warp_min(k1);
    const int c1 = 511 - (int)(k1 & 511);
    unsigned long long k2 = kNone;
#pragma unroll
    for (int s = 0; s < kPer; ++s)
      if (freq[s] && freq[s] <= kMaxCandidate && lane + 32 * s != c1) k2 = min(k2, freq[s] << 9 | (511 - (lane + 32 * s)));
    k2 = warp_min(k2);
    if (k2 == kNone) break;
    const int c2 = 511 - (int)(k2 & 511);
    const unsigned long long f2 = k2 >> 9;
#pragma unroll
    for (int s = 0; s < kPer; ++s) {
      const int j = lane + 32 * s;
      if (j == c1) freq[s] += f2;
      if (j == c2) freq[s] = 0;
      if (root[s] == c1 || root[s] == c2) {
        ++size[s];
        root[s] = c1;
      }
    }
  }
#pragma unroll
  for (int s = 0; s < kPer; ++s)
    if (lane + 32 * s < 257) W.size[lane + 32 * s] = (unsigned char)size[s];
  for (int j = lane; j < 256; j += 32) hc.size[j] = 0;
  for (int j = lane; j <= kMaxLen; j += 32) W.bits[j] = 0;
  __syncwarp();
  if (lane != 0) return;

  for (int j = 0; j < 256; ++j)
    if (W.size[j]) ++W.bits[W.size[j]];
  for (int l = 1, a = 0; l <= kMaxLen; ++l) {   // list positions by unlimited length (a stable counting sort by symbol)
    W.at[l] = a;
    a += W.bits[l];
  }
  ++W.bits[W.size[256]];
  // Annex K.3: move pairs of the longest codes up until no code is longer than 16 bits
  for (int l = kMaxLen; l > 16; --l) {
    while (W.bits[l] > 0) {
      int j = l - 2;
      while (W.bits[j] == 0) --j;
      W.bits[l] -= 2;
      W.bits[l - 1] += 1;
      W.bits[j + 1] += 2;
      W.bits[j] -= 1;
    }
  }
  int l = 16;
  while (W.bits[l] == 0) --l;
  W.bits[l] -= 1;   // the reserved symbol's code: one of the longest
  int nsym = 0;
  for (int j = 0; j < 16; ++j) {
    out.counts[t][j] = (unsigned char)W.bits[j + 1];
    nsym += W.bits[j + 1];
  }
  out.nsym[t] = nsym;
  for (int j = 0; j < 256; ++j)
    if (W.size[j]) out.syms[t][W.at[W.size[j]]++] = (unsigned char)j;
  // Annex C: canonical codes in list order with the limited lengths
  int code = 0, p = 0;
  for (int len = 1; len <= 16; ++len, code <<= 1)
    for (int k = 0; k < W.bits[len]; ++k, ++p, ++code) {
      hc.code[out.syms[t][p]] = (unsigned short)code;
      hc.size[out.syms[t][p]] = (unsigned char)len;
    }
}

// DHT segment k in the order libjpeg writes them, DC 0, AC 0, DC 1, AC 1: its table and its class / id byte
__device__ __forceinline__ int dht_table(int k) { return (k >> 1) + 2 * (k & 1); }
__device__ __forceinline__ int dht_class_id(int k) { return (k & 1) << 4 | k >> 1; }

__global__ void __launch_bounds__(kThreads) jpeg_opt_header_kernel(const __grid_constant__ HeaderList H, JpegScratch S) {
  const int i = blockIdx.x;
  const JpegTables& T = S.tabs[i];
  unsigned char* o = H.out[i];
  int seg[5];   // where each DHT segment starts, then SOS (header bytes without the APP1 / APP2 segments)
  seg[0] = H.sof_end;
#pragma unroll
  for (int k = 0; k < 4; ++k) seg[k + 1] = seg[k] + 2 + 2 + 1 + 16 + T.nsym[dht_table(k)];
  const int len = seg[4] + JPEG_SOS_BYTES;
  for (int j = threadIdx.x; j < len; j += kThreads) {
    unsigned char v;
    if (j < H.sof_end) {
      v = header_byte(H, i, j);
    } else if (j >= seg[4]) {
      v = H.bytes[H.len - JPEG_SOS_BYTES + (j - seg[4])];
    } else {
      int k = 0;
      while (j >= seg[k + 1]) ++k;
      const int t = dht_table(k), r = j - seg[k], n = seg[k + 1] - seg[k] - 2;
      v = r == 0 ? 0xFF : r == 1 ? 0xC4 : r == 2 ? n >> 8 : r == 3 ? n & 0xFF : r == 4 ? dht_class_id(k)
        : r < 21 ? T.counts[t][r - 5] : T.syms[t][r - 21];
    }
    o[header_at(H, j)] = v;
  }
  if (threadIdx.x == 0) S.hdr_len[i] = len + H.meta;
}

__global__ void __launch_bounds__(kThreads) jpeg_opt_bits_kernel(const __grid_constant__ JpegList L, JpegScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= L.blocks) return;
  const int i = image_of(L.im, L.n, &JImg::blk0, g);
  const HuffCodes* T = S.tabs[i].codes;
  const int diff = S.dcdiff[g];
  unsigned bits = nbits(diff);
  block_symbols(L, S, L.im[i], g, [&](int t, int sym) { bits += T[t].size[sym] + (t >= 2 ? sym & 15 : 0); });
  S.bits[g] = bits;
}

}  // namespace

int jpeg_optimize_tables(const JpegList& L, const JpegScratch& S, cudaStream_t st) {
  jpeg_hist_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, S);
  return jpeg_build_tables(S.hist, S.tabs, L.n, 4, st);
}

int jpeg_build_tables(const unsigned long long* hist, JpegTables* tabs, int slots, int ntab, cudaStream_t st) {
  jpeg_table_kernel<<<slots, 32 * ntab, 0, st>>>(hist, tabs, ntab);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

int jpeg_optimize_header(const JpegList& L, const HeaderList& H, const JpegScratch& S, cudaStream_t st) {
  jpeg_opt_header_kernel<<<L.n, kThreads, 0, st>>>(H, S);
  jpeg_opt_bits_kernel<<<grid_of(L.blocks, kThreads), kThreads, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

// PNG encoding of uint8 windows, byte for byte what cv2.imencode(".png", img) writes with no parameters: libpng 1.6 with
// OpenCV's settings (filter Sub on every row, None when the image is 1 pixel wide; IDAT chunks of 8192 bytes; no chunks
// besides IHDR, IDAT and IEND) over zlib 1.3 at level 1, memLevel 8, strategy Z_RLE. tests/util_png.py restates each stage
// in numpy; the comments below name the zlib source a stage follows.
//
// deflate_rle looks back one byte only and matches greedily, so the parse of every maximal run of L equal filtered bytes is
// fixed: one literal, (L - 1) / 258 matches of 258, then r = (L - 1) % 258 as one match (r >= 3) or r literals. A block
// ends every 16383 symbols. Given where the runs start, every stage is a scan, a reduction or a per-block serial step.
// Work is split into tiles of kTile filtered bytes (256 threads x 16 bytes); tiles never span two images. Launches on one
// stream:
//   runs:   per tile, its first and last run start and its Adler-32 sums;
//   carry:  one block: for each tile, the start of the run its first byte is in and the end of the run its last byte is in;
//   count:  per tile, its symbols; exclusive scan -> each tile's first symbol;
//   hist:   per tile, literal/length counts, matches and input bytes of the deflate blocks its symbols fall in;
//   trees:  one thread per deflate block: trees.c's build_tree / gen_bitlen / gen_codes / build_bl_tree and _tr_flush_block's
//           choice of stored, static or dynamic; its code table, header bits and data bits;
//   bits:   per tile, the bits of its symbols (none in stored blocks); exclusive scan;
//   place:  one warp per image: each block's first bit in order (a stored block pads to a byte), Adler-32 of the image;
//   emit:   per tile, each symbol's code at its bit offset into a zeroed word stream (atomicOr; LSB first, so the words'
//           bytes are the stream), or its bytes in a stored block;
//   header: one thread per block: the 3 type bits, the stored LEN / NLEN or the dynamic tree description, END_BLOCK;
//   file:   one warp per IDAT chunk: its bytes and CRC-32; chunk 0 also writes the signature and IHDR, the last one IEND
//           and the file's length.
#include <string.h>

#include <algorithm>
#include <climits>
#include <string>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_scan.cuh"

namespace se {

constexpr int PNG_MAX_BATCH = 32;   // images per call: their descriptors travel as kernel parameters
constexpr int kTileT = 256, kTileV = 16, kTile = kTileT * kTileV;
constexpr int kBlockSyms = 16383;   // (lit_bufsize - 1) symbols per block, lit_bufsize = 1 << (memLevel + 6)
constexpr int kMaxMatch = 258;
constexpr int kChunk = 8192;        // libpng's zbuffer: stream bytes per IDAT chunk
constexpr int kHead = 8 + 25;       // signature and IHDR
constexpr int kLCodes = 286, kDCodes = 30, kBLCodes = 19, kHeapSize = 2 * kLCodes + 1, kEndBlock = 256;
constexpr int kChunkWarps = 4;

// ------------------------------------------------------------------------------------------ tables (trees.c, CRC-32)
struct DeflateTabs {
  unsigned char length_code[256];   // match length - 3 -> length code 0..28 (_length_code)
  unsigned char base_length[29];
  unsigned char extra_lbits[29];
  unsigned char extra_dbits[30];
  unsigned char extra_blbits[19];
  unsigned char bl_order[19];
};
constexpr DeflateTabs deflate_tabs() {
  DeflateTabs t{};
  const unsigned char xl[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
  const unsigned char bo[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  for (int i = 0; i < 29; ++i) t.extra_lbits[i] = xl[i];
  for (int i = 0; i < 30; ++i) t.extra_dbits[i] = (unsigned char)(i < 4 ? 0 : (i - 2) / 2);
  for (int i = 0; i < 19; ++i) {
    t.extra_blbits[i] = (unsigned char)(i == 16 ? 2 : i == 17 ? 3 : i == 18 ? 7 : 0);
    t.bl_order[i] = bo[i];
  }
  int lc = 0;
  for (int code = 0; code < 28; ++code) {
    t.base_length[code] = (unsigned char)lc;
    for (int k = 0; k < (1 << xl[code]); ++k) t.length_code[lc++] = (unsigned char)code;
  }
  t.length_code[255] = 28;   // 258 is code 285, not 284 with extra 31
  t.base_length[28] = 255;
  return t;
}
__constant__ DeflateTabs c_tabs = deflate_tabs();

struct CrcTabs {
  unsigned t[256];
  unsigned shift[9][32];   // shift[k]: the state after 2^k zero bytes, as a GF(2) matrix (column i = image of bit i)
};
constexpr unsigned crc_step(const unsigned* t, unsigned s) { return t[s & 0xFF] ^ (s >> 8); }
constexpr CrcTabs crc_tabs() {
  CrcTabs c{};
  for (unsigned n = 0; n < 256; ++n) {
    unsigned v = n;
    for (int k = 0; k < 8; ++k) v = v & 1 ? 0xEDB88320u ^ (v >> 1) : v >> 1;
    c.t[n] = v;
  }
  for (int i = 0; i < 32; ++i) c.shift[0][i] = crc_step(c.t, 1u << i);
  for (int k = 1; k < 9; ++k)
    for (int i = 0; i < 32; ++i) {
      unsigned v = c.shift[k - 1][i], r = 0;
      for (int b = 0; b < 32; ++b)
        if (v >> b & 1) r ^= c.shift[k - 1][b];
      c.shift[k][i] = r;
    }
  return c;
}
__constant__ CrcTabs c_crc = crc_tabs();

// ------------------------------------------------------------------------------------------ descriptors
struct PImg {   // one image of a call; tile, block, word and chunk indices are the call's
  const unsigned char* src;
  unsigned char* out;
  long long* out_bytes;
  long long pitch;
  long long n;                                   // filtered bytes, h (1 + w c)
  long long pos0;                                // its first filtered byte in call coordinates
  long long tile0, ntiles, blk0, word0, chunk0;  // first tile, block slot, stream word and IDAT chunk slot
  int h, w, rowlen;                              // rowlen = 1 + w c
  unsigned char cmf, flg;                        // zlib header after libpng's window rewrite
};
struct PngList {
  PImg im[PNG_MAX_BATCH];
  int n, c, swap;
  long long tiles, blocks, chunks, bytes;
};
static_assert(sizeof(PngList) <= 4096, "descriptors must fit the kernel parameter space");

enum { kStored = 0, kStatic = 1, kDynamic = 2 };

struct PBlk {   // one deflate block
  unsigned lcode[kLCodes];   // bit-reversed code | length << 16
  unsigned dcode[kDCodes];
  unsigned blcode[kBLCodes];
  int kind, last, lcodes, dcodes, blcodes;
  long long hdr_bits, data_bits, stored_len;   // tree description bits; symbol bits without END_BLOCK; input bytes
  long long bit0, sbit0, byte0;                // (place) first bit; data bits of the blocks before; first input byte
};

struct PState {   // one image
  long long nsym, nblocks, zlen;   // symbols, blocks, zlib stream bytes
  unsigned adler;
};

struct PngScratch {
  long long *first, *last, *run_s, *run_e;   // [tiles]: first / last run start (call coordinates); carries
  unsigned* symcnt;                          // [tiles]
  unsigned long long* symoff;
  unsigned* bitcnt;
  unsigned long long* bitoff;
  unsigned long long *adl_a, *adl_b;         // [tiles]: sum of bytes; sum of (tile bytes - i) * byte_i
  unsigned* hist;                            // [blocks][288]: literal/length counts, [286] matches
  unsigned long long* bbytes;                // [blocks]
  PBlk* blk;                                 // [blocks]
  PState* st;                                // [n]
  unsigned* words;
  unsigned long long* sums;
};

// ------------------------------------------------------------------------------------------ filtered bytes
// The thread's kTileV filtered bytes from image position j0 (fewer at the image's end), and the byte before j0 (-1 at 0).
// A row is its filter byte (1 = Sub, or 0 = None for 1-pixel-wide images), then w c bytes in PNG order (RGB): channel ch
// reads source channel c - 1 - ch when swap (BGR source), ch otherwise; Sub subtracts the same channel of the pixel before.
__device__ __forceinline__ int load_bytes(const PngList& L, const PImg& d, long long j0, unsigned (&f)[kTileV], int& prev) {
  const int c = L.c;
  const int cnt = (int)min((long long)kTileV, d.n - j0);
  long long jj = j0 > 0 ? j0 - 1 : 0;
  long long y = jj / d.rowlen;
  int x = (int)(jj - y * d.rowlen);
  prev = -1;
  for (int k = (j0 > 0 ? -1 : 0); k < cnt; ++k) {
    unsigned v;
    if (x == 0) {
      v = d.w > 1 ? 1u : 0u;
    } else {
      const int i = x - 1, p = i / c, ch = i - p * c, sc = L.swap ? c - 1 - ch : ch;
      const unsigned char* row = d.src + y * d.pitch;
      v = row[p * c + sc];
      if (d.w > 1 && p > 0) v = (v - row[(p - 1) * c + sc]) & 0xFFu;
    }
    if (k < 0) prev = (int)v;
    else f[k] = v;
    if (++x == d.rowlen) {
      x = 0;
      ++y;
    }
  }
  return cnt;
}

// inclusive scans over a block's NT shared values: max from the left in a, min from the right in b
template <int NT>
__device__ __forceinline__ void scan_max_min(long long* a, long long* b) {
  const int t = threadIdx.x;
  for (int o = 1; o < NT; o <<= 1) {
    long long x = a[t], y = b[t];
    if (t >= o) x = max(x, a[t - o]);
    if (t + o < NT) y = min(y, b[t + o]);
    __syncthreads();
    a[t] = x;
    b[t] = y;
    __syncthreads();
  }
}

struct ThreadRuns {   // a thread's bytes, in image coordinates
  unsigned f[kTileV];
  unsigned starts;    // bit k: byte j0 + k starts a run
  long long j0, s0, e1;   // first byte; start of the run of byte j0; end of the run of its last byte
  int cnt;
};

// The thread's bytes and run flags, and (run_s / run_e given) where its first run starts and its last run ends.
__device__ __forceinline__ void thread_runs(const PngList& L, const PImg& d, long long tile, const PngScratch* S, ThreadRuns& R) {
  __shared__ long long sh_last[kTileT], sh_first[kTileT];
  R.j0 = (tile - d.tile0) * kTile + (long long)threadIdx.x * kTileV;
  int prev = -1;
  R.cnt = R.j0 < d.n ? load_bytes(L, d, R.j0, R.f, prev) : 0;
  R.starts = 0;
  long long lastp = -1, firstp = LLONG_MAX;
  for (int k = 0; k < R.cnt; ++k) {
    const bool s = (k == 0 ? prev : (int)R.f[k - 1]) != (int)R.f[k];
    if (s) {
      R.starts |= 1u << k;
      lastp = R.j0 + k;
      if (firstp == LLONG_MAX) firstp = R.j0 + k;
    }
  }
  R.s0 = R.e1 = 0;
  if (!S) return;   // the runs kernel: flags only
  // run start of byte j0: the last start at or before it; run end of the last byte: the first start after it
  sh_last[threadIdx.x] = lastp;
  sh_first[threadIdx.x] = firstp;
  __syncthreads();
  scan_max_min<kTileT>(sh_last, sh_first);
  const long long carry_s = S->run_s[tile] - d.pos0, carry_e = S->run_e[tile] - d.pos0;
  R.s0 = (R.starts & 1) ? R.j0 : max(carry_s, threadIdx.x ? sh_last[threadIdx.x - 1] : -1LL);
  R.e1 = min(carry_e, threadIdx.x + 1 < kTileT ? sh_first[threadIdx.x + 1] : LLONG_MAX);
  __syncthreads();
}

// f(k, len, value): the symbols starting at the thread's bytes in order; len 1 is a literal of byte value, len >= 3 a match
template <class F>
__device__ __forceinline__ void thread_symbols(const ThreadRuns& R, F&& f) {
  long long s = R.s0, e = R.e1;
  for (int k = 0; k < R.cnt; ++k) {
    const long long j = R.j0 + k;
    if (R.starts >> k & 1) s = j;
    if (k == 0 || (R.starts >> k & 1)) {   // the end of this run: the next start in the thread, else e1
      const unsigned later = k + 1 < 32 ? R.starts >> (k + 1) : 0u;
      e = later ? j + 1 + __ffs(later) - 1 : R.e1;
    }
    const long long q = j - s;
    if (q == 0) {
      f(k, 1, R.f[k]);
      continue;
    }
    const long long len = e - s, nfull = (len - 1) / kMaxMatch, r = (len - 1) % kMaxMatch, qq = q - 1;
    if (qq < nfull * kMaxMatch) {
      if (qq % kMaxMatch == 0) f(k, kMaxMatch, R.f[k]);
    } else if (r >= 3) {
      if (qq == nfull * kMaxMatch) f(k, (int)r, R.f[k]);
    } else {
      f(k, 1, R.f[k]);
    }
  }
}

// ------------------------------------------------------------------------------------------ runs and carries
template <class T>
__device__ __forceinline__ T block_sum(T v) {
  __shared__ T part[32];
  for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0)
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += part[i];
  __syncthreads();
  return s;   // in thread 0
}

// per tile: its first and last run start (call coordinates) and its Adler-32 sums
__global__ void __launch_bounds__(kTileT) png_runs_kernel(const __grid_constant__ PngList L, PngScratch S) {
  const long long tile = blockIdx.x;
  const PImg& d = L.im[image_of(L.im, L.n, &PImg::tile0, tile)];
  __shared__ long long lo[kTileT], hi[kTileT];
  ThreadRuns R;
  thread_runs(L, d, tile, nullptr, R);
  long long first = LLONG_MAX, last = -1;
  unsigned long long a = 0, b = 0;
  const long long t0 = (tile - d.tile0) * kTile, tn = min((long long)kTile, d.n - t0);
  for (int k = 0; k < R.cnt; ++k) {
    if (R.starts >> k & 1) {
      first = min(first, d.pos0 + R.j0 + k);
      last = d.pos0 + R.j0 + k;
    }
    a += R.f[k];
    b += (unsigned long long)(tn - (R.j0 + k - t0)) * R.f[k];
  }
  lo[threadIdx.x] = last;
  hi[threadIdx.x] = first;
  __syncthreads();
  scan_max_min<kTileT>(lo, hi);
  a = block_sum(a);
  b = block_sum(b);
  if (threadIdx.x == 0) {
    S.last[tile] = lo[kTileT - 1];
    S.first[tile] = hi[0];
    S.adl_a[tile] = a % 65521u;
    S.adl_b[tile] = b % 65521u;
  }
}

// run_s[t]: the last run start before tile t; run_e[t]: the first run start after it (the call's end past the last). Every
// image's first byte starts a run, so the scans over the call need no image boundaries.
__global__ void __launch_bounds__(1024) png_carry_kernel(long long tiles, long long total, PngScratch S) {
  __shared__ long long a[1024], b[1024];
  long long carry = -1;
  for (long long c0 = 0; c0 < tiles; c0 += 1024) {
    const long long t = c0 + threadIdx.x;
    a[threadIdx.x] = t < tiles ? S.last[t] : -1;
    b[threadIdx.x] = LLONG_MAX;
    __syncthreads();
    scan_max_min<1024>(a, b);
    if (t < tiles) S.run_s[t] = threadIdx.x ? max(carry, a[threadIdx.x - 1]) : carry;
    const long long next = max(carry, a[1023]);
    __syncthreads();
    carry = next;
  }
  carry = total;
  for (long long c1 = tiles; c1 > 0; c1 -= 1024) {
    const long long t = c1 - 1024 + threadIdx.x;   // may be negative in the first chunk
    a[threadIdx.x] = -1;
    b[threadIdx.x] = t >= 0 ? S.first[t] : LLONG_MAX;
    __syncthreads();
    scan_max_min<1024>(a, b);
    if (t >= 0) S.run_e[t] = threadIdx.x + 1 < 1024 ? min(carry, b[threadIdx.x + 1]) : carry;
    const long long next = min(carry, b[0]);
    __syncthreads();
    carry = next;
  }
}

// ------------------------------------------------------------------------------------------ symbols
enum { kCount = 0, kHist = 1, kBits = 2, kEmit = 3 };

__device__ __forceinline__ int lcode_of_len(int len) { return 257 + c_tabs.length_code[len - 3]; }

// bits of one symbol with the block's codes (0 in a stored block)
__device__ __forceinline__ unsigned sym_bits(const PBlk& B, int len, unsigned v) {
  if (B.kind == kStored) return 0;
  if (len == 1) return B.lcode[v] >> 16;
  const int code = c_tabs.length_code[len - 3];
  return (B.lcode[257 + code] >> 16) + c_tabs.extra_lbits[code] + (B.dcode[0] >> 16);
}

__device__ __forceinline__ void put_bits(unsigned* w, unsigned long long pos, unsigned long long val, int len) {
  if (!len) return;
  const unsigned long long v = val << (pos & 31);
  const long long i = (long long)(pos >> 5);
  if ((unsigned)v) atomicOr(w + i, (unsigned)v);
  if ((pos & 31) + len > 32 && (unsigned)(v >> 32)) atomicOr(w + i + 1, (unsigned)(v >> 32));
}

__device__ __forceinline__ void put_byte(unsigned* w, unsigned long long byte_pos, unsigned v) {
  if (v) atomicOr(w + (byte_pos >> 2), v << (8 * (byte_pos & 3)));
}

template <int MODE>
__global__ void __launch_bounds__(kTileT) png_sym_kernel(const __grid_constant__ PngList L, PngScratch S) {
  const long long tile = blockIdx.x;
  const PImg& d = L.im[image_of(L.im, L.n, &PImg::tile0, tile)];
  ThreadRuns R;
  thread_runs(L, d, tile, &S, R);
  if (MODE == kCount) {
    unsigned n = 0;
    thread_symbols(R, [&](int, int, unsigned) { ++n; });
    const unsigned long long t = block_sum((unsigned long long)n);
    if (threadIdx.x == 0) S.symcnt[tile] = (unsigned)t;
    return;
  }
  unsigned n = 0;
  thread_symbols(R, [&](int, int, unsigned) { ++n; });
  unsigned long long total;
  const long long sym0 = (long long)(S.symoff[tile] - S.symoff[d.tile0]) + (long long)block_exclusive_scan<kTileT>(n, &total);
  if (MODE == kHist) {
    __shared__ unsigned sh[2][288];
    __shared__ unsigned long long shb[2];
    const long long tsym0 = (long long)(S.symoff[tile] - S.symoff[d.tile0]), b_lo = tsym0 / kBlockSyms;
    for (int i = threadIdx.x; i < 2 * 288; i += kTileT) (&sh[0][0])[i] = 0;
    if (threadIdx.x < 2) shb[threadIdx.x] = 0;
    __syncthreads();
    long long k = sym0;
    thread_symbols(R, [&](int, int len, unsigned v) {
      const int b = (int)(k++ / kBlockSyms - b_lo);
      atomicAdd(&sh[b][len == 1 ? v : lcode_of_len(len)], 1u);
      if (len > 1) atomicAdd(&sh[b][286], 1u);
      atomicAdd(&shb[b], (unsigned long long)len);
    });
    __syncthreads();
    const long long nb = (tsym0 + (long long)total + kBlockSyms - 1) / kBlockSyms - b_lo;   // blocks the tile touches
    for (int i = threadIdx.x; i < nb * 288; i += kTileT) {
      const unsigned v = sh[i / 288][i % 288];
      if (v) atomicAdd(&S.hist[(d.blk0 + b_lo + i / 288) * 288 + i % 288], v);
    }
    if (threadIdx.x < nb && shb[threadIdx.x]) atomicAdd(&S.bbytes[d.blk0 + b_lo + threadIdx.x], shb[threadIdx.x]);
    return;
  }
  const PBlk* blk = S.blk + d.blk0;
  unsigned bits = 0;
  {
    long long k = sym0;
    thread_symbols(R, [&](int, int len, unsigned v) { bits += sym_bits(blk[k++ / kBlockSyms], len, v); });
  }
  if (MODE == kBits) {
    const unsigned long long t = block_sum((unsigned long long)bits);
    if (threadIdx.x == 0) S.bitcnt[tile] = (unsigned)t;
    return;
  }
  // emit: symbol bits before this thread's in the image, as if all blocks were coded back to back (sbit)
  unsigned long long sbit = (S.bitoff[tile] - S.bitoff[d.tile0]) + block_exclusive_scan<kTileT>(bits, &total);
  unsigned* w = S.words + d.word0;
  long long k = sym0;
  thread_symbols(R, [&](int kk, int len, unsigned v) {
    const PBlk& B = blk[k++ / kBlockSyms];
    if (B.kind == kStored) {   // its bytes at the block's data, byte aligned after LEN / NLEN
      const unsigned long long at = (unsigned long long)((B.bit0 + 3 + 7) >> 3) + 4 + (R.j0 + kk - B.byte0);
      for (int i = 0; i < len; ++i) put_byte(w, at + i, v);
      return;
    }
    const unsigned long long pos = (unsigned long long)(B.bit0 + 3 + B.hdr_bits) + (sbit - (unsigned long long)B.sbit0);
    if (len == 1) {
      const unsigned e = B.lcode[v];
      put_bits(w, pos, e & 0xFFFF, e >> 16);
      sbit += e >> 16;
      return;
    }
    const int code = c_tabs.length_code[len - 3], xb = c_tabs.extra_lbits[code];
    const unsigned e = B.lcode[257 + code], dc = B.dcode[0];
    const unsigned long long x = (unsigned long long)(e & 0xFFFF) | ((unsigned long long)(len - 3 - c_tabs.base_length[code]) << (e >> 16));
    put_bits(w, pos, x, (e >> 16) + xb);
    put_bits(w, pos + (e >> 16) + xb, dc & 0xFFFF, dc >> 16);
    sbit += (e >> 16) + xb + (dc >> 16);
  });
}

// ------------------------------------------------------------------------------------------ trees (trees.c)
struct TreeWork {
  unsigned freq[kHeapSize];
  unsigned short len[kHeapSize], dad[kHeapSize];
  unsigned char depth[kHeapSize];
  short heap[kHeapSize];
  int bl_count[16];
};

__device__ __forceinline__ int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }
__device__ __forceinline__ unsigned bi_reverse(unsigned code, int len) { return len ? __brev(code) >> (32 - len) : 0; }
__device__ __forceinline__ unsigned static_lcode(int n) {
  const unsigned c = n < 144 ? 0x30 + n : n < 256 ? 0x190 + (n - 144) : n < 280 ? n - 256 : 0xC0 + (n - 280);
  return bi_reverse(c, static_llen(n)) | (unsigned)static_llen(n) << 16;
}

__device__ __forceinline__ bool smaller(const TreeWork& W, int n, int m) {
  return W.freq[n] < W.freq[m] || (W.freq[n] == W.freq[m] && W.depth[n] <= W.depth[m]);
}

__device__ void pqdownheap(TreeWork& W, int heap_len, int k) {
  const int v = W.heap[k];
  int j = k << 1;
  while (j <= heap_len) {
    if (j < heap_len && smaller(W, W.heap[j + 1], W.heap[j])) j++;
    if (smaller(W, v, W.heap[j])) break;
    W.heap[k] = W.heap[j];
    k = j;
    j <<= 1;
  }
  W.heap[k] = (short)v;
}

// build_tree, gen_bitlen and gen_codes over W.freq[0..elems): stat 1 = the static literal/length lengths, 2 = the static
// distance lengths (5), 0 = none (bit-length tree). codes[n] = bit-reversed code | length << 16. opt_len / static_len as
// trees.c adds to them.
__device__ void build_tree(TreeWork& W, int elems, int stat, const unsigned char* extra, int base, int max_length, unsigned* codes,
                           int& max_code_out, long long& opt_len, long long& static_len) {
  int heap_len = 0, heap_max = kHeapSize, max_code = -1;
  for (int n = 0; n < elems; ++n) {
    if (W.freq[n]) {
      W.heap[++heap_len] = (short)(max_code = n);
      W.depth[n] = 0;
    } else {
      W.len[n] = 0;
    }
  }
  while (heap_len < 2) {
    const int node = max_code < 2 ? ++max_code : 0;
    W.heap[++heap_len] = (short)node;
    W.freq[node] = 1;
    W.depth[node] = 0;
    opt_len--;
    if (stat) static_len -= stat == 1 ? static_llen(node) : 5;
  }
  for (int k = heap_len / 2; k >= 1; --k) pqdownheap(W, heap_len, k);
  int node = elems;
  do {
    const int n = W.heap[1];
    W.heap[1] = W.heap[heap_len--];
    pqdownheap(W, heap_len, 1);
    const int m = W.heap[1];
    W.heap[--heap_max] = (short)n;
    W.heap[--heap_max] = (short)m;
    W.freq[node] = W.freq[n] + W.freq[m];
    W.depth[node] = (unsigned char)((W.depth[n] >= W.depth[m] ? W.depth[n] : W.depth[m]) + 1);
    W.dad[n] = W.dad[m] = (unsigned short)node;
    W.heap[1] = (short)node++;
    pqdownheap(W, heap_len, 1);
  } while (heap_len >= 2);
  W.heap[--heap_max] = W.heap[1];

  // gen_bitlen
  for (int b = 0; b < 16; ++b) W.bl_count[b] = 0;
  W.len[W.heap[heap_max]] = 0;
  int overflow = 0, h;
  for (h = heap_max + 1; h < kHeapSize; ++h) {
    const int n = W.heap[h];
    int bits = W.len[W.dad[n]] + 1;
    if (bits > max_length) bits = max_length, overflow++;
    W.len[n] = (unsigned short)bits;
    if (n > max_code) continue;
    W.bl_count[bits]++;
    const int xbits = n >= base ? extra[n - base] : 0;
    const long long f = W.freq[n];
    opt_len += f * (bits + xbits);
    if (stat) static_len += f * ((stat == 1 ? static_llen(n) : 5) + xbits);
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (W.bl_count[bits] == 0) bits--;
      W.bl_count[bits]--;
      W.bl_count[bits + 1] += 2;
      W.bl_count[max_length]--;
      overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; bits--) {
      int n = W.bl_count[bits];
      while (n != 0) {
        const int m = W.heap[--h];
        if (m > max_code) continue;
        if (W.len[m] != bits) {
          opt_len += ((long long)bits - W.len[m]) * W.freq[m];
          W.len[m] = (unsigned short)bits;
        }
        n--;
      }
    }
  }
  // gen_codes
  unsigned next_code[16];
  unsigned code = 0;
  for (int bits = 1; bits <= 15; bits++) {
    code = (code + W.bl_count[bits - 1]) << 1;
    next_code[bits] = code;
  }
  for (int n = 0; n < elems; ++n) {
    const int l = n <= max_code ? W.len[n] : 0;
    codes[n] = l ? bi_reverse(next_code[l]++, l) | (unsigned)l << 16 : 0;
  }
  max_code_out = max_code;
}

// scan_tree / send_tree over the code lengths of codes[0..max_code]: f(symbol, extra value, extra bits) per bit-length symbol
template <class F>
__device__ void tree_runs(const unsigned* codes, int max_code, F&& f) {
  int prevlen = -1, nextlen = codes[0] >> 16, count = 0, max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  for (int n = 0; n <= max_code; n++) {
    const int curlen = nextlen;
    nextlen = n + 1 <= max_code ? (int)(codes[n + 1] >> 16) : 0xFFFF;
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      do f(curlen, 0, 0);
      while (--count != 0);
    } else if (curlen != 0) {
      if (curlen != prevlen) {
        f(curlen, 0, 0);
        count--;
      }
      f(16, count - 3, 2);
    } else if (count <= 10) {
      f(17, count - 3, 3);
    } else {
      f(18, count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

__device__ __forceinline__ long long image_syms(const PImg& d, const PngScratch& S) {
  const long long t = d.tile0 + d.ntiles - 1;
  return (long long)(S.symoff[t] + S.symcnt[t] - S.symoff[d.tile0]);
}

// One thread per block slot: the block's trees and _tr_flush_block's choice. A stored block is only chosen when its input
// is at most 1.5 x its literals (stored_len + 4 <= static_lenb needs 8 (match bytes) <= literals + 18 matches), so at most
// 24575 bytes: its data is still in zlib's window and the buf != NULL condition holds.
__global__ void __launch_bounds__(1) png_tree_kernel(const __grid_constant__ PngList L, PngScratch S) {
  __shared__ TreeWork W;   // about 6.4 KB: in shared memory rather than on a per-thread stack
  const long long g = blockIdx.x;
  const PImg& d = L.im[image_of(L.im, L.n, &PImg::blk0, g)];
  const long long nsym = image_syms(d, S), nblocks = nsym / kBlockSyms + 1, b = g - d.blk0;
  if (b >= nblocks) return;
  PBlk& B = S.blk[g];
  const unsigned* hist = S.hist + g * 288;
  long long opt_len = 0, static_len = 0, dummy = 0;
  for (int n = 0; n < kLCodes; ++n) W.freq[n] = hist[n];
  W.freq[kEndBlock] = 1;
  unsigned *lcode = B.lcode, *dcode = B.dcode, *blcode = B.blcode;   // the dynamic codes; a static block overwrites them
  int lmax, dmax, blmax;
  build_tree(W, kLCodes, 1, c_tabs.extra_lbits, 257, 15, lcode, lmax, opt_len, static_len);
  for (int n = 0; n < kDCodes; ++n) W.freq[n] = 0;
  W.freq[0] = hist[286];
  build_tree(W, kDCodes, 2, c_tabs.extra_dbits, 0, 15, dcode, dmax, opt_len, static_len);
  for (int n = 0; n < kBLCodes; ++n) W.freq[n] = 0;
  auto count_bl = [&](int sym, int, int) { W.freq[sym]++; };
  tree_runs(lcode, lmax, count_bl);
  tree_runs(dcode, dmax, count_bl);
  build_tree(W, kBLCodes, 0, c_tabs.extra_blbits, 0, 7, blcode, blmax, opt_len, dummy);
  int max_blindex = kBLCodes - 1;
  for (; max_blindex >= 3; max_blindex--)
    if (blcode[c_tabs.bl_order[max_blindex]] >> 16) break;
  opt_len += 3 * ((long long)max_blindex + 1) + 5 + 5 + 4;
  long long opt_lenb = (opt_len + 3 + 7) >> 3;
  const long long static_lenb = (static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
  const long long stored_len = (long long)S.bbytes[g];
  B.stored_len = stored_len;
  B.last = b == nblocks - 1;
  B.hdr_bits = 0;
  if (stored_len + 4 <= opt_lenb) {
    B.kind = kStored;
    B.data_bits = 0;
    return;
  }
  if (static_lenb == opt_lenb) {
    B.kind = kStatic;
    for (int n = 0; n < kLCodes; ++n) B.lcode[n] = static_lcode(n);
    for (int n = 0; n < kDCodes; ++n) B.dcode[n] = bi_reverse(n, 5) | 5u << 16;
  } else {
    B.kind = kDynamic;
    B.lcodes = lmax + 1;
    B.dcodes = dmax + 1;
    B.blcodes = max_blindex + 1;
    long long hb = 5 + 5 + 4 + 3LL * B.blcodes;
    auto count_hdr = [&](int sym, int, int nb) { hb += (blcode[sym] >> 16) + nb; };
    tree_runs(lcode, lmax, count_hdr);
    tree_runs(dcode, dmax, count_hdr);
    B.hdr_bits = hb;
  }
  long long db = (long long)hist[286] * (B.dcode[0] >> 16);
  for (int n = 0; n < kLCodes; ++n)
    if (hist[n]) db += (long long)hist[n] * ((B.lcode[n] >> 16) + (n > 256 ? c_tabs.extra_lbits[n - 257] : 0));
  B.data_bits = db;
}

// ------------------------------------------------------------------------------------------ place, headers, file
__device__ __forceinline__ unsigned adler_mod(unsigned long long v) { return (unsigned)(v % 65521u); }

// one warp per image: lane 0 places the blocks in order; the lanes fold the tiles' Adler sums in 32 contiguous segments
__global__ void __launch_bounds__(32) png_place_kernel(const __grid_constant__ PngList L, PngScratch S) {
  const PImg& d = L.im[blockIdx.x];
  const int lane = threadIdx.x;
  const long long nsym = image_syms(d, S), nblocks = nsym / kBlockSyms + 1;
  const long long per = (d.ntiles + 31) / 32, t0 = min(d.ntiles, lane * per), t1 = min(d.ntiles, t0 + per);
  unsigned long long A = 0, Bs = 0, n = 0;   // segment sums from a = 0: A = sum of bytes, Bs = sum over its bytes of (n - i) d_i
  for (long long t = t0; t < t1; ++t) {
    const long long tn = min((long long)kTile, d.n - t * kTile);
    Bs = (Bs + (unsigned long long)adler_mod(tn) * A + S.adl_b[d.tile0 + t]) % 65521u;
    A = (A + S.adl_a[d.tile0 + t]) % 65521u;
    n += tn;
  }
  if (lane == 0) {
    unsigned long long bit = 0, sbit = 0, byte0 = 0;
    for (long long b = 0; b < nblocks; ++b) {
      PBlk& B = S.blk[d.blk0 + b];
      B.bit0 = (long long)bit;
      B.sbit0 = (long long)sbit;
      B.byte0 = (long long)byte0;
      if (B.kind == kStored) bit = (((bit + 3 + 7) >> 3) + 4 + B.stored_len) * 8;
      else bit += 3 + B.hdr_bits + B.data_bits + (B.lcode[kEndBlock] >> 16);
      sbit += B.data_bits;
      byte0 += B.stored_len;
    }
    S.st[blockIdx.x].nsym = nsym;
    S.st[blockIdx.x].nblocks = nblocks;
    S.st[blockIdx.x].zlen = 2 + (long long)((bit + 7) >> 3) + 4;
  }
  unsigned long long a = 1, bb = 0;   // lane 0 folds the segments in order
  for (int l = 0; l < 32; ++l) {
    const unsigned long long sA = __shfl_sync(0xffffffffu, A, l), sB = __shfl_sync(0xffffffffu, Bs, l),
                             sn = __shfl_sync(0xffffffffu, n, l);
    bb = (bb + (sn % 65521u) * a + sB) % 65521u;
    a = (a + sA) % 65521u;
  }
  if (lane == 0) S.st[blockIdx.x].adler = (unsigned)((bb << 16) | a);
}

__global__ void __launch_bounds__(32) png_header_kernel(const __grid_constant__ PngList L, PngScratch S) {
  const long long g = (long long)blockIdx.x * 32 + threadIdx.x;
  if (g >= L.blocks) return;
  const int i = image_of(L.im, L.n, &PImg::blk0, g);
  const PImg& d = L.im[i];
  if (g - d.blk0 >= S.st[i].nblocks) return;
  const PBlk& B = S.blk[g];
  unsigned* w = S.words + d.word0;
  unsigned long long pos = (unsigned long long)B.bit0;
  put_bits(w, pos, (unsigned)B.last | (unsigned)B.kind << 1, 3);
  pos += 3;
  if (B.kind == kStored) {
    const unsigned len = (unsigned)B.stored_len;
    put_bits(w, ((pos + 7) >> 3) * 8, len | (~len & 0xFFFFu) << 16, 32);
    return;
  }
  if (B.kind == kDynamic) {
    put_bits(w, pos, B.lcodes - 257, 5);
    put_bits(w, pos + 5, B.dcodes - 1, 5);
    put_bits(w, pos + 10, B.blcodes - 4, 4);
    pos += 14;
    for (int r = 0; r < B.blcodes; ++r, pos += 3) put_bits(w, pos, B.blcode[c_tabs.bl_order[r]] >> 16, 3);
    auto send = [&](int sym, int val, int nb) {
      const unsigned e = B.blcode[sym];
      put_bits(w, pos, e & 0xFFFF, e >> 16);
      pos += e >> 16;
      put_bits(w, pos, (unsigned)val, nb);
      pos += nb;
    };
    tree_runs(B.lcode, B.lcodes - 1, send);
    tree_runs(B.dcode, B.dcodes - 1, send);
  }
  const unsigned e = B.lcode[kEndBlock];
  put_bits(w, (unsigned long long)(B.bit0 + 3 + B.hdr_bits + B.data_bits), e & 0xFFFF, e >> 16);
}

__device__ __forceinline__ unsigned crc_shift(unsigned s, int nbytes) {   // nbytes <= 511 zero bytes
  for (int k = 0; k < 9; ++k)
    if (nbytes >> k & 1) {
      unsigned r = 0;
      for (int b = 0; b < 32; ++b)
        if (s >> b & 1) r ^= c_crc.shift[k][b];
      s = r;
    }
  return s;
}

__device__ __forceinline__ void put_be32(unsigned char* o, unsigned v) {
  o[0] = (unsigned char)(v >> 24);
  o[1] = (unsigned char)(v >> 16);
  o[2] = (unsigned char)(v >> 8);
  o[3] = (unsigned char)v;
}

// One warp per IDAT chunk slot. Each lane copies and CRCs a 256-byte segment of the chunk from state 0; lane 0 folds the
// segments: crc(s, A B) = shift(crc(s, A), |B|) ^ crc(0, B).
__global__ void __launch_bounds__(32 * kChunkWarps) png_file_kernel(const __grid_constant__ PngList L, PngScratch S) {
  __shared__ unsigned tab[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) tab[i] = c_crc.t[i];
  __syncthreads();
  const long long g = (long long)blockIdx.x * kChunkWarps + (threadIdx.x >> 5);
  if (g >= L.chunks) return;
  const int i = image_of(L.im, L.n, &PImg::chunk0, g), lane = threadIdx.x & 31;
  const PImg& d = L.im[i];
  const PState st = S.st[i];
  const long long c = g - d.chunk0, nch = (st.zlen + kChunk - 1) / kChunk;
  if (c >= nch) return;
  const unsigned char* z = reinterpret_cast<const unsigned char*>(S.words + d.word0);
  const long long zb = st.zlen - 6;   // deflate bytes
  const long long z0 = c * kChunk, zn = min((long long)kChunk, st.zlen - z0);
  unsigned char* o = d.out + kHead + c * (kChunk + 12);
  const int seg = kChunk / 32, s0 = lane * seg, s1 = (int)min((long long)s0 + seg, zn);
  unsigned r = 0;
  for (int k = s0; k < s1; ++k) {
    const long long q = z0 + k;
    unsigned v;
    if (q == 0) v = d.cmf;
    else if (q == 1) v = d.flg;
    else if (q - 2 < zb) v = z[q - 2];
    else v = st.adler >> (8 * (3 - (int)(q - 2 - zb))) & 0xFF;
    o[8 + k] = (unsigned char)v;
    r = tab[(r ^ v) & 0xFF] ^ (r >> 8);
  }
  const unsigned char idat[4] = {'I', 'D', 'A', 'T'};
  unsigned crc = 0xFFFFFFFFu;
  for (int k = 0; k < 4; ++k) crc = tab[(crc ^ idat[k]) & 0xFF] ^ (crc >> 8);
  for (int l = 0; l < 32; ++l) {
    const unsigned rl = __shfl_sync(0xffffffffu, r, l);
    const int nl = (int)max(0LL, min((long long)seg, zn - (long long)l * seg));
    if (nl) crc = crc_shift(crc, nl) ^ rl;
  }
  if (lane) return;
  put_be32(o, (unsigned)zn);
  o[4] = 'I', o[5] = 'D', o[6] = 'A', o[7] = 'T';
  put_be32(o + 8 + zn, ~crc);
  if (c == 0) {   // signature and IHDR
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    unsigned char* h = d.out;
    for (int k = 0; k < 8; ++k) h[k] = sig[k];
    put_be32(h + 8, 13);
    const unsigned char body[17] = {'I', 'H', 'D', 'R', (unsigned char)(d.w >> 24), (unsigned char)(d.w >> 16), (unsigned char)(d.w >> 8),
                                    (unsigned char)d.w, (unsigned char)(d.h >> 24), (unsigned char)(d.h >> 16), (unsigned char)(d.h >> 8),
                                    (unsigned char)d.h, 8, (unsigned char)(L.c == 3 ? 2 : 0), 0, 0, 0};
    unsigned hc = 0xFFFFFFFFu;
    for (int k = 0; k < 17; ++k) {
      h[12 + k] = body[k];
      hc = tab[(hc ^ body[k]) & 0xFF] ^ (hc >> 8);
    }
    put_be32(h + 29, ~hc);
  }
  if (c == nch - 1) {   // IEND and the file's length
    unsigned char* e = o + 12 + zn;
    const unsigned char iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    for (int k = 0; k < 12; ++k) e[k] = iend[k];
    *d.out_bytes = (long long)(e + 12 - d.out);
  }
}

// ------------------------------------------------------------------------------------------ host
static long long filtered_bytes(int h, int w, int c) { return (long long)h * (1 + (long long)w * c); }
static long long deflate_max(long long n) { return n + 8 * (n / kBlockSyms + 2) + 8; }
static long long max_blocks(long long n) { return n / kBlockSyms + 1; }
static long long zlib_max(long long n) { return 2 + deflate_max(n) + 4; }
static long long chunks_max(long long n) { return (zlib_max(n) + kChunk - 1) / kChunk; }

long long png_max_bytes(int h, int w, int c) {
  const long long n = filtered_bytes(h, w, c);
  return kHead + zlib_max(n) + 12 * chunks_max(n) + 12;
}

// CMF and FLG: zlib's 0x78 0x01 (level 1 with Z_RLE: FLEVEL 0), then libpng's optimize_cmf: for at most 16384 bytes of data
// the smallest window that covers them, and FCHECK recomputed
static void zlib_header(long long n, unsigned char& cmf, unsigned char& flg) {
  unsigned cinfo = 7;
  if (n <= 16384) {
    unsigned half = 1u << 14;
    do {
      half >>= 1;
      --cinfo;
    } while (cinfo > 0 && n <= half);
  }
  cmf = (unsigned char)(cinfo << 4 | 8);
  flg = (unsigned char)(0x1F - ((unsigned)cmf << 8) % 0x1F);
}

struct PngLayout {
  long long tiles = 0, blocks = 0, words = 0, chunks = 0, bytes = 0;
  size_t first, last, run_s, run_e, symcnt, symoff, bitcnt, bitoff, adl_a, adl_b, hist, bbytes, blk, st, words_at, sums, total;
};

static PngLayout png_layout(const int* hw, int n, int c) {
  PngLayout l;
  for (int i = 0; i < n; ++i) {
    const long long nb = filtered_bytes(hw[2 * i], hw[2 * i + 1], c);
    l.tiles += (nb + kTile - 1) / kTile;
    l.blocks += max_blocks(nb);
    l.words += deflate_max(nb) / 4 + 2;
    l.chunks += chunks_max(nb);
    l.bytes += nb;
  }
  size_t at = 0;
  auto take = [&](size_t bytes) {
    const size_t p = at;
    at += scratch_round(bytes);
    return p;
  };
  const size_t t8 = (size_t)l.tiles * 8, t4 = (size_t)l.tiles * 4;
  l.first = take(t8);
  l.last = take(t8);
  l.run_s = take(t8);
  l.run_e = take(t8);
  l.symcnt = take(t4);
  l.symoff = take(t8);
  l.bitcnt = take(t4);
  l.bitoff = take(t8);
  l.adl_a = take(t8);
  l.adl_b = take(t8);
  l.hist = take((size_t)l.blocks * 288 * 4);
  l.bbytes = take((size_t)l.blocks * 8);
  l.blk = take((size_t)l.blocks * sizeof(PBlk));
  l.st = take((size_t)std::max(n, 1) * sizeof(PState));
  l.words_at = take((size_t)l.words * 4);
  l.sums = take((size_t)std::max((l.tiles + SCAN_TILE - 1) / SCAN_TILE, 1LL) * 8);
  l.total = at;
  return l;
}

}  // namespace se

using namespace se;

extern "C" {

long long se_png_max_bytes(int h, int w, int channels) {
  if (h < 1 || w < 1 || h > kMaxDim || w > kMaxDim || (channels != 1 && channels != 3)) {
    set_error("se_png_max_bytes: sizes must be in [1, 65535] and channels 1 or 3");
    return -1;
  }
  return png_max_bytes(h, w, channels);
}

int se_png_encode_u8(const unsigned char* const* src, const long long* src_pitch, const int* hw, int n, int channels, int swap_rb,
                     unsigned char* out, const long long* out_off, long long* out_bytes_dev, void* scratch, long long* scratch_bytes,
                     void* stream) {
  SE_REQUIRE(n >= 0 && n <= PNG_MAX_BATCH, "n must be in [0, " + std::to_string(PNG_MAX_BATCH) + "] images per call");
  SE_REQUIRE(channels == 1 || channels == 3, "channels must be 1 or 3");
  SE_REQUIRE(swap_rb == 0 || swap_rb == 1, "swap_rb must be 0 or 1");
  SE_REQUIRE(scratch_bytes != nullptr, "scratch_bytes");
  SE_REQUIRE(n == 0 || (src_pitch && hw && out_off), "null size / offset array");
  for (int i = 0; i < n; ++i)
    if (int rc = check_window(i, hw[2 * i], hw[2 * i + 1], src_pitch[i], (long long)channels * hw[2 * i + 1], out_off[i])) return rc;
  const PngLayout lay = png_layout(hw, n, channels);
  SE_SCRATCH(scratch, scratch_bytes, lay.total, n);
  SE_REQUIRE(src && out && out_bytes_dev, "null src / out / out_bytes");
  for (int i = 0; i < n; ++i) SE_REQUIRE(src[i] != nullptr, "null src");
  SE_REQUIRE(lay.tiles < (1LL << 31) && lay.chunks < (1LL << 31) * kChunkWarps, "batch too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;

  PngList L;
  memset(&L, 0, sizeof(L));
  L.n = n;
  L.c = channels;
  L.swap = swap_rb;
  long long tile = 0, blk = 0, word = 0, chunk = 0, pos = 0;
  for (int i = 0; i < n; ++i) {
    const int h = hw[2 * i], w = hw[2 * i + 1];
    const long long nb = filtered_bytes(h, w, channels);
    PImg& d = L.im[i];
    d.src = src[i];
    d.out = out + out_off[i];
    d.out_bytes = out_bytes_dev + i;
    d.pitch = src_pitch[i];
    d.n = nb;
    d.pos0 = pos;
    d.tile0 = tile;
    d.ntiles = (nb + kTile - 1) / kTile;
    d.blk0 = blk;
    d.word0 = word;
    d.chunk0 = chunk;
    d.h = h;
    d.w = w;
    d.rowlen = 1 + w * channels;
    zlib_header(nb, d.cmf, d.flg);
    pos += nb;
    tile += d.ntiles;
    blk += max_blocks(nb);
    word += deflate_max(nb) / 4 + 2;
    chunk += chunks_max(nb);
  }
  L.tiles = tile;
  L.blocks = blk;
  L.chunks = chunk;
  L.bytes = pos;
  unsigned char* s = (unsigned char*)scratch;
  PngScratch S;
  S.first = (long long*)(s + lay.first);
  S.last = (long long*)(s + lay.last);
  S.run_s = (long long*)(s + lay.run_s);
  S.run_e = (long long*)(s + lay.run_e);
  S.symcnt = (unsigned*)(s + lay.symcnt);
  S.symoff = (unsigned long long*)(s + lay.symoff);
  S.bitcnt = (unsigned*)(s + lay.bitcnt);
  S.bitoff = (unsigned long long*)(s + lay.bitoff);
  S.adl_a = (unsigned long long*)(s + lay.adl_a);
  S.adl_b = (unsigned long long*)(s + lay.adl_b);
  S.hist = (unsigned*)(s + lay.hist);
  S.bbytes = (unsigned long long*)(s + lay.bbytes);
  S.blk = (PBlk*)(s + lay.blk);
  S.st = (PState*)(s + lay.st);
  S.words = (unsigned*)(s + lay.words_at);
  S.sums = (unsigned long long*)(s + lay.sums);

  SE_CUDA_OK(cudaMemsetAsync(S.hist, 0, (size_t)L.blocks * 288 * 4, st));
  SE_CUDA_OK(cudaMemsetAsync(S.bbytes, 0, (size_t)L.blocks * 8, st));
  SE_CUDA_OK(cudaMemsetAsync(S.words, 0, (size_t)lay.words * 4, st));
  const unsigned tiles = (unsigned)L.tiles;
  png_runs_kernel<<<tiles, kTileT, 0, st>>>(L, S);
  png_carry_kernel<<<1, 1024, 0, st>>>(L.tiles, L.bytes, S);
  png_sym_kernel<kCount><<<tiles, kTileT, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  int rc = exclusive_scan(S.symcnt, S.symoff, S.sums, L.tiles, st);
  if (rc) return rc;
  png_sym_kernel<kHist><<<tiles, kTileT, 0, st>>>(L, S);
  png_tree_kernel<<<(unsigned)L.blocks, 1, 0, st>>>(L, S);
  png_sym_kernel<kBits><<<tiles, kTileT, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  rc = exclusive_scan(S.bitcnt, S.bitoff, S.sums, L.tiles, st);
  if (rc) return rc;
  png_place_kernel<<<n, 32, 0, st>>>(L, S);
  png_sym_kernel<kEmit><<<tiles, kTileT, 0, st>>>(L, S);
  png_header_kernel<<<grid_of(L.blocks, 32), 32, 0, st>>>(L, S);
  png_file_kernel<<<grid_of(L.chunks, kChunkWarps), 32 * kChunkWarps, 0, st>>>(L, S);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

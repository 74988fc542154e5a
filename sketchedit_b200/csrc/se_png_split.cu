// PNG decoding of large files across the whole GPU: the pixels of se_png_decode_u8 (the same files, arguments and status
// rule), with each file's zlib stream inflated by many warps at once (se_inflate_split.cuh) instead of one.
//
// Six launches per call, every dependency between CTAs at a launch boundary:
//   find:    one warp per chunk of S compressed bytes: chunk 0 starts after the zlib header, chunk k > 0 at the first
//            dynamic-block header in its bits (find_block, 32 candidate bits per step), or is empty;
//   count:   one warp per non-empty chunk: its blocks up to the next non-empty chunk's start, counting bytes (chunk_count);
//   link:    one thread per file: the chunks must join end to start, end with the final block and sum to the file's raw
//            size (chunks_link), which gives each chunk its output offset; otherwise the file's status is nonzero;
//   emit:    one warp per chunk: its blocks again, into 4-byte entries, a literal or the position of a byte before the chunk;
//   resolve: one thread per raw byte: its entry's markers followed back to a literal (resolve_byte), written to the raw
//            filtered scanlines; the Adler-32 sums of the bytes reduced per CTA and added into the file's two sums;
//   rows:    one CTA of kRowWarps warps per file: the Adler-32 against the stream's, then the rows of se_png_dec.cuh, warp w
//            taking the groups of 32 rows g = w, w + kRowWarps, ... each staggered behind the group before it through a
//            progress counter in shared memory (lane 0 of group g reads the last row of group g - 1 as lane 31 writes it).
// A file whose stream has few dynamic blocks has few non-empty chunks and decodes with little parallelism (one warp for a
// single-block stream), but correctly.
#include <string.h>

#include <string>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_inflate_split.cuh"
#include "se_png_dec.cuh"

namespace se {

constexpr int kChunkWarps = 4;     // chunks per CTA in find, count and emit (4 table sets: 22 KB of shared memory)
constexpr int kRowWarps = 32;      // warps of the rows CTA
constexpr int kResolveThreads = 256;
constexpr long long kMaxSplitRaw = 0x7FFFFFFFll;   // entries hold positions in 31 bits

struct SFile {
  long long src_off, src_len, plte_off, raw_off;   // raw_off: the file's raw bytes in scratch, and its entries at 4 times it
  unsigned char* out;
  int chunk0, nchunks;                               // its chunks in the call's chunk list
  int h, w, depth, ctype, npal, mode;
};
struct SState {                    // per file, in scratch: set by link, resolve and rows
  unsigned long long a, b;         // Adler-32 sums of the resolved bytes (resolve)
  long long tail;                  // the bit after the final block (link)
  int status;
};
struct SList {
  const unsigned char* src;
  unsigned char* raw;
  unsigned* ent;
  SplitChunk* chunks;
  SState* st;
  int* status;
  long long S;
  int n, nchunks;
  SFile f[PNG_DECODE_MAX_BATCH];
};

__device__ __forceinline__ long long raw_n_of(const SFile& F) { return raw_bytes(F.h, F.w, F.depth, F.ctype); }

__global__ void __launch_bounds__(32 * kChunkWarps) split_find_kernel(const __grid_constant__ SList L) {
  const int lane = threadIdx.x & 31, g = blockIdx.x * kChunkWarps + (threadIdx.x >> 5);
  if (g >= L.nchunks) return;
  const int i = image_of(L.f, L.n, &SFile::chunk0, g);
  const SFile& F = L.f[i];
  const long long k = g - F.chunk0;
  long long start = 16;
  if (k > 0) {
    long long lo, hi;
    chunk_bits(k, L.S, F.src_len, &lo, &hi);
    start = find_block(L.src + F.src_off, F.src_len, lo, hi, lane, 32);
  }
  if (lane == 0) L.chunks[g] = SplitChunk{start, -1, 0, 0, 0, 0, 0};
}

__global__ void __launch_bounds__(32 * kChunkWarps) split_count_kernel(const __grid_constant__ SList L) {
  __shared__ InflateTabs tabs[kChunkWarps];
  const int lane = threadIdx.x & 31, g = blockIdx.x * kChunkWarps + (threadIdx.x >> 5);
  if (g >= L.nchunks) return;
  SplitChunk c = L.chunks[g];
  if (c.start < 0) return;
  const int i = image_of(L.f, L.n, &SFile::chunk0, g);
  const SFile& F = L.f[i];
  for (int k = g + 1; k < F.chunk0 + F.nchunks; ++k)
    if (L.chunks[k].start >= 0) {
      c.next = L.chunks[k].start;
      break;
    }
  const int st = chunk_count(L.src + F.src_off, F.src_len, raw_n_of(F), c, g == F.chunk0, tabs[threadIdx.x >> 5], lane, 32);
  if (lane == 0) {
    c.status = st;
    L.chunks[g] = c;
  }
}

__global__ void split_link_kernel(const __grid_constant__ SList L) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.n) return;
  const SFile& F = L.f[i];
  long long tail = 0;
  L.st[i] = SState{0, 0, 0, chunks_link(L.chunks + F.chunk0, F.nchunks, raw_n_of(F), &tail)};
  L.st[i].tail = tail;
}

__global__ void __launch_bounds__(32 * kChunkWarps) split_emit_kernel(const __grid_constant__ SList L) {
  __shared__ InflateTabs tabs[kChunkWarps];
  const int lane = threadIdx.x & 31, g = blockIdx.x * kChunkWarps + (threadIdx.x >> 5);
  if (g >= L.nchunks) return;
  const SplitChunk c = L.chunks[g];
  const int i = image_of(L.f, L.n, &SFile::chunk0, g);
  if (c.start < 0 || L.st[i].status) return;
  const SFile& F = L.f[i];
  const int st = chunk_emit(L.src + F.src_off, F.src_len, c, L.ent + F.raw_off, tabs[threadIdx.x >> 5], lane, 32);
  if (lane == 0 && st) atomicCAS(&L.st[i].status, 0, st);
}

// grid (x, file): threads stride over the file's raw bytes.
__global__ void __launch_bounds__(kResolveThreads) split_resolve_kernel(const __grid_constant__ SList L) {
  __shared__ unsigned long long part[2][kResolveThreads / 32];
  __shared__ int skip;
  const SFile& F = L.f[blockIdx.y];
  SState& S = L.st[blockIdx.y];
  if (threadIdx.x == 0) skip = *(volatile int*)&S.status;   // link's or emit's verdict: the entries are incomplete
  __syncthreads();
  if (skip) return;
  const long long n = raw_n_of(F);
  unsigned* e = L.ent + F.raw_off;
  unsigned char* raw = L.raw + F.raw_off;
  unsigned long long a = 0, b = 0;
  bool bad = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = resolve_byte(e, i);
    bad |= v < 0;
    const unsigned d = v < 0 ? 0 : (unsigned)v;
    e[i] = kLiteral | d;   // later chains that reach i stop here
    raw[i] = (unsigned char)d;
    a += d;
    b += (unsigned long long)(n - i) * d;   // byte i is counted in n - i of the running sums (adler32_lanes)
  }
  a %= 65521;
  b %= 65521;
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xFFFFFFFFu, a, o);
    b += __shfl_xor_sync(0xFFFFFFFFu, b, o);
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    part[0][w] = a;
    part[1][w] = b;
  }
  if (bad) atomicCAS(&S.status, 0, (int)INF_LINK);
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long sa = 0, sb = 0;
    for (int k = 0; k < kResolveThreads / 32; ++k) {
      sa += part[0][k];
      sb += part[1][k];
    }
    atomicAdd(&S.a, sa % 65521);
    atomicAdd(&S.b, sb % 65521);
  }
}

// The stagger of the rows CTA: warp `warp` runs group g behind the warp running group g - 1, which publishes in prog[] how
// many pixels of its last row it has written back, as g (npx + 1) + pixels.
struct RowsStagger {
  volatile long long* prog;
  long long g, npx;
  int warp, lane;
  __device__ void before(long long t) {
    if (g == 0 || t >= npx || (t & 63)) return;
    const long long want = (g - 1) * (npx + 1) + (t + 64 < npx ? t + 64 : npx);
    while (prog[(warp + kRowWarps - 1) % kRowWarps] < want) {
    }
    __threadfence_block();
  }
  __device__ void after(long long t, long long done) {
    if (lane == 31 && done > 0 && ((done & 63) == 0 || done == npx) && t - 31 < npx) {
      __threadfence_block();   // the row's bytes before the count that announces them
      prog[warp] = g * (npx + 1) + done;
    }
  }
};

__global__ void __launch_bounds__(32 * kRowWarps) split_rows_kernel(const __grid_constant__ SList L) {
  __shared__ unsigned char pal[768];
  __shared__ long long prog[kRowWarps];
  __shared__ int err_sh;
  const SFile& F = L.f[blockIdx.x];
  const SState& S = L.st[blockIdx.x];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x < kRowWarps) prog[threadIdx.x] = -1;
  if (F.ctype == 3)
    for (int k = threadIdx.x; k < 3 * F.npal; k += blockDim.x) pal[k] = L.src[F.plte_off + k];
  int st = S.status;
  if (st == INF_OK) {
    const long long n = raw_n_of(F), want = stored_adler(L.src + F.src_off, F.src_len, S.tail);
    const unsigned long long a = (S.a % 65521 + 1) % 65521, b = (S.b % 65521 + (unsigned long long)(n % 65521)) % 65521;
    st = want < 0 ? INF_SHORT_INPUT : (long long)(b << 16 | a) == want ? INF_OK : INF_ADLER;
  }
  if (threadIdx.x == 0) err_sh = st;
  __syncthreads();
  if (st == INF_OK) {
    const PRows R{F.out, F.h, F.w, F.depth, F.ctype, F.npal, F.mode};
    const int bpp_bits = channels_of(F.ctype) * F.depth;
    const long long npx = row_bytes(F.w, F.depth, F.ctype) / (bpp_bits < 8 ? 1 : bpp_bits / 8);
    int err = 0;
    for (long long g = warp; g * 32 < F.h; g += kRowWarps) {
      RowsStagger sync{prog, g, npx, warp, lane};
      png_row_group(R, L.raw + F.raw_off, pal, (int)(g * 32), lane, err, sync);
    }
    if (err) atomicCAS(&err_sh, 0, err);
  }
  __syncthreads();
  if (threadIdx.x == 0) L.status[blockIdx.x] = err_sh;
}

}  // namespace se

using namespace se;

extern "C" {

int se_png_split_u8(const unsigned char* src, const long long* src_off, const long long* src_len, const int* info,
                    const long long* plte_off, int n, unsigned char* const* out, int* status_dev, long long chunk_bytes,
                    void* scratch, long long* scratch_bytes, void* stream) {
  if (int rc = png_check_files(src_off, src_len, info, plte_off, n, scratch_bytes)) return rc;
  SE_REQUIRE(chunk_bytes >= 1, "chunk_bytes must be at least 1");
  long long raw = 0, nchunks = 0, max_raw = 0;
  for (int i = 0; i < n; ++i) {
    const long long r = raw_bytes(info[6 * i], info[6 * i + 1], info[6 * i + 2], info[6 * i + 3]);
    SE_REQUIRE(r <= kMaxSplitRaw, "file " + std::to_string(i) + ": " + std::to_string(r) +
                                      " bytes of scanlines, more than the split decoder's 2^31 - 1");
    raw += (r + 15) / 16 * 16;
    max_raw = r > max_raw ? r : max_raw;
    nchunks += src_len[i] / chunk_bytes + 1;
  }
  SE_REQUIRE(nchunks <= 0x7FFFFFFFll, "more than 2^31 - 1 chunks: chunk_bytes is too small");
  // scratch: per file state, chunks, raw filtered scanlines, entries (4 bytes per raw byte)
  const long long st_bytes = ((long long)sizeof(SState) * n + 255) / 256 * 256;
  const long long ch_bytes = ((long long)sizeof(SplitChunk) * nchunks + 255) / 256 * 256;
  SE_SCRATCH(scratch, scratch_bytes, st_bytes + ch_bytes + 5 * raw, n);
  SE_REQUIRE(src && out && status_dev, "null src / out / status");
  for (int i = 0; i < n; ++i) SE_REQUIRE(out[i] != nullptr, "null out");
  if (n == 0) return 0;
  SList L;
  memset(&L, 0, sizeof(L));
  char* s = (char*)scratch;
  L.src = src;
  L.st = (SState*)s;
  L.chunks = (SplitChunk*)(s + st_bytes);
  L.raw = (unsigned char*)(s + st_bytes + ch_bytes);
  L.ent = (unsigned*)(s + st_bytes + ch_bytes + raw);
  L.status = status_dev;
  L.S = chunk_bytes;
  L.n = n;
  L.nchunks = (int)nchunks;
  long long at = 0;
  int c0 = 0;
  for (int i = 0; i < n; ++i) {
    const int* f = info + 6 * i;
    SFile& d = L.f[i];
    d.src_off = src_off[i];
    d.src_len = src_len[i];
    d.raw_off = at;
    d.out = out[i];
    d.chunk0 = c0;
    d.nchunks = (int)(src_len[i] / chunk_bytes + 1);
    d.h = f[0];
    d.w = f[1];
    d.depth = f[2];
    d.ctype = f[3];
    d.npal = f[4];
    d.mode = f[5];
    d.plte_off = d.ctype == 3 ? plte_off[i] : 0;
    at += (raw_bytes(d.h, d.w, d.depth, d.ctype) + 15) / 16 * 16;
    c0 += d.nchunks;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int cblocks = (int)((nchunks + kChunkWarps - 1) / kChunkWarps);
  split_find_kernel<<<cblocks, 32 * kChunkWarps, 0, st>>>(L);
  split_count_kernel<<<cblocks, 32 * kChunkWarps, 0, st>>>(L);
  split_link_kernel<<<(n + 127) / 128, 128, 0, st>>>(L);
  split_emit_kernel<<<cblocks, 32 * kChunkWarps, 0, st>>>(L);
  const long long rblocks = (max_raw + kResolveThreads * 8 - 1) / (kResolveThreads * 8);
  split_resolve_kernel<<<dim3((unsigned)(rblocks < 4096 ? rblocks : 4096), n), kResolveThreads, 0, st>>>(L);
  split_rows_kernel<<<n, 32 * kRowWarps, 0, st>>>(L);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

// Progressive JPEG for se_jpeg_encode_progressive_u8: byte for byte what PIL.Image.save(buf, "JPEG", quality=q,
// subsampling=s, progressive=True) writes, libjpeg-turbo's jcphuff.c coder over jpeg_simple_progression's ten scans, each
// scan with optimal Huffman tables built from its own symbol counts. tests/util_jpeg_progressive.py restates it in numpy.
// After se_jpeg.cu's dct kernel has left the quantised coefficients in scratch, per call (a slot is one block of one scan):
//   prep:   one thread per slot of an AC scan: whether the block codes a symbol (N), whether it ends in an EOB run (T), and
//           the correction bits that trail its last symbol (refinement scans).
//   runs:   one thread per EOB run, started at the scan's first slot and at each N slot: it walks the run's slots in order
//           and places the run's emissions (before the next N slot's first symbol, every 0x7FFF blocks, once the waiting
//           correction bits pass 937, and at the end of the scan) on the slots that emit them.
//   hist:   one thread per slot counts the symbols it emits into its (image, scan)'s two histograms.
//   tables: se_jpeg_opt.cu's Annex K.2 / K.3 builder, one warp per (image, scan, table).
//   bits:   one thread per slot, its bit count with the scan's tables; an exclusive scan over the call.
//   pack:   one thread per slot writes its codes at its bit offset in its (image, scan)'s zeroed word stream by atomicOr,
//           and the correction bits its emissions carry.
//   stuff:  per 64-byte chunk of a stream: count its 0xFF bytes, scan the counts; then one CTA per image writes SOI..SOF2,
//           each scan's DHT segments and SOS at the offsets the scan lengths give, and EOI; then the chunks write their bytes
//           with 0x00 after each 0xFF (each scan's last byte padded with 1-bits).
// hist, bits and pack walk a slot's symbols through one function, prog_symbols, so the counts and the codes agree.
#include <algorithm>
#include <type_traits>

#include "../../include/sketchedit_b200.h"
#include "se_jpeg.h"
#include "se_scan.cuh"

namespace se {

namespace {

constexpr int kThreads = 128;
constexpr int kChunkBytes = 64;
constexpr int kMaxRun = 0x7FFF;                 // jcphuff.c forces an EOB run out at this length
constexpr int kCorrLimit = 1000 - 64 + 1;       // ... and once more than MAX_CORR_BITS - DCTSIZE2 + 1 correction bits wait
constexpr unsigned char kT = 0x80, kN = 0x40;   // slot flags
static_assert(sizeof(JpegList) + sizeof(ProgList) + sizeof(ProgScratch) <= 4096, "descriptors must fit the kernel parameter space");
static_assert(sizeof(HeaderList) + sizeof(ProgList) + sizeof(ProgScratch) <= 4096, "descriptors must fit the kernel parameter space");

struct ScanDef {
  int comp, ss, se, ah, al;   // comp -1: Y, Cb, Cr interleaved
};

// jpeg_simple_progression for three YCbCr components
__host__ __device__ __forceinline__ ScanDef scan_def(int s) {
  switch (s) {
    case 0: return {-1, 0, 0, 0, 1};
    case 1: return {0, 1, 5, 0, 2};
    case 2: return {2, 1, 63, 0, 1};
    case 3: return {1, 1, 63, 0, 1};
    case 4: return {0, 6, 63, 0, 2};
    case 5: return {0, 1, 63, 2, 1};
    case 6: return {-1, 0, 0, 1, 0};
    case 7: return {2, 1, 63, 1, 0};
    case 8: return {1, 1, 63, 1, 0};
    default: return {0, 1, 63, 1, 0};
  }
}

// the slots of scan s: every block of every MCU for the DC scans, else the component's own blocks
__host__ __device__ __forceinline__ long long scan_slots(int h, int w, int sub, int s) {
  const int c = scan_def(s).comp;
  const long long mh = mcu_h(sub), mw = mcu_w(sub);
  const long long mcus = ((h + mh - 1) / mh) * ((w + mw - 1) / mw);
  if (c < 0) return mcus * mcu_blocks(sub);
  if (c > 0) return mcus;   // a chroma block per MCU
  return (long long)((h + 7) / 8) * ((w + 7) / 8);
}

// Most bits one slot of scan s accounts for (DESIGN §7b): a DC first code and value; a DC refinement bit; per AC
// coefficient a code and value (26), a run/1 code, sign and correction bit (18), or a ZRL share (1); and one EOB run (16 + 14).
__host__ __device__ __forceinline__ int slot_max_bits(int s) {
  const ScanDef d = scan_def(s);
  if (d.comp < 0) return d.ah ? 1 : 16 + 11;
  return (d.se - d.ss + 1) * (d.ah ? 18 : 26) + 30;
}
__host__ __device__ __forceinline__ long long scan_words(long long slots, int s) { return (slots * slot_max_bits(s) + 31) / 32; }
__host__ __device__ __forceinline__ long long scan_chunks(long long words) { return (words * 4 + kChunkBytes - 1) / kChunkBytes; }

struct Stream {   // one (image, scan) of the call
  int i, s;
  long long slot0, nslot, word0, chunk0, nchunk;
};

// the stream holding call slot g (by_chunk = false) or call chunk g (true)
__device__ Stream stream_of(const JpegList& L, const ProgList& P, long long g, bool by_chunk) {
  Stream r;
  r.i = by_chunk ? image_of(P.im, L.n, &PImg::chunk0, g) : image_of(P.im, L.n, &PImg::slot0, g);
  const JImg& d = L.im[r.i];
  r.slot0 = P.im[r.i].slot0;
  r.word0 = P.im[r.i].word0;
  r.chunk0 = P.im[r.i].chunk0;
  for (r.s = 0;; ++r.s) {
    r.nslot = scan_slots(d.h, d.w, L.sub, r.s);
    const long long words = scan_words(r.nslot, r.s);
    r.nchunk = scan_chunks(words);
    if (r.s == JPEG_SCANS - 1 || (by_chunk ? g < r.chunk0 + r.nchunk : g < r.slot0 + r.nslot)) break;
    r.slot0 += r.nslot;
    r.word0 += words;
    r.chunk0 += r.nchunk;
  }
  return r;
}

// the MCU-order block (se_jpeg.cu's numbering within the image) of slot p of a scan of component c (-1: interleaved)
__device__ __forceinline__ long long slot_block(const JImg& d, int sub, int c, long long p) {
  if (c < 0) return p;
  const int per = mcu_blocks(sub);
  if (sub == 0) return p * 3 + c;
  if (c > 0) return p * per + per - 3 + c;
  const int bw = (d.w + 7) / 8;
  const long long bx = p % bw, by = p / bw;
  if (sub == 1) return (by * d.mcu_x + (bx >> 1)) * 4 + (bx & 1);
  return ((by >> 1) * d.mcu_x + (bx >> 1)) * 6 + (by & 1) * 2 + (bx & 1);
}

struct Slot {
  Stream st;
  ScanDef sc;
  long long g, e;   // call slot; the block in its image
  const JImg* d;
};

__device__ __forceinline__ Slot slot_at(const JpegList& L, const ProgList& P, long long g) {
  Slot q;
  q.st = stream_of(L, P, g, false);
  q.sc = scan_def(q.st.s);
  q.g = g;
  q.d = &L.im[q.st.i];
  q.e = slot_block(*q.d, L.sub, q.sc.comp, g - q.st.slot0);
  return q;
}

__device__ __forceinline__ int coef_at(const JpegList& L, const ProgScratch& S, const Slot& q, int k) {
  return S.coef[(size_t)k * L.blocks + q.d->blk0 + q.e];
}

// prep: N, T and the trailing correction bits of an AC slot (jcphuff.c encode_mcu_AC_first / encode_mcu_AC_refine)
__global__ void __launch_bounds__(kThreads) jpeg_prog_prep_kernel(const __grid_constant__ JpegList L,
                                                                 const __grid_constant__ ProgList P, ProgScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= P.slots) return;
  const Slot q = slot_at(L, P, g);
  if (q.sc.comp < 0) return;
  int last = 0, eob = 0;   // the last nonzero (first scans) / newly nonzero (refinement) position, 0: none
  for (int k = q.sc.ss; k <= q.sc.se; ++k) {
    const int y = coef_at(L, S, q, k), a = (y < 0 ? -y : y) >> q.sc.al;
    if (a) last = k;
    if (a == 1) eob = k;
  }
  const int at = q.sc.ah ? eob : last;
  unsigned char f = (at ? kN : 0) | (at < q.sc.se ? kT : 0);
  unsigned long long corr = 0;
  if (q.sc.ah) {
    int n = 0;
    for (int k = max(at + 1, q.sc.ss); k <= q.sc.se; ++k) {
      const int y = coef_at(L, S, q, k), a = (y < 0 ? -y : y) >> q.sc.al;
      if (a > 1) {
        corr = corr << 1 | (a & 1);
        ++n;
      }
    }
    f |= (unsigned char)n;
    S.corr[g] = corr;
  }
  S.flags[g] = f;
}

// runs: the thread of a run's first slot walks it; each later N slot starts the next run
__global__ void __launch_bounds__(kThreads) jpeg_prog_runs_kernel(const __grid_constant__ JpegList L,
                                                                 const __grid_constant__ ProgList P, ProgScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= P.slots) return;
  const Stream st = stream_of(L, P, g, false);
  if (scan_def(st.s).comp < 0 || (g != st.slot0 && !(S.flags[g] & kN))) return;
  const long long end = st.slot0 + st.nslot;
  unsigned run = 0, be = 0, from = 0;
  auto visit = [&](long long j, unsigned f) {   // slot j of the walk; true: the run has ended
    if (j != g && (f & kN)) {   // the next run starts here: its first symbol is preceded by this one
      if (run) {
        ProgRun& r = S.runs[j];
        r.pre_run = (unsigned short)run;
        r.pre_be = (unsigned short)be;
        r.pre_from = from;
      }
      return true;
    }
    if (!(f & kT)) return false;
    if (f & 63) {
      if (!be) from = (unsigned)(j - st.slot0);
      be += f & 63;
    }
    if (++run == kMaxRun || be > kCorrLimit || j == end - 1) {   // forced out, or the end of the scan
      ProgRun& r = S.runs[j];
      r.post_run = (unsigned short)run;
      r.post_be = (unsigned short)be;
      r.post_from = from;
      run = be = 0;
    }
    return false;
  };
  // 16 flags per load where aligned. 16 slots that all extend the run (T, not N) and cut it nowhere (the count stays
  // below 0x7FFF, the waiting bits within the limit, the scan goes on) are one step: their correction bits are summed.
  for (long long j = g; j < end;) {
    if ((j & 15) || j + 16 > end) {
      if (visit(j, S.flags[j])) return;
      ++j;
      continue;
    }
    const uint4 v = *reinterpret_cast<const uint4*>(S.flags + j);
    const unsigned w[4] = {v.x, v.y, v.z, v.w};
    const bool step = run + 16 < kMaxRun && j + 16 < end;
    if (step && (v.x & v.y & v.z & v.w) == 0x80808080u && (v.x | v.y | v.z | v.w) == 0x80808080u) {   // no bits: flat blocks
      run += 16;
      j += 16;
      continue;
    }
    if (step && ((v.x & v.y & v.z & v.w) & 0x80808080u) == 0x80808080u && !((v.x | v.y | v.z | v.w) & 0x40404040u)) {
      unsigned sum = 0, first = 16;
#pragma unroll
      for (int k = 3; k >= 0; --k) {
        const unsigned c = w[k] & 0x3F3F3F3Fu;
        sum += (c * 0x01010101u) >> 24;   // the four byte counts (each <= 63) added in the top byte
        if (c) first = 4 * k + (__ffs(c) - 1) / 8;
      }
      if (be + sum <= kCorrLimit) {
        if (!be && sum) from = (unsigned)(j + first - st.slot0);
        be += sum;
        run += 16;
        j += 16;
        continue;
      }
    }
#pragma unroll
    for (int b = 0; b < 16; ++b)
      if (visit(j + b, (w[b >> 2] >> 8 * (b & 3)) & 0xFFu)) return;
    j += 16;
  }
}

// Every code slot q emits, in order: f(t, sym, bits, nb) is Huffman symbol sym of the scan's table t followed by nb value
// bits, or for sym < 0 nb raw bits. With GATHER false an emitted run's correction bits come as one call of their count
// (bits 0); with GATHER true as the bits themselves, one call per slot that holds some.
template <bool GATHER, class F>
__device__ __forceinline__ void prog_symbols(const JpegList& L, const ProgScratch& S, const Slot& q, F&& f) {
  const ScanDef& sc = q.sc;
  if (sc.comp < 0) {
    const int dc = dc_of(*q.d, L.sub, S.coef, q.e) >> sc.al;
    if (sc.ah) {
      f(0, -1, (unsigned long long)(dc & 1), 1);
      return;
    }
    const long long p = prev_same_comp(L.sub, q.e);
    const int diff = dc - (p < 0 ? 0 : dc_of(*q.d, L.sub, S.coef, p) >> sc.al), nb = nbits(diff);
    f(block_at(*q.d, L.sub, q.e).comp ? 1 : 0, nb, (unsigned long long)((diff < 0 ? diff - 1 : diff) & ((1 << nb) - 1)), nb);
    return;
  }
  const int t = sc.comp ? 1 : 0;
  const ProgRun R = S.runs[q.g];
  auto emit = [&](unsigned run, unsigned be, unsigned from) {
    const int nb = 31 - __clz(run);
    f(t, nb << 4, (unsigned long long)(run & ((1u << nb) - 1)), nb);
    if (!be) return;
    if constexpr (!GATHER) {
      f(t, -1, 0ull, (int)be);
    } else {
      for (long long j = q.st.slot0 + from; be; ++j) {
        const int n = S.flags[j] & 63;
        if (!n) continue;
        f(t, -1, S.corr[j], n);
        be -= n;
      }
    }
  };
  bool first = true;
  auto lead = [&]() {   // the run before this block goes out ahead of its first symbol
    if (first && R.pre_run) emit(R.pre_run, R.pre_be, R.pre_from);
    first = false;
  };
  int r = 0;
  if (!sc.ah) {
    for (int k = sc.ss; k <= sc.se; ++k) {
      const int y = coef_at(L, S, q, k), a = (y < 0 ? -y : y) >> sc.al;
      if (!a) {
        ++r;
        continue;
      }
      lead();
      for (; r > 15; r -= 16) f(t, 0xF0, 0ull, 0);
      const int nb = nbits(a);
      f(t, r << 4 | nb, (unsigned long long)((y < 0 ? ~a : a) & ((1 << nb) - 1)), nb);
      r = 0;
    }
  } else {
    int eob = 0;
    for (int k = sc.ss; k <= sc.se; ++k) {
      const int y = coef_at(L, S, q, k);
      if (((y < 0 ? -y : y) >> sc.al) == 1) eob = k;
    }
    unsigned long long br = 0;   // this block's waiting correction bits
    int nbr = 0;
    for (int k = sc.ss; k <= sc.se; ++k) {
      const int y = coef_at(L, S, q, k), a = (y < 0 ? -y : y) >> sc.al;
      if (!a) {
        ++r;
        continue;
      }
      while (r > 15 && k <= eob) {
        lead();
        f(t, 0xF0, 0ull, 0);
        r -= 16;
        if (nbr) f(t, -1, br, nbr);
        br = 0;
        nbr = 0;
      }
      if (a > 1) {
        br = br << 1 | (a & 1);
        ++nbr;
        continue;
      }
      lead();
      f(t, r << 4 | 1, (unsigned long long)(y < 0 ? 0 : 1), 1);
      if (nbr) f(t, -1, br, nbr);
      br = 0;
      nbr = 0;
      r = 0;
    }
  }
  if (R.post_run) emit(R.post_run, R.post_be, R.post_from);   // the trailing correction bits are among the run's
}

__device__ __forceinline__ int stream_key(const Stream& st) { return st.i * JPEG_SCANS + st.s; }

__global__ void __launch_bounds__(kThreads) jpeg_prog_hist_kernel(const __grid_constant__ JpegList L,
                                                                 const __grid_constant__ ProgList P, ProgScratch S) {
  __shared__ unsigned sh[2 * 256];
  for (int j = threadIdx.x; j < 2 * 256; j += kThreads) sh[j] = 0;
  __syncthreads();
  const long long g0 = (long long)blockIdx.x * kThreads, g = g0 + threadIdx.x;
  const int key0 = stream_key(stream_of(L, P, g0, false));
  if (g < P.slots) {
    const Slot q = slot_at(L, P, g);
    const int key = stream_key(q.st);
    unsigned long long* gh = S.hist + (size_t)key * 2 * 256;
    prog_symbols<false>(L, S, q, [&](int t, int sym, unsigned long long, int) {
      if (sym < 0) return;
      if (key == key0)
        atomicAdd(sh + t * 256 + sym, 1u);
      else
        atomicAdd(gh + t * 256 + sym, 1ull);
    });
  }
  __syncthreads();
  unsigned long long* gh = S.hist + (size_t)key0 * 2 * 256;
  for (int j = threadIdx.x; j < 2 * 256; j += kThreads)
    if (sh[j]) atomicAdd(gh + j, (unsigned long long)sh[j]);
}

__global__ void __launch_bounds__(kThreads) jpeg_prog_bits_kernel(const __grid_constant__ JpegList L,
                                                                 const __grid_constant__ ProgList P, ProgScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= P.slots) return;
  const Slot q = slot_at(L, P, g);
  const HuffCodes* T = S.tabs[stream_key(q.st)].codes;
  unsigned bits = 0;
  prog_symbols<false>(L, S, q, [&](int t, int sym, unsigned long long, int nb) { bits += (sym < 0 ? 0 : T[t].size[sym]) + nb; });
  S.bits[g] = bits;
}

__global__ void __launch_bounds__(kThreads) jpeg_prog_pack_kernel(const __grid_constant__ JpegList L,
                                                                 const __grid_constant__ ProgList P, ProgScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= P.slots) return;
  const Slot q = slot_at(L, P, g);
  const HuffCodes* T = S.tabs[stream_key(q.st)].codes;
  const unsigned long long at = S.bitoff[g] - S.bitoff[q.st.slot0];
  unsigned* w = S.words + q.st.word0;
  long long wi = (long long)(at >> 5);
  int n = (int)(at & 31);
  unsigned long long acc = 0;
  prog_symbols<true>(L, S, q, [&](int t, int sym, unsigned long long bits, int nb) {
    if (sym >= 0) {   // code <= 16 bits and value <= 14 bits
      put_bits(acc, n, w, wi, ((unsigned)T[t].code[sym] << nb) | (unsigned)bits, T[t].size[sym] + nb);
      return;
    }
    if (nb > 32) {
      put_bits(acc, n, w, wi, (unsigned)(bits >> 32), nb - 32);
      nb = 32;
    }
    put_bits(acc, n, w, wi, (unsigned)bits, nb);
  });
  if (n) atomicOr(w + wi, (unsigned)(acc << (32 - n)));
}

__device__ __forceinline__ unsigned long long stream_bits(const Stream& st, const ProgScratch& S) {
  const long long last = st.slot0 + st.nslot - 1;
  return S.bitoff[last] + S.bits[last] - S.bitoff[st.slot0];
}

template <bool WRITE>
__global__ void __launch_bounds__(kThreads) jpeg_prog_stuff_kernel(const __grid_constant__ JpegList L,
                                                                  const __grid_constant__ ProgList P, ProgScratch S) {
  const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (g >= P.chunks) return;
  const Stream st = stream_of(L, P, g, true);
  const unsigned long long nbits = stream_bits(st, S);
  const long long nbytes = (long long)((nbits + 7) >> 3);
  const long long j0 = (g - st.chunk0) * kChunkBytes, j1 = min(j0 + kChunkBytes, nbytes);
  const unsigned* w = S.words + st.word0;
  if (!WRITE) {
    unsigned ff = 0;
    for (long long j = j0; j < j1; ++j) ff += stream_byte(w, j, nbits) == 0xFFu;
    S.ffcnt[g] = ff;
    return;
  }
  unsigned char* o = P.im[st.i].out + S.data_at[stream_key(st)] + j0 + (S.ffoff[g] - S.ffoff[st.chunk0]);
  for (long long j = j0; j < j1; ++j) {
    const unsigned v = stream_byte(w, j, nbits);
    *o++ = (unsigned char)v;
    if (v == 0xFFu) *o++ = 0;
  }
}

// the DHT segments of scan s (its tables that code something) and its SOS: byte j, and the length with j < 0
__device__ int scan_header_byte(const JpegTables& T, int s, int j) {
  const ScanDef d = scan_def(s);
  const int ntab = d.comp < 0 ? (d.ah ? 0 : 2) : 1, t0 = d.comp > 0 ? 1 : 0;
  int at = 0;
  for (int k = 0; k < ntab; ++k) {
    const int t = t0 + k, len = 2 + 2 + 1 + 16 + T.nsym[t];
    if (j >= at && j < at + len) {
      const int r = j - at, n = len - 2;
      return r == 0 ? 0xFF : r == 1 ? 0xC4 : r == 2 ? n >> 8 : r == 3 ? n & 0xFF : r == 4 ? (d.comp < 0 ? 0x00 : 0x10) | t
           : r < 21 ? T.counts[t][r - 5] : T.syms[t][r - 21];
    }
    at += len;
  }
  const int nc = d.comp < 0 ? 3 : 1, len = 2 + 2 + 1 + 2 * nc + 3;
  if (j < 0) return at + len;
  const int r = j - at;
  if (r < 5) return r == 0 ? 0xFF : r == 1 ? 0xDA : r == 2 ? 0 : r == 3 ? len - 2 : nc;
  if (r < 5 + 2 * nc) {
    const int c = d.comp < 0 ? (r - 5) >> 1 : d.comp;
    if (!((r - 5) & 1)) return c + 1;
    return d.comp < 0 ? (d.ah || c == 0 ? 0x00 : 0x10) : t0;   // DC: the DC table in the high nibble; AC: the AC table
  }
  const int u = r - 5 - 2 * nc;
  return u == 0 ? d.ss : u == 1 ? d.se : d.ah << 4 | d.al;
}

// one CTA per image: the header before the first scan, each scan's tables and SOS, and EOI, at offsets from the stuffed
// scan lengths; stores where each scan's data goes and the file's length
__global__ void __launch_bounds__(kThreads) jpeg_prog_header_kernel(const __grid_constant__ HeaderList H,
                                                                   const __grid_constant__ ProgList P, ProgScratch S) {
  __shared__ long long hdr_at[JPEG_SCANS + 1];
  const int i = blockIdx.x;
  if (threadIdx.x == 0) {
    long long at = H.sof_end + H.meta, slot = P.im[i].slot0, chunk = P.im[i].chunk0;
    for (int s = 0; s < JPEG_SCANS; ++s) {
      Stream st;
      st.slot0 = slot;
      st.nslot = scan_slots(H.hw[i][0], H.hw[i][1], P.sub, s);
      st.chunk0 = chunk;
      st.nchunk = scan_chunks(scan_words(st.nslot, s));
      const long long lc = st.chunk0 + st.nchunk - 1;
      const long long ff = S.ffoff[lc] + S.ffcnt[lc] - S.ffoff[st.chunk0];
      hdr_at[s] = at;
      at += scan_header_byte(S.tabs[i * JPEG_SCANS + s], s, -1);
      S.data_at[i * JPEG_SCANS + s] = at;
      at += (long long)((stream_bits(st, S) + 7) >> 3) + ff;
      slot += st.nslot;
      chunk += st.nchunk;
    }
    hdr_at[JPEG_SCANS] = at;
    unsigned char* o = P.im[i].out;
    o[at] = 0xFF;
    o[at + 1] = 0xD9;
    *P.im[i].out_bytes = at + 2;
  }
  __syncthreads();
  unsigned char* o = P.im[i].out;
  for (int j = threadIdx.x; j < H.sof_end; j += kThreads)   // SOF0's marker byte becomes SOF2's
    o[header_at(H, j)] = j == H.sof_end - 18 ? 0xC2 : header_byte(H, i, j);
  for (int s = 0; s < JPEG_SCANS; ++s) {
    const JpegTables& T = S.tabs[i * JPEG_SCANS + s];
    const int len = (int)(S.data_at[i * JPEG_SCANS + s] - hdr_at[s]);
    for (int j = threadIdx.x; j < len; j += kThreads) o[hdr_at[s] + j] = (unsigned char)scan_header_byte(T, s, j);
  }
}

}  // namespace

long long jpeg_prog_max_bytes(int h, int w, int subsampling, int sof_end) {
  // the header through SOF2 (sof_end bytes); scan 1's two DC tables (<= 12 symbols each) and SOS; scan 7's SOS; eight AC scans' table
  // (<= 176 symbols: 160 run/size, ZRL and 15 EOB runs) and SOS; EOI
  const long long headers = sof_end + 2 * (21 + 12) + 14 + 14 + 8 * (21 + 176 + 10) + 2;
  long long bits = 0;
  for (int s = 0; s < JPEG_SCANS; ++s) bits += ((scan_slots(h, w, subsampling, s) * slot_max_bits(s) + 7) / 8) * 8;
  return headers + 2 * (bits / 8);   // each scan's bits padded to a byte, every byte possibly followed by 0x00
}

size_t jpeg_prog_layout(const JpegList& L, unsigned char* base, ProgList* P, ProgScratch* S) {
  long long slots = 0, words = 0, chunks = 0;
  for (int i = 0; i < L.n; ++i) {
    PImg& p = P->im[i];
    p.slot0 = slots;
    p.word0 = words;
    p.chunk0 = chunks;
    p.out = L.im[i].out;
    p.out_bytes = L.im[i].out_bytes;
    for (int s = 0; s < JPEG_SCANS; ++s) {
      const long long n = scan_slots(L.im[i].h, L.im[i].w, L.sub, s), wd = scan_words(n, s);
      slots += n;
      words += wd;
      chunks += scan_chunks(wd);
    }
  }
  P->sub = L.sub;
  P->slots = slots;
  P->chunks = chunks;
  const long long tiles = (std::max(slots, chunks) + SCAN_TILE - 1) / SCAN_TILE;
  const size_t streams = (size_t)L.n * JPEG_SCANS;
  size_t at = 0;
  auto take = [&](auto*& ptr, size_t count) {
    ptr = base ? reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(base + at) : nullptr;
    at += scratch_round(count * sizeof(*ptr));
  };
  take(S->flags, slots);
  take(S->corr, slots);
  take(S->runs, slots);
  take(S->hist, streams * 2 * 256);
  take(S->words, words);
  take(S->bits, slots);
  take(S->bitoff, slots);
  take(S->ffcnt, chunks);
  take(S->ffoff, chunks);
  take(S->sums, std::max(tiles, 1LL));
  take(S->tabs, streams);
  take(S->data_at, streams);
  return at;
}

int jpeg_progressive(const JpegList& L, const HeaderList& H, const ProgList& P, const ProgScratch& S, cudaStream_t st) {
  // the run records, histograms and word streams lie together and start zeroed
  SE_CUDA_OK(cudaMemsetAsync(S.runs, 0, (unsigned char*)S.bits - (unsigned char*)S.runs, st));
  const unsigned gs = grid_of(P.slots, kThreads), gc = grid_of(P.chunks, kThreads);
  jpeg_prog_prep_kernel<<<gs, kThreads, 0, st>>>(L, P, S);
  jpeg_prog_runs_kernel<<<gs, kThreads, 0, st>>>(L, P, S);
  jpeg_prog_hist_kernel<<<gs, kThreads, 0, st>>>(L, P, S);
  SE_CUDA_OK(cudaGetLastError());
  int rc = jpeg_build_tables(S.hist, S.tabs, L.n * JPEG_SCANS, 2, st);
  if (rc) return rc;
  jpeg_prog_bits_kernel<<<gs, kThreads, 0, st>>>(L, P, S);
  SE_CUDA_OK(cudaGetLastError());
  if ((rc = exclusive_scan(S.bits, S.bitoff, S.sums, P.slots, st))) return rc;
  jpeg_prog_pack_kernel<<<gs, kThreads, 0, st>>>(L, P, S);
  jpeg_prog_stuff_kernel<false><<<gc, kThreads, 0, st>>>(L, P, S);
  SE_CUDA_OK(cudaGetLastError());
  if ((rc = exclusive_scan(S.ffcnt, S.ffoff, S.sums, P.chunks, st))) return rc;
  jpeg_prog_header_kernel<<<L.n, kThreads, 0, st>>>(H, P, S);
  jpeg_prog_stuff_kernel<true><<<gc, kThreads, 0, st>>>(L, P, S);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace se

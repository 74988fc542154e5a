// The stages of a split inflate: one zlib stream decoded by many groups of lanes at once (se_png_split.cu on the device,
// one group per chunk; tests/test_png_split.py builds them for the host with one lane and runs them in order).
//
// The deflate payload is cut at nominal compressed offsets k S. Chunk 0 starts after the zlib header; chunk k > 0 starts at
// the first bit in [8 k S, 8 (k + 1) S) where a dynamic-Huffman block header with BFINAL = 0 passes every check zlib
// applies (find_block; the block finder of rapidgzip, Knespel and Brunst 2023), or is empty when there is none.
//   count: each non-empty chunk decodes whole blocks from its start until the first block boundary at or after the next
//          non-empty chunk's start, or through the final block, keeping only its end bit and its byte count;
//   link:  the stream is decoded here only if every chunk ends exactly where the next starts, the last ends with the final
//          block and the counts sum to raw_n. Chunk 0 starts at a real block, so by induction every accepted start is one:
//          a false start from the finder can only refuse the stream, never change its bytes;
//   emit:  each chunk decodes again into 4-byte entries at its output offset: kLiteral | byte, or the absolute position of
//          the byte a match reads from before the chunk's start (a match inside the chunk copies entries, such markers
//          included), so no chunk needs the bytes of another;
//   resolve: each byte follows its markers back to a literal. A marker is always below the position that holds it, so
//          the chain ends.
// Everything the one-warp inflate_zlib checks is checked here too (a distance before the stream's start in emit, where
// positions are known), so whatever is accepted, zlib accepts with the same bytes.
#pragma once

#include "se_inflate.cuh"

namespace se {

constexpr unsigned kLiteral = 0x80000000u;   // an emit entry with this bit is a literal byte; without it, a position

struct SplitChunk {
  long long start;   // bit of its first block, or -1: empty
  long long next;    // start of the next non-empty chunk, or -1: none
  long long end;     // bit after its last block
  long long count;   // bytes it decodes to
  long long off;     // where they go in the output (link)
  int final;         // its last block is the stream's final block
  int status;
};

// Whether a dynamic-Huffman block header with BFINAL = 0 that zlib 1.3 accepts starts at bit b of src[0, n): HLIT and HDIST
// in range, a complete code-length code, repeats inside the lengths (a 16 with a length before it), a nonzero end-of-block
// length, and literal/length and distance codes neither over-subscribed nor incomplete, except a single code of 1 bit.
// The checks of inflate_header and huff_build, on code counts alone.
SE_HD inline bool dynamic_header_at(const unsigned char* src, long long n, long long b) {
  BitIn in{src, 0, n, 0ull, 0};
  if (!in.seek(b) || !in.need(17) || in.take(3) != 4) return false;   // BFINAL 0, then BTYPE 2, LSB first
  const int nlit = (int)in.take(5) + 257;
  const int ndist = (int)in.take(5) + 1;
  const int ncode = (int)in.take(4) + 4;
  if (nlit > 286 || ndist > 30) return false;
  const unsigned char order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  unsigned char cl[19] = {0};
  for (int k = 0; k < ncode; ++k) {
    if (!in.need(3)) return false;
    cl[order[k]] = (unsigned char)in.take(3);
  }
  unsigned char count[8] = {0}, sym[19];
  for (int s = 0; s < 19; ++s) count[cl[s]]++;
  int left = 1;
  for (int l = 1; l <= 7; ++l) {
    left = 2 * left - count[l];
    if (left < 0) return false;
  }
  if (left > 0) return false;   // incomplete, or no code at all
  unsigned char offs[8];
  offs[1] = 0;
  for (int l = 1; l < 7; ++l) offs[l + 1] = (unsigned char)(offs[l] + count[l]);
  for (int s = 0; s < 19; ++s)
    if (cl[s]) sym[offs[cl[s]]++] = (unsigned char)s;
  unsigned short litc[16] = {0}, distc[16] = {0};
  int k = 0, prev = 0, litk = 0, distk = 0;   // Kraft sums of the lengths so far, in units of 2^-15
  bool eob = false;
  while (k < nlit + ndist) {
    if (in.cnt < 7) in.refill();
    int s = -1, code = 0, first = 0, index = 0;
    for (int l = 1; l <= 7 && l <= in.cnt; ++l) {   // the canonical decode of huff_slow
      code |= (int)(in.buf >> (l - 1)) & 1;
      if (code - first < count[l]) {
        s = sym[index + code - first];
        in.take(l);
        break;
      }
      index += count[l];
      first = (first + count[l]) << 1;
      code <<= 1;
    }
    if (s < 0) return false;
    int rep = 1, v = s;
    if (s == 16) {
      if (k == 0 || !in.need(2)) return false;
      v = prev;
      rep = 3 + (int)in.take(2);
    } else if (s == 17) {
      if (!in.need(3)) return false;
      v = 0;
      rep = 3 + (int)in.take(3);
    } else if (s == 18) {
      if (!in.need(7)) return false;
      v = 0;
      rep = 11 + (int)in.take(7);
    }
    if (k + rep > nlit + ndist) return false;
    for (; rep > 0; --rep, ++k) {
      if (k < nlit) litc[v]++, litk += v ? 1 << (15 - v) : 0;
      else distc[v]++, distk += v ? 1 << (15 - v) : 0;
      if (k == 256) eob = v != 0;
    }
    if (litk > 1 << 15 || distk > 1 << 15) return false;   // over-subscribed already: most false candidates end here
    prev = v;
  }
  if (!eob) return false;
  for (int c = 0; c < 2; ++c) {
    const unsigned short* cnt = c ? distc : litc;
    int lft = 1, maxlen = 0;
    for (int l = 1; l <= 15; ++l) {
      lft = 2 * lft - cnt[l];
      if (lft < 0) return false;
      if (cnt[l]) maxlen = l;
    }
    if (maxlen > 0 && lft > 0 && maxlen != 1) return false;
  }
  return true;
}

// The first bit in [lo, hi) where dynamic_header_at holds, or -1. On the device the 32 lanes of a warp test 32 bits at once.
SE_HD inline long long find_block(const unsigned char* src, long long n, long long lo, long long hi, int lane, int nl) {
  for (long long b0 = lo; b0 < hi; b0 += nl) {
    const bool ok = b0 + lane < hi && dynamic_header_at(src, n, b0 + lane);
#ifdef __CUDA_ARCH__
    const unsigned any = __ballot_sync(0xFFFFFFFFu, ok);
    if (any) return b0 + __ffs(any) - 1;
#else
    if (ok) return b0 + lane;
#endif
  }
  return -1;
}

// The bits chunk k >= 1 of a stream of n bytes searches: [8 k S, 8 (k + 1) S), after chunk 0's start (bit 16, past the
// zlib header) and before the stream's end.
SE_HD inline void chunk_bits(long long k, long long S, long long n, long long* lo, long long* hi) {
  *lo = 8 * k * S < 17 ? 17 : 8 * k * S;
  *hi = 8 * (k + 1) * S < 8 * n ? 8 * (k + 1) * S : 8 * n;
}

// count's output: bytes only, at most cap of them.
struct CountOut {
  long long out, cap;
  SE_HD int stored(const unsigned char*, unsigned len) { return (out += len) > cap ? INF_LONG_OUTPUT : INF_OK; }
  SE_HD int lit(int) { return ++out > cap ? INF_LONG_OUTPUT : INF_OK; }
  SE_HD int match(long long len, long long) { return (out += len) > cap ? INF_LONG_OUTPUT : INF_OK; }
};

// emit's output: entries e[base, end) of the stream's raw_n, out the next one written; lane 0 writes the literals, all lanes
// the copies. A match byte whose source lies in the chunk copies the source's entry; one before the chunk gets its position.
struct EntryOut {
  unsigned* e;
  long long base, out, end;
  int lane, nl;
  SE_HD int stored(const unsigned char* data, unsigned len) {
    if (out + len > end) return INF_LONG_OUTPUT;
    SE_LANE_SYNC();
    for (unsigned k = lane; k < len; k += nl) e[out + k] = kLiteral | data[k];
    SE_LANE_SYNC();
    out += len;
    return INF_OK;
  }
  SE_HD int lit(int s) {
    if (out >= end) return INF_LONG_OUTPUT;
    if (lane == 0) e[out] = kLiteral | (unsigned)s;
    ++out;
    return INF_OK;
  }
  SE_HD int match(long long len, long long d) {
    if (d > out) return INF_DISTANCE;
    if (out + len > end) return INF_LONG_OUTPUT;
    SE_LANE_SYNC();   // the entries written before are visible to every lane
    for (long long k = lane; k < len; k += nl) {
      const long long s = out - d + (k < d ? k : k % d);   // below out, as in ByteOut::match
      e[out + k] = s >= base ? e[s] : (unsigned)s;
    }
    SE_LANE_SYNC();
    out += len;
    return INF_OK;
  }
};

// Decodes whole blocks of src[0, n) from c.start into `out` until the first block boundary at or after c.next (c.next < 0:
// through the final block). *end is the bit after the last block, *final whether it was the final one.
template <class Out>
SE_HD inline int chunk_blocks(const unsigned char* src, long long n, const SplitChunk& c, InflateTabs& t, Out& out,
                              long long* end, int* final, int lane, int nl) {
  BitIn in{src, 0, n, 0ull, 0};
  if (!in.seek(c.start)) return INF_SHORT_INPUT;
  unsigned last = 0;
  do {
    if (int st = inflate_block(in, t, out, &last, lane, nl)) return st;
  } while (!last && (c.next < 0 || in.bit() < c.next));
  *end = in.bit();
  *final = (int)last;
  return INF_OK;
}

// count for chunk c (first: chunk 0, which also checks the zlib header) of a stream of raw_n bytes: sets c.count, c.end and
// c.final (lane 0) and returns the status.
SE_HD inline int chunk_count(const unsigned char* src, long long n, long long raw_n, SplitChunk& c, bool first, InflateTabs& t,
                             int lane, int nl) {
  if (first && (n < 2 || zlib_header(src[0], src[1]))) return n < 2 ? INF_SHORT_INPUT : INF_HEADER;
  CountOut out{0, raw_n};
  long long end = 0;
  int final = 0;
  const int st = chunk_blocks(src, n, c, t, out, &end, &final, lane, nl);
  if (lane == 0 && st == INF_OK) {
    c.count = out.out;
    c.end = end;
    c.final = final;
  }
  return st;
}

// link over the nc chunks of one stream of raw_n bytes (after count): sets each non-empty chunk's off and *tail, the bit
// after the final block. Returns INF_OK, a chunk's status, or why the chunks do not join.
SE_HD inline int chunks_link(SplitChunk* c, long long nc, long long raw_n, long long* tail) {
  long long off = 0;
  for (long long k = 0; k < nc; ++k) {
    if (c[k].start < 0) continue;
    if (c[k].status) return c[k].status;
    if (c[k].next >= 0 ? (c[k].final || c[k].end != c[k].next) : !c[k].final) return INF_LINK;
    c[k].off = off;
    off += c[k].count;
    if (off > raw_n) return INF_LONG_OUTPUT;
    *tail = c[k].end;
  }
  return off == raw_n ? INF_OK : INF_SHORT_OUTPUT;
}

// emit for a linked chunk c into the stream's entries e.
SE_HD inline int chunk_emit(const unsigned char* src, long long n, const SplitChunk& c, unsigned* e, InflateTabs& t, int lane,
                            int nl) {
  EntryOut out{e, c.off, c.off, c.off + c.count, lane, nl};
  long long end = 0;
  int final = 0;
  const int st = chunk_blocks(src, n, c, t, out, &end, &final, lane, nl);
  return st ? st : out.out == c.off + c.count && end == c.end ? INF_OK : INF_LINK;
}

// The byte at position i of the emitted entries e, or -1 if a marker does not point below its position (never, by
// construction: the check bounds the walk).
SE_HD inline int resolve_byte(const unsigned* e, long long i) {
  unsigned v = e[i];
  while (!(v & kLiteral)) {
    if ((long long)v >= i) return -1;
    i = v;
    v = e[i];
  }
  return (int)(v & 0xFF);
}

// The Adler-32 the stream stores after the byte-aligned bit `tail`, or -1 when the stream ends before it.
SE_HD inline long long stored_adler(const unsigned char* src, long long n, long long tail) {
  const long long at = (tail + 7) >> 3;
  if (at + 4 > n) return -1;
  return (long long)((unsigned)src[at] << 24 | (unsigned)src[at + 1] << 16 | (unsigned)src[at + 2] << 8 | src[at + 3]);
}

}  // namespace se

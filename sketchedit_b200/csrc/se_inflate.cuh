// zlib stream inflation (RFC 1950 / 1951) for the PNG decoder, written once for the device (one warp per stream) and for a
// host build with one lane (tests/test_png_decode.py compiles it with the host compiler and runs malformed streams through
// it). Every lane of a warp runs the same symbol loop on its own copy of the bit buffer, so control flow stays uniform; the
// lanes split only the table fills, the stored-block copies, the match copies and the Adler-32 sum.
//
// The decoder is at least as strict as zlib 1.3's inflate: whatever it accepts, zlib accepts with the same bytes. Anything
// else (a bad header or FDICT, block type 3, LEN != ~NLEN, HLIT > 286 or HDIST > 30, a repeat with nothing before it or past
// the lengths, no end-of-block code, an over-subscribed table or an incomplete one zlib refuses, codes 286-287 or 30-31, a
// distance reaching before the start, too few or too many bytes, a wrong Adler-32) ends with a nonzero status. Every read is
// checked against the stream length, every write against `raw_n`, every table index against its table.
#pragma once

#ifdef __CUDACC__
#define SE_HD __host__ __device__
#else
#define SE_HD
#endif
#ifdef __CUDA_ARCH__
#define SE_LANE_SYNC() __syncwarp()
#else
#define SE_LANE_SYNC() ((void)0)
#endif

namespace se {

enum InflateStatus : int {
  INF_OK = 0,
  INF_HEADER = 1,       // bad zlib header: method, window size, check bits, or FDICT set
  INF_BLOCK = 2,        // block type 3 or a stored block's LEN != ~NLEN
  INF_TABLE = 3,        // bad code lengths: counts, repeats, over-subscribed or refused incomplete tables, no end-of-block
  INF_CODE = 4,         // a code absent from its table, or literal/length 286-287, or distance 30-31
  INF_DISTANCE = 5,     // a distance reaching before the start of the output
  INF_SHORT_INPUT = 6,  // the stream ends before its last block or its Adler-32
  INF_SHORT_OUTPUT = 7, // the last block ends before raw_n bytes
  INF_LONG_OUTPUT = 8,  // the stream holds more than raw_n bytes
  INF_ADLER = 9,        // the Adler-32 differs from the output's
  // set by the PNG stages after inflation
  PNG_FILTER = 10,      // a row's filter type is not 0-4
  PNG_PALETTE = 11,     // a palette index at or past the palette's entries
  // set by the split inflate (se_inflate_split.cuh)
  INF_LINK = 12,        // a chunk ends elsewhere than where the next one starts, or the last one before the final block
};

constexpr int kTabBits = 10;   // first-level lookup: codes of at most 10 bits resolve in one shared-memory read

// A canonical Huffman code: count[len] codes of each length, its symbols sorted by (length, value), and a 2^10 lookup of the
// next 10 stream bits (LSB first) -> symbol | length << 10, or 0 when the code is longer (or absent).
struct Huff {
  unsigned short count[16];
  unsigned short symbol[288];
  unsigned short tab[1 << kTabBits];
};

struct InflateTabs {
  Huff lit, dist;
  unsigned char lens[288 + 32];   // code lengths of the block: literal/length, then distance
};

// The bit-serial canonical decode (RFC 1951 3.2.2) of the first 15 bits of `bits`: the symbol, its length in *len; -1 if no
// code of at most `maxlen` bits matches.
SE_HD inline int huff_slow(const Huff& h, unsigned bits, int maxlen, int* len) {
  int code = 0, first = 0, index = 0;
  for (int l = 1; l <= maxlen; ++l) {
    code |= (bits >> (l - 1)) & 1;
    const int count = h.count[l];
    if (code - first < count) {
      *len = l;
      return h.symbol[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// Builds h from n code lengths (lengths[s] in [0, 15]). `kind`: 0 code-length code, 1 literal/length, 2 distance. Returns
// INF_OK or INF_TABLE, the latter where zlib's inflate_table refuses: over-subscribed, or incomplete unless it is a
// literal/length or distance code whose longest code has 1 bit. All lanes must call it; it ends with the lanes in step.
SE_HD inline int huff_build(Huff& h, const unsigned char* lengths, int n, int kind, int lane, int nl) {
  unsigned short count[16] = {0};
  for (int s = 0; s < n; ++s) count[lengths[s] & 15]++;
  int left = 1, maxlen = 0;
  for (int l = 1; l <= 15; ++l) {
    left <<= 1;
    left -= count[l];
    if (left < 0) return INF_TABLE;
    if (count[l]) maxlen = l;
  }
  if (maxlen > 0 && left > 0 && (kind == 0 || maxlen != 1)) return INF_TABLE;
  SE_LANE_SYNC();   // no lane still decodes with the table this one replaces
  if (lane == 0) {
    unsigned short offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = (unsigned short)(offs[l] + count[l]);
    for (int l = 0; l < 16; ++l) h.count[l] = count[l];
    h.count[0] = 0;
    for (int s = 0; s < n; ++s)
      if (lengths[s]) h.symbol[offs[lengths[s]]++] = (unsigned short)s;
  }
  SE_LANE_SYNC();
  for (int e = lane; e < (1 << kTabBits); e += nl) {
    int len = 0;
    const int s = huff_slow(h, (unsigned)e, kTabBits, &len);
    h.tab[e] = (unsigned short)(s < 0 ? 0 : (s | len << kTabBits));
  }
  SE_LANE_SYNC();
  return INF_OK;
}

// The stream's bits, LSB first, in a 64-bit buffer refilled 8 bytes at a time; reads stop at the stream's end.
struct BitIn {
  const unsigned char* p;
  long long pos, n;
  unsigned long long buf;
  int cnt;
  SE_HD void refill() {
    if (cnt <= 56 && pos + 8 <= n) {   // 8 independent loads; the bytes past the whole ones taken are the stream's next bits
      unsigned long long v = 0;
      for (int i = 0; i < 8; ++i) v |= (unsigned long long)p[pos + i] << (8 * i);
      const int k = (63 - cnt) >> 3;
      buf |= v << cnt;
      pos += k;
      cnt += 8 * k;
      return;
    }
    while (cnt <= 56 && pos < n) {
      buf |= (unsigned long long)p[pos++] << cnt;
      cnt += 8;
    }
  }
  // false when fewer than k bits remain in the stream
  SE_HD bool need(int k) {
    if (cnt < k) refill();
    return cnt >= k;
  }
  SE_HD unsigned take(int k) {   // k <= cnt
    const unsigned v = (unsigned)(buf & ((1ull << k) - 1));
    buf >>= k;
    cnt -= k;
    return v;
  }
  SE_HD long long bit() const { return pos * 8 - cnt; }   // the offset of the next bit in the stream
  // moves to bit b of the stream (b >= 0); false when b is past its end
  SE_HD bool seek(long long b) {
    pos = b >> 3;
    buf = 0;
    cnt = 0;
    if (pos > n || !need((int)(b & 7))) return false;
    take((int)(b & 7));
    return true;
  }
};

// One symbol of h; -INF_CODE or -INF_SHORT_INPUT on failure.
SE_HD inline int huff_decode(const Huff& h, BitIn& in) {
  if (in.cnt < 15) in.refill();   // a refill leaves 56 bits or more: one per several symbols
  const unsigned bits = (unsigned)(in.buf & 0x7FFF);
  int len;
  int s;
  const unsigned e = h.tab[bits & ((1u << kTabBits) - 1)];
  if (e) {
    s = (int)(e & ((1u << kTabBits) - 1));
    len = (int)(e >> kTabBits);
  } else {
    s = huff_slow(h, bits, 15, &len);
    if (s < 0) return in.cnt >= 15 ? -INF_CODE : -INF_SHORT_INPUT;
  }
  if (len > in.cnt) return -INF_SHORT_INPUT;
  in.take(len);
  return s;
}

// RFC 1951 3.2.5: base and extra bits of length code lc (0-28) and distance code dc (0-29)
SE_HD inline int len_extra(int lc) { return lc < 8 || lc == 28 ? 0 : (lc - 4) >> 2; }
SE_HD inline int len_base(int lc) { return lc < 8 ? 3 + lc : lc == 28 ? 258 : ((4 + ((lc - 4) & 3)) << len_extra(lc)) + 3; }
SE_HD inline int dist_extra(int dc) { return dc < 4 ? 0 : (dc >> 1) - 1; }
SE_HD inline int dist_base(int dc) { return dc < 4 ? dc + 1 : ((2 | (dc & 1)) << dist_extra(dc)) + 1; }

// Adler-32 of raw[0, n), lanes splitting the bytes; every lane returns the sum.
SE_HD inline unsigned adler32_lanes(const unsigned char* raw, long long n, int lane, int nl) {
  const unsigned long long M = 65521;
  unsigned long long a = 0, b = 0;
  int k = 0;
  for (long long i = lane; i < n; i += nl) {
    const unsigned d = raw[i];
    a += d;
    b += (unsigned long long)(n - i) * d;   // byte i is counted in n - i of the running sums
    if (++k == 4096) {
      a %= M;
      b %= M;
      k = 0;
    }
  }
  a %= M;
  b %= M;
#ifdef __CUDA_ARCH__
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xFFFFFFFFu, a, o);
    b += __shfl_xor_sync(0xFFFFFFFFu, b, o);
  }
#endif
  a = (a + 1) % M;
  b = (b + (unsigned long long)(n % (long long)M)) % M;
  return (unsigned)(b << 16 | a);
}

// Reads one block's header at in's position into *last and *type. A stored block leaves in byte-aligned at its LEN bytes of
// data, LEN in *stored; a Huffman block leaves its tables in t. All lanes call it and get the same result.
SE_HD inline int inflate_header(BitIn& in, InflateTabs& t, unsigned* last, unsigned* type, unsigned* stored, int lane, int nl) {
  if (!in.need(3)) return INF_SHORT_INPUT;
  *last = in.take(1);
  *type = in.take(2);
  if (*type == 0) {
    in.take(in.cnt & 7);
    if (!in.need(32)) return INF_SHORT_INPUT;
    const unsigned len = in.take(16), nlen = in.take(16);
    if (len != (~nlen & 0xFFFF)) return INF_BLOCK;
    *stored = len;
    return INF_OK;
  }
  if (*type == 3) return INF_BLOCK;
  if (*type == 1) {
    SE_LANE_SYNC();   // no lane still reads the previous block's lengths
    for (int s = lane; s < 288 + 32; s += nl) t.lens[s] = (unsigned char)(s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5);
    SE_LANE_SYNC();
    if (huff_build(t.lit, t.lens, 288, 1, lane, nl) || huff_build(t.dist, t.lens + 288, 32, 2, lane, nl)) return INF_TABLE;
    return INF_OK;
  }
  if (!in.need(14)) return INF_SHORT_INPUT;
  const int nlit = (int)in.take(5) + 257;
  const int ndist = (int)in.take(5) + 1;
  const int ncode = (int)in.take(4) + 4;
  if (nlit > 286 || ndist > 30) return INF_TABLE;
  const unsigned char order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  unsigned char cl[19] = {0};
  for (int k = 0; k < ncode; ++k) {
    if (!in.need(3)) return INF_SHORT_INPUT;
    cl[order[k]] = (unsigned char)in.take(3);
  }
  if (huff_build(t.lit, cl, 19, 0, lane, nl)) return INF_TABLE;
  int k = 0;
  while (k < nlit + ndist) {
    const int s = huff_decode(t.lit, in);
    if (s < 0) return -s;
    if (s < 16) {
      t.lens[k++] = (unsigned char)s;
      continue;
    }
    int rep, v = 0;
    if (s == 16) {
      if (k == 0) return INF_TABLE;
      if (!in.need(2)) return INF_SHORT_INPUT;
      v = t.lens[k - 1];
      rep = 3 + (int)in.take(2);
    } else if (s == 17) {
      if (!in.need(3)) return INF_SHORT_INPUT;
      rep = 3 + (int)in.take(3);
    } else {
      if (!in.need(7)) return INF_SHORT_INPUT;
      rep = 11 + (int)in.take(7);
    }
    if (k + rep > nlit + ndist) return INF_TABLE;
    while (rep--) t.lens[k++] = (unsigned char)v;
  }
  if (t.lens[256] == 0) return INF_TABLE;
  if (huff_build(t.lit, t.lens, nlit, 1, lane, nl) || huff_build(t.dist, t.lens + nlit, ndist, 2, lane, nl)) return INF_TABLE;
  return INF_OK;
}

// One block at in's position, its bytes handed to `out`: out.stored(data, len) for a stored block, out.lit(byte) and
// out.match(len, dist) for a Huffman block's symbols; each returns INF_OK or the status that ends the decode. *last is the
// block's BFINAL. All lanes call it and get the same result.
template <class Out>
SE_HD inline int inflate_block(BitIn& in, InflateTabs& t, Out& out, unsigned* last, int lane, int nl) {
  unsigned type = 0, stored = 0;
  if (int st = inflate_header(in, t, last, &type, &stored, lane, nl)) return st;
  if (type == 0) {
    const long long at = in.pos - in.cnt / 8;   // the bit buffer holds whole bytes now: rewind it into the stream
    if (at + stored > in.n) return INF_SHORT_INPUT;
    if (int st = out.stored(in.p + at, stored)) return st;
    in.pos = at + stored;
    in.buf = 0;
    in.cnt = 0;
    return INF_OK;
  }
  for (;;) {
    const int s = huff_decode(t.lit, in);
    if (s < 0) return -s;
    if (s < 256) {
      if (int st = out.lit(s)) return st;
      continue;
    }
    if (s == 256) return INF_OK;
    const int lc = s - 257;
    if (lc >= 29) return INF_CODE;
    const int lx = len_extra(lc);
    if (!in.need(lx)) return INF_SHORT_INPUT;
    const long long len = len_base(lc) + in.take(lx);
    const int dc = huff_decode(t.dist, in);
    if (dc < 0) return -dc;
    if (dc >= 30) return INF_CODE;
    const int dx = dist_extra(dc);
    if (!in.need(dx)) return INF_SHORT_INPUT;
    const long long d = dist_base(dc) + in.take(dx);
    if (int st = out.match(len, d)) return st;
  }
}

// inflate_block's output into raw[0, raw_n), out bytes written so far; lane 0 writes the literals, all lanes the copies.
struct ByteOut {
  unsigned char* raw;
  long long raw_n, out;
  int lane, nl;
  SE_HD int stored(const unsigned char* data, unsigned len) {
    if (out + len > raw_n) return INF_LONG_OUTPUT;
    SE_LANE_SYNC();
    for (unsigned k = lane; k < len; k += nl) raw[out + k] = data[k];
    SE_LANE_SYNC();
    out += len;
    return INF_OK;
  }
  SE_HD int lit(int s) {
    if (out >= raw_n) return INF_LONG_OUTPUT;
    if (lane == 0) raw[out] = (unsigned char)s;
    ++out;
    return INF_OK;
  }
  SE_HD int match(long long len, long long d) {
    if (d > out) return INF_DISTANCE;
    if (out + len > raw_n) return INF_LONG_OUTPUT;
    SE_LANE_SYNC();   // the literals lane 0 just wrote are visible to every lane
    // byte k of the match is byte k mod d of the d bytes before it: no lane reads a byte this copy writes
    for (long long k = lane; k < len; k += nl) raw[out + k] = raw[out - d + (k < d ? k : k % d)];
    SE_LANE_SYNC();
    out += len;
    return INF_OK;
  }
};

// The zlib header's check (RFC 1950): 0 when CMF, FLG name deflate with a window of at most 32 KB, no preset dictionary.
SE_HD inline int zlib_header(unsigned cmf, unsigned flg) {
  return (cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 0x20) ? INF_HEADER : INF_OK;
}

// Inflates the zlib stream src[0, n) into raw[0, raw_n). Returns INF_OK only when the stream is a complete zlib stream
// whose last block ends at exactly raw_n bytes and whose Adler-32 matches; bytes after the Adler-32 are ignored.
// `t` is scratch for the tables (shared memory on the device); all lanes of the group call it and get the same result.
SE_HD inline int inflate_zlib(const unsigned char* src, long long n, unsigned char* raw, long long raw_n, InflateTabs& t,
                              int lane, int nl) {
  BitIn in{src, 0, n, 0ull, 0};
  if (!in.need(16)) return INF_SHORT_INPUT;
  const unsigned cmf = in.take(8), flg = in.take(8);
  if (zlib_header(cmf, flg)) return INF_HEADER;
  ByteOut out{raw, raw_n, 0, lane, nl};
  for (unsigned last = 0; !last;)
    if (int st = inflate_block(in, t, out, &last, lane, nl)) return st;
  SE_LANE_SYNC();
  if (out.out != raw_n) return INF_SHORT_OUTPUT;
  in.take(in.cnt & 7);
  if (!in.need(32)) return INF_SHORT_INPUT;
  unsigned want = 0;
  for (int k = 0; k < 4; ++k) want = want << 8 | in.take(8);
  return adler32_lanes(raw, raw_n, lane, nl) == want ? INF_OK : INF_ADLER;
}

}  // namespace se

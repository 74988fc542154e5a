// Baseline JPEG encoding of uint8 RGB windows on the GPU (se_jpeg.cu), byte for byte what PIL.Image.save(buf, "JPEG",
// quality=q, subsampling=s[, optimize=True]) writes with libjpeg-turbo for s = 0 (4:4:4) and s = 2 (4:2:0), and what
// save(buf, "JPEG", qtables=T, subsampling=s, exif=E, icc_profile=I) writes for 1 to 4 8-bit tables T and s = 0, 1 (4:2:2)
// or 2 (se_jpeg_encode_tables_u8). The optimal Huffman tables of optimize=True are built by the kernels of se_jpeg_opt.cu.
#pragma once
#include "se_common.cuh"

namespace se {

constexpr int JPEG_MAX_BATCH = 32;          // images per call: their descriptors travel as kernel parameters
constexpr int JPEG_HEADER_BYTES = 623;      // SOI, APP0, 2 DQT, SOF0, 4 DHT, SOS: the header of the quality entries
constexpr int JPEG_HEADER_MAX = 692;        // ... with 3 DQT, the most a call writes besides its APP1 / APP2 segments
constexpr int JPEG_MAX_BLOCK_BITS = 1664;   // 64 x (16-bit code + 10 value bits) >= DC (<= 16 + 11) + 63 AC (see DESIGN §7b)
constexpr int JPEG_APP0_END = 20;           // SOI and the JFIF APP0; a call's APP1 / APP2 segments follow
constexpr int JPEG_SOS_BYTES = 14;          // the SOS segment that ends the header
constexpr int JPEG_DHT_BYTES = 432;         // the four Annex K DHT segments

// header bytes of a call with nq DQT segments and meta bytes of APP1 / APP2 segments: through SOF0, and in all
__host__ __device__ constexpr int jpeg_sof_end(int nq, long long meta) { return (int)(JPEG_APP0_END + meta) + 69 * nq + 19; }
__host__ __device__ constexpr long long jpeg_header_bytes(int nq, long long meta) {
  return jpeg_sof_end(nq, meta) + JPEG_DHT_BYTES + JPEG_SOS_BYTES;
}
static_assert(jpeg_header_bytes(2, 0) == JPEG_HEADER_BYTES && jpeg_header_bytes(3, 0) == JPEG_HEADER_MAX, "header layout");

// MCU geometry of a subsampling 0 (4:4:4, 8x8: Y Cb Cr), 1 (4:2:2, 16x8: Y0 Y1 Cb Cr) or 2 (4:2:0, 16x16: Y0..Y3 Cb Cr)
__host__ __device__ __forceinline__ int mcu_blocks(int sub) { return sub == 2 ? 6 : sub == 1 ? 4 : 3; }
__host__ __device__ __forceinline__ int mcu_w(int sub) { return sub ? 16 : 8; }
__host__ __device__ __forceinline__ int mcu_h(int sub) { return sub == 2 ? 16 : 8; }
// block e's MCU, e / mcu_blocks(sub), as divisions by constants (a 64-bit division by a variable is a long subroutine)
__host__ __device__ __forceinline__ long long mcu_of(int sub, long long e) { return sub == 2 ? e / 6 : sub == 1 ? e / 4 : e / 3; }

// se_jpeg_max_bytes without the checks: the header (header_bytes of them), JPEG_MAX_BLOCK_BITS per block doubled for 0xFF
// stuffing, and EOI
long long jpeg_max_bytes(int h, int w, int subsampling, long long header_bytes = JPEG_HEADER_BYTES);

struct HuffCodes {   // symbol -> canonical code and its length (0: not in the table)
  unsigned short code[256];
  unsigned char size[256];
};

// One image's optimal tables, [0] DC luma, [1] DC chroma, [2] AC luma, [3] AC chroma: the codes, and the DHT contents (code
// counts per length 1..16, then the nsym symbols by code length).
struct JpegTables {
  HuffCodes codes[4];
  unsigned char counts[4][16];
  unsigned char syms[4][256];
  int nsym[4];
};

struct JImg {   // one image of a call; block, word and chunk indices are the call's (all images' arrays concatenated)
  const unsigned char* src;
  unsigned char* out;
  long long* out_bytes;
  long long pitch;
  long long blk0, word0, chunk0;   // its first block, word and stuffing chunk
  int h, w, mcu_x;                 // image size; MCUs per row
};
struct JpegList {
  JImg im[JPEG_MAX_BATCH];
  int n, sub;   // images; subsampling (0, 1 or 2)
  int hdr;      // header bytes of each file (baseline Annex K tables)
  long long blocks, chunks;
};

struct JpegScratch {   // the call's scratch arrays
  short* coef;                 // [64][blocks], zigzag order; [0] the quantised DC
  unsigned* bits;              // [blocks]: AC bits (dct), then all bits of the block (bits, or opt_bits with optimal tables)
  int* dcdiff;                 // [blocks]
  unsigned long long* bitoff;  // [blocks], exclusive scan of bits over the call
  unsigned* words;             // the bit streams, word0 of each image on
  unsigned* ffcnt;             // [chunks]
  unsigned long long* ffoff;   // [chunks], exclusive scan of ffcnt over the call
  unsigned long long* sums;    // scan tile sums
  // optimize only, else null: the Annex K Huffman tables and the header of L.hdr bytes are used
  unsigned long long* hist;    // [n][4][256] symbol counts per image and table
  JpegTables* tabs;            // [n] optimal tables
  int* hdr_len;                // [n] header bytes, where the entropy-coded data starts
};

// The call's header without its APP1 / APP2 segments, for a 1x1 image: SOI, APP0, the DQTs, SOF0, the DHTs, SOS. In a file
// the segments (meta bytes, copied there by the host entry) follow APP0, so byte j >= JPEG_APP0_END lies at j + meta.
struct HeaderList {
  unsigned char bytes[JPEG_HEADER_MAX];
  int len, sof_end, meta;   // bytes used; those through SOF0; the APP1 / APP2 bytes after APP0 in the file
  unsigned char* out[JPEG_MAX_BATCH];
  unsigned short hw[JPEG_MAX_BATCH][2];
};
static_assert(sizeof(HeaderList) <= 4096, "header descriptors must fit the kernel parameter space");

// header byte j of image i (j < H.sof_end, or of SOS) with its height and width in SOF0
__host__ __device__ __forceinline__ unsigned char header_byte(const HeaderList& H, int i, int j) {
  const int at = H.sof_end - 14;   // SOF0's height and width
  if (j >= at && j < at + 4) {
    const int x = H.hw[i][(j - at) >> 1];
    return (unsigned char)((j - at) & 1 ? x : x >> 8);
  }
  return H.bytes[j];
}
// where header byte j goes in the file
__host__ __device__ __forceinline__ long long header_at(const HeaderList& H, int j) { return j < JPEG_APP0_END ? j : j + H.meta; }

#ifdef __CUDACC__
// Block e of an image in scan order: its component (0 Y, 1 Cb, 2 Cr) and block column / row in that component's plane.
// A 4:2:0 MCU holds luma blocks (0,0), (0,1), (1,0), (1,1), then Cb and Cr; a 4:2:2 MCU luma blocks (0,0), (0,1), then Cb
// and Cr; a 4:4:4 MCU holds Y, Cb, Cr.
struct BlockAt {
  int comp, bx, by;
  bool dummy;   // a 4:2:0 or 4:2:2 luma block wholly outside the image
};
__device__ __forceinline__ BlockAt block_at(const JImg& d, int sub, long long e) {
  const int per = mcu_blocks(sub), nl = per - 2;
  const long long mcu = mcu_of(sub, e);
  const int k = (int)(e - mcu * per), mx = (int)(mcu % d.mcu_x), my = (int)(mcu / d.mcu_x);
  BlockAt b;
  if (sub && k < nl) {
    b.comp = 0;
    b.bx = 2 * mx + (k & 1);
    b.by = (sub == 2 ? 2 : 1) * my + (k >> 1);
    b.dummy = b.bx * 8 >= d.w || b.by * 8 >= d.h;
  } else {
    b.comp = k - nl + 1;
    b.bx = mx;
    b.by = my;
    b.dummy = false;
  }
  return b;
}

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// the quantised DC of block e's component that block e + 1 of that component codes its difference against: a dummy takes
// the DC of the block before it in the MCU (block 0 of an MCU is never a dummy)
__device__ __forceinline__ int dc_of(const JImg& d, int sub, const short* dc, long long e) {
  while (block_at(d, sub, e).dummy) --e;
  return dc[d.blk0 + e];
}

__device__ __forceinline__ long long prev_same_comp(int sub, long long e) {   // -1: the component's first block
  const int per = mcu_blocks(sub), nl = per - 2;
  const int k = (int)(e - mcu_of(sub, e) * per);
  if (k > 0 && k < nl) return e - 1;
  return e - (k == 0 ? per - nl + 1 : per);
}

// appends len <= 32 bits to a 64-bit accumulator holding n < 32 bits; full words go to w[*wi] by atomicOr
__device__ __forceinline__ void put_bits(unsigned long long& acc, int& n, unsigned* w, long long& wi, unsigned code, int len) {
  acc = (acc << len) | code;
  n += len;
  if (n >= 32) {
    n -= 32;
    atomicOr(w + wi++, (unsigned)(acc >> n));
  }
}

// byte j of a stream, the last one padded with 1-bits
__device__ __forceinline__ unsigned stream_byte(const unsigned* w, long long j, unsigned long long nbits) {
  unsigned v = (w[j >> 2] >> (24 - 8 * (j & 3))) & 0xFFu;
  if (j == (long long)((nbits - 1) >> 3) && (nbits & 7)) v |= 0xFFu >> (nbits & 7);
  return v;
}
#endif

// se_jpeg_opt.cu, each only enqueues on `st`. jpeg_optimize_tables: from the coefficients and DC differences in S, count
// each image's symbols into S.hist (zeroed by the caller) and build its optimal tables into S.tabs. jpeg_optimize_header:
// write each image's header with its tables and its length to S.hdr_len, and every block's bit count with those tables
// to S.bits.
int jpeg_optimize_tables(const JpegList& L, const JpegScratch& S, cudaStream_t st);
int jpeg_optimize_header(const JpegList& L, const HeaderList& H, const JpegScratch& S, cudaStream_t st);
// the optimal tables of `slots` histogram sets hist[slot][ntab][256] (ntab <= 4) into tabs[slot].codes[0 .. ntab)
int jpeg_build_tables(const unsigned long long* hist, JpegTables* tabs, int slots, int ntab, cudaStream_t st);

// ---- progressive (se_jpeg_prog.cu): the ten scans of jpeg_simple_progression, each coded with its own optimal tables.
// A slot is one block of one scan; an image's slots run scan by scan, and each (image, scan) has its own bit stream.
constexpr int JPEG_SCANS = 10;

struct PImg {   // one image of a progressive call: its first slot, stream word and stuffing chunk, and its file
  long long slot0, word0, chunk0;
  unsigned char* out;
  long long* out_bytes;
};
struct ProgList {
  PImg im[JPEG_MAX_BATCH];
  long long slots, chunks;
  int sub;
};

struct ProgRun {   // the EOB runs a slot emits before its first coded symbol (pre) and after its last (post)
  unsigned short pre_run, pre_be, post_run, post_be;   // run length (0: none) and the correction bits that go with it
  unsigned pre_from, post_from;                         // the stream's first slot holding those bits
};

struct ProgScratch {
  const short* coef;             // se_jpeg.cu's [64][blocks] zigzag coefficients
  unsigned char* flags;          // [slots] AC scans: bit 7 the block ends in an EOB run, bit 6 it codes a symbol, bits 0-5
                                 // its trailing correction bits
  unsigned long long* corr;      // [slots] those bits, the first in the highest place
  ProgRun* runs;                 // [slots]
  unsigned* bits;                // [slots] bit count
  unsigned long long* bitoff;    // [slots] exclusive scan of bits over the call
  unsigned* words;               // the bit streams
  unsigned* ffcnt;               // [chunks]
  unsigned long long* ffoff;     // [chunks]
  unsigned long long* sums;      // scan tile sums
  unsigned long long* hist;      // [n][JPEG_SCANS][2][256]
  JpegTables* tabs;              // [n][JPEG_SCANS], tables 0 (luma) and 1 (chroma)
  long long* data_at;            // [n][JPEG_SCANS] where each scan's data starts in the file
};

// The call's slot, word and chunk layout into P (images' sizes from L) and, with base != null, S's arrays at base; returns
// the scratch bytes. S.coef is the caller's.
size_t jpeg_prog_layout(const JpegList& L, unsigned char* base, ProgList* P, ProgScratch* S);
// a true bound of the progressive file of an h x w image whose header through SOF2 is sof_end bytes (DESIGN §7b)
long long jpeg_prog_max_bytes(int h, int w, int subsampling, int sof_end = jpeg_sof_end(2, 0));
// Enqueues the progressive coder on `st` after se_jpeg.cu's dct kernel: writes each image's file and byte count.
int jpeg_progressive(const JpegList& L, const HeaderList& H, const ProgList& P, const ProgScratch& S, cudaStream_t st);

}  // namespace se

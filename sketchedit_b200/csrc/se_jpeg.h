// Baseline JPEG encoding of uint8 RGB windows on the GPU (se_jpeg.cu), byte for byte what PIL.Image.save(buf, "JPEG",
// quality=q, subsampling=s[, optimize=True]) writes with libjpeg-turbo for s = 0 (4:4:4) and s = 2 (4:2:0). The optimal
// Huffman tables of optimize=True are built by the kernels of se_jpeg_opt.cu.
#pragma once
#include "se_common.cuh"

namespace se {

constexpr int JPEG_MAX_BATCH = 32;          // images per call: their descriptors travel as kernel parameters
constexpr int JPEG_HEADER_BYTES = 623;      // SOI, APP0, 2 DQT, SOF0, 4 DHT, SOS
constexpr int JPEG_MAX_BLOCK_BITS = 1664;   // 64 x (16-bit code + 10 value bits) >= DC (<= 16 + 11) + 63 AC (see DESIGN §7b)
constexpr int JPEG_SOF_END = 177;           // header bytes before the first DHT: SOI, APP0, 2 DQT, SOF0
constexpr int JPEG_SOS_BYTES = 14;          // the SOS segment that ends the header
constexpr int kSofHeightAt = 163;           // byte offsets of SOF0's height and width in the header

// se_jpeg_max_bytes without the checks: the header, JPEG_MAX_BLOCK_BITS per block doubled for 0xFF stuffing, and EOI
long long jpeg_max_bytes(int h, int w, int subsampling);

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
  int n, sub;   // images; subsampling (0 or 2)
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
  // optimize only, else null: the Annex K tables and the 623-byte header are used
  unsigned long long* hist;    // [n][4][256] symbol counts per image and table
  JpegTables* tabs;            // [n] optimal tables
  int* hdr_len;                // [n] header bytes, where the entropy-coded data starts
};

struct HeaderList {
  unsigned char bytes[JPEG_HEADER_BYTES];   // the Annex K header of a 1x1 image at the call's quality and subsampling
  unsigned char* out[JPEG_MAX_BATCH];
  unsigned short hw[JPEG_MAX_BATCH][2];
};
static_assert(sizeof(HeaderList) <= 4096, "header descriptors must fit the kernel parameter space");

// header byte j of image i (j < JPEG_SOF_END, or of SOS) with its height and width in SOF0
__host__ __device__ __forceinline__ unsigned char header_byte(const HeaderList& H, int i, int j) {
  if (j >= kSofHeightAt && j < kSofHeightAt + 4) {
    const int x = H.hw[i][(j - kSofHeightAt) >> 1];
    return (unsigned char)((j - kSofHeightAt) & 1 ? x : x >> 8);
  }
  return H.bytes[j];
}

#ifdef __CUDACC__
// Block e of an image in scan order: its component (0 Y, 1 Cb, 2 Cr) and block column / row in that component's plane.
// A 4:2:0 MCU holds luma blocks (0,0), (0,1), (1,0), (1,1), then Cb and Cr; a 4:4:4 MCU holds Y, Cb, Cr.
struct BlockAt {
  int comp, bx, by;
  bool dummy;   // a 4:2:0 luma block wholly outside the image
};
__device__ __forceinline__ BlockAt block_at(const JImg& d, int sub, long long e) {
  const int per = sub == 2 ? 6 : 3;
  const long long mcu = e / per;
  const int k = (int)(e - mcu * per), mx = (int)(mcu % d.mcu_x), my = (int)(mcu / d.mcu_x);
  BlockAt b;
  if (sub == 2 && k < 4) {
    b.comp = 0;
    b.bx = 2 * mx + (k & 1);
    b.by = 2 * my + (k >> 1);
    b.dummy = b.bx * 8 >= d.w || b.by * 8 >= d.h;
  } else {
    b.comp = sub == 2 ? k - 3 : k;
    b.bx = mx;
    b.by = my;
    b.dummy = false;
  }
  return b;
}

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }
#endif

// se_jpeg_opt.cu, each only enqueues on `st`. jpeg_optimize_tables: from the coefficients and DC differences in S, count
// each image's symbols into S.hist (zeroed by the caller) and build its optimal tables into S.tabs. jpeg_optimize_header:
// write each image's header with its tables and its length to S.hdr_len, and every block's bit count with those tables
// to S.bits.
int jpeg_optimize_tables(const JpegList& L, const JpegScratch& S, cudaStream_t st);
int jpeg_optimize_header(const JpegList& L, const HeaderList& H, const JpegScratch& S, cudaStream_t st);

}  // namespace se

// PNG decoding into uint8 pixels, pixel for pixel what np.asarray(Image.open(f).convert(mode)) gives for mode "RGB" or "L"
// (Pillow 12), for non-interlaced files of colour types 0 (depths 1/2/4/8), 2 (8), 3 (1/2/4/8), 4 (8) and 6 (8). The host
// parses the container (sketchedit_b200/pngfile.py) and passes each file's IDAT payloads as one zlib stream; tests/
// util_png_decode.py restates the stages below in numpy.
//
// One warp per file, one launch:
//   inflate: se_inflate.cuh into the file's raw filtered scanlines (scratch), then Adler-32 over them;
//   rows:    a wavefront over 32 rows at a time (se_png_dec.cuh): lane j reconstructs row r0 + j one pixel behind lane
//            j - 1; each reconstructed pixel is unpacked, looked up in the palette, converted to the requested mode and stored.
// Files of many megabytes decode faster across the whole GPU: se_png_split.cu.
// The file's status word is 0 only when every stage succeeded; any other value sends the file to Pillow.
#include <string.h>

#include <string>

#include "../../include/sketchedit_b200.h"
#include "se_common.cuh"
#include "se_inflate.cuh"
#include "se_png_dec.cuh"

namespace se {

struct PDec {
  long long src_off, src_len, plte_off, raw_off;
  unsigned char* out;
  int h, w, depth, ctype, npal, mode;   // mode: output bytes per pixel, 1 ("L") or 3 ("RGB")
};
struct PDecList {
  const unsigned char* src;
  unsigned char* raw;
  int* status;
  int n;
  PDec f[PNG_DECODE_MAX_BATCH];
};

__global__ void __launch_bounds__(32) png_decode_kernel(const __grid_constant__ PDecList L) {
  __shared__ InflateTabs tabs;
  __shared__ unsigned char pal[768];
  const int lane = threadIdx.x;
  const PDec& F = L.f[blockIdx.x];
  if (F.ctype == 3)
    for (int k = lane; k < 3 * F.npal; k += 32) pal[k] = L.src[F.plte_off + k];
  unsigned char* raw = L.raw + F.raw_off;
  int st = inflate_zlib(L.src + F.src_off, F.src_len, raw, raw_bytes(F.h, F.w, F.depth, F.ctype), tabs, lane, 32);
  __syncwarp();
  if (st == INF_OK) {
    const PRows R{F.out, F.h, F.w, F.depth, F.ctype, F.npal, F.mode};
    RowsAlone alone;
    int err = 0;
    for (int r0 = 0; r0 < F.h; r0 += 32) png_row_group(R, raw, pal, r0, lane, err, alone);
    // the first of the lanes' errors in lane order
    const unsigned any = __ballot_sync(0xFFFFFFFFu, err != 0);
    if (any) st = __shfl_sync(0xFFFFFFFFu, err, __ffs(any) - 1);
  }
  if (lane == 0) L.status[blockIdx.x] = st;
}

}  // namespace se

using namespace se;

extern "C" {

int se_png_decode_u8(const unsigned char* src, const long long* src_off, const long long* src_len, const int* info,
                     const long long* plte_off, int n, unsigned char* const* out, int* status_dev,
                     void* scratch, long long* scratch_bytes, void* stream) {
  if (int rc = png_check_files(src_off, src_len, info, plte_off, n, scratch_bytes)) return rc;
  long long need = 0;
  for (int i = 0; i < n; ++i) need += (raw_bytes(info[6 * i], info[6 * i + 1], info[6 * i + 2], info[6 * i + 3]) + 15) / 16 * 16;
  SE_SCRATCH(scratch, scratch_bytes, need, n);
  SE_REQUIRE(src && out && status_dev, "null src / out / status");
  for (int i = 0; i < n; ++i) SE_REQUIRE(out[i] != nullptr, "null out");
  PDecList L;
  memset(&L, 0, sizeof(L));
  L.src = src;
  L.raw = (unsigned char*)scratch;
  L.status = status_dev;
  L.n = n;
  long long at = 0;
  for (int i = 0; i < n; ++i) {
    const int* f = info + 6 * i;
    PDec& d = L.f[i];
    d.src_off = src_off[i];
    d.src_len = src_len[i];
    d.raw_off = at;
    d.out = out[i];
    d.h = f[0];
    d.w = f[1];
    d.depth = f[2];
    d.ctype = f[3];
    d.npal = f[4];
    d.mode = f[5];
    d.plte_off = d.ctype == 3 ? plte_off[i] : 0;
    at += (raw_bytes(d.h, d.w, d.depth, d.ctype) + 15) / 16 * 16;
  }
  png_decode_kernel<<<n, 32, 0, (cudaStream_t)stream>>>(L);
  SE_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"

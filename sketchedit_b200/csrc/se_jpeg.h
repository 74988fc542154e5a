// Baseline JPEG encoding of uint8 RGB windows on the GPU (se_jpeg.cu), byte for byte what PIL.Image.save(buf, "JPEG",
// quality=q, subsampling=s) writes with libjpeg-turbo for s = 0 (4:4:4) and s = 2 (4:2:0).
#pragma once
#include "se_common.cuh"

namespace se {

constexpr int JPEG_MAX_BATCH = 32;          // images per call: their descriptors travel as kernel parameters
constexpr int JPEG_HEADER_BYTES = 623;      // SOI, APP0, 2 DQT, SOF0, 4 DHT, SOS
constexpr int JPEG_MAX_BLOCK_BITS = 1664;   // 64 x (16-bit code + 10 value bits) >= DC (<= 11 + 11) + 63 AC

// se_jpeg_max_bytes without the checks: the header, JPEG_MAX_BLOCK_BITS per block doubled for 0xFF stuffing, and EOI
long long jpeg_max_bytes(int h, int w, int subsampling);

}  // namespace se

// deflate_encode.h — the Deflate encoder of deflate_encode.cu as an internal entry point: the strips of a raster in
// device memory (convention in include/aerial_mapper_b200.h, amb_deflate_strips_device).  The Cloud-Optimized GeoTIFF
// (raster_pyramid.cu) compresses its stacked tiles with it, one tile per strip.
#pragma once

#include "amb_context.h"

namespace amb {

constexpr unsigned kAdlerMod = 65521u;

// Adler-32 of n bytes b_i from partial sums of segments: a = 1 + sum b_i, b = n + sum (n - i) b_i (mod 65521).  Start
// with *a = 1, *b = n % 65521; a segment at offset o with S = sum b_i and W = sum (i - o) b_i over its bytes adds
// (n - o) S - W to b.  The Adler-32 is (b << 16) | a.
__host__ __device__ __forceinline__ void adler_add_segment(unsigned long long n, unsigned long long o,
                                                           unsigned long long S, unsigned long long W,
                                                           unsigned long long* a, unsigned long long* b) {
  S %= kAdlerMod;
  W %= kAdlerMod;
  const unsigned long long rest = (n - o) % kAdlerMod;
  *a = (*a + S) % kAdlerMod;
  *b = (*b + rest * S % kAdlerMod + kAdlerMod - W) % kAdlerMod;
}

struct DeflateShape {
  const unsigned char* img;
  unsigned long long stride;     // bytes between raster rows
  int32_t w, h;
  int32_t spp, bps;              // samples per pixel, bytes per sample
  int32_t predict;               // 1: the TIFF predictor of the format; 0: the bytes as they are (a COG's 1-bit masks)
  unsigned long long row_bytes;  // predicted bytes per row = w * spp * bps
  int32_t rps;                   // rows per strip
  int32_t n_strips;
  int32_t segs;                  // segments per full strip
  int32_t blocks;                // blocks per full strip
  int32_t win_bytes, prev_bytes; // the match kernel's shared memory: the largest window and its segment's chain links,
                                 // each rounded up to 16 bytes (strips shorter than a window take less)
};

struct DeflateParams {
  DeflateShape s;
  unsigned long long n_bytes;  // predicted bytes of the whole raster
  unsigned long long bound;    // the largest file
};

// AMB_OK, AMB_ERR_INVALID_ARGUMENT or AMB_ERR_UNSUPPORTED (a strip over 4 GiB, which TIFF cannot count).  predictor
// false: no predictor (TIFF Predictor 1), for 8-bit formats only.
int deflate_params(int32_t w, int32_t h, int format, int32_t rps, DeflateParams* p, bool predictor = true);

// The strips of the w x h raster at d_img (rows row_stride bytes apart), ordered after earlier work on the context's
// stream; synchronous, with the capacity contract of amb_deflate_strips_device.  Arguments are checked by the caller.
int deflate_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, DeflateParams p, void* host_out,
                   size_t capacity, size_t* size, uint32_t* strip_bytes);

}  // namespace amb

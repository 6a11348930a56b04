// jpeg_encode.h — the baseline JPEG encoder of jpeg_encode.cu as internal entry points for the JPEG tiles of a
// Cloud-Optimized GeoTIFF (raster_pyramid.cu; convention in include/aerial_mapper_b200.h, amb_cog_jpeg_tiles_device):
// the stacked T x T tiles are encoded as one image with one restart interval per tile, and every interval is written
// out as an abbreviated stream of its own.
#pragma once

#include <vector>

#include "amb_context.h"

namespace amb {

struct JpegParams {
  int32_t w, h;
  int channels, quality, sampling;
  int32_t interval;
  int bpm, mcus_x, mcus_y, kind;
  unsigned long long n_mcu, n_seg;
};

// The stacked tiles of side `tile` (a multiple of 16), n_tiles of them: an image tile wide and n_tiles * tile high with
// one restart interval per tile.  No 65535 limit on the height or the interval, which only the JPEG file format of
// amb_jpeg_encode_device has.  AMB_OK or AMB_ERR_UNSUPPORTED (channels, quality, sampling).
int jpeg_tile_params(int32_t tile, long long n_tiles, int channels, int quality, int sampling, JpegParams* p);

// The largest output of jpeg_tiles_encode for p: every tile's header, data and EOI
unsigned long long jpeg_tiles_bound(const JpegParams& p);

// SOI, the DQT and DHT segments of the file amb_jpeg_encode_device writes, EOI: the TIFF JPEGTables stream
std::vector<unsigned char> jpeg_tables_stream(int channels, int quality);

// Every restart interval of the image at d_img (rows row_stride bytes apart) as an abbreviated stream: SOI, SOF0 of a
// tile, SOS, the interval's stuffed entropy-coded bytes without its RST marker, EOI; back to back in host_out, with
// each stream's length in tile_bytes[n_seg].  Synchronous, with the capacity contract of amb_jpeg_encode_device.
int jpeg_tiles_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, const JpegParams& p,
                      void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes);

}  // namespace amb

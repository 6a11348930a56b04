// jpeg_header.h — the JPEG marker parser (jpeg_header.cc), the only code that reads markers: amb_jpeg_info and the
// decoder (jpeg_decode.cu) take the frame, the tables and the scan's position from it.  Host only.
#pragma once

#include <cstddef>
#include <cstdint>

struct amb_ctx;

namespace amb {

struct JpegHuffTable {
  bool present = false;
  uint8_t bits[16];    // codes of length 1..16
  uint8_t vals[256];
};

struct JpegFrame {
  int32_t width = 0, height = 0;
  int components = 0;          // 1 or 3
  int sampling = 0;            // amb_jpeg_sampling of the luma factors (AMB_JPEG_444 for gray)
  int hmax = 1, vmax = 1;      // the luma factors (1 for gray: a one-component scan has one-block MCUs)
  int restart_interval = 0;    // MCUs, 0 = none
  int comp_h[3] = {1, 1, 1}, comp_v[3] = {1, 1, 1};
  int comp_tq[3] = {0, 0, 0};  // quantisation table of each component
  int comp_td[3] = {0, 0, 0}, comp_ta[3] = {0, 0, 0};  // DC / AC Huffman table of each component (scan order = frame order)
  uint16_t quant[4][64];       // natural order
  bool quant_present[4] = {false, false, false, false};
  JpegHuffTable dc[4], ac[4];
  size_t scan_begin = 0;       // first byte of the entropy-coded data (the scan runs to the first marker other than RSTn)
};

// AMB_OK, AMB_ERR_INVALID_ARGUMENT (not a JPEG stream, or a malformed header) or AMB_ERR_UNSUPPORTED (a JPEG outside the
// set include/aerial_mapper_b200.h states).  Reads data[0, bytes) only.
int jpeg_parse(const unsigned char* data, size_t bytes, JpegFrame* f);

// jpeg_decode.cu: rows [row0[i], row1[i]) of every frame (all columns; none where row1 <= row0), decoded into the context's
// `frames` buffer; band_ptr[i] is row row0[i] of frame i, rows band_pitch[i] bytes apart.  Returns the first failing
// frame's status.
struct JpegBands {
  const void* const* files;
  const size_t* file_bytes;
  const JpegFrame* headers;
  const int32_t* row0;
  const int32_t* row1;
  size_t n;
  int channels;
};
int jpeg_decode_bands(amb_ctx* ctx, const JpegBands& in, unsigned char** band_ptr, int* band_pitch);

}  // namespace amb

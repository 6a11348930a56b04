// jpeg_header.cc — JPEG markers up to the first scan (convention and supported set in include/aerial_mapper_b200.h,
// "JPEG frames decoded on the device").  The checks of the tables are libjpeg-turbo's (jdmarker.c, jdhuff.c
// jpeg_make_d_derived_tbl): a stream cv2.imread rejects is rejected here too.
#include "jpeg_header.h"

#include <cstring>

#include "../../include/aerial_mapper_b200.h"

namespace amb {
namespace {

const uint8_t kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                              41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                              30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

int be16(const unsigned char* p) { return (p[0] << 8) | p[1]; }

// The EXIF orientation of an APP1 payload, 0 if it has none (or the TIFF structure is unreadable, which cv2 ignores too)
int exif_orientation(const unsigned char* p, size_t n) {
  if (n < 14 || std::memcmp(p, "Exif\0\0", 6) != 0) return 0;
  const unsigned char* t = p + 6;
  const size_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I')
    le = true;
  else if (t[0] == 'M' && t[1] == 'M')
    le = false;
  else
    return 0;
  auto u16 = [&](size_t o) { return le ? (t[o] | (t[o + 1] << 8)) : ((t[o] << 8) | t[o + 1]); };
  auto u32 = [&](size_t o) {
    return le ? (uint32_t(t[o]) | (uint32_t(t[o + 1]) << 8) | (uint32_t(t[o + 2]) << 16) | (uint32_t(t[o + 3]) << 24))
              : ((uint32_t(t[o]) << 24) | (uint32_t(t[o + 1]) << 16) | (uint32_t(t[o + 2]) << 8) | uint32_t(t[o + 3]));
  };
  const uint32_t ifd = u32(4);
  if (ifd > tn || tn - ifd < 2) return 0;
  const int count = u16(ifd);
  for (int e = 0; e < count; ++e) {
    const size_t o = ifd + 2 + 12 * static_cast<size_t>(e);
    if (o + 12 > tn) return 0;
    if (u16(o) == 0x0112) return u16(o + 2) == 3 ? u16(o + 8) : 0;
  }
  return 0;
}

// jdhuff.c jpeg_make_d_derived_tbl: at most 256 codes, and no length may hold more codes than it has room for
bool huffman_table_valid(const JpegHuffTable& t, bool dc) {
  int total = 0;
  for (int l = 0; l < 16; ++l) total += t.bits[l];
  if (total > 256) return false;
  long code = 0;
  for (int l = 1; l <= 16; ++l) {
    code += t.bits[l - 1];
    if (code >= (1L << l)) return false;  // (the all-ones code of a length is reserved)
    code <<= 1;
  }
  if (dc)
    for (int i = 0; i < total; ++i)
      if (t.vals[i] > 15) return false;
  return true;
}

}  // namespace

int jpeg_parse(const unsigned char* d, size_t n, JpegFrame* f) {
  if (!d || !f || n < 4 || d[0] != 0xff || d[1] != 0xd8) return AMB_ERR_INVALID_ARGUMENT;
  *f = JpegFrame();
  bool have_sof = false, jfif = false;
  uint8_t comp_id[3] = {0, 0, 0};
  size_t i = 2;
  for (;;) {
    if (i + 2 > n || d[i] != 0xff) return AMB_ERR_INVALID_ARGUMENT;
    while (i + 1 < n && d[i + 1] == 0xff) ++i;  // fill bytes
    if (i + 2 > n) return AMB_ERR_INVALID_ARGUMENT;
    const int m = d[i + 1];
    i += 2;
    if (m == 0xd9 || m == 0xd8 || m == 0x01 || (m >= 0xd0 && m <= 0xd7) || m == 0x00) return AMB_ERR_INVALID_ARGUMENT;
    if (i + 2 > n) return AMB_ERR_INVALID_ARGUMENT;
    const size_t len = static_cast<size_t>(be16(d + i));
    if (len < 2 || i + len > n) return AMB_ERR_INVALID_ARGUMENT;
    const unsigned char* p = d + i + 2;
    const size_t pn = len - 2;
    if (m == 0xc0 || m == 0xc1) {  // baseline / extended sequential, Huffman
      if (have_sof || pn < 6) return AMB_ERR_INVALID_ARGUMENT;
      have_sof = true;
      if (p[0] != 8) return AMB_ERR_UNSUPPORTED;
      f->height = be16(p + 1);
      f->width = be16(p + 3);
      f->components = p[5];
      if (f->height == 0) return AMB_ERR_UNSUPPORTED;  // the height would come from a DNL marker
      if (f->width == 0 || f->components == 0 || pn != 6 + 3 * static_cast<size_t>(f->components))
        return AMB_ERR_INVALID_ARGUMENT;
      if (f->components != 1 && f->components != 3) return AMB_ERR_UNSUPPORTED;
      for (int c = 0; c < f->components; ++c) {
        comp_id[c] = p[6 + 3 * c];
        f->comp_h[c] = p[7 + 3 * c] >> 4;
        f->comp_v[c] = p[7 + 3 * c] & 15;
        f->comp_tq[c] = p[8 + 3 * c];
        if (f->comp_h[c] < 1 || f->comp_h[c] > 4 || f->comp_v[c] < 1 || f->comp_v[c] > 4 || f->comp_tq[c] > 3)
          return AMB_ERR_INVALID_ARGUMENT;
      }
    } else if ((m >= 0xc2 && m <= 0xcb && m != 0xc4 && m != 0xc8) || (m >= 0xcd && m <= 0xcf) || m == 0xcc ||
               m == 0xdc) {
      return AMB_ERR_UNSUPPORTED;  // progressive, lossless, hierarchical, arithmetic coding (and DAC), DNL
    } else if (m == 0xdb) {  // DQT
      size_t o = 0;
      while (o < pn) {
        const int pq = p[o] >> 4, tq = p[o] & 15;
        if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > pn) return AMB_ERR_INVALID_ARGUMENT;
        for (int k = 0; k < 64; ++k)
          f->quant[tq][kNatural[k]] = static_cast<uint16_t>(pq ? be16(p + o + 1 + 2 * k) : p[o + 1 + k]);
        f->quant_present[tq] = true;
        o += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xc4) {  // DHT
      size_t o = 0;
      while (o < pn) {
        if (o + 17 > pn) return AMB_ERR_INVALID_ARGUMENT;
        const int tc = p[o] >> 4, th = p[o] & 15;
        if (tc > 1 || th > 3) return AMB_ERR_INVALID_ARGUMENT;
        JpegHuffTable& t = tc ? f->ac[th] : f->dc[th];
        int count = 0;
        for (int l = 0; l < 16; ++l) count += p[o + 1 + l];
        if (count > 256 || o + 17 + count > pn) return AMB_ERR_INVALID_ARGUMENT;
        std::memcpy(t.bits, p + o + 1, 16);
        std::memset(t.vals, 0, sizeof(t.vals));
        std::memcpy(t.vals, p + o + 17, count);
        t.present = true;
        o += 17 + count;
      }
    } else if (m == 0xdd) {  // DRI
      if (pn != 2) return AMB_ERR_INVALID_ARGUMENT;
      f->restart_interval = be16(p);
    } else if (m == 0xe0) {
      // jdmarker.c examine_app0 counts a JFIF marker only with its 14 bytes of payload (APP0_DATA_LEN)
      if (pn >= 14 && std::memcmp(p, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xe1) {
      const int o = exif_orientation(p, pn);
      if (o != 0 && o != 1) return AMB_ERR_UNSUPPORTED;  // cv2.imread would rotate or mirror the image
    } else if (m == 0xee) {
      // Adobe colour transforms; examine_app14 counts the marker only with its 12 bytes of payload (APP14_DATA_LEN)
      if (pn >= 12 && std::memcmp(p, "Adobe", 5) == 0) return AMB_ERR_UNSUPPORTED;
    } else if (m == 0xda) {  // SOS: the frame must be complete, and this one scan must carry every component
      if (!have_sof || pn < 1) return AMB_ERR_INVALID_ARGUMENT;
      const int ns = p[0];
      if (ns < 1 || ns > 4 || pn != 4 + 2 * static_cast<size_t>(ns)) return AMB_ERR_INVALID_ARGUMENT;
      if (ns != f->components) return AMB_ERR_UNSUPPORTED;  // multi-scan sequential
      for (int c = 0; c < ns; ++c) {
        if (p[1 + 2 * c] != comp_id[c]) return AMB_ERR_UNSUPPORTED;  // a scan order other than the frame's
        f->comp_td[c] = p[2 + 2 * c] >> 4;
        f->comp_ta[c] = p[2 + 2 * c] & 15;
        if (f->comp_td[c] > 3 || f->comp_ta[c] > 3) return AMB_ERR_INVALID_ARGUMENT;
      }
      const unsigned char* q = p + 1 + 2 * ns;
      if (q[0] != 0 || q[1] != 63 || q[2] != 0) return AMB_ERR_UNSUPPORTED;  // not a sequential spectral selection
      f->scan_begin = i + len;
      break;
    }
    // APPn, COM and other segments are skipped
    i += len;
  }
  // colour space: libjpeg takes three components as RGB (no conversion) when neither JFIF nor Adobe says otherwise and
  // the component ids spell R, G, B
  if (f->components == 3 && !jfif && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')
    return AMB_ERR_UNSUPPORTED;
  if (f->components == 3) {
    for (int c = 1; c < 3; ++c)
      if (f->comp_h[c] != 1 || f->comp_v[c] != 1) return AMB_ERR_UNSUPPORTED;
    const int h = f->comp_h[0], v = f->comp_v[0];
    if (h == 1 && v == 1)
      f->sampling = AMB_JPEG_444;
    else if (h == 2 && v == 1)
      f->sampling = AMB_JPEG_422;
    else if (h == 2 && v == 2)
      f->sampling = AMB_JPEG_420;
    else
      return AMB_ERR_UNSUPPORTED;  // 4:1:1, 4:4:0 and others
    f->hmax = h;
    f->vmax = v;
  } else {
    f->sampling = AMB_JPEG_444;
    f->comp_h[0] = f->comp_v[0] = 1;  // a one-component scan is not interleaved: one block per MCU, whatever the factors
  }
  for (int c = 0; c < f->components; ++c) {
    if (!f->quant_present[f->comp_tq[c]]) return AMB_ERR_INVALID_ARGUMENT;
    const JpegHuffTable& dc = f->dc[f->comp_td[c]];
    const JpegHuffTable& ac = f->ac[f->comp_ta[c]];
    // a stream that leaves out its (standard) tables is refused rather than given libjpeg-turbo's defaults
    if (!dc.present || !ac.present) return AMB_ERR_UNSUPPORTED;
    if (!huffman_table_valid(dc, true) || !huffman_table_valid(ac, false)) return AMB_ERR_INVALID_ARGUMENT;
  }
  return AMB_OK;
}

}  // namespace amb

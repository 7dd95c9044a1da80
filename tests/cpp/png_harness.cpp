// CPU harness of the PNG decoder: xivo_b200/csrc/png.cuh compiled with g++ (the same container walk, inflate, unfilter and
// conversion code the kernels run, with one lane instead of a warp).  Driven by tests/test_png_logic.py through ctypes.
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../xivo_b200/csrc/png.cuh"

using namespace xb;

extern "C" {

// container walk: 0 or -1 with the reason copied to why
int ph_info(const uint8_t* p, size_t n, int* geo /*rows, cols, channels, bit_depth, n_idat*/, char* why, int why_n) {
  png::Info I;
  const char* w = "";
  const int rc = png::parse(p, n, I, &w, [](size_t, size_t) {});
  snprintf(why, why_n, "%s", rc ? w : "");
  geo[0] = I.rows;
  geo[1] = I.cols;
  geo[2] = I.channels;
  geo[3] = I.bit_depth;
  geo[4] = I.n_idat;
  return rc;
}

// raw zlib stream -> exactly cap bytes; returns the decoder status
int ph_inflate(const uint8_t* in, size_t n, uint8_t* out, size_t cap) {
  png::Huff lit, dst;
  uint8_t lens[320];
  return png::inflate(in, n, out, cap, lit, dst, lens, png::SerialLanes());
}

// whole file -> rows x cols x oc bytes (out must hold them); -1 = container refusal, else the decoder status
int ph_decode(const uint8_t* p, size_t n, int oc, uint8_t* out) {
  png::Info I;
  const char* w = "";
  std::vector<uint8_t> z;
  if (png::parse(p, n, I, &w, [&](size_t off, size_t len) { z.insert(z.end(), p + off, p + off + len); })) return -1;
  const size_t rowbytes = (size_t)I.cols * I.bpp, stride = rowbytes + 1;
  std::vector<uint8_t> raw(I.raw_bytes());
  if (int s = ph_inflate(z.data(), z.size(), raw.data(), raw.size())) return s;
  for (int r = 0; r < I.rows; ++r) {
    uint8_t* cur = raw.data() + (size_t)r * stride;
    if (int s = png::unfilter_row(cur + 1, r ? cur + 1 - stride : nullptr, cur[0], rowbytes, I.bpp)) return s;
    for (int x = 0; x < I.cols; ++x) png::convert_px(cur + 1 + (size_t)x * I.bpp, I.channels, I.bit_depth / 8, oc, out + ((size_t)r * I.cols + x) * oc);
  }
  return 0;
}

const char* ph_status_text(int s) { return png::status_text(s); }
}

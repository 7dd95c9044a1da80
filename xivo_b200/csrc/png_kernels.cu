// PNG decoding on the device (DESIGN §2 "PNG ingest", §4 "png_inflate_kernel / png_unfilter_kernel").  The host walks the chunks and
// packs every frame's IDAT payloads back to back; png_inflate_kernel inflates one frame per warp into a scratch buffer of filtered
// scanlines, png_unfilter_kernel undoes the row filters in place (one warp per frame, 32 rows as a skewed wavefront) and writes the
// cv::imread conversion (BGR / grey, high byte of 16-bit samples, alpha stripped).  The decoding logic itself is png.cuh, which the CPU
// harness compiles with g++.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/xivo_b200.h"
#include "common.cuh"
#include "ctx.h"
#include "kernels.h"
#include "png.cuh"
#include "prof.h"

namespace xb {
extern std::atomic<unsigned long long> g_launches;

namespace {
constexpr int kPngWarps = 4;  // frames per block

// W of png::inflate for a full warp
struct WarpLanes {
  static constexpr int n = 32;
  int lane;
  __host__ __device__ void sync() const {
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
  }
  __host__ __device__ uint32_t sum(uint32_t v) const {
#ifdef __CUDA_ARCH__
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
  }
};

__global__ void __launch_bounds__(kPngWarps * 32) png_inflate_kernel(const uint8_t* __restrict__ in, uint8_t* scratch,
                                                                       const PngFrameDesc* __restrict__ fr, int n, int* status) {
  __shared__ png::Huff lit[kPngWarps], dst[kPngWarps];
  __shared__ uint8_t lens[kPngWarps][320];
  const int wid = threadIdx.x >> 5, f = blockIdx.x * kPngWarps + wid;
  if (f >= n) return;
  const PngFrameDesc d = fr[f];
  const size_t cap = (size_t)d.rows * (1 + (size_t)d.cols * d.bpp);
  const WarpLanes w{(int)(threadIdx.x & 31)};
  const int s = png::inflate(in + d.in_off, (size_t)d.in_len, scratch + d.scratch_off, cap, lit[wid], dst[wid], lens[wid], w);
  if (w.lane == 0) status[f] = s;
}

// Rows r0 .. r0 + 31 of one frame, lane i on row r0 + i, one byte behind lane i - 1: at step t lane i undoes byte x = t - i, whose
// up value lane i - 1 produced at step t - 1 (one shuffle); up-left and left are the up values received / bytes produced BPP steps ago,
// kept in two BPP-deep register shift lines.  Lane 0 reads its up row from memory (finished in the previous group).
template <int BPP>
__device__ bool unfilter_group(uint8_t* img, int rows, size_t rowbytes, int r0, int lane) {
  const size_t stride = rowbytes + 1;
  const int r = r0 + lane;
  const bool valid = r < rows;
  uint8_t* row = img + (size_t)(valid ? r : 0) * stride;
  const int ft = valid ? row[0] : 0;
  const uint8_t* above = (lane == 0 && r > 0) ? img + (size_t)(r - 1) * stride + 1 : nullptr;
  uint32_t mine[BPP], ups[BPP];
#pragma unroll
  for (int k = 0; k < BPP; ++k) mine[k] = ups[k] = 0;
  uint32_t last = 0;
  const long long steps = (long long)rowbytes + 31;
  for (long long t = 0; t < steps; ++t) {
    uint32_t b = __shfl_up_sync(0xffffffffu, last, 1);
    const long long x = t - lane;
    const bool act = valid && x >= 0 && x < (long long)rowbytes;
    if (lane == 0) b = (above && act) ? above[x] : 0;
    uint32_t out = 0;
    if (act) {
      const uint32_t a = x >= BPP ? mine[BPP - 1] : 0, c = x >= BPP ? ups[BPP - 1] : 0;
      out = (row[1 + x] + png::predict(ft, a, b, c)) & 255u;
      row[1 + x] = (uint8_t)out;
    }
#pragma unroll
    for (int k = BPP - 1; k > 0; --k) {
      mine[k] = mine[k - 1];
      ups[k] = ups[k - 1];
    }
    mine[0] = out;
    ups[0] = b;
    last = out;
  }
  return valid && ft > 4;
}

__global__ void __launch_bounds__(kPngWarps * 32) png_unfilter_kernel(uint8_t* scratch, uint8_t* out, const PngFrameDesc* __restrict__ fr, int n,
                                                                        int* status) {
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, f = blockIdx.x * kPngWarps + wid;
  if (f >= n || status[f] != png::kOk) return;
  const PngFrameDesc d = fr[f];
  uint8_t* img = scratch + d.scratch_off;
  const size_t rowbytes = (size_t)d.cols * d.bpp, stride = rowbytes + 1;
  bool bad = false;
  for (int r0 = 0; r0 < d.rows; r0 += 32) {
    switch (d.bpp) {
      case 1: bad |= unfilter_group<1>(img, d.rows, rowbytes, r0, lane); break;
      case 2: bad |= unfilter_group<2>(img, d.rows, rowbytes, r0, lane); break;
      case 3: bad |= unfilter_group<3>(img, d.rows, rowbytes, r0, lane); break;
      case 4: bad |= unfilter_group<4>(img, d.rows, rowbytes, r0, lane); break;
      case 6: bad |= unfilter_group<6>(img, d.rows, rowbytes, r0, lane); break;
      default: bad |= unfilter_group<8>(img, d.rows, rowbytes, r0, lane); break;
    }
    __syncwarp();
    const int r1 = min(r0 + 32, d.rows);
    for (int r = r0; r < r1; ++r) {
      const uint8_t* src = img + (size_t)r * stride + 1;
      uint8_t* o = out + d.out_off + (size_t)r * d.cols * d.oc;
      for (int px = lane; px < d.cols; px += 32) png::convert_px(src + (size_t)px * d.bpp, d.channels, d.bps, d.oc, o + (size_t)px * d.oc);
    }
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) status[f] = png::kFilter;
}
}  // namespace

int launch_png_decode(cudaStream_t st, const uint8_t* in, uint8_t* scratch, uint8_t* out, const PngFrameDesc* fr, int n, int* status) {
  if (n <= 0) return 0;
  const int blocks = (n + kPngWarps - 1) / kPngWarps;
  {
    ProfScope ps("png_inflate_kernel", st);
    png_inflate_kernel<<<blocks, kPngWarps * 32, 0, st>>>(in, scratch, fr, n, status);
  }
  {
    ProfScope ps("png_unfilter_kernel", st);
    png_unfilter_kernel<<<blocks, kPngWarps * 32, 0, st>>>(scratch, out, fr, n, status);
  }
  g_launches += 2;
  XB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace xb

using namespace xb;

extern "C" {

int xivo_png_info(const uint8_t* png_data, size_t n, int* rows, int* cols, int* channels, int* bit_depth) {
  png::Info I;
  const char* why = "";
  if (png::parse(png_data, n, I, &why, [](size_t, size_t) {})) {
    set_error("png: %s", why);
    return XIVO_ERR_ARG;
  }
  if (rows) *rows = I.rows;
  if (cols) *cols = I.cols;
  if (channels) *channels = I.channels;
  if (bit_depth) *bit_depth = I.bit_depth;
  return XIVO_OK;
}

int xivo_decode_png(xivo_ctx* ctx, int n, const uint8_t* const* png_data, const size_t* png_bytes, int channels, uint8_t* const* out) {
  if (!ctx) {
    set_error("null ctx");
    return XIVO_ERR_ARG;
  }
  XB_REQUIRE(n >= 0 && (n == 0 || (png_data && png_bytes && out)), "decode_png: bad arguments");
  if (channels != 1 && channels != 3) {
    set_error("decode_png: channels must be 1 or 3, got %d", channels);
    return XIVO_ERR_ARG;
  }
  if (n == 0) return XIVO_OK;
  XB_CUDA(cudaSetDevice(ctx->device));
  // container walk and IDAT packing on the host: every refusal is reported before anything is uploaded
  std::vector<PngFrameDesc> fr(n);
  std::vector<uint8_t> blob;
  unsigned long long scratch = 0, outb = 0;
  for (int i = 0; i < n; ++i) {
    png::Info I;
    const char* why = "";
    const uint8_t* p = png_data[i];
    const size_t start = blob.size();
    if (!p || png::parse(p, png_bytes[i], I, &why, [&](size_t off, size_t len) { blob.insert(blob.end(), p + off, p + off + len); })) {
      set_error("png frame %d: %s", i, p ? why : "null data");
      return XIVO_ERR_ARG;
    }
    if (channels == 1 && I.channels > 2) {
      set_error("png frame %d: 1-channel output needs a grey or grey + alpha PNG (colour type %d)", i, I.color_type);
      return XIVO_ERR_ARG;
    }
    PngFrameDesc& d = fr[i];
    d.in_off = start;
    d.in_len = blob.size() - start;
    d.rows = I.rows;
    d.cols = I.cols;
    d.bpp = I.bpp;
    d.channels = I.channels;
    d.bps = I.bit_depth / 8;
    d.oc = channels;
    d.scratch_off = scratch;
    d.out_off = outb;
    scratch += I.raw_bytes();
    outb += (unsigned long long)I.rows * I.cols * channels;
  }
  cudaStream_t st = ctx->stream;
  DevBuf<uint8_t> din(std::max<size_t>(blob.size(), 1)), dscr(scratch), dout(outb);
  DevBuf<PngFrameDesc> dfr(n);
  DevBuf<int> dst(n);
  XB_REQUIRE(din.ok() && dscr.ok() && dout.ok() && dfr.ok() && dst.ok(), "cudaMalloc failed");
  if (!blob.empty()) XB_CUDA(cudaMemcpyAsync(din.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfr.p, fr.data(), sizeof(PngFrameDesc) * n, cudaMemcpyHostToDevice, st));
  if (int rc = launch_png_decode(st, din.p, dscr.p, dout.p, dfr.p, n, dst.p)) return rc;
  std::vector<int> status(n);
  XB_CUDA(cudaMemcpyAsync(status.data(), dst.p, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i)
    if (status[i] != png::kOk) {
      set_error("png frame %d: %s", i, png::status_text(status[i]));
      return XIVO_ERR_ARG;
    }
  for (int i = 0; i < n; ++i)
    XB_CUDA(cudaMemcpyAsync(out[i], dout.p + fr[i].out_off, (size_t)fr[i].rows * fr[i].cols * channels, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

}  // extern "C"

// Tracker kernels (HOT LOOP 1 of SURVEY.md §3.2): image pyramid, FAST-9/16 score + NMS,
// pyramidal Lucas-Kanade.  Integer / fixed-point semantics follow OpenCV exactly
// (the arithmetic the reference calls at /root/reference/src/tracker.cpp:224, :493, :526);
// float math in LK is compiled with -fmad=false so it rounds like the scalar CPU code.
//
// All kernels take a batch dimension (blockIdx.z or .y = independent sequence) because the
// only way a 640x480 frame fills an H100 (132 SMs) is by processing many sequences per launch.
#include <cuda.h>
#include <algorithm>
#include <cstdlib>
#include "kernels.h"
#include "prof.h"

namespace xb {

// ------------------------------------------------------------------------------------------
// pyrDown: 5-tap [1 4 6 4 1] separable, BORDER_REFLECT_101, (sum+128)>>8   (cv::pyrDown, u8)
// Replaces cv::buildOpticalFlowPyramid's per-level pyrDown (tracker.cpp:476,493).  Scharr
// derivatives are NOT materialised: the LK kernel recomputes them from the staged patch.
// Tile: 32x8 output pixels; input region (2*32+3)x(2*8+3) staged in shared memory.
// ------------------------------------------------------------------------------------------
// One launch copies one frame per sequence: src[z] -> dst + (off ? off[z] : z * stride).  Replaces B
// cudaMemcpyAsync calls (the API cost, not the bytes, is what matters at 0.3 MB per frame).
__global__ void __launch_bounds__(256) gather_frames_kernel(const uint8_t* const* __restrict__ src, uint8_t* __restrict__ dst,
                                                           unsigned long long stride, const unsigned long long* __restrict__ off,
                                                           size_t bytes) {
  const unsigned long long o = off ? off[blockIdx.y] : (unsigned long long)blockIdx.y * stride;
  if (o == ~0ull) return;
  const uint8_t* __restrict__ s = src[blockIdx.y];
  uint8_t* __restrict__ t = dst + o;
  const size_t i0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
  const size_t step = (size_t)gridDim.x * blockDim.x * 16;
  if (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(t)) & 15) == 0) {
    size_t i = i0;
    for (; i + 3 * step + 16 <= bytes; i += 4 * step) {  // four loads in flight per thread: what matters when the source is host memory behind PCIe
      const uint4 v0 = *reinterpret_cast<const uint4*>(s + i), v1 = *reinterpret_cast<const uint4*>(s + i + step);
      const uint4 v2 = *reinterpret_cast<const uint4*>(s + i + 2 * step), v3 = *reinterpret_cast<const uint4*>(s + i + 3 * step);
      *reinterpret_cast<uint4*>(t + i) = v0;
      *reinterpret_cast<uint4*>(t + i + step) = v1;
      *reinterpret_cast<uint4*>(t + i + 2 * step) = v2;
      *reinterpret_cast<uint4*>(t + i + 3 * step) = v3;
    }
    for (; i + 16 <= bytes; i += step) *reinterpret_cast<uint4*>(t + i) = *reinterpret_cast<const uint4*>(s + i);
    if (blockIdx.x == 0 && threadIdx.x < (bytes & 15)) t[(bytes & ~(size_t)15) + threadIdx.x] = s[(bytes & ~(size_t)15) + threadIdx.x];
  } else {
    for (size_t i = i0; i < bytes; i += step)
      for (int k = 0; k < 16 && i + k < bytes; ++k) t[i + k] = s[i + k];
  }
}
int launch_gather_frames(cudaStream_t st, const uint8_t* const* src, uint8_t* dst, unsigned long long stride, const unsigned long long* off,
                         size_t bytes, int batch, int max_chunks, int threads) {
  ProfScope ps("gather_frames", st);
  // max_chunks: CTAs per frame.  Host sources (pinned memory read over PCIe): a few small CTAs with four loads in flight per thread already
  // saturate the link and leave the SMs' thread slots to the
  // kernels of the other batches while they wait.
  threads = threads < 32 ? 32 : (threads > 256 ? 256 : (threads & ~31));
  const int chunks = (int)std::min<size_t>(max_chunks < 1 ? 1 : max_chunks, (bytes + (size_t)threads * 16 - 1) / ((size_t)threads * 16));
  gather_frames_kernel<<<dim3(chunks, batch), threads, 0, st>>>(src, dst, stride, off, bytes);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// cv::normalize(image, img_, 0, 255, NORM_MINMAX) (tracker.cpp:343-344, :465-467), in place on one frame per sequence.
// min / max are taken over all channels together; OpenCV then runs convertTo with
//   scale = 255 * (max - min > DBL_EPSILON ? 1 / (max - min) : 0), shift = -min * scale   (double, rounded to float)
//   out = saturate_u8(rint(fmaf(v, scale, shift)))
// which is bit-exact against cv2 over every (min, max, v).  Two launches: per-CTA partial min / max, then every CTA of a frame
// folds its frame's partials and remaps its share.  A frame starts anywhere (ring slot b * ring_n + slot of a frame of odd size):
// the bytes before its first and after its last 16-byte boundary go through CTA 0 one per thread.
// ------------------------------------------------------------------------------------------
constexpr int NM_THREADS = 256;
static int normalize_chunks(size_t bytes) {
  const size_t per = (size_t)NM_THREADS * 16 * 4;  // four 16-byte words per thread before a CTA loops
  return (int)std::min<size_t>(kNormMaxChunks, std::max<size_t>(1, (bytes + per - 1) / per));
}
// [head | 16-byte aligned body of nv words | tail] of a frame at p
struct FrameSplit {
  size_t head, nv, tail0;
  __device__ FrameSplit(const uint8_t* p, size_t bytes) {
    head = (16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15;
    if (head > bytes) head = bytes;
    nv = (bytes - head) >> 4;
    tail0 = head + nv * 16;
  }
};
__device__ __forceinline__ unsigned bytes_min(unsigned w) { return min(min(w & 255u, (w >> 8) & 255u), min((w >> 16) & 255u, w >> 24)); }
__device__ __forceinline__ unsigned bytes_max(unsigned w) { return max(max(w & 255u, (w >> 8) & 255u), max((w >> 16) & 255u, w >> 24)); }

__global__ void __launch_bounds__(NM_THREADS) minmax_partial_kernel(uint8_t* const* __restrict__ frames, size_t bytes, unsigned* __restrict__ part) {
  const uint8_t* __restrict__ p = frames[blockIdx.y];
  if (!p) return;
  const FrameSplit s(p, bytes);
  const uint4* __restrict__ body = reinterpret_cast<const uint4*>(p + s.head);
  unsigned mn = 0xffffffffu, mx = 0;  // four byte lanes each
  for (size_t i = (size_t)blockIdx.x * NM_THREADS + threadIdx.x; i < s.nv; i += (size_t)gridDim.x * NM_THREADS) {
    const uint4 v = body[i];
    mn = __vminu4(__vminu4(mn, v.x), __vminu4(v.y, __vminu4(v.z, v.w)));
    mx = __vmaxu4(__vmaxu4(mx, v.x), __vmaxu4(v.y, __vmaxu4(v.z, v.w)));
  }
  if (blockIdx.x == 0) {
    const size_t t = threadIdx.x;
    if (t < s.head) { const unsigned b = p[t] * 0x01010101u; mn = __vminu4(mn, b); mx = __vmaxu4(mx, b); }
    if (s.tail0 + t < bytes) { const unsigned b = p[s.tail0 + t] * 0x01010101u; mn = __vminu4(mn, b); mx = __vmaxu4(mx, b); }
  }
  unsigned lo = __reduce_min_sync(0xffffffffu, bytes_min(mn)), hi = __reduce_max_sync(0xffffffffu, bytes_max(mx));
  __shared__ unsigned wlo[NM_THREADS / 32], whi[NM_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { wlo[warp] = lo; whi[warp] = hi; }
  __syncthreads();
  if (warp == 0) {
    lo = __reduce_min_sync(0xffffffffu, lane < NM_THREADS / 32 ? wlo[lane] : 255u);
    hi = __reduce_max_sync(0xffffffffu, lane < NM_THREADS / 32 ? whi[lane] : 0u);
    if (lane == 0) part[(size_t)blockIdx.y * kNormMaxChunks + blockIdx.x] = lo | hi << 8;
  }
}

__device__ __forceinline__ unsigned remap4(unsigned w, float scale, float shift) {
  unsigned r = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int q = __float2int_rn(__fmaf_rn((float)((w >> (8 * k)) & 255u), scale, shift));
    r |= (unsigned)min(max(q, 0), 255) << (8 * k);
  }
  return r;
}

__global__ void __launch_bounds__(NM_THREADS) normalize_remap_kernel(uint8_t* const* __restrict__ frames, size_t bytes, const unsigned* __restrict__ part) {
  uint8_t* __restrict__ p = frames[blockIdx.y];
  if (!p) return;
  // every warp folds the frame's gridDim.x partials itself (at most two per lane): no shared memory, no barrier
  const unsigned* pp = part + (size_t)blockIdx.y * kNormMaxChunks;
  const unsigned lane = threadIdx.x & 31;
  unsigned lo = 255, hi = 0;
  for (unsigned c = lane; c < gridDim.x; c += 32) { lo = min(lo, pp[c] & 255u); hi = max(hi, pp[c] >> 8); }
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  const double scale_d = 255.0 * (hi > lo ? 1.0 / (double)(hi - lo) : 0.0);  // integer min / max: max - min > DBL_EPSILON <=> max > min
  const double shift_d = 0.0 - (double)lo * scale_d;
  const float scale = __double2float_rn(scale_d), shift = __double2float_rn(shift_d);
  const FrameSplit s(p, bytes);
  uint4* __restrict__ body = reinterpret_cast<uint4*>(p + s.head);
  for (size_t i = (size_t)blockIdx.x * NM_THREADS + threadIdx.x; i < s.nv; i += (size_t)gridDim.x * NM_THREADS) {
    uint4 v = body[i];
    v.x = remap4(v.x, scale, shift); v.y = remap4(v.y, scale, shift); v.z = remap4(v.z, scale, shift); v.w = remap4(v.w, scale, shift);
    body[i] = v;
  }
  if (blockIdx.x == 0) {
    const size_t t = threadIdx.x;
    if (t < s.head) p[t] = (uint8_t)remap4(p[t], scale, shift);
    if (s.tail0 + t < bytes) p[s.tail0 + t] = (uint8_t)remap4(p[s.tail0 + t], scale, shift);
  }
}

int launch_normalize_minmax(cudaStream_t st, uint8_t* const* frames, size_t bytes, int batch, unsigned* part) {
  if (batch <= 0 || bytes == 0) return 0;
  ProfScope ps("normalize_minmax", st);
  const dim3 grid(normalize_chunks(bytes), batch);
  minmax_partial_kernel<<<grid, NM_THREADS, 0, st>>>(frames, bytes, part);
  normalize_remap_kernel<<<grid, NM_THREADS, 0, st>>>(frames, bytes, part);
  XB_CUDA(cudaGetLastError());
  return 0;
}

constexpr int PD_TX = 32, PD_TY = 8;

template <int CN>
__global__ void __launch_bounds__(PD_TX* PD_TY) pyrdown_kernel(uint8_t* __restrict__ pyr, unsigned long long pyr_stride,
                                                                const unsigned long long* __restrict__ seq_off, PyrDesc d,
                                                                int lvl_src, const uint8_t* const* __restrict__ frame0) {
  const int srows = d.rows[lvl_src], scols = d.cols[lvl_src];
  const int drows = d.rows[lvl_src + 1], dcols = d.cols[lvl_src + 1];
  const unsigned long long soff = seq_off ? seq_off[blockIdx.z] : (unsigned long long)blockIdx.z * pyr_stride;
  if (soff == ~0ull) return;  // inactive sequence
  // frame0 (level 0 only): the new frame still lives outside the pyramid (the estimator's frame ring); this
  // pass then also writes the level-0 copy from its staged tile, so the frame is read once instead of being
  // copied into place first
  const bool ingest = frame0 != nullptr && lvl_src == 0;
  const uint8_t* __restrict__ src = ingest ? frame0[blockIdx.z] : pyr + soff + d.off[lvl_src];
  uint8_t* __restrict__ dst = pyr + soff + d.off[lvl_src + 1];
  constexpr int RW = 2 * PD_TX + 3, RH = 2 * PD_TY + 3;
  __shared__ uint8_t tile[RH][RW * CN + 1];
  __shared__ unsigned short hsum[RH][PD_TX * CN];
  const int ox = blockIdx.x * PD_TX, oy = blockIdx.y * PD_TY;
  const int tid = threadIdx.y * PD_TX + threadIdx.x;
  const int sx0 = 2 * ox - 2, sy0 = 2 * oy - 2;
  for (int i = tid; i < RH * RW; i += PD_TX * PD_TY) {
    int ry = i / RW, rx = i - ry * RW;
    int sy = reflect101(sy0 + ry, srows), sx = reflect101(sx0 + rx, scols);
    const uint8_t* p = src + ((size_t)sy * scols + sx) * CN;
#pragma unroll
    for (int c = 0; c < CN; ++c) tile[ry][rx * CN + c] = p[c];
  }
  __syncthreads();
  if (ingest) {  // interior of the staged region = this CTA's 2 PD_TX x 2 PD_TY block of level 0
    uint8_t* __restrict__ l0 = pyr + soff + d.off[0];
    for (int i = tid; i < 2 * PD_TY * 2 * PD_TX * CN; i += PD_TX * PD_TY) {
      const int ry = i / (2 * PD_TX * CN), r = i - ry * (2 * PD_TX * CN);
      const int gy = 2 * oy + ry, gx = 2 * ox + r / CN;
      if (gy < srows && gx < scols) l0[((size_t)gy * scols + 2 * ox) * CN + r] = tile[ry + 2][2 * CN + r];
    }
  }
  // horizontal pass for all RH rows
  for (int i = tid; i < RH * PD_TX * CN; i += PD_TX * PD_TY) {
    int ry = i / (PD_TX * CN), r = i - ry * (PD_TX * CN);
    int x = r / CN, c = r - x * CN;
    const uint8_t* t = &tile[ry][(2 * x) * CN + c];
    int s = t[0] + t[4 * CN] + 4 * (t[CN] + t[3 * CN]) + 6 * t[2 * CN];
    hsum[ry][r] = (unsigned short)s;
  }
  __syncthreads();
  const int x = ox + threadIdx.x, y = oy + threadIdx.y;
  if (x < dcols && y < drows) {
#pragma unroll
    for (int c = 0; c < CN; ++c) {
      int r = threadIdx.x * CN + c, ry = 2 * threadIdx.y;
      int s = hsum[ry][r] + hsum[ry + 4][r] + 4 * (hsum[ry + 1][r] + hsum[ry + 3][r]) + 6 * hsum[ry + 2][r];
      dst[((size_t)y * dcols + x) * CN + c] = (uint8_t)((s + 128) >> 8);
    }
  }
}

// XIVO_PYRDOWN_GENERIC=1 routes single-channel levels through the byte-wise kernel (parity tests compare the two)
static bool force_generic_pyrdown() {
  const char* e = getenv("XIVO_PYRDOWN_GENERIC");
  return e && e[0] == '1';
}

// Single-channel fast path (cols of the source level a multiple of 4).  A CTA produces a 64 x 32 output tile:
// the (2*64+8) x (2*32+3) source region is staged as 32-bit words (byte-wise with REFLECT_101 only for words
// that touch the image border), a thread owns 2 x 4 outputs, forms the horizontal [1 4 6 4 1] sums of its
// 11 source rows with byte-permute + dp4a, and combines them vertically in registers.  ~35 thread
// instructions per output pixel instead of ~400 for the byte-wise kernel above; same integers.
constexpr int PV_TX = 64, PV_TY = 32, PV_THREADS = 256;
constexpr int PV_WORDS = (2 * PV_TX + 8) / 4;  // 34 words: source columns [2 ox - 4, 2 ox + 132)
constexpr int PV_ROWS = 2 * PV_TY + 3;         // 67 rows:  source rows    [2 oy - 2, 2 oy + 65)
__global__ void __launch_bounds__(PV_THREADS) pyrdown_vec_kernel(uint8_t* __restrict__ pyr, unsigned long long pyr_stride,
                                                                 const unsigned long long* __restrict__ seq_off, PyrDesc d, int lvl_src,
                                                                 const uint8_t* const* __restrict__ frame0) {
  const int srows = d.rows[lvl_src], scols = d.cols[lvl_src];
  const int drows = d.rows[lvl_src + 1], dcols = d.cols[lvl_src + 1];
  const unsigned long long soff = seq_off ? seq_off[blockIdx.z] : (unsigned long long)blockIdx.z * pyr_stride;
  if (soff == ~0ull) return;  // inactive sequence
  const bool ingest = frame0 != nullptr && lvl_src == 0;
  const uint8_t* __restrict__ src = ingest ? frame0[blockIdx.z] : pyr + soff + d.off[lvl_src];
  uint8_t* __restrict__ dst = pyr + soff + d.off[lvl_src + 1];
  __shared__ unsigned tile[PV_ROWS][PV_WORDS + 1];
  const int ox = blockIdx.x * PV_TX, oy = blockIdx.y * PV_TY;
  const int tid = threadIdx.x;
  const int sx0 = 2 * ox - 4, sy0 = 2 * oy - 2;
  const bool aligned = (reinterpret_cast<uintptr_t>(src) & 3) == 0;
  for (int i = tid; i < PV_ROWS * PV_WORDS; i += PV_THREADS) {
    const int ry = i / PV_WORDS, rw = i - ry * PV_WORDS;
    const int sx = sx0 + 4 * rw;
    if (sx >= scols + 4 || sy0 + ry >= srows + 4) { tile[ry][rw] = 0; continue; }  // feeds no valid output
    const int sy = reflect101(sy0 + ry, srows);
    const uint8_t* row = src + (size_t)sy * scols;
    unsigned w;
    if (aligned && sx >= 0 && sx + 3 < scols) {
      w = *reinterpret_cast<const unsigned*>(row + sx);
    } else {
      w = (unsigned)row[reflect101(sx, scols)] | ((unsigned)row[reflect101(sx + 1, scols)] << 8) |
          ((unsigned)row[reflect101(sx + 2, scols)] << 16) | ((unsigned)row[reflect101(sx + 3, scols)] << 24);
    }
    tile[ry][rw] = w;
  }
  __syncthreads();
  if (ingest) {  // level-0 copy of this CTA's 128 x 64 source block (words 1..32 of rows 2..65)
    uint8_t* __restrict__ l0 = pyr + soff + d.off[0];
    const bool dal = ((reinterpret_cast<uintptr_t>(l0) | (size_t)scols) & 3) == 0;
    for (int i = tid; i < 2 * PV_TY * 2 * PV_TX / 4; i += PV_THREADS) {
      const int ry = i >> 5, rw = i & 31;
      const int gy = 2 * oy + ry, gx = 2 * ox + 4 * rw;
      if (gy >= srows || gx >= scols) continue;
      const unsigned w = tile[ry + 2][rw + 1];
      uint8_t* q = l0 + (size_t)gy * scols + gx;
      if (dal && gx + 3 < scols) *reinterpret_cast<unsigned*>(q) = w;
      else
        for (int k = 0; k < 4 && gx + k < scols; ++k) q[k] = (uint8_t)(w >> (8 * k));
    }
  }
  const int tx = tid & 31, ty = tid >> 5;  // outputs x = ox + 2 tx (+1), y = oy + 4 ty (+0..3)
  int h0[11], h1[11];
#pragma unroll
  for (int r = 0; r < 11; ++r) {
    const unsigned w0 = tile[8 * ty + r][tx], w1 = tile[8 * ty + r][tx + 1], w2 = tile[8 * ty + r][tx + 2];
    // source bytes (relative to word tx): output 0 uses bytes 2..6, output 1 bytes 4..8
    const unsigned a = __byte_perm(w0, w1, 0x5432);
    h0[r] = __dp4a(a, 0x04060401u, __dp4a(w1, 0x00010000u, 0u));
    h1[r] = __dp4a(w1, 0x04060401u, __dp4a(w2, 0x00000001u, 0u));
  }
  const int x = ox + 2 * tx;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int y = oy + 4 * ty + j;
    if (y >= drows || x >= dcols) continue;
    const int s0 = h0[2 * j] + h0[2 * j + 4] + 4 * (h0[2 * j + 1] + h0[2 * j + 3]) + 6 * h0[2 * j + 2];
    const int s1 = h1[2 * j] + h1[2 * j + 4] + 4 * (h1[2 * j + 1] + h1[2 * j + 3]) + 6 * h1[2 * j + 2];
    uint8_t* q = dst + (size_t)y * dcols + x;
    q[0] = (uint8_t)((s0 + 128) >> 8);
    if (x + 1 < dcols) q[1] = (uint8_t)((s1 + 128) >> 8);
  }
}

// TMA variant of the single-channel pass (source level with cols % 16 == 0, sources at a uniform stride: the frame ring or the
// pyramid buffer of a batch).  The (2*64+32) x (2*32+3) byte source box of a CTA arrives by ONE cp.async.bulk.tensor issued by one
// thread (3-D tensor map {cols, rows, image}; coordinates outside the image are zero-filled by the TMA unit), completion on an
// mbarrier: the ~540 thread instructions per CTA-thread that pyrdown_vec_kernel spends on addresses, border tests and word
// assembly disappear (ncu, round 2 start: 82 % issue-active at 7 % of DRAM peak).  BORDER_REFLECT_101 only concerns the CTAs on the
// image rim, which patch their halo rows / columns inside shared memory after the box has landed.  The arithmetic that follows is
// pyrdown_vec_kernel's (byte-permute + dp4a on the same words), so the output is bit-identical.
// Box geometry: the innermost start coordinate times the element size is kept a multiple of 16 bytes, while negative (aligned)
// coordinates and boxes that stick out of the tensor are fine.  So the box starts at column 2 ox - 16 and is 160 bytes wide.
constexpr int PT_LEAD = 16;                  // source column of tile byte 0 = 2 ox - PT_LEAD
constexpr int PT_BOXW = 2 * PV_TX + 32;      // 160 bytes: source columns [2 ox - 16, 2 ox + 144)
constexpr int PT_WORDS = PT_BOXW / 4;        // 40 words per staged row
constexpr int PT_W0 = (PT_LEAD - 4) / 4;     // tile word that holds source columns 2 ox - 4 .. 2 ox - 1 (word 0 of pyrdown_vec_kernel's tile)
constexpr int PT_BOX_BYTES = PT_BOXW * PV_ROWS;

__device__ __forceinline__ unsigned smem_addr_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(PV_THREADS) pyrdown_tma_kernel(const __grid_constant__ CUtensorMap src_map, const int* __restrict__ src_img,
                                                                 uint8_t* __restrict__ pyr, unsigned long long pyr_stride,
                                                                 const unsigned long long* __restrict__ seq_off, PyrDesc d, int lvl_src, int ingest) {
  const int srows = d.rows[lvl_src], scols = d.cols[lvl_src];
  const int drows = d.rows[lvl_src + 1], dcols = d.cols[lvl_src + 1];
  const unsigned long long soff = seq_off ? seq_off[blockIdx.z] : (unsigned long long)blockIdx.z * pyr_stride;
  if (soff == ~0ull) return;  // inactive sequence
  uint8_t* __restrict__ dst = pyr + soff + d.off[lvl_src + 1];
  __shared__ __align__(128) unsigned tile[PV_ROWS][PT_WORDS];
  __shared__ __align__(8) unsigned long long mbar;
  const int ox = blockIdx.x * PV_TX, oy = blockIdx.y * PV_TY;
  const int tid = threadIdx.x;
  const int sx0 = 2 * ox - PT_LEAD, sy0 = 2 * oy - 2;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr_u32(&mbar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid < 32) {  // warp-uniform branch, one elected lane issues (the canonical form: TMA is a warp-level instruction on a uniform path)
    const int z = src_img[blockIdx.z];
    unsigned leader = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(leader));
    if (leader) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(&mbar)), "r"(PT_BOX_BYTES) : "memory");
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                   ::"r"(smem_addr_u32(&tile[0][0])), "l"(reinterpret_cast<unsigned long long>(&src_map)), "r"(sx0), "r"(sy0), "r"(z),
                     "r"(smem_addr_u32(&mbar))
                   : "memory");
    }
  }
  {  // every thread waits for the box (phase 0 of the barrier)
    unsigned done = 0;
    while (!done) {
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_addr_u32(&mbar)) : "memory");
    }
  }
  // BORDER_REFLECT_101 for the rim CTAs (the TMA unit zero-filled what lies outside the image): columns first, then whole rows
  const bool rim_x = sx0 < 0 || sx0 + PT_BOXW > scols, rim_y = sy0 < 0 || sy0 + PV_ROWS > srows;
  if (rim_x) {
    uint8_t* tb = reinterpret_cast<uint8_t*>(&tile[0][0]);
    for (int i = tid; i < PV_ROWS * 8; i += PV_THREADS) {  // the 4 columns left of the image and the first 4 past its right edge
      const int ry = i >> 3, k = i & 7;
      const int sx = k < 4 ? k - 4 : scols + (k - 4);
      const int rx = sx - sx0;
      if (rx < 0 || rx >= PT_BOXW) continue;
      const int rsx = reflect101(sx, scols) - sx0;
      if (rsx >= 0 && rsx < PT_BOXW) tb[ry * PT_BOXW + rx] = tb[ry * PT_BOXW + rsx];
    }
    __syncthreads();
  }
  if (rim_y) {
    for (int i = tid; i < PV_ROWS * PT_WORDS; i += PV_THREADS) {
      const int ry = i / PT_WORDS, rw = i - ry * PT_WORDS;
      const int sy = sy0 + ry;
      if (sy >= 0 && sy < srows) continue;
      const int rsy = reflect101(sy, srows) - sy0;
      if (rsy >= 0 && rsy < PV_ROWS && sy < srows + 4) tile[ry][rw] = tile[rsy][rw];
    }
    __syncthreads();
  }
  if (ingest) {  // level-0 copy of this CTA's 128 x 64 source block (bytes 16 .. 143 of rows 2 .. 65), 16 bytes per store
    uint8_t* __restrict__ l0 = pyr + soff + d.off[0];
    for (int i = tid; i < 2 * PV_TY * (2 * PV_TX / 16); i += PV_THREADS) {
      const int ry = i >> 3, q = i & 7;
      const int gy = 2 * oy + ry, gx = 2 * ox + 16 * q;
      if (gy >= srows || gx >= scols) continue;
      const unsigned* t = &tile[ry + 2][PT_LEAD / 4 + 4 * q];
      *reinterpret_cast<uint4*>(l0 + (size_t)gy * scols + gx) = make_uint4(t[0], t[1], t[2], t[3]);  // cols % 16 == 0: whole chunks only
    }
  }
  const int tx = tid & 31, ty = tid >> 5;  // outputs x = ox + 2 tx (+1), y = oy + 4 ty (+0..3)
  int h0[11], h1[11];
#pragma unroll
  for (int r = 0; r < 11; ++r) {
    const unsigned w0 = tile[8 * ty + r][PT_W0 + tx], w1 = tile[8 * ty + r][PT_W0 + tx + 1], w2 = tile[8 * ty + r][PT_W0 + tx + 2];
    const unsigned a = __byte_perm(w0, w1, 0x5432);
    h0[r] = __dp4a(a, 0x04060401u, __dp4a(w1, 0x00010000u, 0u));
    h1[r] = __dp4a(w1, 0x04060401u, __dp4a(w2, 0x00000001u, 0u));
  }
  const int x = ox + 2 * tx;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int y = oy + 4 * ty + j;
    if (y >= drows || x >= dcols) continue;
    const int s0 = h0[2 * j] + h0[2 * j + 4] + 4 * (h0[2 * j + 1] + h0[2 * j + 3]) + 6 * h0[2 * j + 2];
    const int s1 = h1[2 * j] + h1[2 * j + 4] + 4 * (h1[2 * j + 1] + h1[2 * j + 3]) + 6 * h1[2 * j + 2];
    uint8_t* q = dst + (size_t)y * dcols + x;
    q[0] = (uint8_t)((s0 + 128) >> 8);
    if (x + 1 < dcols) q[1] = (uint8_t)((s1 + 128) >> 8);
  }
}

// Tensor map {cols, rows, n_img} over u8 images that lie `img_stride` bytes apart, box box_w x box_h x 1 (0 = the pyrDown box), zero fill.
// cuTensorMapEncodeTiled is fetched from the driver at run time (the library does not link libcuda).
int make_pyr_tensor_map(CUtensorMap* out, const uint8_t* base, int rows, int cols, unsigned long long img_stride, unsigned long long n_img, int box_w, int box_h) {
  if (box_w <= 0) box_w = PT_BOXW;
  if (box_h <= 0) box_h = PV_ROWS;
  XB_REQUIRE((box_w & 15) == 0 && box_w <= 256 && box_h <= 256, "tensor map: box width must be a multiple of 16 bytes, extents <= 256");
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    XB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    XB_REQUIRE(fn && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled is not available from this driver");
    encode = reinterpret_cast<EncodeFn>(fn);
  }
  XB_REQUIRE((cols & 15) == 0 && (img_stride & 15) == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0, "pyramid tensor map: 16-byte alignment");
  const cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)n_img};
  const cuuint64_t strides[2] = {(cuuint64_t)cols, (cuuint64_t)img_stride};  // bytes, dimensions 1 and 2
  const cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  XB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed");
  return 0;
}

// One pyrDown pass lvl -> lvl + 1 through the TMA kernel.  src_img (device): image index of every sequence inside the tensor map.
int launch_pyrdown_tma(cudaStream_t st, const CUtensorMap& map, const int* src_img, uint8_t* pyr, unsigned long long pyr_stride,
                       const unsigned long long* seq_off, const PyrDesc& d, int lvl, int ingest, int batch) {
  dim3 vgrid((d.cols[lvl + 1] + PV_TX - 1) / PV_TX, (d.rows[lvl + 1] + PV_TY - 1) / PV_TY, batch);
  pyrdown_tma_kernel<<<vgrid, PV_THREADS, 0, st>>>(map, src_img, pyr, pyr_stride, seq_off, d, lvl, ingest);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// one pass lvl -> lvl + 1 with the thread-staged kernels (any channel count / width)
int launch_pyrdown_level(cudaStream_t st, uint8_t* pyr, unsigned long long pyr_stride, const unsigned long long* seq_off, const PyrDesc& d,
                         int batch, const uint8_t* const* frame0, int l) {
  dim3 grid((d.cols[l + 1] + PD_TX - 1) / PD_TX, (d.rows[l + 1] + PD_TY - 1) / PD_TY, batch);
  dim3 block(PD_TX, PD_TY);
  if (d.cn == 1 && (d.cols[l] & 3) == 0 && !force_generic_pyrdown()) {
    dim3 vgrid((d.cols[l + 1] + PV_TX - 1) / PV_TX, (d.rows[l + 1] + PV_TY - 1) / PV_TY, batch);
    pyrdown_vec_kernel<<<vgrid, PV_THREADS, 0, st>>>(pyr, pyr_stride, seq_off, d, l, frame0);
  } else if (d.cn == 1) pyrdown_kernel<1><<<grid, block, 0, st>>>(pyr, pyr_stride, seq_off, d, l, frame0);
  else pyrdown_kernel<3><<<grid, block, 0, st>>>(pyr, pyr_stride, seq_off, d, l, frame0);
  XB_CUDA(cudaGetLastError());
  return 0;
}

int launch_build_pyramid(cudaStream_t st, uint8_t* pyr, unsigned long long pyr_stride, const unsigned long long* seq_off,
                         const PyrDesc& d, int batch, const uint8_t* const* frame0) {
  ProfScope ps("pyrdown", st);
  if (d.n_levels == 1 && frame0) {  // no pyrDown pass to ride on: plain gather copy into level 0
    if (int rc = launch_gather_frames(st, frame0, pyr, pyr_stride, seq_off, (size_t)d.rows[0] * d.cols[0] * d.cn, batch)) return rc;
  }
  for (int l = 0; l + 1 < d.n_levels; ++l)
    if (int rc = launch_pyrdown_level(st, pyr, pyr_stride, seq_off, d, batch, frame0, l)) return rc;
  return 0;
}

// ------------------------------------------------------------------------------------------
// FAST-9/16 + cornerScore + 3x3 non-max suppression (cv::FastFeatureDetector, TYPE_9_16).
// One CTA = 64x16 output pixels.  Stage (64+12)x(16+8) grey pixels (ring radius 3 + NMS 1,
// pair-aligned columns), compute the score on (64+4)x(16+2), suppress, append packed keypoints
// with an atomic cursor.  For 3-channel input the BGR->grey fixed-point conversion (cv2 4.13
// 15-bit coefficients) is fused into the tile load, so the image is read exactly once from HBM.
// Output: packed (y<<20 | x<<8 | score); order is arbitrary (host sorts on the composite key).
// ------------------------------------------------------------------------------------------
constexpr int FT_TX = 64, FT_TY = 16, FT_THREADS = 256;
constexpr int FT_RH = FT_TY + 8;  // pixel region rows
constexpr int FT_SH = FT_TY + 2;  // score region rows

// A thread scores two horizontally adjacent pixels at once.  The grey tile is kept as 16-bit values so a pixel
// pair is one 32-bit word; ring values of the pair are word loads (even column offsets) or a byte-permute of two
// words (odd offsets); all min/max run on s16x2 pairs (3-input where it helps).  No compass pre-test and no arc
// bit-mask: the corner decision is "best > thr" on the cornerScore value, which is what the 9-arc test evaluates
// (the C oracle, oracle/tracker_oracle.c, decides the same way).  ~70 thread instructions per pixel on textured
// frames instead of ~400 for one pixel per thread with the arc test.
constexpr int FP_SW = FT_TX + 4;          // score region width (pairs aligned): image x = ox - 2 + sx
constexpr int FP_RW = FT_TX + 12;         // tile width: image x = ox - 6 + rx (even origin, ring radius 3 on both sides)
__device__ __forceinline__ unsigned pk_min(unsigned a, unsigned b) { return __vmins2(a, b); }
__device__ __forceinline__ unsigned pk_max(unsigned a, unsigned b) { return __vmaxs2(a, b); }
__device__ __forceinline__ unsigned pk_min3(unsigned a, unsigned b, unsigned c) { return __vimin3_s16x2(a, b, c); }
__device__ __forceinline__ unsigned pk_max3(unsigned a, unsigned b, unsigned c) { return __vimax3_s16x2(a, b, c); }

// scores + NMS + keypoint append of one 64 x 16 tile whose grey values are staged as 16-bit pixels (shared by the thread-staged and the TMA kernel)
__device__ __forceinline__ void fast_pair_tile(const unsigned short (*tile)[FP_RW], short (*score)[FP_SW], int ox, int oy, int rows, int cols, int thr,
                                               int nonmax, unsigned* __restrict__ kp_out, int max_kp, int* __restrict__ kp_count) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  // pair (sx, sx + 1), sx even: image x = ox - 2 + sx, tile column rx = sx + 4; score row sy: image y = oy - 1 + sy, tile row sy + 3
  for (int t = threadIdx.x; t < FT_SH * (FP_SW / 2); t += FT_THREADS) {
    const int sy = t / (FP_SW / 2), sx = 2 * (t - sy * (FP_SW / 2));
    const int gy = oy - 1 + sy, gx = ox - 2 + sx;
    unsigned out = 0;
    if (gy >= 3 && gy < rows - 3 && gx + 1 >= 3 && gx < cols - 3) {
      const int ry = sy + 3, rx = sx + 4;
      auto W = [&](int dy, int dx) -> unsigned { return *reinterpret_cast<const unsigned*>(&tile[ry + dy][rx + dx]); };  // dx even
      // words of each ring row: columns rx-4 .. rx+5 as needed
      unsigned p[16];
      {
        const unsigned a = W(3, -2), b = W(3, 0), c = W(3, 2);
        p[15] = __byte_perm(a, b, 0x5432); p[0] = b; p[1] = __byte_perm(b, c, 0x5432);
      }
      p[14] = W(2, -2); p[2] = W(2, 2);
      {
        const unsigned a = W(1, -4), b = W(1, -2), c = W(1, 2), d2 = W(1, 4);
        p[13] = __byte_perm(a, b, 0x5432); p[3] = __byte_perm(c, d2, 0x5432);
      }
      unsigned vv;
      {
        const unsigned a = W(0, -4), b = W(0, -2), c = W(0, 2), d2 = W(0, 4);
        p[12] = __byte_perm(a, b, 0x5432); p[4] = __byte_perm(c, d2, 0x5432);
        vv = W(0, 0);
      }
      {
        const unsigned a = W(-1, -4), b = W(-1, -2), c = W(-1, 2), d2 = W(-1, 4);
        p[11] = __byte_perm(a, b, 0x5432); p[5] = __byte_perm(c, d2, 0x5432);
      }
      p[10] = W(-2, -2); p[6] = W(-2, 2);
      {
        const unsigned a = W(-3, -2), b = W(-3, 0), c = W(-3, 2);
        p[9] = __byte_perm(a, b, 0x5432); p[8] = b; p[7] = __byte_perm(b, c, 0x5432);
      }
      // min / max over the 16 circular 9-arcs: windows of 3, then 3 + 3 + 3
      unsigned n3[16], x3[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        n3[k] = pk_min3(p[k], p[(k + 1) & 15], p[(k + 2) & 15]);
        x3[k] = pk_max3(p[k], p[(k + 1) & 15], p[(k + 2) & 15]);
      }
      unsigned arc_min_max = 0u, arc_max_min = 0x00ff00ffu;
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const unsigned a_mn = pk_min3(n3[k], n3[(k + 3) & 15], n3[(k + 6) & 15]);
        const unsigned a_mx = pk_max3(x3[k], x3[(k + 3) & 15], x3[(k + 6) & 15]);
        arc_min_max = pk_max(arc_min_max, a_mn);
        arc_max_min = pk_min(arc_max_min, a_mx);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int x = gx + h;
        const int v = (vv >> (16 * h)) & 0xffff;
        const int dark = v - (int)((arc_max_min >> (16 * h)) & 0xffff), bright = (int)((arc_min_max >> (16 * h)) & 0xffff) - v;
        const int best = dark > bright ? dark : bright;
        const int sc = (best > thr && x >= 3 && x < cols - 3) ? best - 1 : 0;
        out |= (unsigned)(sc & 0xffff) << (16 * h);
      }
    }
    *reinterpret_cast<unsigned*>(&score[sy][sx]) = out;
  }
  __syncthreads();
  for (int py = ty; py < FT_TY; py += 8) {
    const int gy = oy + py;
    for (int px = tx; px < FT_TX; px += 32) {
      const int gx = ox + px;
      if (gx >= cols || gy >= rows) continue;
      const int cx = px + 2, cy = py + 1;
      const int s = score[cy][cx];
      if (s <= 0) continue;
      bool keep = true;
      if (nonmax) {
        keep = s > score[cy - 1][cx - 1] && s > score[cy - 1][cx] && s > score[cy - 1][cx + 1] && s > score[cy][cx - 1] &&
               s > score[cy][cx + 1] && s > score[cy + 1][cx - 1] && s > score[cy + 1][cx] && s > score[cy + 1][cx + 1];
      }
      if (keep) {
        const int idx = atomicAdd(&kp_count[blockIdx.z], 1);
        if (idx < max_kp) kp_out[(size_t)blockIdx.z * max_kp + idx] = ((unsigned)gy << 20) | ((unsigned)gx << 8) | (unsigned)s;
      }
    }
  }
}

template <int CN>
__global__ void __launch_bounds__(FT_THREADS) fast_pair_kernel(const uint8_t* __restrict__ img, unsigned long long img_stride,
                                                               const unsigned long long* __restrict__ seq_off, int rows, int cols,
                                                               int thr, int nonmax, unsigned* __restrict__ kp_out, int max_kp,
                                                               int* __restrict__ kp_count, const int* __restrict__ need) {
  __shared__ __align__(8) unsigned short tile[FT_RH][FP_RW];
  __shared__ short score[FT_SH][FP_SW];
  const unsigned long long soff = seq_off ? seq_off[blockIdx.z] : (unsigned long long)blockIdx.z * img_stride;
  if (soff == ~0ull) return;  // inactive sequence
  if (need && need[blockIdx.z] <= 0) return;
  const uint8_t* __restrict__ src = img + soff;
  const int ox = blockIdx.x * FT_TX, oy = blockIdx.y * FT_TY;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int gx0 = ox - 6, gy0 = oy - 4;
  for (int ry = ty; ry < FT_RH; ry += 8) {
    const int gy = gy0 + ry;
    for (int rx = tx; rx < FP_RW; rx += 32) {
      const int gx = gx0 + rx;
      int val = 0;
      if (gx >= 0 && gx < cols && gy >= 0 && gy < rows) {
        const uint8_t* p = src + ((size_t)gy * cols + gx) * CN;
        if (CN == 1) val = p[0];
        else val = (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15;
      }
      tile[ry][rx] = (unsigned short)val;
    }
  }
  __syncthreads();
  fast_pair_tile(tile, score, ox, oy, rows, cols, thr, nonmax, kp_out, max_kp, kp_count);
}

// TMA variant (single channel, cols % 16 == 0, images at a uniform stride inside one buffer: the level-0 images of a batch's pyramids).
// The 96 x 24 byte box [ox - 16, ox + 80) x [oy - 4, oy + 20) of a CTA arrives by one cp.async.bulk.tensor; what lies outside the image
// is zero-filled by the TMA unit, which is exactly the value the thread-staged kernel stores there (FAST never scores a pixel closer
// than 3 to the border, so the fill value is never compared).  The bytes are then widened to the 16-bit tile the packed scoring works
// on; everything after that is fast_pair_tile, so the keypoints are identical.
constexpr int FTM_BOXW = 96, FTM_LEAD = 16;  // tile byte 0 = image column ox - 16 (16-byte aligned start)
__global__ void __launch_bounds__(FT_THREADS) fast_pair_tma_kernel(const __grid_constant__ CUtensorMap img_map, unsigned long long img_stride,
                                                                   const unsigned long long* __restrict__ seq_off, int rows, int cols, int thr,
                                                                   int nonmax, unsigned* __restrict__ kp_out, int max_kp, int* __restrict__ kp_count,
                                                                   const int* __restrict__ need) {
  __shared__ __align__(128) uint8_t box[FT_RH][FTM_BOXW];
  __shared__ __align__(8) unsigned short tile[FT_RH][FP_RW];
  __shared__ short score[FT_SH][FP_SW];
  __shared__ __align__(8) unsigned long long mbar;
  const unsigned long long soff = seq_off ? seq_off[blockIdx.z] : (unsigned long long)blockIdx.z * img_stride;
  if (soff == ~0ull) return;  // inactive sequence
  if (need && need[blockIdx.z] <= 0) return;
  const int ox = blockIdx.x * FT_TX, oy = blockIdx.y * FT_TY;
  const int tid = threadIdx.x;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr_u32(&mbar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid < 32) {
    const int z = (int)(soff / img_stride);  // image index of this sequence's level 0 inside the map
    unsigned leader = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(leader));
    if (leader) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr_u32(&mbar)), "r"(FT_RH * FTM_BOXW) : "memory");
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                   ::"r"(smem_addr_u32(&box[0][0])), "l"(reinterpret_cast<unsigned long long>(&img_map)), "r"(ox - FTM_LEAD), "r"(oy - 4), "r"(z),
                     "r"(smem_addr_u32(&mbar))
                   : "memory");
    }
  }
  {
    unsigned done = 0;
    while (!done) {
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_addr_u32(&mbar)) : "memory");
    }
  }
  // widen: tile column rx (image x = ox - 6 + rx) = box byte rx + 10; two pixels per 32-bit store
  for (int i = tid; i < FT_RH * (FP_RW / 2); i += FT_THREADS) {
    const int ry = i / (FP_RW / 2), rp = i - ry * (FP_RW / 2);
    const unsigned two = *reinterpret_cast<const unsigned short*>(&box[ry][2 * rp + FTM_LEAD - 6]);
    *reinterpret_cast<unsigned*>(&tile[ry][2 * rp]) = __byte_perm(two, 0u, 0x4140);
  }
  __syncthreads();
  fast_pair_tile(tile, score, ox, oy, rows, cols, thr, nonmax, kp_out, max_kp, kp_count);
}

int make_fast_tensor_map(CUtensorMap* out, const uint8_t* base, int rows, int cols, unsigned long long img_stride, unsigned long long n_img) {
  return make_pyr_tensor_map(out, base, rows, cols, img_stride, n_img, FTM_BOXW, FT_RH);
}

int launch_fast_detect(cudaStream_t st, const uint8_t* img, unsigned long long img_stride, const unsigned long long* seq_off,
                       int rows, int cols, int cn, int thr, int nonmax, unsigned* kp_out, int max_kp, int* kp_count, int batch, const int* need,
                       const CUtensorMap* tma_map, unsigned long long tma_img_stride, bool count_is_zero) {
  XB_REQUIRE(rows < 4096 && cols < 4096, "FAST: image dimension must be < 4096 (12-bit packed coordinates)");
  XB_REQUIRE(thr >= 0 && thr < 255, "FAST: threshold out of range");
  if (!count_is_zero) XB_CUDA(cudaMemsetAsync(kp_count, 0, sizeof(int) * batch, st));
  ProfScope ps("fast_detect", st);
  dim3 grid((cols + FT_TX - 1) / FT_TX, (rows + FT_TY - 1) / FT_TY, batch);
  if (tma_map && cn == 1 && tma_img_stride) {
    fast_pair_tma_kernel<<<grid, FT_THREADS, 0, st>>>(*tma_map, tma_img_stride, seq_off, rows, cols, thr, nonmax, kp_out, max_kp, kp_count, need);
  } else {
    if (cn == 1) fast_pair_kernel<1><<<grid, FT_THREADS, 0, st>>>(img, img_stride, seq_off, rows, cols, thr, nonmax, kp_out, max_kp, kp_count, need);
    else fast_pair_kernel<3><<<grid, FT_THREADS, 0, st>>>(img, img_stride, seq_off, rows, cols, thr, nonmax, kp_out, max_kp, kp_count, need);
  }
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Pyramidal Lucas-Kanade (cv::calcOpticalFlowPyrLK / LKTrackerInvoker restated).
// One warp per feature walks the levels coarse -> fine.  Per level the warp stages the
// (win+3)^2 patch of the previous image in shared memory, derives the Scharr gradients from it
// (OpenCV materialises them; we never write them to HBM), builds the fixed-point template
// (14-bit bilinear weights, 5 guard bits) and iterates; window sums are exact integers reduced
// with warp shuffles, then converted to float once (OpenCV sums float SIMD lanes; the integer
// sum is the value those floats approximate).
// ------------------------------------------------------------------------------------------
constexpr int LK_WARPS = 4;
constexpr int LK_MAX_WIN = 21;

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
// Exact warp sum of per-lane int32 partials (the total may need 37 bits): the 16-bit halves are reduced separately with the
// hardware warp reduction (redux.sync, 2 instructions) instead of 5 shuffle + 64-bit add rounds; v = (v >> 16) * 65536 + (v & 0xffff).
__device__ __forceinline__ long long warp_sum_i32_exact(int v) {
  const int slo = __reduce_add_sync(0xffffffffu, v & 0xffff);
  const int shi = __reduce_add_sync(0xffffffffu, v >> 16);
  return ((long long)shi << 16) + slo;
}

struct LKParams {
  int win, max_iter, use_initial_flow, max_pts;
  float eps_sq_f;  // unused (double compare below)
  double eps_sq, min_eig;
};

template <int CN>
__global__ void __launch_bounds__(LK_WARPS * 32) lk_kernel(const uint8_t* __restrict__ prev_pyr, const uint8_t* __restrict__ next_pyr,
                                                          unsigned long long pyr_stride,
                                                          const unsigned long long* __restrict__ prev_off,
                                                          const unsigned long long* __restrict__ next_off, PyrDesc d,
                                                          const float* __restrict__ prev_pts, float* __restrict__ next_pts,
                                                          uint8_t* __restrict__ status, float* __restrict__ err,
                                                          const int* __restrict__ npts, LKParams prm) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seq = blockIdx.y;
  const int p = blockIdx.x * LK_WARPS + warp;
  if (p >= npts[seq]) return;  // whole warp exits together
  const int win = prm.win;
  const int RW = win + 3;  // staged region side (patch + bilinear + Scharr halo)
  const int DW = win + 1;  // derivative tile side
  // per-warp shared memory carve-up
  const int reg_bytes = ((RW * RW * CN + 15) / 16) * 16;
  const int dt_elems = DW * DW * CN * 2;
  const int iw_elems = win * win * CN;
  const int per_warp = reg_bytes + 2 * (dt_elems + iw_elems * 3);
  uint8_t* region = smem_raw + (size_t)warp * (((per_warp + 15) / 16) * 16);
  short* dtile = reinterpret_cast<short*>(region + reg_bytes);
  short* Iw = dtile + dt_elems;
  short* dIw = Iw + iw_elems;

  const uint8_t* __restrict__ ppyr = prev_pyr + (prev_off ? prev_off[seq] : (unsigned long long)seq * pyr_stride);
  const uint8_t* __restrict__ npyr = next_pyr + (next_off ? next_off[seq] : (unsigned long long)seq * pyr_stride);
  const size_t pi = (size_t)seq * prm.max_pts + p;
  const float ppx = prev_pts[2 * pi], ppy = prev_pts[2 * pi + 1];
  float outx = next_pts[2 * pi], outy = next_pts[2 * pi + 1];
  int st = 1;
  float errv = 0.f;
  const float half = (win - 1) * 0.5f;
  const float FLT_SCALE = 1.f / (1 << 20);
  const int max_level = d.n_levels - 1;

  for (int level = max_level; level >= 0; --level) {
    const int rows = d.rows[level], cols = d.cols[level];
    const uint8_t* __restrict__ I = ppyr + d.off[level];
    const uint8_t* __restrict__ J = npyr + d.off[level];
    const float scale = (float)(1. / (1 << level));
    float px = ppx * scale, py = ppy * scale;
    float nx, ny;
    if (level == max_level) {
      if (prm.use_initial_flow) { nx = outx * scale; ny = outy * scale; }
      else { nx = px; ny = py; }
    } else {
      nx = outx * 2.f;
      ny = outy * 2.f;
    }
    outx = nx;
    outy = ny;
    px -= half;
    py -= half;
    const int ipx = (int)floorf(px), ipy = (int)floorf(py);
    if (ipx < -win || ipx >= cols || ipy < -win || ipy >= rows) {
      if (level == 0) { st = 0; errv = 0.f; }
      continue;
    }
    float a = px - ipx, b = py - ipy;
    int iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    int iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
    int iw10 = __float2int_rn((1.f - a) * b * 16384.f);
    int iw11 = 16384 - iw00 - iw01 - iw10;

    __syncwarp();
    // stage region: origin (ipx-1, ipy-1), REFLECT_101 == reads of OpenCV's padded level
    for (int i = lane; i < RW * RW; i += 32) {
      int ry = i / RW, rx = i - ry * RW;
      int sy = reflect101(ipy - 1 + ry, rows), sx = reflect101(ipx - 1 + rx, cols);
      const uint8_t* q = I + ((size_t)sy * cols + sx) * CN;
#pragma unroll
      for (int c = 0; c < CN; ++c) region[i * CN + c] = q[c];
    }
    __syncwarp();
    // Scharr derivatives on the (win+1)^2 grid; zero outside the image (BORDER_CONSTANT)
    for (int i = lane; i < DW * DW; i += 32) {
      int ty = i / DW, tx = i - ty * DW;
      int X = ipx + tx, Y = ipy + ty;
      bool inside = (X >= 0 && X < cols && Y >= 0 && Y < rows);
      const uint8_t* r0 = region + ((ty)*RW + tx) * CN;  // row Y-1, col X-1
      const uint8_t* r1 = r0 + RW * CN;
      const uint8_t* r2 = r1 + RW * CN;
#pragma unroll
      for (int c = 0; c < CN; ++c) {
        int dx = 0, dy = 0;
        if (inside) {
          int t0l = (r0[c] + r2[c]) * 3 + r1[c] * 10;
          int t0r = (r0[2 * CN + c] + r2[2 * CN + c]) * 3 + r1[2 * CN + c] * 10;
          int t1l = r2[c] - r0[c], t1c = r2[CN + c] - r0[CN + c], t1r = r2[2 * CN + c] - r0[2 * CN + c];
          dx = t0r - t0l;
          dy = (t1r + t1l) * 3 + t1c * 10;
        }
        dtile[(i * CN + c) * 2] = (short)dx;
        dtile[(i * CN + c) * 2 + 1] = (short)dy;
      }
    }
    __syncwarp();
    // template + structure tensor
    int sA11 = 0, sA12 = 0, sA22 = 0;  // per-lane partials fit int32 (<= 22 terms of < 1.7e7)
    long long lA11 = 0, lA12 = 0, lA22 = 0;
    for (int i = lane; i < win * win; i += 32) {
      int y = i / win, x = i - y * win;
      const uint8_t* q = region + ((y + 1) * RW + (x + 1)) * CN;
      const short* dq = dtile + (y * DW + x) * CN * 2;
#pragma unroll
      for (int c = 0; c < CN; ++c) {
        int ival = descale(q[c] * iw00 + q[CN + c] * iw01 + q[RW * CN + c] * iw10 + q[RW * CN + CN + c] * iw11, 9);
        int ix = descale(dq[2 * c] * iw00 + dq[2 * (CN + c)] * iw01 + dq[2 * (DW * CN + c)] * iw10 + dq[2 * (DW * CN + CN + c)] * iw11, 14);
        int iy = descale(dq[2 * c + 1] * iw00 + dq[2 * (CN + c) + 1] * iw01 + dq[2 * (DW * CN + c) + 1] * iw10 +
                             dq[2 * (DW * CN + CN + c) + 1] * iw11,
                         14);
        Iw[i * CN + c] = (short)ival;
        dIw[(i * CN + c) * 2] = (short)ix;
        dIw[(i * CN + c) * 2 + 1] = (short)iy;
        sA11 += ix * ix;
        sA12 += ix * iy;
        sA22 += iy * iy;
      }
      // flush partials every sample group to stay inside int32 for any CN/win
      lA11 += sA11; lA12 += sA12; lA22 += sA22;
      sA11 = sA12 = sA22 = 0;
    }
    lA11 = warp_sum_ll(lA11);
    lA12 = warp_sum_ll(lA12);
    lA22 = warp_sum_ll(lA22);
    __syncwarp();
    const float A11 = __ll2float_rn(lA11) * FLT_SCALE, A12 = __ll2float_rn(lA12) * FLT_SCALE, A22 = __ll2float_rn(lA22) * FLT_SCALE;
    float D = A11 * A22 - A12 * A12;
    const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * win * win);
    if ((double)minEig < prm.min_eig || D < 1.1920928955078125e-7f) {
      if (level == 0) st = 0;
      continue;
    }
    D = 1.f / D;
    nx -= half;
    ny -= half;
    float pdx = 0.f, pdy = 0.f;
    for (int j = 0; j < prm.max_iter; ++j) {
      const int inx = (int)floorf(nx), iny = (int)floorf(ny);
      if (inx < -win || inx >= cols || iny < -win || iny >= rows) {
        if (level == 0) st = 0;
        break;
      }
      a = nx - inx;
      b = ny - iny;
      iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
      iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
      iw10 = __float2int_rn((1.f - a) * b * 16384.f);
      iw11 = 16384 - iw00 - iw01 - iw10;
      const bool interior = (inx >= 0 && iny >= 0 && inx + win < cols && iny + win < rows);
      long long lb1 = 0, lb2 = 0;
      for (int i = lane; i < win * win; i += 32) {
        int y = i / win, x = i - y * win;
        int X0 = inx + x, X1 = X0 + 1, Y0 = iny + y, Y1 = Y0 + 1;
        if (!interior) {
          X0 = reflect101(X0, cols); X1 = reflect101(X1, cols);
          Y0 = reflect101(Y0, rows); Y1 = reflect101(Y1, rows);
        }
        const uint8_t* q00 = J + ((size_t)Y0 * cols + X0) * CN;
        const uint8_t* q01 = J + ((size_t)Y0 * cols + X1) * CN;
        const uint8_t* q10 = J + ((size_t)Y1 * cols + X0) * CN;
        const uint8_t* q11 = J + ((size_t)Y1 * cols + X1) * CN;
        int s1 = 0, s2 = 0;
#pragma unroll
        for (int c = 0; c < CN; ++c) {
          int diff = descale(__ldg(q00 + c) * iw00 + __ldg(q01 + c) * iw01 + __ldg(q10 + c) * iw10 + __ldg(q11 + c) * iw11, 9) -
                     Iw[i * CN + c];
          s1 += diff * dIw[(i * CN + c) * 2];
          s2 += diff * dIw[(i * CN + c) * 2 + 1];
        }
        lb1 += s1;
        lb2 += s2;
      }
      lb1 = warp_sum_ll(lb1);
      lb2 = warp_sum_ll(lb2);
      const float b1 = __ll2float_rn(lb1) * FLT_SCALE, b2 = __ll2float_rn(lb2) * FLT_SCALE;
      const float dx = (A12 * b2 - A22 * b1) * D;
      const float dy = (A12 * b1 - A11 * b2) * D;
      nx += dx;
      ny += dy;
      outx = nx + half;
      outy = ny + half;
      if ((double)dx * dx + (double)dy * dy <= prm.eps_sq) break;
      if (j > 0 && fabs((double)(dx + pdx)) < 0.01 && fabs((double)(dy + pdy)) < 0.01) {
        outx -= dx * 0.5f;
        outy -= dy * 0.5f;
        break;
      }
      pdx = dx;
      pdy = dy;
    }
    if (st && level == 0) {
      // default-flags error measure: mean |J - I| over the window / 32 (lkpyramid.cpp tail)
      const float fx = outx - half, fy = outy - half;
      const int inx = (int)floorf(fx), iny = (int)floorf(fy);
      if (inx < -win || inx >= cols || iny < -win || iny >= rows) {
        st = 0;
        continue;
      }
      const float aa = fx - inx, bb = fy - iny;
      iw00 = __float2int_rn((1.f - aa) * (1.f - bb) * 16384.f);
      iw01 = __float2int_rn(aa * (1.f - bb) * 16384.f);
      iw10 = __float2int_rn((1.f - aa) * bb * 16384.f);
      iw11 = 16384 - iw00 - iw01 - iw10;
      long long le = 0;
      for (int i = lane; i < win * win; i += 32) {
        int y = i / win, x = i - y * win;
        int X0 = reflect101(inx + x, cols), X1 = reflect101(inx + x + 1, cols);
        int Y0 = reflect101(iny + y, rows), Y1 = reflect101(iny + y + 1, rows);
#pragma unroll
        for (int c = 0; c < CN; ++c) {
          int diff = descale(J[((size_t)Y0 * cols + X0) * CN + c] * iw00 + J[((size_t)Y0 * cols + X1) * CN + c] * iw01 +
                                 J[((size_t)Y1 * cols + X0) * CN + c] * iw10 + J[((size_t)Y1 * cols + X1) * CN + c] * iw11,
                             9) -
                     Iw[i * CN + c];
          le += abs(diff);
        }
      }
      le = warp_sum_ll(le);
      errv = __ll2float_rn(le) * 1.f / (float)(32 * win * CN * win);
    }
  }
  if (lane == 0) {
    next_pts[2 * pi] = outx;
    next_pts[2 * pi + 1] = outy;
    status[pi] = (uint8_t)st;
    if (err) err[pi] = errv;
  }
}

// Single-channel fast path for win <= 15.  Same arithmetic as lk_kernel<1> (every window sum is an exact
// integer, so the lane <-> pixel assignment is free): a half-warp spans one window row (16 columns,
// the 16th only feeds the bilinear neighbour), the two half-warps take consecutive rows, and a lane
// keeps its <= 8 template samples (I, Ix, Iy) in registers for the whole level.  Per iteration a lane
// loads 2 bytes per sample slot (rows y, y+1 of its column) and gets the x+1 neighbours by shuffle,
// instead of 4 loads + 3 shared-memory reads; no integer divisions remain in the loops.
// (6 CTAs of 4 warps per SM at 80 registers; a 64-register cap for 8 CTAs spills a few words.)
template <int WIN>
__global__ void __launch_bounds__(LK_WARPS * 32, 6) lk_kernel_fast(const uint8_t* __restrict__ prev_pyr, const uint8_t* __restrict__ next_pyr,
                                                               unsigned long long pyr_stride,
                                                               const unsigned long long* __restrict__ prev_off,
                                                               const unsigned long long* __restrict__ next_off, PyrDesc d,
                                                               const float* __restrict__ prev_pts, float* __restrict__ next_pts,
                                                               uint8_t* __restrict__ status, float* __restrict__ err,
                                                               const int* __restrict__ npts, LKParams prm) {
  static_assert(WIN >= 3 && WIN <= 15 && (WIN & 1), "fast LK path: odd window up to 15");
  constexpr int RW = WIN + 3, DW = WIN + 1, NS = (WIN + 1) / 2;
  constexpr int RPW = (RW + 3) / 4, RP = 4 * RPW;  // region row pitch: whole words (the interior staging path stores words)
  constexpr int REG_BYTES = ((RP * RW + 15) / 16) * 16;
  constexpr int PER_WARP = ((REG_BYTES + DW * DW * 2 * 2 + 15) / 16) * 16;
  __shared__ __align__(16) uint8_t smem_raw[LK_WARPS * PER_WARP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seq = blockIdx.y;
  const int p = blockIdx.x * LK_WARPS + warp;
  if (p >= npts[seq]) return;  // whole warp exits together
  uint8_t* region = smem_raw + warp * PER_WARP;
  short* dtile = reinterpret_cast<short*>(region + REG_BYTES);
  const int r = lane >> 4, c = lane & 15;
  const int cx = c < WIN ? c : WIN;  // column offset this lane loads (clamped: lanes past the window only feed neighbours)

  const uint8_t* __restrict__ ppyr = prev_pyr + (prev_off ? prev_off[seq] : (unsigned long long)seq * pyr_stride);
  const uint8_t* __restrict__ npyr = next_pyr + (next_off ? next_off[seq] : (unsigned long long)seq * pyr_stride);
  const size_t pi = (size_t)seq * prm.max_pts + p;
  const float ppx = prev_pts[2 * pi], ppy = prev_pts[2 * pi + 1];
  float outx = next_pts[2 * pi], outy = next_pts[2 * pi + 1];
  int st = 1;
  float errv = 0.f;
  const float half = (WIN - 1) * 0.5f;
  const float FLT_SCALE = 1.f / (1 << 20);
  const int max_level = d.n_levels - 1;

  for (int level = max_level; level >= 0; --level) {
    const int rows = d.rows[level], cols = d.cols[level];
    const uint8_t* __restrict__ I = ppyr + d.off[level];
    const uint8_t* __restrict__ J = npyr + d.off[level];
    const float scale = (float)(1. / (1 << level));
    float px = ppx * scale, py = ppy * scale;
    float nx, ny;
    if (level == max_level) {
      if (prm.use_initial_flow) { nx = outx * scale; ny = outy * scale; }
      else { nx = px; ny = py; }
    } else {
      nx = outx * 2.f;
      ny = outy * 2.f;
    }
    outx = nx;
    outy = ny;
    px -= half;
    py -= half;
    const int ipx = (int)floorf(px), ipy = (int)floorf(py);
    if (ipx < -WIN || ipx >= cols || ipy < -WIN || ipy >= rows) {
      if (level == 0) { st = 0; errv = 0.f; }
      continue;
    }
    float a = px - ipx, b = py - ipy;
    int iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
    int iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
    int iw10 = __float2int_rn((1.f - a) * b * 16384.f);
    int iw11 = 16384 - iw00 - iw01 - iw10;

    __syncwarp();
    // Is the whole (WIN+3)^2 region inside the level?  (Almost always: then no border rule applies and every derivative is inside.)
    const bool reg_interior = ipx >= 1 && ipy >= 1 && ipx + WIN + 1 < cols && ipy + WIN + 1 < rows;
    if (reg_interior) {
      // lane l < RW stages row l: the words that cover its RW bytes, funnel-shifted so that the row starts at byte 0 of its pitch
      if (lane < RW) {
        const uint8_t* a = I + (size_t)(ipy - 1 + lane) * cols + (ipx - 1);
        const unsigned sh = (unsigned)(reinterpret_cast<uintptr_t>(a) & 3);
        const unsigned* aw = reinterpret_cast<const unsigned*>(a - sh);
        unsigned w[RPW + 1];
#pragma unroll
        for (int j = 0; j < RPW; ++j) w[j] = __ldg(aw + j);
        w[RPW] = (sh + RW > 4 * RPW) ? __ldg(aw + RPW) : 0u;  // the last word is needed only when the shift pushes the row into it
        unsigned* rw_ = reinterpret_cast<unsigned*>(region) + lane * RPW;
#pragma unroll
        for (int j = 0; j < RPW; ++j) rw_[j] = __funnelshift_r(w[j], w[j + 1], 8 * sh);
      }
      __syncwarp();
      // Scharr on the (WIN+1)^2 grid, separable: lane x < RW walks down column x keeping three pixels, S = 3 a + 10 b + 3 c (vertical
      // smoothing) and D = c - a (vertical difference); dx = S[x+2] - S[x], dy = 3 D[x] + 10 D[x+1] + 3 D[x+2] come from shuffles.
      {
        const int x = lane < RW ? lane : RW - 1;
        int pa = region[x], pb = region[RP + x];
#pragma unroll
        for (int ty = 0; ty < DW; ++ty) {
          const int pc = region[(ty + 2) * RP + x];
          const int S = (pa + pc) * 3 + pb * 10, D = pc - pa;
          const int S2 = __shfl_down_sync(0xffffffffu, S, 2), D1 = __shfl_down_sync(0xffffffffu, D, 1), D2 = __shfl_down_sync(0xffffffffu, D, 2);
          const int dx = S2 - S, dy = (D2 + D) * 3 + D1 * 10;
          if (lane < DW) reinterpret_cast<unsigned*>(dtile)[ty * DW + lane] = ((unsigned)dx & 0xffffu) | ((unsigned)dy << 16);
          pa = pb;
          pb = pc;
        }
      }
    } else {
      // stage region: origin (ipx-1, ipy-1), REFLECT_101 == reads of OpenCV's padded level
      for (int i = lane; i < RW * RW; i += 32) {
        const int ry = i / RW, rx = i - ry * RW;
        const int sy = reflect101(ipy - 1 + ry, rows), sx = reflect101(ipx - 1 + rx, cols);
        region[ry * RP + rx] = I[(size_t)sy * cols + sx];
      }
      __syncwarp();
      // Scharr derivatives on the (win+1)^2 grid; zero outside the image (BORDER_CONSTANT)
      for (int i = lane; i < DW * DW; i += 32) {
        const int ty = i / DW, tx = i - ty * DW;
        const int X = ipx + tx, Y = ipy + ty;
        const bool inside = (X >= 0 && X < cols && Y >= 0 && Y < rows);
        const uint8_t* r0 = region + ty * RP + tx;  // row Y-1, col X-1
        const uint8_t* r1 = r0 + RP;
        const uint8_t* r2 = r1 + RP;
        int dx = 0, dy = 0;
        if (inside) {
          const int t0l = (r0[0] + r2[0]) * 3 + r1[0] * 10;
          const int t0r = (r0[2] + r2[2]) * 3 + r1[2] * 10;
          const int t1l = r2[0] - r0[0], t1c = r2[1] - r0[1], t1r = r2[2] - r0[2];
          dx = t0r - t0l;
          dy = (t1r + t1l) * 3 + t1c * 10;
        }
        dtile[i * 2] = (short)dx;
        dtile[i * 2 + 1] = (short)dy;
      }
    }
    __syncwarp();
    // template + structure tensor: slot s of this lane is window pixel (y = 2 s + r, x = c)
    // Ix | Iy << 16 in one register (|Ix|, |Iy| <= 4080) to raise occupancy: 80 registers -> 6 CTAs/SM, measured 17 % faster than
    // keeping Ix and Iy in separate registers
    int tI[NS], tX[NS];
    int pA11 = 0, pA12 = 0, pA22 = 0;  // per-lane partials: <= 8 samples of |Ix|, |Iy| <= 4080 -> < 2^27
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const int y = 2 * s + r;
      int ival = 0, ix = 0, iy = 0;
      if (c < WIN && y < WIN) {
        const uint8_t* q = region + (y + 1) * RP + (c + 1);
        const unsigned* dq = reinterpret_cast<const unsigned*>(dtile) + (y * DW + c);  // packed (dx | dy << 16)
        const unsigned d00 = dq[0], d01 = dq[1], d10 = dq[DW], d11 = dq[DW + 1];
        ival = descale(q[0] * iw00 + q[1] * iw01 + q[RP] * iw10 + q[RP + 1] * iw11, 9);
        ix = descale((int)(short)(d00 & 0xffffu) * iw00 + (int)(short)(d01 & 0xffffu) * iw01 + (int)(short)(d10 & 0xffffu) * iw10 + (int)(short)(d11 & 0xffffu) * iw11, 14);
        iy = descale(((int)d00 >> 16) * iw00 + ((int)d01 >> 16) * iw01 + ((int)d10 >> 16) * iw10 + ((int)d11 >> 16) * iw11, 14);
      }
      tI[s] = ival;
      tX[s] = (ix & 0xffff) | (iy << 16);
      pA11 += ix * ix;
      pA12 += ix * iy;
      pA22 += iy * iy;
    }
    const long long lA11 = warp_sum_i32_exact(pA11), lA12 = warp_sum_i32_exact(pA12), lA22 = warp_sum_i32_exact(pA22);
    const float A11 = __ll2float_rn(lA11) * FLT_SCALE, A12 = __ll2float_rn(lA12) * FLT_SCALE, A22 = __ll2float_rn(lA22) * FLT_SCALE;
    float D = A11 * A22 - A12 * A12;
    const float minEig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * WIN * WIN);
    if ((double)minEig < prm.min_eig || D < 1.1920928955078125e-7f) {
      if (level == 0) st = 0;
      continue;
    }
    D = 1.f / D;
    nx -= half;
    ny -= half;
    float pdx = 0.f, pdy = 0.f;
    // Raw bytes of J under this lane's slots: rows y = 2 s + r and y + 1 (clamped to the window: only the last
    // slot of the upper half-warp would step past it) at column inx + cx.  The interior case (whole window inside
    // the image: almost every iteration) is branch-free so the 2 NS loads issue back to back; the border case
    // applies REFLECT_101 per coordinate.  Lanes outside the window fetch junk that meets a zero template gradient.
    auto fetch = [&](int inx, int iny, bool interior, int (&v0)[NS], int (&v1)[NS]) {
      if (interior) {
        const uint8_t* __restrict__ q = J + (size_t)(iny + r) * cols + (inx + cx);
        const size_t two_rows = 2 * (size_t)cols;
        const size_t last_off = r == 1 ? 0 : (size_t)cols;  // the last slot of the upper half-warp would step past the window
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          v0[s] = __ldg(q);
          v1[s] = __ldg(q + (s == NS - 1 ? last_off : (size_t)cols));
          q += two_rows;
        }
      } else {
        const int X = reflect101(inx + cx, cols);
#pragma unroll
        for (int s = 0; s < NS; ++s) {
          const int Y0 = reflect101(iny + min(2 * s + r, WIN), rows), Y1 = reflect101(iny + min(2 * s + r + 1, WIN), rows);
          v0[s] = __ldg(J + (size_t)Y0 * cols + X);
          v1[s] = __ldg(J + (size_t)Y1 * cols + X);
        }
      }
    };
    auto bilinear = [&](int v0, int v1) -> int {
      const int v0r = __shfl_down_sync(0xffffffffu, v0, 1), v1r = __shfl_down_sync(0xffffffffu, v1, 1);
      return descale(v0 * iw00 + v0r * iw01 + v1 * iw10 + v1r * iw11, 9);
    };
    for (int j = 0; j < prm.max_iter; ++j) {
      const int inx = (int)floorf(nx), iny = (int)floorf(ny);
      if (inx < -WIN || inx >= cols || iny < -WIN || iny >= rows) {
        if (level == 0) st = 0;
        break;
      }
      a = nx - inx;
      b = ny - iny;
      iw00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
      iw01 = __float2int_rn(a * (1.f - b) * 16384.f);
      iw10 = __float2int_rn((1.f - a) * b * 16384.f);
      iw11 = 16384 - iw00 - iw01 - iw10;
      const bool interior = (inx >= 0 && iny >= 0 && inx + WIN < cols && iny + WIN < rows);
      int pb1 = 0, pb2 = 0;  // per-lane partials: <= 8 samples of |diff| <= 8160 times |I'| <= 4080 -> < 2^29
      int v0[NS], v1[NS];
      fetch(inx, iny, interior, v0, v1);
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int diff = bilinear(v0[s], v1[s]) - tI[s];
        pb1 += diff * (int)(short)(tX[s] & 0xffff);
        pb2 += diff * (tX[s] >> 16);
      }
      const long long lb1 = warp_sum_i32_exact(pb1), lb2 = warp_sum_i32_exact(pb2);
      const float b1 = __ll2float_rn(lb1) * FLT_SCALE, b2 = __ll2float_rn(lb2) * FLT_SCALE;
      const float dx = (A12 * b2 - A22 * b1) * D;
      const float dy = (A12 * b1 - A11 * b2) * D;
      nx += dx;
      ny += dy;
      outx = nx + half;
      outy = ny + half;
      if ((double)dx * dx + (double)dy * dy <= prm.eps_sq) break;
      if (j > 0 && fabs((double)(dx + pdx)) < 0.01 && fabs((double)(dy + pdy)) < 0.01) {
        outx -= dx * 0.5f;
        outy -= dy * 0.5f;
        break;
      }
      pdx = dx;
      pdy = dy;
    }
    if (st && level == 0) {
      // default-flags error measure: mean |J - I| over the window / 32 (lkpyramid.cpp tail)
      const float fx = outx - half, fy = outy - half;
      const int inx = (int)floorf(fx), iny = (int)floorf(fy);
      if (inx < -WIN || inx >= cols || iny < -WIN || iny >= rows) {
        st = 0;
        continue;
      }
      const float aa = fx - inx, bb = fy - iny;
      iw00 = __float2int_rn((1.f - aa) * (1.f - bb) * 16384.f);
      iw01 = __float2int_rn(aa * (1.f - bb) * 16384.f);
      iw10 = __float2int_rn((1.f - aa) * bb * 16384.f);
      iw11 = 16384 - iw00 - iw01 - iw10;
      int pe = 0;
      int v0[NS], v1[NS];
      fetch(inx, iny, false, v0, v1);
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        const int diff = bilinear(v0[s], v1[s]) - tI[s];
        if (c < WIN && 2 * s + r < WIN) pe += abs(diff);
      }
      const long long le = warp_sum_i32_exact(pe);
      errv = __ll2float_rn(le) * 1.f / (float)(32 * WIN * WIN);
    }
  }
  if (lane == 0) {
    next_pts[2 * pi] = outx;
    next_pts[2 * pi + 1] = outy;
    status[pi] = (uint8_t)st;
    if (err) err[pi] = errv;
  }
}

template <int WIN>
static void launch_lk_fast(dim3 grid, cudaStream_t st, const uint8_t* prev_pyr, const uint8_t* next_pyr, unsigned long long pyr_stride,
                           const unsigned long long* prev_off, const unsigned long long* next_off, const PyrDesc& d, const float* prev_pts,
                           float* next_pts, uint8_t* status, float* err, const int* npts_dev, const LKParams& prm) {
  lk_kernel_fast<WIN><<<grid, LK_WARPS * 32, 0, st>>>(prev_pyr, next_pyr, pyr_stride, prev_off, next_off, d, prev_pts, next_pts, status, err, npts_dev, prm);
}

// XIVO_LK_GENERIC=1 routes single-channel frames through the generic kernel (parity tests compare the two)
static bool prm_force_generic_lk() {
  const char* e = getenv("XIVO_LK_GENERIC");
  return e && e[0] == '1';
}

size_t lk_smem_bytes(int win, int cn) {
  const int RW = win + 3, DW = win + 1;
  const int reg_bytes = ((RW * RW * cn + 15) / 16) * 16;
  const int per_warp = reg_bytes + 2 * (DW * DW * cn * 2 + win * win * cn * 3);
  return (size_t)LK_WARPS * (((per_warp + 15) / 16) * 16);
}

int launch_lk_track(cudaStream_t st, const uint8_t* prev_pyr, const uint8_t* next_pyr, unsigned long long pyr_stride,
                    const unsigned long long* prev_off, const unsigned long long* next_off, const PyrDesc& d, const float* prev_pts, float* next_pts, uint8_t* status, float* err,
                    const int* npts_dev, int max_pts, int batch, int win, int max_iter, double eps, int use_initial_flow,
                    double min_eig) {
  XB_REQUIRE(win >= 3 && win <= LK_MAX_WIN && (win & 1), "LK: win_size must be odd and in [3, 21]");
  XB_REQUIRE(d.cn == 1 || d.cn == 3, "LK: 1 or 3 channels");
  LKParams prm;
  prm.win = win;
  prm.max_iter = max_iter < 0 ? 0 : (max_iter > 100 ? 100 : max_iter);
  double e = eps < 0 ? 0 : (eps > 10 ? 10 : eps);
  prm.eps_sq = e * e;
  prm.eps_sq_f = (float)prm.eps_sq;
  prm.min_eig = min_eig;
  prm.use_initial_flow = use_initial_flow;
  prm.max_pts = max_pts;
  size_t smem = lk_smem_bytes(win, d.cn);
  dim3 grid((max_pts + LK_WARPS - 1) / LK_WARPS, batch);
  ProfScope ps("lk_track", st);
  const bool generic = prm_force_generic_lk();
  if (d.cn == 1 && win <= 15 && !generic) {
    switch (win) {
#define XB_LK_CASE(W) case W: launch_lk_fast<W>(grid, st, prev_pyr, next_pyr, pyr_stride, prev_off, next_off, d, prev_pts, next_pts, status, err, npts_dev, prm); break;
      XB_LK_CASE(3) XB_LK_CASE(5) XB_LK_CASE(7) XB_LK_CASE(9) XB_LK_CASE(11) XB_LK_CASE(13) XB_LK_CASE(15)
#undef XB_LK_CASE
    }
  } else if (d.cn == 1) {
    static size_t attr1 = 0;
    if (smem > attr1) { XB_CUDA(cudaFuncSetAttribute(lk_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr1 = smem; }
    lk_kernel<1><<<grid, LK_WARPS * 32, smem, st>>>(prev_pyr, next_pyr, pyr_stride, prev_off, next_off, d, prev_pts, next_pts, status, err, npts_dev, prm);
  } else {
    static size_t attr3 = 0;
    if (smem > attr3) { XB_CUDA(cudaFuncSetAttribute(lk_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr3 = smem; }
    lk_kernel<3><<<grid, LK_WARPS * 32, smem, st>>>(prev_pyr, next_pyr, pyr_stride, prev_off, next_off, d, prev_pts, next_pts, status, err, npts_dev, prm);
  }
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Descriptor path (/root/reference/src/tracker.cpp:231-292, :341-460, :530-565; popcount distance src/fastbrief.cpp:53-93):
// BRIEF-32 at given keypoints and the Hamming matrix of the cross-checked brute-force matcher.  Semantics: oracle/tracker_oracle.c
// (orc_brief, orc_bf_match_crosscheck); the 256 test pairs are the own table of brief_pattern.h (opencv_contrib's is not available).
// brief_kernel: one warp per keypoint.  The 56 x 56 neighbourhood (48-pixel patch + 9 x 9 box) is staged in shared memory as grey
// bytes (BGR converted with FAST's coefficients), then summed separably into 48 x 48 box sums (u16: 81 * 255 < 65536); lane l
// evaluates tests 8 l .. 8 l + 7 = byte l of the descriptor, so a descriptor is one coalesced 32-byte store.
// ------------------------------------------------------------------------------------------
}  // namespace xb
#include "brief_pattern.h"
namespace xb {
__constant__ signed char c_brief_pattern[256][4];
constexpr int BR_WARPS = 3, BR_R = 28;                 // 56 x 56 staged region: keypoint pixel +- 28 (27 suffices; 28 keeps rows 8-byte sized)
constexpr int BR_W = 2 * BR_R;                         // 56
constexpr int BR_S = 48;                               // box-sum image: offsets -24 .. 23 (tests reach +-19)
template <int CN>
__global__ void __launch_bounds__(BR_WARPS * 32) brief_kernel(const uint8_t* __restrict__ img, unsigned long long img_stride,
                                                              const unsigned long long* __restrict__ seq_off, int rows, int cols,
                                                              const float* __restrict__ kp_xy, const int* __restrict__ nkp, int max_kp,
                                                              uint8_t* __restrict__ desc, uint8_t* __restrict__ valid) {
  __shared__ uint8_t patch[BR_WARPS][BR_W][BR_W];
  __shared__ unsigned short hsum[BR_WARPS][BR_W][BR_S];
  __shared__ unsigned short box[BR_WARPS][BR_S][BR_S];
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.x * BR_WARPS + warp;
  const unsigned long long soff = seq_off ? seq_off[b] : (unsigned long long)b * img_stride;
  if (soff == ~0ull || k >= nkp[b]) return;  // warp-uniform
  const uint8_t* __restrict__ src = img + soff;
  const size_t ki = (size_t)b * max_kp + k;
  const float fx = kp_xy[2 * ki], fy = kp_xy[2 * ki + 1];
  const bool ok = fx >= XB_BRIEF_BORDER && fx < cols - XB_BRIEF_BORDER && fy >= XB_BRIEF_BORDER && fy < rows - XB_BRIEF_BORDER;
  uint8_t* __restrict__ d = desc + ki * XB_BRIEF_BYTES;
  if (!ok) {  // KeyPointsFilter::runByImageBorder drops the keypoint
    d[lane] = 0;
    if (lane == 0) valid[ki] = 0;
    return;
  }
  const int cx = (int)(fx + 0.5f), cy = (int)(fy + 0.5f);
  // stage rows cy - 28 .. cy + 27, columns cx - 28 .. cx + 27 (inside the image: cx, cy >= 28 and <= dim - 28)
  for (int i = lane; i < BR_W * BR_W; i += 32) {
    const int ry = i / BR_W, rx = i - ry * BR_W;
    const int gy = min(max(cy - BR_R + ry, 0), rows - 1), gx = min(max(cx - BR_R + rx, 0), cols - 1);
    const uint8_t* p = src + ((size_t)gy * cols + gx) * CN;
    patch[warp][ry][rx] = CN == 1 ? p[0] : (uint8_t)((p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15);
  }
  __syncwarp();
  // horizontal 9-sums: hsum[ry][sx] = sum patch[ry][sx + 0 .. sx + 8], sx = 0 .. 47 <-> offset sx - 24 (box centre at column sx + 4 = cx - 24 + sx)
  for (int i = lane; i < BR_W * BR_S; i += 32) {
    const int ry = i / BR_S, sx = i - ry * BR_S;
    int s = 0;
#pragma unroll
    for (int q = 0; q < 9; ++q) s += patch[warp][ry][sx + q];
    hsum[warp][ry][sx] = (unsigned short)s;
  }
  __syncwarp();
  for (int i = lane; i < BR_S * BR_S; i += 32) {
    const int sy = i / BR_S, sx = i - sy * BR_S;
    int s = 0;
#pragma unroll
    for (int q = 0; q < 9; ++q) s += hsum[warp][sy + q][sx];
    box[warp][sy][sx] = (unsigned short)s;
  }
  __syncwarp();
  // box[sy][sx] = 9 x 9 sum centred at pixel (cx - 24 + sx, cy - 24 + sy): offset (dx, dy) -> box[dy + 24][dx + 24]
  unsigned byte = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const signed char* t = c_brief_pattern[8 * lane + q];
    const int a = box[warp][t[1] + 24][t[0] + 24], c2 = box[warp][t[3] + 24][t[2] + 24];
    byte |= (unsigned)(a < c2) << (7 - q);
  }
  d[lane] = (uint8_t)byte;
  if (lane == 0) valid[ki] = 1;
}

int launch_brief(cudaStream_t st, const uint8_t* img, unsigned long long img_stride, const unsigned long long* seq_off, int rows, int cols, int cn,
                 const float* kp_xy, const int* nkp, int max_kp, uint8_t* desc, uint8_t* valid, int batch) {
  XB_REQUIRE(cn == 1 || cn == 3, "BRIEF: 1 or 3 channels");
  static bool uploaded = false;
  if (!uploaded) {  // (one device per process in this library)
    XB_CUDA(cudaMemcpyToSymbol(c_brief_pattern, kBriefPattern, sizeof(kBriefPattern)));
    uploaded = true;
  }
  ProfScope ps("brief", st);
  dim3 grid((max_kp + BR_WARPS - 1) / BR_WARPS, batch);
  if (cn == 1) brief_kernel<1><<<grid, BR_WARPS * 32, 0, st>>>(img, img_stride, seq_off, rows, cols, kp_xy, nkp, max_kp, desc, valid);
  else brief_kernel<3><<<grid, BR_WARPS * 32, 0, st>>>(img, img_stride, seq_off, rows, cols, kp_xy, nkp, max_kp, desc, valid);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// Nearest train descriptor of every query and nearest query of every train (first index on ties), Hamming distance over 32-byte
// descriptors: what cv::BFMatcher(NORM_HAMMING, crossCheck) needs.  One warp per query row (best train) / per train row (best query);
// a lane strides over the other side, keeps (distance, index) packed as distance << 16 | index, and the warp reduces with min.
__global__ void __launch_bounds__(128) hamming_nearest_kernel(const uint8_t* __restrict__ a, const int* __restrict__ na, int max_a,
                                                              const uint8_t* __restrict__ bdesc, const int* __restrict__ nb, int max_b,
                                                              int* __restrict__ best_idx, int* __restrict__ best_dist) {
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 4 + warp;
  if (i >= na[s]) return;
  const uint4* qa = reinterpret_cast<const uint4*>(a + ((size_t)s * max_a + i) * 32);
  const uint4 q0 = qa[0], q1 = qa[1];
  unsigned best = 0xffffffffu;
  const int n = nb[s];
  for (int j = lane; j < n; j += 32) {
    const uint4* tb = reinterpret_cast<const uint4*>(bdesc + ((size_t)s * max_b + j) * 32);
    const uint4 t0 = tb[0], t1 = tb[1];
    const unsigned dist = __popc(q0.x ^ t0.x) + __popc(q0.y ^ t0.y) + __popc(q0.z ^ t0.z) + __popc(q0.w ^ t0.w) + __popc(q1.x ^ t1.x) + __popc(q1.y ^ t1.y) +
                          __popc(q1.z ^ t1.z) + __popc(q1.w ^ t1.w);
    best = min(best, (dist << 16) | (unsigned)j);  // equal distances: the smaller index wins (j < 65536)
  }
  best = __reduce_min_sync(0xffffffffu, best);
  if (lane == 0) {
    best_idx[(size_t)s * max_a + i] = n > 0 ? (int)(best & 0xffffu) : -1;
    best_dist[(size_t)s * max_a + i] = n > 0 ? (int)(best >> 16) : -1;
  }
}

int launch_hamming_nearest(cudaStream_t st, const uint8_t* a, const int* na, int max_a, const uint8_t* b, const int* nb, int max_b, int* best_idx,
                           int* best_dist, int batch) {
  XB_REQUIRE(max_b < 65536, "Hamming matcher: at most 65535 descriptors per side");
  ProfScope ps("hamming_nearest", st);
  hamming_nearest_kernel<<<dim3((max_a + 3) / 4, batch), 128, 0, st>>>(a, na, max_a, b, nb, max_b, best_idx, best_dist);
  XB_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// Device-side tracker decisions: Tracker::UpdateLK's accept loop (tracker.cpp:571-589) and Tracker::DetectLK's greedy selection
// (tracker.cpp:224-229, :295-328) without a host round trip.  Both walk a list in order while a mask of claimed pixels grows, so each
// sequence is one CTA whose warp 0 does the sequential walk (the 15 x 15 mask-out of one feature is spread over the lanes);
// the mask lives in shared memory as a bitmap (bit = pixel still free).  Same arithmetic as the host code they replace
// (estimator_host.cpp.inc: mask_out / mask_valid; tracker_host.cpp.inc: Estimator::tracker_detect_select): truncation for the validity test, round-half-even
// for the block corners, the displacement test in double precision.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mask_reset(unsigned* m, int stride, const TrackDecideCfg& c, int tid, int nthr) {
  for (int i = tid; i < c.rows * stride; i += nthr) {
    const int y = i / stride, w = i - y * stride;
    unsigned v = 0u;
    const int x0 = c.margin, x1 = c.cols - c.margin - 1;  // free columns [x0, x1] of the rows [margin, rows - margin)
    if (y >= c.margin && y < c.rows - c.margin && x1 >= x0) {
      const int lo = max(x0, 32 * w), hi = min(x1, 32 * w + 31);
      if (hi >= lo) v = (0xffffffffu >> (31 - (hi - 32 * w))) & (0xffffffffu << (lo - 32 * w));
    }
    m[i] = v;
  }
}
// clear the block [x0, x1] x [y0, y1] (already clipped); lanes split the rows; atomic = several blocks may be cleared concurrently
__device__ __forceinline__ void mask_clear_block(unsigned* m, int stride, int x0, int y0, int x1, int y1, int lane, int nlanes, bool atomic) {
  if (x1 < x0) return;
  for (int y = y0 + lane; y <= y1; y += nlanes) {
    for (int w = x0 >> 5; w <= (x1 >> 5); ++w) {
      const int lo = max(x0, 32 * w) - 32 * w, hi = min(x1, 32 * w + 31) - 32 * w;
      const unsigned bits = (0xffffffffu >> (31 - hi)) & (0xffffffffu << lo);
      if (atomic) atomicAnd(&m[y * stride + w], ~bits);
      else m[y * stride + w] &= ~bits;
    }
  }
}
__device__ __forceinline__ void block_of(double x, double y, const TrackDecideCfg& c, int* x0, int* y0, int* x1, int* y1) {
  const int h = c.mask_half;
  *x0 = max(__double2int_rn(x - h), 0);
  *y0 = max(__double2int_rn(y - h), 0);
  *x1 = min(__double2int_rn(x + h), c.cols - 1);
  *y1 = min(__double2int_rn(y + h), c.rows - 1);
}
__device__ __forceinline__ bool mask_free(const unsigned* m, int stride, const TrackDecideCfg& c, double x, double y) {
  const int col = (int)x, row = (int)y;
  if (col < 0 || col >= c.cols || row < 0 || row >= c.rows) return false;
  return (m[row * stride + (col >> 5)] >> (col & 31)) & 1u;
}

// kind[b]: 1 = first frame (detection only), 2 = tracked by LK, 3 = empty list (nothing to do), 0 = inactive.
// Outputs: stat[b][i] = feature i keeps its track; need[b] = features the detection should add (0 = none).
// The reference walks the list while a mask of claimed pixels grows (tracker.cpp:571-589).  The mask only ever loses the margin band and
// the (2 mask_half + 1)^2 blocks of the tracks accepted so far, so "pixel of track i still free" == "inside the margin band and in no
// block of an earlier ACCEPTED track": all threads build the bit matrix C[i] = {j : block(j) contains pixel(i)}, then warp 0 resolves the
// order dependence with one AND + vote per track (lane l keeps word l of the accepted set) instead of clearing bitmap blocks.
__global__ void __launch_bounds__(128) track_accept_kernel(TrackDecideCfg c, const int* __restrict__ kind, const int* __restrict__ npts,
                                                           const float* __restrict__ pts0, const float* __restrict__ pts1,
                                                           const uint8_t* __restrict__ lkst, uint8_t* __restrict__ stat, int* __restrict__ need,
                                                           int* __restrict__ kp_count) {
  extern __shared__ unsigned acc_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (kp_count && tid == 0) kp_count[b] = 0;  // the keypoint cursor of the detection that follows in the stream (saves its memset call)
  const int k = kind[b];
  if (k == 1) { if (tid == 0) need[b] = c.num_max; return; }
  if (k != 2) { if (tid == 0) need[b] = 0; return; }
  const int n = min(npts[b], c.max_pts);
  const int nw = (c.max_pts + 31) >> 5;  // <= 32 (launch_track_accept)
  int* px = reinterpret_cast<int*>(acc_smem);
  int* py = px + c.max_pts;
  int* bx0 = py + c.max_pts;
  int* by0 = bx0 + c.max_pts;
  int* bx1 = by0 + c.max_pts;
  int* by1 = bx1 + c.max_pts;
  unsigned* C = reinterpret_cast<unsigned*>(by1 + c.max_pts);
  uint8_t* sok = reinterpret_cast<uint8_t*>(C + (size_t)c.max_pts * nw);
  {
    const float2* p0 = reinterpret_cast<const float2*>(pts0 + (size_t)b * c.max_pts * 2);
    const float2* p1 = reinterpret_cast<const float2*>(pts1 + (size_t)b * c.max_pts * 2);
    for (int i = tid; i < n; i += blockDim.x) {
      const float2 a = p0[i], q = p1[i];
      bool ok = lkst[(size_t)b * c.max_pts + i] != 0;
      const double x = (double)q.x, y = (double)q.y;
      const int col = (int)x, row = (int)y;
      if (ok) {
        const double dx = (double)a.x - x, dy = (double)a.y - y;
        // mask_valid on the fresh mask (inside the image and the margin band) + the displacement test
        ok = col >= 0 && col < c.cols && row >= 0 && row < c.rows && row >= c.margin && row < c.rows - c.margin && col >= c.margin &&
             col <= c.cols - c.margin - 1 && sqrt(dx * dx + dy * dy) < c.max_disp;
      }
      int x0, y0, x1, y1;
      block_of(x, y, c, &x0, &y0, &x1, &y1);
      px[i] = col; py[i] = row;
      bx0[i] = x0; by0[i] = y0; bx1[i] = x1; by1[i] = y1;
      sok[i] = ok ? 1 : 0;
    }
  }
  __syncthreads();
  for (int item = tid; item < n * nw; item += blockDim.x) {
    const int i = item / nw, w = item - i * nw;
    unsigned bits = 0u;
    if (32 * w < i && sok[i]) {  // only earlier tracks can have claimed the pixel
      const int x = px[i], y = py[i], jend = min(32, i - 32 * w);
      for (int jj = 0; jj < jend; ++jj) {
        const int j = 32 * w + jj;
        if (x >= bx0[j] && x <= bx1[j] && y >= by0[j] && y <= by1[j]) bits |= 1u << jj;
      }
    }
    C[item] = bits;
  }
  __syncthreads();
  if (tid < 32) {
    unsigned acc = 0u;  // lane l: tracks 32 l .. 32 l + 31 accepted so far
    int num_valid = 0;
    for (int i = 0; i < n; ++i) {
      if (!sok[i]) continue;  // warp-uniform
      const unsigned cw = tid < nw ? C[i * nw + tid] : 0u;
      const bool claimed = __any_sync(0xffffffffu, (cw & acc) != 0u);
      if (!claimed) {
        if (tid == (i >> 5)) acc |= 1u << (i & 31);
        ++num_valid;
      } else if (tid == 0) {
        sok[i] = 0;
      }
    }
    if (tid == 0) need[b] = num_valid < c.num_min ? c.num_max - num_valid : 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) stat[(size_t)b * c.max_pts + i] = sok[i];
}
size_t track_accept_smem_bytes(int max_pts) { return (size_t)max_pts * (6 * 4 + ((max_pts + 31) / 32) * 4 + 1) + 16; }

// Greedy selection of new features from the FAST keypoints of the sequences with need[b] > 0, in the order (score descending, y, x).
// kp: packed (y << 20 | x << 8 | score), rewritten in place as sort keys ((255 - score) << 24 | y << 12 | x; unique per pixel).
// The candidates are consumed in sorted chunks of at most SEL_CAP keys: a 4-pass radix select finds the chunk's largest key, the chunk is
// gathered and bitonic-sorted in shared memory, warp 0 walks it.  new_kp[b][j] = packed (y << 20 | x << 8 | score) of the j-th pick.
constexpr int SEL_CAP = 1024, SEL_THREADS = 256;
__global__ void __launch_bounds__(SEL_THREADS) track_select_kernel(TrackDecideCfg c, const int* __restrict__ kind, const int* __restrict__ npts,
                                                                   const float* __restrict__ pts1, const uint8_t* __restrict__ stat,
                                                                   const int* __restrict__ need, unsigned* __restrict__ kp,
                                                                   const int* __restrict__ kp_count, unsigned* __restrict__ new_kp,
                                                                   int* __restrict__ n_new) {
  extern __shared__ unsigned tmask[];
  __shared__ unsigned chunk[SEL_CAP];
  __shared__ int hist[256];
  __shared__ int s_cnt, s_budget, s_stop, s_nnew;
  __shared__ unsigned s_prefix, s_last;
  const int b = blockIdx.x, tid = threadIdx.x;
  int budget = need[b];
  if (budget <= 0) { if (tid == 0) n_new[b] = 0; return; }
  const int stride = (c.cols + 31) >> 5;
  mask_reset(tmask, stride, c, tid, SEL_THREADS);
  __syncthreads();
  if (kind[b] == 2) {  // the pixels claimed by the tracks that survived (any order: the union is what matters)
    const int n = npts[b];
    const float* p1 = pts1 + (size_t)b * c.max_pts * 2;
    for (int i = tid >> 4; i < n; i += SEL_THREADS >> 4) {
      if (!stat[(size_t)b * c.max_pts + i]) continue;
      int x0, y0, x1, y1;
      block_of((double)p1[2 * i], (double)p1[2 * i + 1], c, &x0, &y0, &x1, &y1);
      mask_clear_block(tmask, stride, x0, y0, x1, y1, tid & 15, 16, true);
    }
  }
  __syncthreads();
  unsigned* keys = kp + (size_t)b * c.max_kp;
  const int n = min(kp_count[b], c.max_kp);
  // KeyPointsFilter::runByPixelsMask + key conversion; candidates on claimed pixels get the key ~0 (never selected: valid keys are
  // < 2^32 - 1 because x < 4096)
  for (int i = tid; i < n; i += SEL_THREADS) {
    const unsigned k = keys[i];
    const int x = (k >> 8) & 0xfff, y = k >> 20, sc = k & 0xff;
    const bool free_px = (tmask[y * stride + (x >> 5)] >> (x & 31)) & 1u;
    keys[i] = free_px ? (((unsigned)(255 - sc) << 24) | ((unsigned)y << 12) | (unsigned)x) : 0xffffffffu;
  }
  if (tid == 0) { s_last = 0u; s_stop = 0; s_nnew = 0; s_budget = budget; }
  __syncthreads();
  bool first = true;
  for (;;) {
    // ---- the SEL_CAP-th smallest key among those > s_last (or the largest if fewer remain): MSB-first radix select
    // the first chunk is small: the budget is a few dozen picks and the best-scored candidates are rarely all on claimed pixels, so one short
    // sort usually ends the walk; later chunks are full-sized (the chunking does not change the order in which candidates are visited)
    const int cap = first ? SEL_CAP / 4 : SEL_CAP;
    const unsigned last = s_last;
    unsigned prefix = 0u;
    int want = cap;  // rank (1-based) still to be found inside the current prefix
    bool exhausted = false;
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      for (int i = tid; i < 256; i += SEL_THREADS) hist[i] = 0;
      __syncthreads();
      const unsigned pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
      for (int i = tid; i < n; i += SEL_THREADS) {
        const unsigned k = keys[i];
        if (k == 0xffffffffu || (!first && k <= last) ) continue;
        if ((k & pmask) == prefix) atomicAdd(&hist[(k >> shift) & 0xff], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int acc = 0, d = 0, total = 0;
        for (int q = 0; q < 256; ++q) total += hist[q];
        if (total == 0) { s_cnt = -1; }
        else {
          if (want > total) want = total;  // fewer than SEL_CAP remain: take them all (rank = total)
          for (d = 0; d < 256; ++d) { if (acc + hist[d] >= want) break; acc += hist[d]; }
          s_prefix = prefix | ((unsigned)d << shift);
          s_cnt = want - acc;
        }
      }
      __syncthreads();
      if (s_cnt < 0) { exhausted = true; break; }
      prefix = s_prefix;
      want = s_cnt;
      __syncthreads();
    }
    if (exhausted) break;
    const unsigned kth = prefix;  // all keys in (last, kth] form the chunk (<= SEL_CAP of them, keys are unique)
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    for (int i = tid; i < n; i += SEL_THREADS) {
      const unsigned k = keys[i];
      if (k == 0xffffffffu || (!first && k <= last) || k > kth) continue;
      const int pos = atomicAdd(&s_cnt, 1);
      if (pos < cap) chunk[pos] = k;
    }
    __syncthreads();
    const int m = min(s_cnt, cap);
    for (int i = m + tid; i < cap; i += SEL_THREADS) chunk[i] = 0xffffffffu;
    __syncthreads();
    for (int k2 = 2; k2 <= cap; k2 <<= 1)  // bitonic sort, ascending
      for (int j = k2 >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < cap; i += SEL_THREADS) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned a = chunk[i], bb = chunk[ixj];
            const bool up = (i & k2) == 0;
            if ((a > bb) == up) { chunk[i] = bb; chunk[ixj] = a; }
          }
        }
        __syncthreads();
      }
    // ---- greedy walk (warp 0)
    if (tid < 32) {
      int bud = s_budget, nn = s_nnew, stop = 0;
      for (int i = 0; i < m && !stop; ++i) {
        const unsigned k = chunk[i];
        const int x = k & 0xfff, y = (k >> 12) & 0xfff, sc = 255 - (int)(k >> 24);
        const bool free_px = (tmask[y * stride + (x >> 5)] >> (x & 31)) & 1u;
        if (free_px) {
          if (tid == 0 && nn < c.max_new) new_kp[(size_t)b * c.max_new + nn] = ((unsigned)y << 20) | ((unsigned)x << 8) | (unsigned)sc;
          ++nn;
          int x0, y0, x1, y1;
          block_of((double)x, (double)y, c, &x0, &y0, &x1, &y1);
          __syncwarp();
          mask_clear_block(tmask, stride, x0, y0, x1, y1, tid, 32, false);
          __syncwarp();
          --bud;
        }
        if (bud <= 0 || sc < 5) stop = 1;  // tracker.cpp:326 (and the host's `s < 5` cut: OpenCV scores below 5 are never asked for)
      }
      if (tid == 0) { s_budget = bud; s_nnew = nn; s_stop = stop; s_last = kth; }
    }
    __syncthreads();
    first = false;
    if (s_stop || m == 0) break;
  }
  if (tid == 0) n_new[b] = min(s_nnew, c.max_new);
}

size_t track_mask_bytes(int rows, int cols) { return (size_t)rows * ((cols + 31) / 32) * sizeof(unsigned); }

int launch_track_accept(cudaStream_t st, const TrackDecideCfg& c, const int* kind, const int* npts, const float* pts0, const float* pts1,
                        const uint8_t* lkst, uint8_t* stat, int* need, int batch, int* kp_count_to_zero) {
  const size_t smem = track_accept_smem_bytes(c.max_pts);
  XB_REQUIRE(c.max_pts <= 1024 && smem <= 200 * 1024, "track_accept: more than 1024 tracks per sequence");
  static size_t attr = 0;
  if (smem > attr) { XB_CUDA(cudaFuncSetAttribute(track_accept_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  ProfScope ps("track_accept", st);
  track_accept_kernel<<<batch, 128, smem, st>>>(c, kind, npts, pts0, pts1, lkst, stat, need, kp_count_to_zero);
  XB_CUDA(cudaGetLastError());
  return 0;
}
int launch_track_select(cudaStream_t st, const TrackDecideCfg& c, const int* kind, const int* npts, const float* pts1, const uint8_t* stat,
                        const int* need, unsigned* kp, const int* kp_count, unsigned* new_kp, int* n_new, int batch) {
  const size_t smem = track_mask_bytes(c.rows, c.cols);
  XB_REQUIRE(smem <= 200 * 1024, "track_select: image too large for the shared-memory mask");
  static size_t attr = 0;
  if (smem > attr) { XB_CUDA(cudaFuncSetAttribute(track_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  ProfScope ps("track_select", st);
  track_select_kernel<<<batch, SEL_THREADS, smem, st>>>(c, kind, npts, pts1, stat, need, kp, kp_count, new_kp, n_new);
  XB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace xb

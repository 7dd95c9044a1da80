// Shared device/host helpers for the xivo_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace xb {

// last error text returned by xivo_last_error()
void set_error(const char* fmt, ...);

#define XB_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess) {                                                              \
      xb::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return -2;                                                                          \
    }                                                                                     \
  } while (0)

#define XB_REQUIRE(cond, msg)                                  \
  do {                                                         \
    if (!(cond)) {                                             \
      xb::set_error("%s:%d %s", __FILE__, __LINE__, msg);      \
      return -1;                                               \
    }                                                          \
  } while (0)

__host__ __device__ inline int reflect101(int i, int n) {
  // BORDER_REFLECT_101, single reflection is enough for |overshoot| < n (callers guarantee it);
  // loop kept for tiny levels.
  if (n == 1) return 0;
  while (i < 0 || i >= n) i = (i < 0) ? -i : 2 * (n - 1) - i;
  return i;
}

// ---- image pyramid descriptor (levels stored unpadded, back to back, 16-byte aligned) ----
constexpr int kMaxPyrLevels = 8;
struct PyrDesc {
  int n_levels;  // number of stored levels = maxLevel reached + 1
  int cn;        // channels (1 or 3), interleaved
  int rows[kMaxPyrLevels];
  int cols[kMaxPyrLevels];
  unsigned long long off[kMaxPyrLevels];  // byte offset of level l inside one pyramid
  unsigned long long total;               // bytes of one pyramid (16-byte aligned)
};

inline PyrDesc make_pyr_desc(int rows, int cols, int cn, int win, int max_level) {
  // Level count follows cv::buildOpticalFlowPyramid: stop when the next level would be <= win.
  PyrDesc d;
  memset(&d, 0, sizeof(d));
  d.cn = cn;
  int r = rows, c = cols;
  unsigned long long off = 0;
  int l = 0;
  for (;; ++l) {
    d.rows[l] = r;
    d.cols[l] = c;
    d.off[l] = off;
    off += ((unsigned long long)r * c * cn + 15ull) & ~15ull;
    int nr = (r + 1) / 2, nc = (c + 1) / 2;
    if (l == max_level || l == kMaxPyrLevels - 1 || nc <= win || nr <= win) break;
    r = nr;
    c = nc;
  }
  d.n_levels = l + 1;
  d.total = off;
  return d;
}

// ---- tiny fp64 3x3 algebra used by the per-feature kernels (row-major) ----
struct M3 { double m[9]; };
struct V3 { double v[3]; };

__host__ __device__ inline M3 m3_mul(const M3& a, const M3& b) {
  M3 c;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
  return c;
}
__host__ __device__ inline M3 m3_t(const M3& a) {
  M3 c;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c.m[3 * i + j] = a.m[3 * j + i];
  return c;
}
__host__ __device__ inline M3 m3_neg(const M3& a) {
  M3 c;
  for (int i = 0; i < 9; ++i) c.m[i] = -a.m[i];
  return c;
}
__host__ __device__ inline M3 m3_add(const M3& a, const M3& b) {
  M3 c;
  for (int i = 0; i < 9; ++i) c.m[i] = a.m[i] + b.m[i];
  return c;
}
__host__ __device__ inline V3 m3_mulv(const M3& a, const V3& x) {
  V3 y;
  for (int i = 0; i < 3; ++i) y.v[i] = a.m[3 * i] * x.v[0] + a.m[3 * i + 1] * x.v[1] + a.m[3 * i + 2] * x.v[2];
  return y;
}
__host__ __device__ inline V3 v3_add(const V3& a, const V3& b) { return V3{{a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]}}; }
__host__ __device__ inline V3 v3_sub(const V3& a, const V3& b) { return V3{{a.v[0] - b.v[0], a.v[1] - b.v[1], a.v[2] - b.v[2]}}; }
__host__ __device__ inline M3 m3_hat(const V3& w) {
  return M3{{0.0, -w.v[2], w.v[1], w.v[2], 0.0, -w.v[0], -w.v[1], w.v[0], 0.0}};
}
__host__ __device__ inline M3 m3_eye() { return M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }

// 2x3 times 3x3
struct M23 { double m[6]; };
__host__ __device__ inline M23 m23_mul(const M23& a, const M3& b) {
  M23 c;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) c.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
  return c;
}

// ---- camera (pinhole = 0, equidistant = 3; enum values of DistortionType,
//      /root/reference/common/camera_base.h:13-18) ----
struct CameraParams {
  int model, rows, cols;
  double fx, fy, cx, cy, k0, k1, k2, k3;
};

// Project normalised camera coordinates to pixels + 2x2 Jacobian.
// pinhole:  /root/reference/common/camera_pinhole.h:17-37
// equidist: /root/reference/common/camera_equidist.h:23-95
__host__ __device__ inline void camera_project(const CameraParams& c, double x, double y, double* u, double* v, double J[4]) {
  if (c.model == 0) {
    *u = c.fx * x + c.cx;
    *v = c.fy * y + c.cy;
    J[0] = c.fx; J[1] = 0; J[2] = 0; J[3] = c.fy;
    return;
  }
  double n2 = x * x + y * y, n = sqrt(n2), n3 = n2 + 1;
  double th = atan2(n, 1.0), phi = atan2(y, x);
  double th2 = th * th, th3 = th2 * th, th4 = th3 * th, th5 = th3 * th2, th6 = th5 * th, th7 = th5 * th2, th8 = th7 * th,
         th9 = th7 * th2;
  double r = th + c.k0 * th3 + c.k1 * th5 + c.k2 * th7 + c.k3 * th9;
  double cp = cos(phi), sp = sin(phi);
  *u = c.fx * r * cp + c.cx;
  *v = c.fy * r * sp + c.cy;
  double dphi_dx = -y / n2, dphi_dy = x / n2;
  double dth_dx = x / n3 / n, dth_dy = y / n3 / n;
  double dr = 1 + c.k0 * 3 * th2 + c.k1 * 5 * th4 + c.k2 * 7 * th6 + c.k3 * 9 * th8;
  J[0] = c.fx * cp * dr * dth_dx - c.fx * r * sp * dphi_dx;
  J[1] = c.fx * cp * dr * dth_dy - c.fx * r * sp * dphi_dy;
  J[2] = c.fy * sp * dr * dth_dx + c.fy * r * cp * dphi_dx;
  J[3] = c.fy * sp * dr * dth_dy + c.fy * r * cp * dphi_dy;
}

}  // namespace xb

// C-ABI layer, kernel-level entry points (include/xivo_b200.h).  Host buffers in, host
// buffers out; everything in between is the CUDA kernels of tracker_kernels.cu / ekf_kernels.cu.
#include <stdarg.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "../../include/xivo_b200.h"
#include "ctx.h"
#include "homography.h"
#include "kernels.h"

namespace xb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
std::atomic<unsigned long long> g_launches{0};
}  // namespace xb

using namespace xb;

#define API_BEGIN             \
  if (!ctx) {                 \
    set_error("null ctx");    \
    return XIVO_ERR_ARG;      \
  }                           \
  XB_CUDA(cudaSetDevice(ctx->device));

static CameraParams cam_from(const double* c) {
  CameraParams p;
  p.model = (int)c[0];
  p.rows = (int)c[1];
  p.cols = (int)c[2];
  p.fx = c[3]; p.fy = c[4]; p.cx = c[5]; p.cy = c[6];
  p.k0 = c[7]; p.k1 = c[8]; p.k2 = c[9]; p.k3 = c[10];
  return p;
}

extern "C" {

const char* xivo_last_error(void) { return g_err; }
int xivo_version(void) { return 100; }
unsigned long long xivo_launch_count(void) { return g_launches.load(); }
void* xivo_ctx_stream(xivo_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int xivo_ctx_create(int device, xivo_ctx** out) {
  if (!out) { set_error("null out"); return XIVO_ERR_ARG; }
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    set_error("no CUDA device available (%s); xivo_b200 has no CPU path", e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
    return XIVO_ERR_CUDA;
  }
  if (device < 0 || device >= n) { set_error("device %d out of range [0,%d)", device, n); return XIVO_ERR_ARG; }
  XB_CUDA(cudaSetDevice(device));
  xivo_ctx* c = new xivo_ctx();
  c->device = device;
  XB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  *out = c;
  return XIVO_OK;
}

void xivo_ctx_destroy(xivo_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  cudaStreamDestroy(ctx->stream);
  delete ctx;
}

unsigned long long xivo_pyramid_layout(int rows, int cols, int cn, int win, int max_level, int* n_levels, int* level_rows,
                                       int* level_cols, unsigned long long* level_off) {
  PyrDesc d = make_pyr_desc(rows, cols, cn, win, max_level);
  if (n_levels) *n_levels = d.n_levels;
  for (int l = 0; l < d.n_levels; ++l) {
    if (level_rows) level_rows[l] = d.rows[l];
    if (level_cols) level_cols[l] = d.cols[l];
    if (level_off) level_off[l] = d.off[l];
  }
  return d.total;
}

int xivo_build_pyramid(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, int win, int max_level, uint8_t* out) {
  API_BEGIN;
  XB_REQUIRE(img && out && rows > 0 && cols > 0 && (cn == 1 || cn == 3), "build_pyramid: bad arguments");
  PyrDesc d = make_pyr_desc(rows, cols, cn, win, max_level);
  DevBuf<uint8_t> pyr(d.total);
  XB_REQUIRE(pyr.ok(), "cudaMalloc failed");
  cudaStream_t st = ctx->stream;
  XB_CUDA(cudaMemcpyAsync(pyr.p, img, (size_t)rows * cols * cn, cudaMemcpyHostToDevice, st));
  // levels whose rows are 16-byte multiples go through the TMA pass (pyrdown_tma_kernel) like in the estimator; XIVO_PYRDOWN_TMA=0 keeps
  // the thread-staged kernels (the parity tests run both against the oracle)
  const char* tv = getenv("XIVO_PYRDOWN_TMA");
  const char* gv = getenv("XIVO_PYRDOWN_GENERIC");
  const bool tma = cn == 1 && !(tv && tv[0] == '0') && !(gv && gv[0] == '1');
  DevBuf<int> zero(1);
  XB_REQUIRE(zero.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemsetAsync(zero.p, 0, sizeof(int), st));
  for (int l = 0; l + 1 < d.n_levels; ++l) {
    CUtensorMap map;
    if (tma && (d.cols[l] & 15) == 0 && (d.off[l] & 15) == 0 && make_pyr_tensor_map(&map, pyr.p + d.off[l], d.rows[l], d.cols[l], d.total, 1) == 0) {
      if (int rc = launch_pyrdown_tma(st, map, zero.p, pyr.p, d.total, nullptr, d, l, 0, 1)) return rc;
    } else if (int rc = launch_pyrdown_level(st, pyr.p, d.total, nullptr, d, 1, nullptr, l)) return rc;
  }
  g_launches += d.n_levels - 1;
  XB_CUDA(cudaMemcpyAsync(out, pyr.p, d.total, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

int xivo_fast_detect(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, int threshold, int nonmax, int* kp_xy,
                     int* kp_score, int max_kp, int* n_kp) {
  API_BEGIN;
  XB_REQUIRE(img && kp_xy && kp_score && n_kp && max_kp > 0 && (cn == 1 || cn == 3), "fast_detect: bad arguments");
  cudaStream_t st = ctx->stream;
  const int cap = std::max(max_kp, 1 << 16);
  DevBuf<uint8_t> dimg((size_t)rows * cols * cn);
  DevBuf<unsigned> dkp(cap);
  DevBuf<int> dcnt(1);
  XB_REQUIRE(dimg.ok() && dkp.ok() && dcnt.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemcpyAsync(dimg.p, img, (size_t)rows * cols * cn, cudaMemcpyHostToDevice, st));
  // single-channel images with 16-byte rows are tiled by TMA (fast_pair_tma_kernel) like in the estimator; XIVO_FAST_TMA=0 = thread-staged tiles
  const char* fv = getenv("XIVO_FAST_TMA");
  CUtensorMap map;
  const bool tma = cn == 1 && (cols & 15) == 0 && !(fv && fv[0] == '0') && make_fast_tensor_map(&map, dimg.p, rows, cols, (size_t)rows * cols, 1) == 0;
  int rc = launch_fast_detect(st, dimg.p, (size_t)rows * cols * cn, nullptr, rows, cols, cn, threshold, nonmax, dkp.p, cap, dcnt.p, 1, nullptr,
                              tma ? &map : nullptr, (size_t)rows * cols);
  if (rc) return rc;
  g_launches += 1;
  int cnt = 0;
  XB_CUDA(cudaMemcpyAsync(&cnt, dcnt.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  const int got = std::min(cnt, cap);
  std::vector<unsigned> kp(got);
  if (got) XB_CUDA(cudaMemcpy(kp.data(), dkp.p, sizeof(unsigned) * got, cudaMemcpyDeviceToHost));
  std::sort(kp.begin(), kp.end());  // packed (y, x, score): ascending == raster order
  *n_kp = cnt;
  for (int i = 0; i < std::min(got, max_kp); ++i) {
    kp_xy[2 * i] = xb::kp_x(kp[i]);
    kp_xy[2 * i + 1] = xb::kp_y(kp[i]);
    kp_score[i] = xb::kp_score(kp[i]);
  }
  return XIVO_OK;
}

int xivo_brief_describe(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, const float* kp_xy, int n, uint8_t* desc, uint8_t* valid) {
  API_BEGIN;
  XB_REQUIRE(img && rows > 0 && cols > 0 && (cn == 1 || cn == 3) && n >= 0 && (n == 0 || (kp_xy && desc && valid)), "brief_describe: bad arguments");
  if (n == 0) return XIVO_OK;
  cudaStream_t st = ctx->stream;
  DevBuf<uint8_t> dimg((size_t)rows * cols * cn), ddesc((size_t)n * 32), dvalid(n);
  DevBuf<float> dkp((size_t)n * 2);
  DevBuf<int> dn(1);
  XB_REQUIRE(dimg.ok() && ddesc.ok() && dvalid.ok() && dkp.ok() && dn.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemcpyAsync(dimg.p, img, (size_t)rows * cols * cn, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dkp.p, kp_xy, sizeof(float) * 2 * n, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dn.p, &n, sizeof(int), cudaMemcpyHostToDevice, st));
  if (int rc = launch_brief(st, dimg.p, 0, nullptr, rows, cols, cn, dkp.p, dn.p, n, ddesc.p, dvalid.p, 1)) return rc;
  g_launches += 1;
  XB_CUDA(cudaMemcpyAsync(desc, ddesc.p, (size_t)n * 32, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(valid, dvalid.p, n, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

int xivo_hamming_match(xivo_ctx* ctx, const uint8_t* query, int nq, const uint8_t* train, int nt, int* out3, int* n_out) {
  API_BEGIN;
  XB_REQUIRE(n_out && nq >= 0 && nt >= 0 && (nq == 0 || query) && (nt == 0 || train) && (nq == 0 || out3), "hamming_match: bad arguments");
  *n_out = 0;
  if (nq == 0 || nt == 0) return XIVO_OK;
  cudaStream_t st = ctx->stream;
  DevBuf<uint8_t> dq((size_t)nq * 32), dt((size_t)nt * 32);
  DevBuf<int> dn(2), bt(nq), bd(nq), bq(nt), bqd(nt);
  XB_REQUIRE(dq.ok() && dt.ok() && dn.ok() && bt.ok() && bd.ok() && bq.ok() && bqd.ok(), "cudaMalloc failed");
  const int n2[2] = {nq, nt};
  XB_CUDA(cudaMemcpyAsync(dq.p, query, (size_t)nq * 32, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dt.p, train, (size_t)nt * 32, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dn.p, n2, sizeof(n2), cudaMemcpyHostToDevice, st));
  if (int rc = launch_hamming_nearest(st, dq.p, dn.p, nq, dt.p, dn.p + 1, nt, bt.p, bd.p, 1)) return rc;   // nearest train of every query
  if (int rc = launch_hamming_nearest(st, dt.p, dn.p + 1, nt, dq.p, dn.p, nq, bq.p, bqd.p, 1)) return rc;  // nearest query of every train
  g_launches += 2;
  std::vector<int> hbt(nq), hbd(nq), hbq(nt);
  XB_CUDA(cudaMemcpyAsync(hbt.data(), bt.p, sizeof(int) * nq, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(hbd.data(), bd.p, sizeof(int) * nq, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(hbq.data(), bq.p, sizeof(int) * nt, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  int m = 0;
  for (int i = 0; i < nq; ++i)
    if (hbt[i] >= 0 && hbq[hbt[i]] == i) { out3[3 * m] = i; out3[3 * m + 1] = hbt[i]; out3[3 * m + 2] = hbd[i]; ++m; }
  *n_out = m;
  return XIVO_OK;
}

int xivo_lk_track(xivo_ctx* ctx, const uint8_t* prev, const uint8_t* next, int rows, int cols, int cn, const float* prev_pts,
                  float* next_pts, uint8_t* status, float* err, int npts, int win, int max_level, int max_iter, double eps,
                  int use_initial_flow, double min_eig_threshold) {
  API_BEGIN;
  XB_REQUIRE(prev && next && prev_pts && next_pts && status && npts >= 0 && (cn == 1 || cn == 3), "lk_track: bad arguments");
  if (npts == 0) return XIVO_OK;
  cudaStream_t st = ctx->stream;
  PyrDesc d = make_pyr_desc(rows, cols, cn, win, max_level);
  DevBuf<uint8_t> pyr(2 * d.total);
  DevBuf<float> dp0(2 * (size_t)npts), dp1(2 * (size_t)npts), derr(npts);
  DevBuf<uint8_t> dst(npts);
  DevBuf<int> dn(1);
  XB_REQUIRE(pyr.ok() && dp0.ok() && dp1.ok() && derr.ok() && dst.ok() && dn.ok(), "cudaMalloc failed");
  const size_t ib = (size_t)rows * cols * cn;
  XB_CUDA(cudaMemcpyAsync(pyr.p, prev, ib, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(pyr.p + d.total, next, ib, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dp0.p, prev_pts, sizeof(float) * 2 * npts, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dp1.p, next_pts, sizeof(float) * 2 * npts, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dn.p, &npts, sizeof(int), cudaMemcpyHostToDevice, st));
  int rc = launch_build_pyramid(st, pyr.p, d.total, nullptr, d, 2);  // prev and next as a batch of two
  if (rc) return rc;
  rc = launch_lk_track(st, pyr.p, pyr.p + d.total, 0, nullptr, nullptr, d, dp0.p, dp1.p, dst.p, derr.p, dn.p, npts, 1, win, max_iter, eps,
                       use_initial_flow, min_eig_threshold);
  if (rc) return rc;
  g_launches += d.n_levels;
  XB_CUDA(cudaMemcpyAsync(next_pts, dp1.p, sizeof(float) * 2 * npts, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(status, dst.p, npts, cudaMemcpyDeviceToHost, st));
  if (err) XB_CUDA(cudaMemcpyAsync(err, derr.p, sizeof(float) * npts, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

// Uploads the per-filter tables of one filter and runs the Jacobian/gate kernel.
struct FeatTables {
  DevBuf<CameraParams> cam{1};
  DevBuf<double> X{kPoseDoubles}, groups, fx, fxp, P, R{1};
  DevBuf<int> fref, fsind, nfeat{1};
  DevBuf<FeatJac> jac;
  EkfLayout lay;
  bool ok() const { return cam.ok() && X.ok() && groups.ok() && fx.ok() && fxp.ok() && fref.ok() && fsind.ok() && jac.ok() && P.ok(); }
};

static int upload_tables(cudaStream_t st, FeatTables& t, int G, int F, const double* camera, const double* X24,
                         const double* groups, int n, const double* feat_x, const double* feat_xp, const int* feat_ref,
                         const int* feat_sind, const double* P, double R) {
  XB_REQUIRE(G > 0 && F > 0 && n >= 0 && n <= F, "need 0 <= n <= F");
  for (int i = 0; i < n; ++i)
    XB_REQUIRE(feat_ref[i] >= 0 && feat_ref[i] < G && feat_sind[i] >= 0 && feat_sind[i] < F, "slot index out of range");
  t.lay = EkfLayout{G, F};
  const int N = t.lay.N();
  t.groups.alloc((size_t)G * kGroupDoubles);
  t.fx.alloc((size_t)F * 3);
  t.fxp.alloc((size_t)F * 2);
  t.fref.alloc(F);
  t.fsind.alloc(F);
  t.jac.alloc(F);
  t.P.alloc((size_t)N * N);
  XB_REQUIRE(t.ok(), "cudaMalloc failed");
  CameraParams cp = cam_from(camera);
  XB_CUDA(cudaMemcpyAsync(t.cam.p, &cp, sizeof(cp), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(t.X.p, X24, sizeof(double) * kPoseDoubles, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(t.groups.p, groups, sizeof(double) * G * kGroupDoubles, cudaMemcpyHostToDevice, st));
  if (n) {
    XB_CUDA(cudaMemcpyAsync(t.fx.p, feat_x, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, st));
    XB_CUDA(cudaMemcpyAsync(t.fxp.p, feat_xp, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, st));
    XB_CUDA(cudaMemcpyAsync(t.fref.p, feat_ref, sizeof(int) * n, cudaMemcpyHostToDevice, st));
    XB_CUDA(cudaMemcpyAsync(t.fsind.p, feat_sind, sizeof(int) * n, cudaMemcpyHostToDevice, st));
  }
  XB_CUDA(cudaMemcpyAsync(t.nfeat.p, &n, sizeof(int), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(t.R.p, &R, sizeof(double), cudaMemcpyHostToDevice, st));
  if (P) XB_CUDA(cudaMemcpyAsync(t.P.p, P, sizeof(double) * N * N, cudaMemcpyHostToDevice, st));
  else XB_CUDA(cudaMemsetAsync(t.P.p, 0, sizeof(double) * N * N, st));
  return 0;
}

int xivo_jacobian_batch(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups, int n,
                        const double* feat_x, const double* feat_xp, const int* feat_ref_sind, const int* feat_sind,
                        const double* P, double R, double* J_dense, double* inn, double* mh) {
  API_BEGIN;
  XB_REQUIRE(camera && X24 && groups && (n == 0 || (feat_x && feat_xp && feat_ref_sind && feat_sind)), "jacobian_batch: null input");
  cudaStream_t st = ctx->stream;
  FeatTables t;
  int rc = upload_tables(st, t, G, F, camera, X24, groups, n, feat_x, feat_xp, feat_ref_sind, feat_sind, P, R);
  if (rc) return rc;
  const int N = t.lay.N();
  DevBuf<double> Jd(J_dense ? (size_t)F * 2 * N : 0);
  XB_REQUIRE(Jd.ok(), "cudaMalloc failed");
  rc = launch_jacobian_gate(st, t.lay, t.cam.p, t.X.p, t.groups.p, t.fx.p, t.fxp.p, t.fref.p, t.fsind.p, t.nfeat.p, t.P.p, t.R.p,
                            t.jac.p, J_dense ? Jd.p : nullptr, nullptr, 1);
  if (rc) return rc;
  g_launches += 1;
  std::vector<FeatJac> hj(n);
  if (n) XB_CUDA(cudaMemcpyAsync(hj.data(), t.jac.p, sizeof(FeatJac) * n, cudaMemcpyDeviceToHost, st));
  if (J_dense && n) XB_CUDA(cudaMemcpyAsync(J_dense, Jd.p, sizeof(double) * n * 2 * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    if (inn) { inn[2 * i] = hj[i].inn[0]; inn[2 * i + 1] = hj[i].inn[1]; }
    if (mh) mh[i] = P ? hj[i].mh : -1.0;
  }
  return XIVO_OK;
}

int xivo_mh_gate(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups, int n,
                 const double* feat_x, const double* feat_xp, const int* feat_ref_sind, const int* feat_sind, const double* P,
                 double R, double* mh) {
  if (!P || !mh) { set_error("mh_gate: P and mh are required"); return XIVO_ERR_ARG; }
  return xivo_jacobian_batch(ctx, G, F, camera, X24, groups, n, feat_x, feat_xp, feat_ref_sind, feat_sind, P, R, nullptr, nullptr, mh);
}

int xivo_ekf_update(xivo_ctx* ctx, int N, int M, const double* H, double* P, const double* inn, const double* diagR, double* err) {
  return xivo_ekf_update_ex(ctx, N, M, H, P, inn, diagR, err, 0);
}

int xivo_ekf_update_ex(xivo_ctx* ctx, int N, int M, const double* H, double* P, const double* inn, const double* diagR, double* err,
                       unsigned flags) {
  return xivo_ekf_update_batch(ctx, N, M, 1, H, P, inn, diagR, err, flags, 1);
}

// `batch` independent filters with the same (N, M): H (batch x M x N), P (batch x N x N, in/out), inn / diagR (batch x M), err (batch x N).
// repeat > 1 applies the same update `repeat` times to the ORIGINAL P (restored on the device before every pass) and returns the result of
// one application: with the in-library profiler on (xivo_profile_enable) the report then holds `repeat` samples of ekf_gain / ekf_cov.
int xivo_ekf_update_batch(xivo_ctx* ctx, int N, int M, int batch, const double* H, double* P, const double* inn, const double* diagR, double* err,
                          unsigned flags, int repeat) {
  API_BEGIN;
  XB_REQUIRE((flags & ~(unsigned)XIVO_UPDATE_TF32X3) == 0, "ekf_update: unknown flags");
  XB_REQUIRE(N > 0 && M >= 0 && batch > 0 && repeat >= 1 && P && err && (M == 0 || (H && inn && diagR)), "ekf_update: bad arguments");
  if (M == 0) {
    for (size_t i = 0; i < (size_t)batch * N; ++i) err[i] = 0.0;
    return XIVO_OK;
  }
  cudaStream_t st = ctx->stream;
  const size_t nb = (size_t)batch;
  DevBuf<double> dH(nb * M * N), dP(nb * N * N), dP0(repeat > 1 ? nb * N * N : 0), dinn(nb * M), dR(nb * M), derr(nb * N), dHP(nb * M * N), dKt(nb * M * N);
  XB_REQUIRE(dH.ok() && dP.ok() && dP0.ok() && dinn.ok() && dR.ok() && derr.ok() && dHP.ok() && dKt.ok(), "cudaMalloc failed");
  const bool tensor = (flags & XIVO_UPDATE_TF32X3) != 0;
  const bool v1 = getenv("XIVO_TC_V1") && getenv("XIVO_TC_V1")[0] == '1';
  TcOperands tc;
  DevBuf<uint32_t> dKt32, dHP32;
  if (tensor && !v1) {  // second formulation: TF32 hi / lo operand buffers written by the gain kernel, staged by TMA in the downdate kernel
    const size_t words = tc_operand_words(N, M, batch);
    dKt32.alloc(words); dHP32.alloc(words);
    XB_REQUIRE(dKt32.ok() && dHP32.ok(), "cudaMalloc failed");
    XB_CUDA(cudaMemsetAsync(dKt32.p, 0, words * 4, st));
    XB_CUDA(cudaMemsetAsync(dHP32.p, 0, words * 4, st));
    if (int rc = tc_operands_init(&tc, N, M, batch, dKt32.p, dHP32.p)) return rc;
  }
  XB_CUDA(cudaMemcpyAsync(dH.p, H, sizeof(double) * nb * M * N, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dP.p, P, sizeof(double) * nb * N * N, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dinn.p, inn, sizeof(double) * nb * M, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dR.p, diagR, sizeof(double) * nb * M, cudaMemcpyHostToDevice, st));
  if (repeat > 1) XB_CUDA(cudaMemcpyAsync(dP0.p, dP.p, sizeof(double) * nb * N * N, cudaMemcpyDeviceToDevice, st));
  for (int it = 0; it < repeat; ++it) {
    if (it) XB_CUDA(cudaMemcpyAsync(dP.p, dP0.p, sizeof(double) * nb * N * N, cudaMemcpyDeviceToDevice, st));
    int rc = launch_ekf_update_dense(st, N, M, dH.p, dR.p, dinn.p, dP.p, derr.p, dHP.p, dKt.p, batch, tensor ? 1 : 0, tensor && !v1 ? &tc : nullptr);
    if (rc) return rc;
    g_launches += 2;
  }
  XB_CUDA(cudaMemcpyAsync(P, dP.p, sizeof(double) * nb * N * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(err, derr.p, sizeof(double) * nb * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  if (tensor) XB_REQUIRE(ekf_cov_tc_fault(st) == 0, "ekf_update: the tensor-core downdate timed out waiting for its MMAs");
  return XIVO_OK;
}

int xivo_filter_update(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups, int n,
                       const double* feat_x, const double* feat_xp, const int* feat_ref_sind, const int* feat_sind,
                       const int* sel, int nsel, double R, double* P, double* err, double* H_dense) {
  API_BEGIN;
  XB_REQUIRE(P && err && nsel >= 0 && nsel <= n && (nsel == 0 || sel), "filter_update: bad arguments");
  for (int i = 0; i < nsel; ++i) XB_REQUIRE(sel[i] >= 0 && sel[i] < n, "filter_update: sel out of range");
  cudaStream_t st = ctx->stream;
  FeatTables t;
  int rc = upload_tables(st, t, G, F, camera, X24, groups, n, feat_x, feat_xp, feat_ref_sind, feat_sind, P, R);
  if (rc) return rc;
  const int N = t.lay.N(), Mmax = 2 * F;
  DevBuf<int> dsel(F), dnsel(1);
  DevBuf<double> derr(N), dHP((size_t)Mmax * N), dKt((size_t)Mmax * N), dH(H_dense ? (size_t)Mmax * N : 0);
  XB_REQUIRE(dsel.ok() && dnsel.ok() && derr.ok() && dHP.ok() && dKt.ok() && dH.ok(), "cudaMalloc failed");
  if (nsel) XB_CUDA(cudaMemcpyAsync(dsel.p, sel, sizeof(int) * nsel, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dnsel.p, &nsel, sizeof(int), cudaMemcpyHostToDevice, st));
  rc = launch_jacobian_gate(st, t.lay, t.cam.p, t.X.p, t.groups.p, t.fx.p, t.fxp.p, t.fref.p, t.fsind.p, t.nfeat.p, t.P.p, t.R.p,
                            t.jac.p, nullptr, nullptr, 1);
  if (rc) return rc;
  rc = launch_ekf_update(st, t.lay, t.jac.p, dsel.p, dnsel.p, t.R.p, t.P.p, derr.p, dHP.p, dKt.p, H_dense ? dH.p : nullptr, 1);
  if (rc) return rc;
  g_launches += 3;
  XB_CUDA(cudaMemcpyAsync(P, t.P.p, sizeof(double) * N * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(err, derr.p, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
  if (H_dense && nsel) XB_CUDA(cudaMemcpyAsync(H_dense, dH.p, sizeof(double) * 2 * nsel * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

// Packs n edit ops (xivo_cov_edit format) into out, checking them against the state dimension.
static int pack_edits(int N, const int* ops, const double* blk, int n, EditOp* out) {
  for (int i = 0; i < n; ++i) {
    EditOp& h = out[i];
    h.type = ops[4 * i]; h.a = ops[4 * i + 1]; h.b = ops[4 * i + 2]; h.n = ops[4 * i + 3];
    XB_REQUIRE(h.type >= 0 && h.type <= 2, "filter_update_batch: unknown edit op");
    const int w = h.type == 2 ? 3 : h.n;
    XB_REQUIRE(w >= 0 && h.a >= 0 && h.a + w <= N && (h.type != 1 || (h.b >= 0 && h.b + w <= N)), "filter_update_batch: edit op out of range");
    for (int k = 0; k < 9; ++k) h.blk[k] = (blk && h.type == 2) ? blk[9 * i + k] : 0.0;
  }
  return 0;
}

// The gate + update phases of Batch (estimator.cu: process_visual) for `batch` filters, `npass` times on the same device buffers.
int xivo_filter_update_batch(xivo_ctx* ctx, int G, int F, int batch, int npass, const double* camera, const double* X24, const double* groups,
                             const int* nfeat, const double* feat_x, const double* feat_xp, const int* feat_ref, const int* feat_sind,
                             const double* Rmeas, const double* P, const int* pre_nops, const int* pre_ops, const double* pre_blk,
                             const int* nsel, const int* sel, const int* post_nops, const int* post_ops, const double* post_blk, unsigned flags,
                             double* P_out, double* err, double* mh, double* diag) {
  API_BEGIN;
  XB_REQUIRE((flags & ~(unsigned)(XIVO_UPDATE_TF32X3 | XIVO_UPDATE_FULL_J)) == 0, "filter_update_batch: unknown flags");
  XB_REQUIRE(G > 0 && F > 0 && batch > 0 && npass > 0 && camera && X24 && groups && nfeat && feat_x && feat_xp && feat_ref && feat_sind && Rmeas &&
                 P && pre_nops && nsel && sel && post_nops && P_out && err && mh && diag,
             "filter_update_batch: bad arguments");
  const EkfLayout lay{G, F};
  const int N = lay.N(), Mmax = 2 * F;
  const size_t nb = (size_t)batch, NN = (size_t)N * N;
  for (int b = 0; b < batch; ++b) {
    XB_REQUIRE(nfeat[b] >= 0 && nfeat[b] <= F, "filter_update_batch: need 0 <= nfeat <= F");
    for (int i = 0; i < nfeat[b]; ++i) {
      const size_t fi = (size_t)b * F + i;
      XB_REQUIRE(feat_ref[fi] >= 0 && feat_ref[fi] < G && feat_sind[fi] >= 0 && feat_sind[fi] < F, "filter_update_batch: slot index out of range");
    }
  }
  // edit lists of every pass, packed in (pass, filter) order; first* / n*: npass x batch
  std::vector<int> first_pre(npass * nb), first_post(npass * nb);
  int npre = 0, npost = 0;
  for (size_t q = 0; q < npass * nb; ++q) {
    XB_REQUIRE(pre_nops[q] >= 0 && post_nops[q] >= 0 && nsel[q] >= 0 && nsel[q] <= nfeat[q % nb], "filter_update_batch: bad counts");
    for (int k = 0; k < nsel[q]; ++k) XB_REQUIRE(sel[q * F + k] >= 0 && sel[q * F + k] < nfeat[q % nb], "filter_update_batch: sel out of range");
    first_pre[q] = npre; npre += pre_nops[q];
    first_post[q] = npost; npost += post_nops[q];
  }
  XB_REQUIRE((npre == 0 || pre_ops) && (npost == 0 || post_ops), "filter_update_batch: null edit list");
  std::vector<EditOp> hops(std::max(1, npre + npost));
  if (int rc = pack_edits(N, pre_ops, pre_blk, npre, hops.data())) return rc;
  if (int rc = pack_edits(N, post_ops, post_blk, npost, hops.data() + npre)) return rc;
  for (int& f : first_post) f += npre;
  std::vector<CameraParams> hcam(nb);
  for (size_t b = 0; b < nb; ++b) hcam[b] = cam_from(camera + 11 * b);

  cudaStream_t st = ctx->stream;
  DevBuf<CameraParams> dcam(nb);
  DevBuf<double> dX(nb * kPoseDoubles), dgroups(nb * G * kGroupDoubles), dfx(nb * F * 3), dfxp(nb * F * 2), dR(nb), dP(nb * NN), derr(nb * N),
      dmh(nb * F), ddiag(nb * N), dHP(nb * Mmax * N), dKt(nb * Mmax * N);
  DevBuf<int> dfref(nb * F), dfsind(nb * F), dnfeat(nb), dsel(npass * nb * F), dnsel(npass * nb), dfirst(4 * npass * nb);
  DevBuf<FeatJac> djac(nb * F);
  DevBuf<EditOp> dops(hops.size());
  XB_REQUIRE(dcam.ok() && dX.ok() && dgroups.ok() && dfx.ok() && dfxp.ok() && dR.ok() && dP.ok() && derr.ok() && dmh.ok() && ddiag.ok() && dHP.ok() &&
                 dKt.ok() && dfref.ok() && dfsind.ok() && dnfeat.ok() && dsel.ok() && dnsel.ok() && dfirst.ok() && djac.ok() && dops.ok(),
             "cudaMalloc failed");
  const bool tensor = (flags & XIVO_UPDATE_TF32X3) != 0, full_j = (flags & XIVO_UPDATE_FULL_J) != 0;
  const bool v1 = getenv("XIVO_TC_V1") && getenv("XIVO_TC_V1")[0] == '1';
  TcOperands tc;
  DevBuf<uint32_t> dKt32, dHP32;
  if (tensor && !v1) {  // as Batch: allocated and zeroed once; each update rewrites only the k-blocks its M covers
    const size_t words = tc_operand_words(N, Mmax, batch);
    dKt32.alloc(words); dHP32.alloc(words);
    XB_REQUIRE(dKt32.ok() && dHP32.ok(), "cudaMalloc failed");
    XB_CUDA(cudaMemsetAsync(dKt32.p, 0, words * 4, st));
    XB_CUDA(cudaMemsetAsync(dHP32.p, 0, words * 4, st));
    if (int rc = tc_operands_init(&tc, N, Mmax, batch, dKt32.p, dHP32.p)) return rc;
  }
  // [pre nops | pre first | post nops | post first], each npass x batch
  std::vector<int> hfirst(4 * npass * nb);
  for (size_t q = 0; q < npass * nb; ++q) {
    hfirst[q] = pre_nops[q]; hfirst[npass * nb + q] = first_pre[q];
    hfirst[2 * npass * nb + q] = post_nops[q]; hfirst[3 * npass * nb + q] = first_post[q];
  }
  XB_CUDA(cudaMemcpyAsync(dcam.p, hcam.data(), sizeof(CameraParams) * nb, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dX.p, X24, sizeof(double) * nb * kPoseDoubles, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dgroups.p, groups, sizeof(double) * nb * G * kGroupDoubles, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfx.p, feat_x, sizeof(double) * nb * F * 3, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfxp.p, feat_xp, sizeof(double) * nb * F * 2, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfref.p, feat_ref, sizeof(int) * nb * F, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfsind.p, feat_sind, sizeof(int) * nb * F, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dnfeat.p, nfeat, sizeof(int) * nb, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dR.p, Rmeas, sizeof(double) * nb, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dP.p, P, sizeof(double) * nb * NN, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dsel.p, sel, sizeof(int) * npass * nb * F, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dnsel.p, nsel, sizeof(int) * npass * nb, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dfirst.p, hfirst.data(), sizeof(int) * hfirst.size(), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dops.p, hops.data(), sizeof(EditOp) * hops.size(), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemsetAsync(dmh.p, 0, sizeof(double) * nb * F, st));  // the gate writes features < nfeat only
  for (int p = 0; p < npass; ++p) {
    const size_t q = (size_t)p * nb;
    const int* pre_n = dfirst.p + q;
    const int* pre_f = dfirst.p + npass * nb + q;
    const int* post_n = dfirst.p + 2 * npass * nb + q;
    const int* post_f = dfirst.p + 3 * npass * nb + q;
    int rc = launch_jacobian_gate(st, lay, dcam.p, dX.p, dgroups.p, dfx.p, dfxp.p, dfref.p, dfsind.p, dnfeat.p, dP.p, dR.p, djac.p, nullptr, dmh.p,
                                  batch, dops.p, pre_f, pre_n, ddiag.p);
    if (rc) return rc;
    rc = launch_ekf_update(st, lay, djac.p, dsel.p + q * F, dnsel.p + q, dR.p, dP.p, derr.p, dHP.p, dKt.p, nullptr, batch, tensor ? 1 : 0, dops.p,
                           post_f, post_n, tensor && !v1 ? &tc : nullptr, full_j ? 1 : 0);
    if (rc) return rc;
    g_launches += 3;
    XB_CUDA(cudaMemcpyAsync(P_out + q * NN, dP.p, sizeof(double) * nb * NN, cudaMemcpyDeviceToHost, st));
    XB_CUDA(cudaMemcpyAsync(err + q * N, derr.p, sizeof(double) * nb * N, cudaMemcpyDeviceToHost, st));
    XB_CUDA(cudaMemcpyAsync(mh + q * F, dmh.p, sizeof(double) * nb * F, cudaMemcpyDeviceToHost, st));
    XB_CUDA(cudaMemcpyAsync(diag + q * N, ddiag.p, sizeof(double) * nb * N, cudaMemcpyDeviceToHost, st));
  }
  XB_CUDA(cudaStreamSynchronize(st));
  if (tensor) XB_REQUIRE(ekf_cov_tc_fault(st) == 0, "filter_update_batch: the tensor-core downdate timed out waiting for its MMAs");
  return XIVO_OK;
}

int xivo_subfilter_batch(xivo_ctx* ctx, const double* camera, const double* X24, int n, const double* x, const double* P33,
                         const double* xp, const double* ref, const double* outlier_counter, double Rtri, double mh_thresh,
                         double* x_out, double* P33_out, double* outlier_counter_out) {
  API_BEGIN;
  XB_REQUIRE(camera && X24 && n >= 0, "subfilter_batch: bad arguments");
  if (n == 0) return XIVO_OK;
  cudaStream_t st = ctx->stream;
  std::vector<SubfilterIn> hin(n);
  for (int i = 0; i < n; ++i) {
    memcpy(hin[i].x, x + 3 * i, 24);
    memcpy(hin[i].P, P33 + 9 * i, 72);
    memcpy(hin[i].xp, xp + 2 * i, 16);
    memcpy(hin[i].ref, ref + 12 * i, 96);
    hin[i].outlier_counter = outlier_counter[i];
    hin[i].filter = 0;
    hin[i].pad = 0;
  }
  DevBuf<SubfilterIn> din(n);
  DevBuf<SubfilterOut> dout(n);
  DevBuf<CameraParams> dcam(1);
  DevBuf<double> dX(kPoseDoubles);
  XB_REQUIRE(din.ok() && dout.ok() && dcam.ok() && dX.ok(), "cudaMalloc failed");
  CameraParams cp = cam_from(camera);
  XB_CUDA(cudaMemcpyAsync(dcam.p, &cp, sizeof(cp), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dX.p, X24, sizeof(double) * kPoseDoubles, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(din.p, hin.data(), sizeof(SubfilterIn) * n, cudaMemcpyHostToDevice, st));
  int rc = launch_subfilter(st, dcam.p, dX.p, din.p, dout.p, n, Rtri, mh_thresh);
  if (rc) return rc;
  g_launches += 1;
  std::vector<SubfilterOut> hout(n);
  XB_CUDA(cudaMemcpyAsync(hout.data(), dout.p, sizeof(SubfilterOut) * n, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    memcpy(x_out + 3 * i, hout[i].x, 24);
    memcpy(P33_out + 9 * i, hout[i].P, 72);
    outlier_counter_out[i] = hout[i].outlier_counter;
  }
  return XIVO_OK;
}

int xivo_oos_project(xivo_ctx* ctx, int G, int F, const double* camera, const double* gbc12, int nf, int k, const double* Xs,
                     const double* obs_pose, const int* obs_sind, const double* obs_xp, double* Hf, double* Hx, double* inn,
                     double* Hx_proj, double* inn_proj) {
  API_BEGIN;
  XB_REQUIRE(camera && gbc12 && nf >= 0 && Xs && obs_pose && obs_sind && obs_xp && Hf && Hx && inn && Hx_proj && inn_proj,
             "oos_project: null argument");
  if (nf == 0) return XIVO_OK;
  for (int i = 0; i < nf * k; ++i) XB_REQUIRE(obs_sind[i] >= 0 && obs_sind[i] < G, "oos_project: group slot out of range");
  cudaStream_t st = ctx->stream;
  EkfLayout lay{G, F};
  const int N = lay.N(), R2 = 2 * k;
  DevBuf<CameraParams> dcam(1);
  DevBuf<double> dg(12), dXs((size_t)nf * 3), dpose((size_t)nf * k * 12), dxp((size_t)nf * k * 2), dHf((size_t)nf * R2 * 3),
      dHx((size_t)nf * R2 * N), dinn((size_t)nf * R2), dHp((size_t)nf * R2 * N), dip((size_t)nf * R2);
  DevBuf<int> dsind((size_t)nf * k);
  XB_REQUIRE(dcam.ok() && dg.ok() && dXs.ok() && dpose.ok() && dxp.ok() && dHf.ok() && dHx.ok() && dinn.ok() && dHp.ok() &&
                 dip.ok() && dsind.ok(),
             "cudaMalloc failed");
  CameraParams cp = cam_from(camera);
  XB_CUDA(cudaMemcpyAsync(dcam.p, &cp, sizeof(cp), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dg.p, gbc12, 96, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dXs.p, Xs, sizeof(double) * nf * 3, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dpose.p, obs_pose, sizeof(double) * nf * k * 12, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dxp.p, obs_xp, sizeof(double) * nf * k * 2, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dsind.p, obs_sind, sizeof(int) * nf * k, cudaMemcpyHostToDevice, st));
  int rc = launch_oos(st, lay, dcam.p, dg.p, dXs.p, dpose.p, dsind.p, dxp.p, k, nf, dHf.p, dHx.p, dinn.p, dHp.p, dip.p);
  if (rc) return rc;
  g_launches += 1;
  XB_CUDA(cudaMemcpyAsync(Hf, dHf.p, sizeof(double) * nf * R2 * 3, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(Hx, dHx.p, sizeof(double) * nf * R2 * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(inn, dinn.p, sizeof(double) * nf * R2, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(Hx_proj, dHp.p, sizeof(double) * nf * R2 * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaMemcpyAsync(inn_proj, dip.p, sizeof(double) * nf * R2, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

int xivo_cov_edit(xivo_ctx* ctx, int N, double* P, const int* ops, const double* blk, int nops) {
  API_BEGIN;
  XB_REQUIRE(N > 0 && P && nops >= 0 && (nops == 0 || ops), "cov_edit: bad arguments");
  if (nops == 0) return XIVO_OK;
  std::vector<EditOp> h(nops);
  for (int i = 0; i < nops; ++i) {
    h[i].type = ops[4 * i];
    h[i].a = ops[4 * i + 1];
    h[i].b = ops[4 * i + 2];
    h[i].n = ops[4 * i + 3];
    XB_REQUIRE(h[i].type >= 0 && h[i].type <= 2, "cov_edit: unknown op");
    const int n = h[i].type == 2 ? 3 : h[i].n;
    XB_REQUIRE(h[i].a >= 0 && h[i].a + n <= N && (h[i].type != 1 || (h[i].b >= 0 && h[i].b + n <= N)), "cov_edit: range");
    for (int k = 0; k < 9; ++k) h[i].blk[k] = (blk && h[i].type == 2) ? blk[9 * i + k] : 0.0;
  }
  cudaStream_t st = ctx->stream;
  DevBuf<double> dP((size_t)N * N);
  DevBuf<EditOp> dops(nops);
  DevBuf<int> dn(1);
  XB_REQUIRE(dP.ok() && dops.ok() && dn.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemcpyAsync(dP.p, P, sizeof(double) * N * N, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dops.p, h.data(), sizeof(EditOp) * nops, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dn.p, &nops, sizeof(int), cudaMemcpyHostToDevice, st));
  int rc = launch_cov_edit(st, N, dP.p, dops.p, dn.p, nops, 1);
  if (rc) return rc;
  g_launches += 1;
  XB_CUDA(cudaMemcpyAsync(P, dP.p, sizeof(double) * N * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

int xivo_cov_propagate(xivo_ctx* ctx, int N, double* P, const double* Phi, const double* Pmm) {
  API_BEGIN;
  XB_REQUIRE(N >= 23 && P && Phi && Pmm, "cov_propagate: bad arguments");
  cudaStream_t st = ctx->stream;
  DevBuf<double> dP((size_t)N * N), dPhi(529), dPmm(529);
  XB_REQUIRE(dP.ok() && dPhi.ok() && dPmm.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemcpyAsync(dP.p, P, sizeof(double) * N * N, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dPhi.p, Phi, sizeof(double) * 529, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dPmm.p, Pmm, sizeof(double) * 529, cudaMemcpyHostToDevice, st));
  int rc = launch_cov_propagate(st, N, dP.p, dPhi.p, dPmm.p, nullptr, 1);
  if (rc) return rc;
  g_launches += 1;
  XB_CUDA(cudaMemcpyAsync(P, dP.p, sizeof(double) * N * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

int xivo_imu_cov_propagate(xivo_ctx* ctx, int N, double* P, int nstages, const double* stage16, const double* g3, const double* qimu12,
                           const double* qmodel23, int stages_per_step) {
  API_BEGIN;
  XB_REQUIRE(N >= 23 && P && nstages >= 0 && nstages <= kMaxStages && (nstages == 0 || stage16) && g3 && qimu12 && qmodel23 &&
                 (stages_per_step == 7 || stages_per_step == 4) && nstages % stages_per_step == 0,
             "imu_cov_propagate: bad arguments");
  if (nstages == 0) return XIVO_OK;
  static_assert(sizeof(ImuStage) == 16 * sizeof(double), "ImuStage layout");
  // The kernel reads one record per sub-step and rebuilds the rotation and rates of its other stages: the sub-step takes R, the rates
  // and h of its first stage, and the rate slopes from the stage whose rates lie furthest from them (cin = 1 for Prince-Dormand, 1/2 for RK4).
  const bool pd = stages_per_step == 7;
  const int nsteps = nstages / stages_per_step, sfar = pd ? 5 : 1;
  double cs_far, cin_far;
  imu_stage_coef(pd, sfar, &cs_far, &cin_far);
  std::vector<ImuStep> steps(nsteps);
  for (int k = 0; k < nsteps; ++k) {
    const double* s0 = stage16 + (size_t)16 * stages_per_step * k;
    const double* sf = s0 + 16 * sfar;
    ImuStep& r = steps[k];
    memcpy(r.R, s0, 72); memcpy(r.gc, s0 + 9, 24); memcpy(r.ac, s0 + 12, 24);
    r.h = s0[15];
    const double t = cin_far * fabs(r.h);
    for (int e = 0; e < 3; ++e) {
      r.dgc[e] = t > 0 ? (sf[9 + e] - s0[9 + e]) / t : 0.0;
      r.dac[e] = t > 0 ? (sf[12 + e] - s0[12 + e]) / t : 0.0;
    }
  }
  cudaStream_t st = ctx->stream;
  ImuConst ic;
  memcpy(ic.g, g3, 24); memcpy(ic.qimu, qimu12, 96); memcpy(ic.qmodel, qmodel23, 184);
  ic.stages_per_step = stages_per_step; ic.pad = 0;
  const int zero = 0;
  DevBuf<double> dP((size_t)N * N);
  DevBuf<ImuStep> dS(nsteps);
  DevBuf<ImuConst> dC(1);
  DevBuf<int> dn(1), df(1);
  XB_REQUIRE(dP.ok() && dS.ok() && dC.ok() && dn.ok() && df.ok(), "cudaMalloc failed");
  XB_CUDA(cudaMemcpyAsync(dP.p, P, sizeof(double) * N * N, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dS.p, steps.data(), sizeof(ImuStep) * nsteps, cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dC.p, &ic, sizeof(ic), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(dn.p, &nsteps, sizeof(int), cudaMemcpyHostToDevice, st));
  XB_CUDA(cudaMemcpyAsync(df.p, &zero, sizeof(int), cudaMemcpyHostToDevice, st));
  int rc = launch_imu_cov_propagate(st, N, dP.p, dS.p, df.p, dn.p, dC.p, 1);
  if (rc) return rc;
  g_launches += 1;
  XB_CUDA(cudaMemcpyAsync(P, dP.p, sizeof(double) * N * N, cudaMemcpyDeviceToHost, st));
  XB_CUDA(cudaStreamSynchronize(st));
  return XIVO_OK;
}

// Host-side entry point (no device work): the tracker's homography outlier mask, see include/xivo_b200.h.
int xivo_find_homography_mask(const float* pts0, const float* pts1, int n, int method, double reproj_thresh, int max_iters, double confidence,
                              uint8_t* mask, int* ok) {
  if (!pts0 || !pts1 || !mask || n < 0 || (method != xb::homography::kLMEDS && method != xb::homography::kRANSAC)) {
    set_error("find_homography_mask: bad arguments (method must be 4 = LMEDS or 8 = RANSAC)");
    return XIVO_ERR_ARG;
  }
  std::vector<uint8_t> m;
  const bool good = xb::homography::find_homography_mask(pts0, pts1, n, method, reproj_thresh, max_iters, confidence, m);
  for (int i = 0; i < n; ++i) mask[i] = m[i];
  if (ok) *ok = good ? 1 : 0;
  return 0;
}

}  // extern "C"

/*
 * xivo_b200.h — C ABI of the CUDA-native (H100, sm_90a) XIVO inner loop.
 *
 * The reference (ucla-vision/xivo) has no FFI/plugin layer: its boundary is the C++ class API
 * (src/estimator.h:115-231, src/tracker.h:25-54) and the pybind11 module
 * (pybind11/pyxivo.cpp:332-398).  This header is the thin C layer those would bind to; every
 * entry point names the reference interface it replaces (paths relative to the reference
 * repository root).  Conventions:
 *   - plain pointers and sizes only; all matrices row-major, fp64 unless stated;
 *   - every function returns 0 on success, a negative code on failure (the reference's
 *     LOG(FATAL)/throw sites are mapped to codes; nothing throws across this boundary) and
 *     xivo_last_error() describes the failure;
 *   - buffers are HOST memory: each call copies in, runs the CUDA kernels, copies out;
 *   - there is no CPU implementation behind this interface: without a CUDA device every
 *     call fails with XIVO_ERR_CUDA.
 */
#ifndef XIVO_B200_H_
#define XIVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XIVO_OK 0
#define XIVO_ERR_ARG (-1)   /* invalid argument (reference: CHECK / LOG(FATAL) on bad config) */
#define XIVO_ERR_CUDA (-2)  /* CUDA runtime failure, incl. "no device" */
#define XIVO_ERR_STATE (-3) /* call not valid in the current state (reference: throw std::invalid_argument) */
#define XIVO_ERR_SLOTS (-4) /* out of group/feature slots (reference: throw std::runtime_error, estimator.cpp:821,844) */

typedef struct xivo_ctx xivo_ctx; /* one CUDA device + stream + scratch */

/* Camera description shared by all entry points: {model, rows, cols, fx, fy, cx, cy, k0, k1, k2, k3}
 * model 0 = pinhole (common/camera_pinhole.h), 3 = equidistant (common/camera_equidist.h);
 * values of DistortionType, common/camera_base.h:13-18. */
#define XIVO_CAMERA_DOUBLES 11

const char* xivo_last_error(void);
int xivo_version(void);
int xivo_ctx_create(int device, xivo_ctx** out);
void xivo_ctx_destroy(xivo_ctx* ctx);
/* number of kernels this library has launched in the calling process (for bench.py's gpu_launches) */
unsigned long long xivo_launch_count(void);
/* the cudaStream_t every kernel of this context is launched on (so callers can bracket work with CUDA events) */
void* xivo_ctx_stream(xivo_ctx* ctx);

/* ---------------------------------------------------------------------------------------------
 * Kernel-level entry points (parity-test surface; SURVEY.md §8b).
 * ------------------------------------------------------------------------------------------- */

/* Bytes / level geometry of the pyramid cv::buildOpticalFlowPyramid would produce for these
 * arguments (levels stop when the next one would be <= win).  Replaces the pyramid built at
 * src/tracker.cpp:476,493.  Levels are stored unpadded, back to back, 16-byte aligned. */
unsigned long long xivo_pyramid_layout(int rows, int cols, int cn, int win, int max_level, int* n_levels,
                                       int* level_rows /*[8]*/, int* level_cols /*[8]*/,
                                       unsigned long long* level_off /*[8]*/);

/* img: rows x cols x cn uint8 (cn = 1 or 3, interleaved).  out: xivo_pyramid_layout() bytes. */
int xivo_build_pyramid(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, int win, int max_level,
                       uint8_t* out);

/* BRIEF-32 descriptors at the given keypoints; replaces extractor_->compute() (src/tracker.cpp:231-234, :361-363, :536-545) for the
 * "BRIEF" descriptor.  kp_xy: n (x, y) float pairs.  desc: n x 32 bytes, valid: n flags; keypoints closer than 28 px to the image border are
 * dropped by OpenCV's extractor: they get valid = 0 and a zero descriptor here, the caller compacts.  3-channel input is converted to grey.
 * The 256 test pairs are this library's own table (xivo_b200/csrc/brief_pattern.h): opencv_contrib's is not vendored in the reference. */
int xivo_brief_describe(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, const float* kp_xy, int n, uint8_t* desc,
                        uint8_t* valid);

/* cv::BFMatcher(NORM_HAMMING, crossCheck = true).knnMatch(query, train, 1, noArray(), compactResult = true) for 32-byte descriptors;
 * replaces matcher_->knnMatch at src/tracker.cpp:261-262, :378-379 and the popcount distance of src/fastbrief.cpp:53-93.
 * out3: up to nq (queryIdx, trainIdx, distance) triples in query order; *n_out their number. */
int xivo_hamming_match(xivo_ctx* ctx, const uint8_t* query, int nq, const uint8_t* train, int nt, int* out3, int* n_out);

/* FAST-9/16 + non-max suppression; replaces detector_->detect() at src/tracker.cpp:224 for the
 * "FAST" detector (src/tracker.cpp:39-42).  3-channel input is converted to grey first, as
 * OpenCV does.  Output is raster ordered (y major) like OpenCV's; kp_xy = (x, y) pairs.
 * *n_kp receives the total found (may exceed max_kp; only max_kp are stored). */
int xivo_fast_detect(xivo_ctx* ctx, const uint8_t* img, int rows, int cols, int cn, int threshold, int nonmax,
                     int* kp_xy, int* kp_score, int max_kp, int* n_kp);

/* Pyramidal Lucas-Kanade; replaces cv::calcOpticalFlowPyrLK at src/tracker.cpp:526-528
 * (criteria COUNT|EPS, default minEigThreshold 1e-4, flags = OPTFLOW_USE_INITIAL_FLOW when
 * use_initial_flow).  next_pts is in/out (initial guess -> result).  Multi-channel images are
 * tracked on all channels, like the reference which feeds the 8UC3 cv::imread result. */
int xivo_lk_track(xivo_ctx* ctx, const uint8_t* prev, const uint8_t* next, int rows, int cols, int cn,
                  const float* prev_pts, float* next_pts, uint8_t* status, float* err, int npts, int win,
                  int max_level, int max_iter, double eps, int use_initial_flow, double min_eig_threshold);

/* In-state measurement Jacobians for n features of one filter; replaces
 * Estimator::ComputeInstateJacobians -> Feature::ComputeJacobian (src/update.cpp:24-32,
 * src/feature.cpp:542-656).  G/F are the compile-time kMaxGroup/kMaxFeature of the reference
 * (src/core.h:92-105); N = 23 + 6G + 3F.
 *   X24     : Rsb(9) Tsb(3) Rbc(9) Tbc(3)
 *   groups  : G x {Rsb(9) Tsb(3)} indexed by state slot (Group::sind)
 *   feat_*  : local state x (X/Z, Y/Z, log Z), last pixel measurement, reference-group slot, own slot
 *   P       : N x N covariance or NULL (then mh is not computed and set to -1)
 * Outputs: J_dense n x 2 x N (Feature::J_), inn n x 2 (Feature::inn_), mh n = Mahalanobis
 * distance of Estimator::MHGating (src/update.cpp:60-69) with measurement variance R. */
int xivo_jacobian_batch(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups,
                        int n, const double* feat_x, const double* feat_xp, const int* feat_ref_sind,
                        const int* feat_sind, const double* P, double R, double* J_dense, double* inn, double* mh);

/* Same inputs, distances only (Estimator::MHGating, src/update.cpp:50-69). */
int xivo_mh_gate(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups, int n,
                 const double* feat_x, const double* feat_xp, const int* feat_ref_sind, const int* feat_sind,
                 const double* P, double R, double* mh);

/* Dense EKF measurement update; replaces Estimator::UpdateJosephForm (src/estimator.cpp:1257-1288).
 * H: M x N, P: N x N (in/out), inn: M, diagR: M, err: N (= K inn). */
int xivo_ekf_update(xivo_ctx* ctx, int N, int M, const double* H, double* P, const double* inn, const double* diagR,
                    double* err);

/* Same update with options.  XIVO_UPDATE_TF32X3: the rank-M covariance downdate P -= K (H P) runs on the
 * tensor cores (wgmma.mma_async .tf32, operands split hi+lo = "3xTF32", fp32 accumulator in registers) instead of
 * fp64 CUDA cores: the "fp32 covariance" mode (BASELINE configs[2]); gain, innovation and the storage of P stay
 * fp64.  Tolerance vs the fp64 update, elementwise: |dP_ij| <= 1e-5 * sqrt(P_ii P_jj) (tests/test_gpu_ekf.py, tests/test_gpu_ekf_batch.py).
 * Measured on an H100 80GB HBM3 (400 W limit) with estimator-like H (feature Jacobians sharing group columns) and variances from 1e-8 to
 * 1: at most 1.3e-6 for ekf_cov_tc2_kernel and 2.2e-6 for the first kernel (N = 299, M up to 124), consistent with the 3xTF32 product
 * error 2^-22 sum_k |K_ik||HP_kj| (up to 1.2e-6 of sqrt(P_ii P_jj) on these inputs) plus the fp32 accumulation. */
#define XIVO_UPDATE_TF32X3 1u
int xivo_ekf_update_ex(xivo_ctx* ctx, int N, int M, const double* H, double* P, const double* inn, const double* diagR,
                       double* err, unsigned flags);
/* The same update for `batch` independent filters of one (N, M) in a single launch pair: H (batch x M x N), P (batch x N x N, in / out),
 * inn, diagR (batch x M), err (batch x N).  repeat > 1 re-applies the update to the original P `repeat` times on the device (kernel timing
 * through xivo_profile_enable / xivo_profile_report) and returns the result of one application.
 * Replaces: a loop of Estimator::UpdateJosephForm calls (/root/reference/src/estimator.cpp:1257-1288), one per filter. */
int xivo_ekf_update_batch(xivo_ctx* ctx, int N, int M, int batch, const double* H, double* P, const double* inn, const double* diagR,
                          double* err, unsigned flags, int repeat);

/* Production form of the update: Jacobians -> stack H for the selected features with
 * Feature::FillJacobianBlock semantics (src/feature.cpp:658-684) -> update; replaces
 * Estimator::FilterUpdate (src/update.cpp:120-153) up to AbsorbError.  sel: nsel indices into the
 * feature arrays, in update order.  H_dense (2*nsel x N) may be NULL. */
int xivo_filter_update(xivo_ctx* ctx, int G, int F, const double* camera, const double* X24, const double* groups,
                       int n, const double* feat_x, const double* feat_xp, const int* feat_ref_sind,
                       const int* feat_sind, const int* sel, int nsel, double R, double* P, double* err,
                       double* H_dense);

/* The gate and update phases of the estimator for `batch` filters of one layout (G, F), run `npass` times in a row on the same device
 * buffers, with the launches and arguments Estimator batches use (Jacobian / gate kernel with the pre-gate edit list, then the gain and
 * downdate kernels with the post-gate edit list).  The TF32 operand buffers of XIVO_UPDATE_TF32X3 are zeroed once per call, not between
 * passes, as in a running estimator.
 *   per filter b     : camera (11), X24 (24), groups (G x 12), nfeat[b] <= F features in feat_x (F x 3), feat_xp (F x 2),
 *                      feat_ref / feat_sind (F), Rmeas[b], the initial covariance P (N x N)
 *   per pass p and b : pre_nops[p * batch + b] ops of the pre-gate list, post_nops[...] of the post-gate list, nsel[p * batch + b]
 *                      indices into the feature table at sel + (p * batch + b) * F.  The ops of both lists are packed in (pass, filter)
 *                      order, in the xivo_cov_edit format (4 ints + 9 doubles each)
 *   flags            : XIVO_UPDATE_TF32X3, XIVO_UPDATE_FULL_J (stack the rows of J unchanged, as the 1-point RANSAC update does,
 *                      instead of Feature::FillJacobianBlock's layout); XIVO_TC_V1=1 in the environment selects the first tensor-core kernel
 * Outputs after every pass: P_out (npass x batch x N x N), err (npass x batch x N; NaN where S was not positive definite, the filter's P
 * then keeps its post-gate value), mh (npass x batch x F; 0 beyond nfeat), diag (npass x batch x N: diag(P) after the pre-gate edits). */
#define XIVO_UPDATE_FULL_J 2u
int xivo_filter_update_batch(xivo_ctx* ctx, int G, int F, int batch, int npass, const double* camera, const double* X24,
                             const double* groups, const int* nfeat, const double* feat_x, const double* feat_xp, const int* feat_ref,
                             const int* feat_sind, const double* Rmeas, const double* P, const int* pre_nops, const int* pre_ops,
                             const double* pre_blk, const int* nsel, const int* sel, const int* post_nops, const int* post_ops,
                             const double* post_blk, unsigned flags, double* P_out, double* err, double* mh, double* diag);

/* Depth sub-filter for n not-in-state features; replaces Feature::SubfilterUpdate
 * (src/feature.cpp:246-297).  ref: n x {Rsb(9) Tsb(3)} of each feature's reference group. */
int xivo_subfilter_batch(xivo_ctx* ctx, const double* camera, const double* X24, int n, const double* x,
                         const double* P33, const double* xp, const double* ref, const double* outlier_counter,
                         double Rtri, double mh_thresh, double* x_out, double* P33_out, double* outlier_counter_out);

/* OOS / MSCKF Jacobian blocks and left-nullspace projection for nf features with k observations
 * each; replaces Feature::ComputeOOSJacobian[Internal] + SlowGivens (src/oos.cpp:8-89,
 * src/helpers.cpp:13-23).  Hx_proj: nf x 2k x N (first 2k-3 rows valid), inn_proj: nf x 2k. */
int xivo_oos_project(xivo_ctx* ctx, int G, int F, const double* camera, const double* gbc12, int nf, int k,
                     const double* Xs, const double* obs_pose, const int* obs_sind, const double* obs_xp,
                     double* Hf, double* Hx, double* inn, double* Hx_proj, double* inn_proj);

/* Tracker-level outlier rejection: the inlier mask of cv::findHomography(pts0, pts1, method, reproj_thresh, mask, max_iters,
 * confidence) as Tracker::OutlierRejection calls it (src/tracker.cpp:705-753, :131-150); method 4 = cv::LMEDS, 8 = cv::RANSAC.
 * pts0 / pts1: n x 2 float (cv::Point2f).  Host-side work (a few dozen four-point hypotheses), no context needed.
 * mask[i] = 1 for inliers of the Levenberg-Marquardt-refined model at reproj_thresh (OpenCV 4.x semantics); *ok = 0 when no
 * model was found (mask all zero). */
int xivo_find_homography_mask(const float* pts0, const float* pts1, int n, int method, double reproj_thresh, int max_iters,
                              double confidence, uint8_t* mask, int* ok);

/* PNG frames, decoded as cv::imread decodes them for the reference (pybind11/pyxivo.cpp:81-85, :119-123; src/app/vio.cpp:72).
 * Accepted: colour types 0 (grey), 2 (RGB), 4 (grey + alpha), 6 (RGBA) at 8 or 16 bits, not interlaced.  Refused with XIVO_ERR_ARG
 * and the reason in xivo_last_error(): palette images, bit depths 1/2/4, Adam7 interlace, a bad signature, a missing or misplaced
 * IHDR, a missing IDAT or IEND, a chunk running past the end of the data, zero or oversized (> 16384 px a side) dimensions.
 * Ancillary chunks (gAMA, sRGB, tRNS, tEXt, ...) are skipped, as imread's colour and grey outputs ignore them.  The zlib header and
 * Adler-32 are checked and the inflated length must equal rows x (1 + cols x bytes per pixel); chunk CRCs are not checked (libpng
 * checks them).
 *
 * xivo_png_info: host-only container walk, no context.  channels = samples per pixel of the file (1, 2, 3, 4), bit_depth 8 or 16. */
int xivo_png_info(const uint8_t* png, size_t n, int* rows, int* cols, int* channels, int* bit_depth);
/* Decodes n PNGs of any geometry in one launch pair (png_inflate_kernel, png_unfilter_kernel) into host buffers out[i] of
 * rows x cols x channels bytes.  channels = 3: cv::imread(path) (IMREAD_COLOR): BGR, grey replicated, alpha stripped, 16-bit samples
 * keep their high byte.  channels = 1: IMREAD_GRAYSCALE of grey and grey + alpha files (colour files are refused).  If any frame
 * fails, nothing is written and XIVO_ERR_ARG names the frame index and the reason. */
int xivo_decode_png(xivo_ctx* ctx, int n, const uint8_t* const* png, const size_t* png_bytes, int channels, uint8_t* const* out);

/* Covariance slot surgery; replaces AddGroupToState / AddFeatureToState+FillCovarianceBlock /
 * RemoveGroupFromState / RemoveFeatureFromState / FixFeatureXY / SwitchRefGroup
 * (src/estimator.cpp:739-846, :1362-1391, :1474-1478, src/feature.cpp:753-776).
 * ops: nops x {type, a, b, n} ints; blk: nops x 9 doubles (type 2 only).
 *   type 0: zero rows+cols [a, a+n)   1: copy rows then cols b->a (n wide)   2: P[a:a+3,a:a+3] = blk */
int xivo_cov_edit(xivo_ctx* ctx, int N, double* P, const int* ops, const double* blk, int nops);

/* Covariance side of Estimator::Propagate (src/estimator.cpp:539-592, src/princedormand.cpp:208-215):
 * P[0:23,0:23] <- Pmm, P[0:23,23:] <- Phi P[0:23,23:] (+ symmetric strip). */
int xivo_cov_propagate(xivo_ctx* ctx, int N, double* P, const double* Phi, const double* Pmm);

/* Covariance side of Estimator::Propagate (src/estimator.cpp:539-592 with PrinceDormand / RK4
 * sub-stepping, src/princedormand.cpp:85-221, src/rk4.cpp:35-103): P[0:23,0:23], the motion/structure
 * strips of P, and + Qmodel per Propagate call.  The nominal state is a short sequential chain that the
 * caller integrates; for every Runge-Kutta stage it passes what the motion Jacobian
 * (ComputeMotionJacobianAt, src/estimator.cpp:614-702) depends on:
 *   stage16 : nstages x {Rsb(9), Cg*gyro-bg (3), Ca*accel-ba (3), h}; h = sub-step length on the first
 *             stage of each sub-step, negative when that sub-step closes a Propagate call.  The records
 *             must come from one such integration: the device rebuilds the Rsb of the later stages of a
 *             sub-step from its first stage (as the integrator composes them), and their rates from the
 *             first stage's and the slope between stage 0 and stage 5 (Prince-Dormand) / 1 (RK4)
 *   qimu12 / qmodel23 : diagonals of Qimu (gyro, accel, gyro bias, accel bias) and Qmodel
 *   stages_per_step : 7 (Prince-Dormand) or 4 (RK4) */
int xivo_imu_cov_propagate(xivo_ctx* ctx, int N, double* P, int nstages, const double* stage16, const double* g3,
                           const double* qimu12, const double* qmodel23, int stages_per_step);

/* ---------------------------------------------------------------------------------------------
 * Estimator-level entry points (handle based; one handle = a batch of independent estimators
 * that advance in lock-step, so B sequences share every kernel launch).  Mirrors
 * Estimator::{InertialMeas, VisualMeas, VisualMeasPointCloud, ...} (src/estimator.h:131-231).
 * Declared in xivo_b200_estimator.h.
 * ------------------------------------------------------------------------------------------- */

#ifdef __cplusplus
}
#endif
#endif /* XIVO_B200_H_ */

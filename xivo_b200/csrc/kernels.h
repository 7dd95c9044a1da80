// Internal launcher declarations shared by the C-ABI layer and the host estimator.
// Every launcher works on DEVICE pointers, takes a batch dimension (independent sequences /
// filters) and enqueues on the given stream without synchronising.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "hostmath.h"

namespace xb {

// ---------------- tracker (tracker_kernels.cu) ----------------
// seq_off (device, optional): per-sequence byte offset of the pyramid / image; ~0ull = skip that sequence.
int launch_build_pyramid(cudaStream_t st, uint8_t* pyr, unsigned long long pyr_stride, const unsigned long long* seq_off,
                         const PyrDesc& d, int batch, const uint8_t* const* frame0 = nullptr);
int launch_pyrdown_level(cudaStream_t st, uint8_t* pyr, unsigned long long pyr_stride, const unsigned long long* seq_off, const PyrDesc& d,
                         int batch, const uint8_t* const* frame0, int lvl);
// TMA pass (tracker_kernels.cu: pyrdown_tma_kernel): single channel, source level with cols % 16 == 0, images at a uniform stride
int make_pyr_tensor_map(CUtensorMap* out, const uint8_t* base, int rows, int cols, unsigned long long img_stride, unsigned long long n_img, int box_w = 0,
                        int box_h = 0);
// box of fast_pair_tma_kernel over the level-0 images of a pyramid buffer (image i at base + i * img_stride)
int make_fast_tensor_map(CUtensorMap* out, const uint8_t* base, int rows, int cols, unsigned long long img_stride, unsigned long long n_img);
int launch_pyrdown_tma(cudaStream_t st, const CUtensorMap& map, const int* src_img, uint8_t* pyr, unsigned long long pyr_stride,
                       const unsigned long long* seq_off, const PyrDesc& d, int lvl, int ingest, int batch);
int launch_gather_frames(cudaStream_t st, const uint8_t* const* src, uint8_t* dst, unsigned long long stride, const unsigned long long* off,
                         size_t bytes, int batch, int max_chunks = 64, int threads = 256);
// need (device, optional): per-sequence gate written by the accept kernel; a sequence with need <= 0 is skipped
int launch_fast_detect(cudaStream_t st, const uint8_t* img, unsigned long long img_stride, const unsigned long long* seq_off,
                       int rows, int cols, int cn, int thr, int nonmax, unsigned* kp_out, int max_kp, int* kp_count, int batch,
                       const int* need = nullptr, const CUtensorMap* tma_map = nullptr, unsigned long long tma_img_stride = 0,
                       bool count_is_zero = false /*kp_count was cleared by an earlier kernel of the stream (track_accept)*/);
// A keypoint of launch_fast_detect is packed as y << 20 | x << 8 | score: ascending order is raster order within a score.
inline int kp_x(unsigned k) { return (k >> 8) & 0xfff; }
inline int kp_y(unsigned k) { return k >> 20; }
inline int kp_score(unsigned k) { return k & 0xff; }
// Descriptor path (tracker.cpp:231-292, :341-460, :530-565): BRIEF-32 at given keypoints (kp_xy: batch x max_kp x 2 floats, nkp: batch counts;
// desc: batch x max_kp x 32 bytes, valid: 0 for keypoints closer than 28 px to the border) and, for the cross-checked brute-force matcher,
// the nearest descriptor of side b for every descriptor of side a (index and Hamming distance; -1 when b is empty; first index on ties).
int launch_brief(cudaStream_t st, const uint8_t* img, unsigned long long img_stride, const unsigned long long* seq_off, int rows, int cols, int cn,
                 const float* kp_xy, const int* nkp, int max_kp, uint8_t* desc, uint8_t* valid, int batch);
int launch_hamming_nearest(cudaStream_t st, const uint8_t* a, const int* na, int max_a, const uint8_t* b, const int* nb, int max_b, int* best_idx,
                           int* best_dist, int batch);
// Device-side tracker decisions (accept loop of Tracker::UpdateLK, greedy selection of Tracker::DetectLK); tracker_kernels.cu
struct TrackDecideCfg {
  int rows, cols, margin, mask_half, num_min, num_max, max_pts, max_kp, max_new;
  double max_disp;
};
size_t track_mask_bytes(int rows, int cols);
size_t track_accept_smem_bytes(int max_pts);
int launch_track_accept(cudaStream_t st, const TrackDecideCfg& c, const int* kind, const int* npts, const float* pts0, const float* pts1,
                        const uint8_t* lkst, uint8_t* stat, int* need, int batch, int* kp_count_to_zero = nullptr);
int launch_track_select(cudaStream_t st, const TrackDecideCfg& c, const int* kind, const int* npts, const float* pts1, const uint8_t* stat,
                        const int* need, unsigned* kp, const int* kp_count, unsigned* new_kp, int* n_new, int batch);
size_t lk_smem_bytes(int win, int cn);
int launch_lk_track(cudaStream_t st, const uint8_t* prev_pyr, const uint8_t* next_pyr, unsigned long long pyr_stride,
                    const unsigned long long* prev_off, const unsigned long long* next_off, const PyrDesc& d, const float* prev_pts, float* next_pts, uint8_t* status, float* err,
                    const int* npts_dev, int max_pts, int batch, int win, int max_iter, double eps, int use_initial_flow,
                    double min_eig);

// ---------------- PNG frames (png_kernels.cu) ----------------
// one frame of a decode launch: its zlib stream at in + in_off (in_len bytes, the IDAT payloads back to back), its rows x (1 + cols x bpp)
// bytes of filtered scanlines at scratch + scratch_off, its rows x cols x oc output bytes at out + out_off
struct PngFrameDesc {
  unsigned long long in_off, scratch_off, out_off;
  unsigned long long in_len;
  int rows, cols;
  int bpp, channels, bps, oc;  // bytes per pixel, samples per pixel, bytes per sample, output channels
};
// png_inflate_kernel + png_unfilter_kernel for n frames; status[i] = png::kOk or the png.cuh status of frame i
int launch_png_decode(cudaStream_t st, const uint8_t* in, uint8_t* scratch, uint8_t* out, const PngFrameDesc* fr, int n, int* status);

// ---------------- EKF (ekf_kernels.cu) ----------------
// Error-state layout, /root/reference/src/core.h:40-105 (default build: no online calibration).
struct EkfLayout {
  int G, F;
  __host__ __device__ int N() const { return 23 + 6 * G + 3 * F; }
  __host__ __device__ int goff(int s) const { return 23 + 6 * s; }
  __host__ __device__ int foff(int s) const { return 23 + 6 * G + 3 * s; }
};
constexpr int kJacNnz = 21;  // non-zero columns of one feature's 2xN Jacobian

// Per-feature output of the Jacobian/gate kernel (compact form of Feature::J_, inn_).
struct FeatJac {
  double J[2][kJacNnz];  // columns: Wsb(3) Tsb(3) Wbc(3) Tbc(3) Wsbr(3) Tsbr(3) x(3)
  double inn[2];
  double mh;  // Mahalanobis distance r^T (J P J^T + R)^-1 r
  int goff, foff;
};

// Covariance edit list (AddGroupToState / AddFeatureToState / Remove* / FixFeatureXY / SwitchRefGroup): applied by cov_edit_kernel or, packed,
// at the start of the Jacobian / gate kernel and of the gain kernel.
struct EditOp {
  int type;  // 0 = zero rows+cols [a, a+n); 1 = copy rows then cols b -> a (n wide); 2 = set 3x3 block at (a, a)
  int a, b, n;
  double blk[9];
};

// Motion + calibration state the Jacobians need: Rsb(9) Tsb(3) Rbc(9) Tbc(3), row-major.
constexpr int kPoseDoubles = 24;
constexpr int kGroupDoubles = 12;  // Rsb(9) Tsb(3) of a group slot

int launch_jacobian_gate(cudaStream_t st, EkfLayout lay, const CameraParams* cam /*device, per filter*/,
                         const double* X /*B x 24*/, const double* groups /*B x G x 12*/, const double* feat_x /*B x F x 3*/,
                         const double* feat_xp /*B x F x 2*/, const int* feat_ref /*B x F*/, const int* feat_sind /*B x F*/,
                         const int* nfeat /*B*/, double* P /*B x N x N*/, const double* Rmeas /*B*/,
                         FeatJac* out /*B x F*/, double* J_dense /*B x F x 2 x N or null*/, double* mh_out /*B x F or null*/,
                         int batch, const EditOp* ops = nullptr /*packed edit lists applied to P first*/, const int* ops_first = nullptr /*B*/,
                         const int* nops = nullptr /*B*/, double* diag_out = nullptr /*B x N: diag(P) after the edits*/);

struct TcOperands;  // TF32 operand buffers + tensor maps of the tensor-core downdate (below)
// Stack H (FillJacobianBlock semantics) for the selected features and do the measurement update.
//   sel: B x F indices into the feature table, nsel: B counts (M = 2*nsel)
// scratch: HP (B x 2F x N), Kt (B x 2F x N).  Outputs: err (B x N), P updated in place.
int launch_ekf_update(cudaStream_t st, EkfLayout lay, const FeatJac* jac, const int* sel, const int* nsel,
                      const double* Rmeas /*B*/, double* P, double* err, double* HP, double* Kt, double* H_dense /*or null*/,
                      int batch, int tensor_core = 0, const EditOp* ops = nullptr /*packed edit lists applied to P first*/,
                      const int* ops_first = nullptr /*B*/, const int* nops = nullptr /*B*/, const TcOperands* tc = nullptr /*tensor_core: second formulation*/,
                      int full_j = 0 /*stack the rows of J() unchanged instead of FillJacobianBlock's layout (1-point RANSAC)*/);

// Dense-input variant used by the kernel-level C ABI (arbitrary H, diagR), same kernels underneath.
int launch_ekf_update_dense(cudaStream_t st, int N, int M, const double* H, const double* diagR, const double* inn, double* P,
                            double* err, double* HP, double* Kt, int batch, int tensor_core = 0, const TcOperands* tc = nullptr);

// Tensor-core (wgmma, 3xTF32, fp32 accumulator in registers) form of the downdate P -= Kt^T HP (ekf_tc_kernels.cu);
// selected by tensor_core != 0 in the two launchers above.  ekf_cov_tc_fault: 1 if a kernel ever gave up waiting
// for its MMAs (never expected), -1 on a CUDA error.
int launch_ekf_cov_tc(cudaStream_t st, int N, const int* nsel, int Mdense, int Mmax, const double* HP, const double* Kt, double* P,
                      int batch);
// Second formulation (ekf_cov_tc2_kernel): the gain kernel also writes K^T and HP as TF32 hi/lo words in the wgmma canonical K-major layout
// [filter][hi|lo][k/4][state column (Npad)][4]; the downdate kernel stages them by TMA.
struct TcOperands {
  uint32_t* kt32 = nullptr;
  uint32_t* hp32 = nullptr;
  int Npad = 0, KCmax = 0, batch = 0;
  CUtensorMap mapA, mapB;
};
int tc_npad(int N);
int tc_kcmax(int Mmax);
size_t tc_operand_words(int N, int Mmax, int batch);  // 32-bit words of ONE operand buffer
int tc_operands_init(TcOperands* t, int N, int Mmax, int batch, uint32_t* kt32, uint32_t* hp32);
int launch_ekf_cov_tc2(cudaStream_t st, int N, const int* nsel, int Mdense, const TcOperands& t, double* P, int batch);
int ekf_cov_tc_fault(cudaStream_t st);

// Covariance edit list (AddGroupToState / AddFeatureToState / Remove* / FixFeatureXY / SwitchRefGroup).
int launch_cov_edit(cudaStream_t st, int N, double* P, const EditOp* ops /*B x max_ops, or packed with first*/, const int* nops /*B*/, int max_ops,
                    int batch, const int* first = nullptr /*B*/);

// Propagation: P[0:23,0:23] <- Pmm ; P[0:23,23:] <- Phi P[0:23,23:] and the symmetric strip.
int launch_cov_propagate(cudaStream_t st, int N, double* P, const double* Phi /*B x 23 x 23*/, const double* Pmm /*B x 23 x 23*/,
                         const unsigned char* active /*B or null*/, int batch);

// [err | Pmm | diag(P)] per filter, 2N+529 doubles each.
int launch_pack_state(cudaStream_t st, int N, const double* P, const double* err, double* out, int batch);

// P of filters [first, first + count) <- identity with the filter's motion block Pmm[b] (B x 23 x 23) in the top-left corner.
int launch_cov_init(cudaStream_t st, int N, double* P, const double* Pmm, int first, int count);

// Depth sub-filter, thread per feature (Feature::SubfilterUpdate).
struct SubfilterIn {
  double x[3], P[9], xp[2], ref[kGroupDoubles], outlier_counter;
  int filter;  // which filter (sequence) the feature belongs to
  int pad;
};
struct SubfilterOut {
  double x[3], P[9], outlier_counter;
};
int launch_subfilter(cudaStream_t st, const CameraParams* cam /*per filter*/, const double* X /*B x 24*/, const SubfilterIn* in,
                     SubfilterOut* out, int n, double Rtri, double mh_thresh);

// OOS / MSCKF: per-observation blocks + left-nullspace projection (Householder), one CTA per feature.
int launch_oos(cudaStream_t st, EkfLayout lay, const CameraParams* cam, const double* Rbc_Tbc /*12*/, const double* Xs /*nf x 3*/,
               const double* obs_pose /*nf x k x 12*/, const int* obs_sind /*nf x k*/, const double* obs_xp /*nf x k x 2*/,
               int k, int nf, double* Hf /*nf x 2k x 3*/, double* Hx /*nf x 2k x N*/, double* inn /*nf x 2k*/,
               double* Hx_proj /*nf x 2k x N scratch; first 2k-3 rows valid*/, double* inn_proj /*nf x 2k; first 2k-3 valid*/);

}  // namespace xb

namespace xb {
// ---------------- IMU covariance propagation on device (ekf_kernels.cu) ----------------
// The nominal motion state is a short, strictly sequential fp64 chain (sin/cos, quaternion
// renormalisation) — a CPU core runs it ~30x faster than one GPU thread — so the host integrates it and
// records what the motion Jacobian depends on.  The device does the covariance algebra (23x23 block +
// strips) of all filters in parallel from those records.
struct ImuStage {  // one Runge-Kutta stage (public ABI of xivo_imu_cov_propagate; the estimator's full records)
  double R[9];   // Rsb at the stage
  double gc[3];  // calibrated gyro  Cg*gyro - bg
  double ac[3];  // calibrated accel Ca*accel - ba
  double h;      // sub-step length, stored on the FIRST stage of each sub-step; negative = this sub-step closes a
                 // Propagate call (add Qmodel afterwards, src/estimator.cpp:590)
};
// One Runge-Kutta sub-step in the form the kernel reads: what the device cannot derive.  Stage s of the sub-step has the rates
// gc + dgc * (cin_s |h|), ac + dac * (cin_s |h|) and the rotation so3_normalize(R so3_exp(gc_s * cs_s |h|)) (stage 0: R itself),
// with the cs / cin of Estimator::nominal_step (imu_stage_coef); the kernel rebuilds them in parallel.  22 doubles per sub-step
// instead of 7 x 16 (Prince-Dormand) or 4 x 16 (RK4).
struct ImuStep {
  double R[9];    // Rsb at the start of the sub-step
  double gc[3];   // calibrated gyro  Cg*gyro - bg at the start of the sub-step
  double ac[3];   // calibrated accel Ca*accel - ba at the start of the sub-step
  double dgc[3];  // Cg * slope_gyro
  double dac[3];  // Ca * slope_accel
  double h;       // sub-step length; negative = this sub-step closes a Propagate call (as ImuStage::h)
};
// (cs, cin) of stage s >= 1: the stage composes the rotation over cs*h with the rates at cin*h (Prince-Dormand: cin = cs; RK4 of
// the reference: cin = 1/2 for every stage, rk4.cpp:79)
__host__ __device__ inline void imu_stage_coef(bool pd, int s, double* cs, double* cin) {
  *cs = pd ? (s == 1 ? 2.0 / 9 : s == 2 ? 3.0 / 9 : s == 3 ? 5.0 / 9 : s == 4 ? 6.0 / 9 : 1.0) : (s < 3 ? 0.5 : 1.0);
  *cin = pd ? *cs : 0.5;
}
// Rotation and calibrated rates of stage s of a sub-step record, as Estimator::nominal_step composes them when it writes one record
// per stage (the kernel rebuilds every stage this way)
__host__ __device__ inline void imu_stage_from_step(const ImuStep& r, int s, bool pd, M3* R, V3* gc, V3* ac) {
  for (int e = 0; e < 9; ++e) R->m[e] = r.R[e];
  for (int e = 0; e < 3; ++e) { gc->v[e] = r.gc[e]; ac->v[e] = r.ac[e]; }
  if (s == 0) return;
  double cs, cin;
  imu_stage_coef(pd, s, &cs, &cin);
  const double h = fabs(r.h);
  for (int e = 0; e < 3; ++e) { gc->v[e] += r.dgc[e] * (cin * h); ac->v[e] += r.dac[e] * (cin * h); }
  *R = so3_normalize(m3_mul(*R, so3_exp(v3_scale(*gc, cs * h))));
}
constexpr int kMaxStages = 1024;  // per filter between two flushes (one Propagate call with dt = 40 ms needs 140)
constexpr int kMaxSteps = kMaxStages / 4;  // the same capacity in sub-steps (RK4: 4 stages per sub-step; Prince-Dormand uses 146)
struct ImuConst {  // per filter
  double g[3], qimu[12], qmodel[23];
  int stages_per_step;  // 7 = Prince-Dormand, 4 = RK4
  int pad;
};
// steps: packed; filter b reads steps[first[b] .. first[b] + nsteps[b])
int launch_imu_cov_propagate(cudaStream_t st, int N, double* P, const ImuStep* steps, const int* first /*B*/, const int* nsteps /*B*/,
                             const ImuConst* cst /*B*/, int batch);
}  // namespace xb

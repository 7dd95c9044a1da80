/*
 * xivo_b200_estimator.h — estimator-level C ABI (handle based).
 *
 * Mirrors the reference's public class API for the hot path — Estimator::{InertialMeas,
 * VisualMeas, VisualMeasTrackerOnly, VisualMeasPointCloud, VisualMeasPointCloudTrackerOnly} and the
 * read-back accessors (src/estimator.h:131-231), which pybind11/pyxivo.cpp:332-398 exposes to
 * Python — with two deliberate differences forced by the reference's design:
 *   - de-singletonised: the reference allows one estimator per process (static singletons,
 *     src/factory.cpp:18-22); here one handle holds `n_seq` independent estimators that advance
 *     in lock-step, so that every CUDA launch and host<->device sync is shared by all sequences
 *     (the filter is sequential per stream; batching sequences is the only parallel axis);
 *   - kMaxGroup / kMaxFeature (compile-time -DEKF_MAX_GROUPS / -DEKF_MAX_FEATURES in the
 *     reference, src/core.h:92-105) are creation-time arguments.
 * cfg_json is the text of a reference config (cfg/NAME.json, JSON with comments).  "camera_cfg" and
 * "tracker_cfg" may be embedded objects or paths, as in src/factory.cpp:31-45.
 * All functions return 0 or a negative XIVO_ERR_* code (include/xivo_b200.h); nothing throws.
 */
#ifndef XIVO_B200_ESTIMATOR_H_
#define XIVO_B200_ESTIMATOR_H_

#include "xivo_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct xivo_batch xivo_batch;

/* CreateSystem / CreateSystemTrackerOnly (src/factory.cpp:17-122) for n_seq sequences.
 * Unless tracker_only, an update of 2 * max_features rows must fit the update kernels' shared memory on an H100: max_features <= 77,
 * and <= 64 with "covariance_update": "tf32x3" (no such bound under XIVO_TC_V1=1); a larger value is refused with XIVO_ERR_ARG. */
int xivo_batch_create(xivo_ctx* ctx, const char* cfg_json, int n_seq, int max_groups, int max_features,
                      int tracker_only, xivo_batch** out);
void xivo_batch_destroy(xivo_batch* b);
int xivo_batch_size(const xivo_batch* b);
int xivo_batch_state_dim(const xivo_batch* b); /* kFullSize = 23 + 6 G + 3 F */
/* Kept for ABI compatibility: always 1 for a valid handle (0 for NULL).  A config with "lanes" > 1 is refused at creation. */
int xivo_batch_lanes(const xivo_batch* b);

/* Estimator::InertialMeas (src/estimator.cpp:1036-1046), one sample per sequence.
 * ts_ns[n_seq], gyro[n_seq*3], accel[n_seq*3]. */
int xivo_batch_inertial_meas(xivo_batch* b, const uint64_t* ts_ns, const double* gyro, const double* accel);

/* Estimator::VisualMeas / VisualMeasTrackerOnly (src/estimator.cpp:943-979), one frame per sequence.
 * imgs[n_seq]: rows x cols x channels uint8, tightly packed (pyxivo.cpp:97-108 requires the same).
 * The pixels are copied to the device before the call returns control of the buffers: unlike the
 * reference (which keeps a shallow cv::Mat header for up to 10 queued messages) the caller may
 * reuse the memory immediately when it is pinned, and after the call returns otherwise. */
int xivo_batch_visual_meas(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* imgs, int rows, int cols,
                           int channels, int tracker_only);

/* xivo_batch_visual_meas with the frames given as PNG files (png[s]: png_bytes[s] bytes), decoded on the device the way cv::imread(path)
 * decodes them for the reference (pybind11/pyxivo.cpp:81-85, src/app/vio.cpp:72; formats and refusals: xivo_decode_png in xivo_b200.h).
 * channels = 3: the BGR imread result; 1: the grey sample of grey / grey + alpha files.  Every frame must have the batch geometry and
 * camera_cfg rows / cols (same checks as xivo_batch_visual_meas); colour type and bit depth may differ between sequences and frames.
 * The host walks the chunks and packs the image data of all sequences into one pinned upload; png_inflate_kernel and png_unfilter_kernel
 * decode it straight into the frame-ring slots the tracker reads.  A refused frame (container refusal on the host, corrupt deflate data,
 * Adler-32 or length mismatch on the device) returns XIVO_ERR_ARG naming the frame and the reason before any message is pushed: no
 * sequence changes and the handle stays usable.  The caller's buffers are free when the call returns.  Pending
 * xivo_batch_prefetch_frames uploads are dropped, as for any call with other buffers. */
int xivo_batch_visual_meas_png(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* png, const size_t* png_bytes, int channels,
                               int tracker_only);

/* Same, with the frames already resident in device memory (imgs_dev[s] are device pointers on this
 * context's GPU); used to measure the device-resident throughput. */
int xivo_batch_visual_meas_device(xivo_batch* b, const uint64_t* ts_ns, const uint8_t* const* imgs_dev, int rows, int cols,
                                  int channels, int tracker_only);

/* One lock-step "frame step": n_imu InertialMeas calls followed by one VisualMeas call per sequence,
 * with exactly the semantics of issuing them one by one (same message heap), in a single call so that
 * the per-call overhead is paid once.  imu_ts: n_imu x n_seq, gyro/accel: n_imu x n_seq x 3.
 * on_device != 0: imgs are device pointers. */
int xivo_batch_step(xivo_batch* b, int n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel,
                    const uint64_t* frame_ts, const uint8_t* const* imgs, int rows, int cols, int channels, int on_device);

/* Per-sequence input for one call, for sequences whose message patterns differ (start times, lengths, IMU samples per frame, dropped
 * frames).  Sequence s receives n_imu[s] InertialMeas, in the order given, then at most one VisualMeas (or VisualMeasTrackerOnly).  Its IMU
 * rows are at offset sum(n_imu[0..s-1]) of imu_ts / gyro (x 3) / accel (x 3).  imgs[s] == NULL (or imgs == NULL): no frame for s;
 * frame_ts[s] is read only where there is a frame.  A sequence with n_imu[s] == 0 and no frame is not touched.
 * After the call every sequence is bit-identical to sequence 0 of a one-sequence handle (same config, G, F, tracker_only) given the same
 * messages one at a time; xivo_batch_step is the case where every sequence has the same n_imu and a frame.  Only the sequences with a
 * frame take a ring slot, so one frame per sequence per call keeps the ring bound.  on_device != 0: imgs are device pointers.  Pending
 * xivo_batch_prefetch_frames uploads are dropped, as for any call with other buffers.
 * Refused with XIVO_ERR_ARG naming the sequence before any message is pushed (nothing changes): a negative n_imu, NULL IMU arrays while
 * some n_imu[s] > 0, a frame geometry other than the handle's.  XIVO_ERR_STATE once an earlier call on the handle failed. */
int xivo_batch_feed(xivo_batch* b, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel,
                    const uint64_t* frame_ts, const uint8_t* const* imgs, int rows, int cols, int channels, int on_device, int tracker_only);
/* The same, with frames as PNG files (png[s] == NULL: no frame for s), decoded on the device as in xivo_batch_visual_meas_png; only the
 * present frames are parsed, uploaded and decoded.  A refused or corrupt file of any sequence returns XIVO_ERR_ARG naming it before any
 * message is pushed: no sequence changes and the handle stays usable. */
int xivo_batch_feed_png(xivo_batch* b, const int* n_imu, const uint64_t* imu_ts, const double* gyro, const double* accel,
                        const uint64_t* frame_ts, const uint8_t* const* png, const size_t* png_bytes, int channels, int tracker_only);

/* Optional streaming hint: start the host->device copy of the NEXT frame of every sequence now, so that it
 * overlaps the step that is still being computed (the reference decouples acquisition from estimation the same
 * way, with its message queue: /root/reference/src/estimator_process.cpp).  Up to two prefetched frames may
 * be pending (the one the next call consumes and the one after it), consumed oldest first: an
 * xivo_batch_step / xivo_batch_visual_meas call that is given exactly the host pointers of the oldest one uses
 * its copy instead of uploading again; a call with any other buffers drops every pending prefetch.  The
 * buffers must stay valid and unchanged until the call that consumes them returns.  Results are identical
 * with and without the hint. */
int xivo_batch_prefetch_frames(xivo_batch* b, const uint8_t* const* imgs, int rows, int cols, int channels);

/* How device-accessible (pinned / registered) host frames are brought into the device frame ring:
 * XIVO_INGEST_ZERO_COPY: one gather launch per call, the SMs read the host memory over PCIe (initial value
 * when XIVO_ZEROCOPY=1);
 * XIVO_INGEST_COPY_ENGINE (default): the copy engine on the copy stream, one pitched copy per run of evenly
 * spaced source frames, else one cudaMemcpyAsync per frame.  Process-wide, takes effect at
 * the next visual_meas / step call, results are identical.  Returns the previous mode; any other argument
 * only queries.  Pageable host frames always take the copy-engine path. */
#define XIVO_INGEST_ZERO_COPY 0
#define XIVO_INGEST_COPY_ENGINE 1
int xivo_set_frame_ingest(int mode);

/* Per-kernel CUDA-event timing + host<->device byte counters (bench.py's roofline / e2e fields).
 * on: 0 off, 1 kernels + batch-level host phases, 2 additionally per-sequence host scopes (slow). */
void xivo_profile_enable(int on);
void xivo_profile_reset(void);
int xivo_profile_report(char* json_out, int capacity);

/* Estimator::VisualMeasPointCloud[TrackerOnly] (src/estimator.cpp:982-1032).
 * n_pts[n_seq]; ids[s]: n_pts[s] ints; xp_depth[s]: n_pts[s] x 3 (x, y, depth) row-major. */
int xivo_batch_visual_meas_pointcloud(xivo_batch* b, const uint64_t* ts_ns, const int* n_pts, const int* const* ids,
                                      const double* const* xp_depth, int tracker_only);

/* ---- read-back (estimator_accessors.cpp); `seq` selects the sequence ------------------------ */
int xivo_get_gsb(xivo_batch* b, int seq, double out12[12]); /* 3x4 row-major [R|T], Estimator::gsb */
int xivo_get_gbc(xivo_batch* b, int seq, double out12[12]);
int xivo_get_gsc(xivo_batch* b, int seq, double out12[12]);
int xivo_get_motion(xivo_batch* b, int seq, double Vsb[3], double bg[3], double ba[3], double Rsg[9]);
int xivo_get_P(xivo_batch* b, int seq, double* out /* N x N */); /* Estimator::P() */
int xivo_get_Pstate(xivo_batch* b, int seq, double out81[81]);   /* Estimator::Pstate(): top-left 9x9 */
/* counters: {num_instate_features, num_instate_groups, gauge_group, num_mh_rejected,
 *            num_tracker_failed, num_tracker_new_detections, vision_counter, imu_counter,
 *            MeasurementUpdateInitialized, VisionInitialized, num_tracked, sticky_error} */
#define XIVO_NUM_COUNTERS 12
int xivo_get_counters(xivo_batch* b, int seq, int out[XIVO_NUM_COUNTERS]);
int xivo_get_time_ns(xivo_batch* b, int seq, uint64_t* ts); /* Estimator::ts() */
/* tracked_features_no_descriptor(): ids and last pixel positions of Tracker::features_. */
int xivo_get_tracked_features(xivo_batch* b, int seq, int* ids, double* xy, int* status, int max_n, int* n);
/* tracked_features(): the descriptor column of the reference's (id, pixel, descriptor) tuples (pybind11/pyxivo.cpp:377-393; Feature::descriptor(),
 * src/feature.h:50).  desc: max_n x 32 bytes (BRIEF-32), has: max_n flags (0 = the feature carries no descriptor: extract_descriptor off),
 * same order as xivo_get_tracked_features. */
int xivo_get_tracked_descriptors(xivo_batch* b, int seq, uint8_t* desc, uint8_t* has, int max_n, int* n);
/* InstateFeatureIDs/Sinds/Positions(Xs)/x and reference group ids. */
int xivo_get_instate_features(xivo_batch* b, int seq, int* ids, int* sinds, int* ref_group_ids, double* Xs3,
                              double* x3, int max_n, int* n);
/* InstateGroupIDs/Sinds/Poses (3x4 row-major each). */
int xivo_get_instate_groups(xivo_batch* b, int seq, int* ids, int* sinds, double* gsb12, int max_n, int* n);
/* The per-feature accessors of src/estimator_accessors.cpp in one call (any output pointer may be NULL):
 * InstateFeature{IDs, Sinds, RefGroups, Positions (cached Xs), Xc, xc, Preds, Meas, Covs (upper triangle of the 3x3 block)}.
 * n_output < 0: the no-argument overloads (the features of the last update; slot order here, raw-pointer order in the reference);
 * n_output >= 0: the (int n_output) overloads: every in-state feature of the graph sorted by the Frobenius norm of its covariance
 * block (FeatureCovComparison, src/estimator.cpp:1451-1455), the first min(count, n_output) rows.  *n = rows available. */
int xivo_get_instate_feature_table(xivo_batch* b, int seq, int n_output, int* ids, int* sinds, int* ref_group_ids, double* Xs3,
                                   double* Xc3, double* xc3, double* pred2, double* meas2, double* cov6, int max_n, int* n);
/* InstateGroup{IDs, Sinds, Poses, Covs}: the in-state groups as the last update saw them (Graph::GetInstateGroups order);
 * pose7 = qx qy qz qw Tx Ty Tz per group (MatX7, estimator_accessors.cpp), cov36 = the full 6x6 block of P row-major (the reference's
 * InstateGroupCovs keeps six entries of it, see xivo_b200/pyxivo.py). */
int xivo_get_instate_group_table(xivo_batch* b, int seq, int* ids, int* sinds, double* pose7, double* cov36, int max_n, int* n);
/* Estimator::Ca / Cg / td (src/estimator.h:173-175) and Camera GetIntrinsics / GetDistortionType (pybind11/pyxivo.cpp:285-291):
 * Ca9, Cg9 row-major; intrinsics9 = fx fy cx cy k0 k1 k2 k3 0; distortion_type 0 pinhole, 3 equidistant. */
int xivo_get_calibration(xivo_batch* b, int seq, double* Ca9, double* Cg9, double* td, double* intrinsics9, int* distortion_type);
int xivo_get_just_dropped(xivo_batch* b, int seq, int* ids, int max_n, int* n); /* Estimator::JustDroppedFeatureIDs */
/* {num_tracker_outlier_rejected, num_tracker_failed_to_track, num_tracker_new_detections, num_oneptransac_rejected} */
int xivo_get_tracker_counters(xivo_batch* b, int seq, int out[4]);
int xivo_scale_init_velocity(xivo_batch* b, int seq, double scale); /* Estimator::ScaleInitVelocity: Vsb /= scale */
int xivo_init_with_sim_depths(xivo_batch* b); /* Estimator::InitWithSimDepths; a handle-level switch that reset sequences inherit */

/* Sequence `seq` starts over as a freshly created estimator: empty message heap, clocks cleared,
 * gravity / vision / update not initialised, tracker not initialised, feature and group ids from
 * their initial values, counters and error zero, its block of P = the initial covariance.
 * From this call on the sequence is bit-identical to sequence 0 of a new one-sequence handle
 * (same config, G, F, tracker_only) fed the same messages; every other sequence continues
 * bit-identically to a run without the call, its queued messages and frames included.
 * The sequence's pending heap messages are discarded (their frame ring slots become free), and
 * pending xivo_batch_prefetch_frames uploads are dropped for the whole handle.
 * cfg_json == NULL: the handle's creation config; otherwise a config of its own, which must agree
 * with the handle on every batch-wide setting: the layout (G, F) and tracker_only,
 * "covariance_update", "use_1pt_RANSAC", "subfilter" {"visual_meas_std", "MH_thresh"}, every key of
 * "tracker_cfg", "camera_cfg" {"rows", "cols"} and "message_buffer_size".  Everything else
 * (camera model and intrinsics, X incl. Rbc / Tbc, P, Qimu, Qmodel, visual_meas_std, the
 * integration method, gating and feature-management thresholds, ...) may differ per sequence.
 * Per-sequence configs from the start: create the handle with any compatible config, then reset
 * every sequence with its own before the first message.
 * Returns XIVO_ERR_ARG for a NULL handle, `seq` out of range, a config that does not parse or that
 * differs in a batch-wide setting (xivo_last_error names the first such key); XIVO_ERR_STATE once an
 * earlier call on the handle failed (such a call stops mid-frame for every sequence).  A refused
 * call changes nothing.  On a handle that isolates failures only a handle-wide failure refuses it:
 * a failed sequence is reset like any other and runs again.
 */
int xivo_batch_reset_sequence(xivo_batch* b, int seq, const char* cfg_json);
const char* xivo_batch_error(xivo_batch* b, int seq);

/* Failure isolation, off by default.  Off: the first error of any sequence ends the call for every sequence mid-frame and every later
 * call on the handle is refused.  On: a failure of one sequence is confined to that sequence --
 *   - what counts as its failure: its estimator's sticky error (out of feature or group slots, non-finite Mahalanobis distances, an
 *     innovation covariance that is not positive definite, a message of the wrong kind), an exception thrown by its host state machine,
 *     or one of its per-sequence capacities exceeded (its track list over the tracker's point table, its sub-filter list, its share of
 *     the covariance edit list);
 *   - in the call where it fails, the sequence leaves every later phase of the frame, and the call returns XIVO_SEQ_FAILED when every
 *     other sequence finished it normally;
 *   - afterwards its messages are dropped by every message call (not queued, no ring slot, its PNG not parsed), its state getters
 *     return XIVO_ERR_STATE with its message, and every other sequence continues bit-identically to a run without it;
 *   - xivo_batch_reset_sequence brings it back, bit-identical from then on to sequence 0 of a new one-sequence handle.
 * Handle-wide failures (CUDA errors, overflow of a buffer the sequences share, an exception while packing PNG frames) still fail the
 * handle as a whole: the call returns the error and later calls, reset included, are refused with XIVO_ERR_STATE.
 * Refused with XIVO_ERR_STATE on a handle that has failed as a whole, and turning isolation off while a sequence is failed. */
int xivo_batch_isolate_failures(xivo_batch* b, int on);
/* *code = 0 for a running sequence, else its error code; msg (msg_cap bytes, NUL-terminated, may be NULL) its message.
 * XIVO_ERR_ARG for a NULL handle or code, or `seq` out of range. */
int xivo_batch_sequence_status(const xivo_batch* b, int seq, int* code, char* msg, int msg_cap);

#ifdef __cplusplus
}
#endif
#endif

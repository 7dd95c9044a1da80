"""pyxivo-compatible Python surface over the estimator-level C ABI (include/xivo_b200_estimator.h).

`Estimator` mirrors the method names of the reference's pybind11 module
(/root/reference/pybind11/pyxivo.cpp:332-398) for the hot path; `Batch` is the lock-step
multi-sequence form that the GPU needs to be kept busy.  ctypes plumbing only — all computation
happens in libxivo_b200.so.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

from . import capi
from .capi import XivoError, _check, _p
from .sim import strip_json_comments


def _resolve_cfg(cfg, base_dir=None) -> str:
    """Accepts a path, a JSON(-with-comments) string or a dict; inlines camera_cfg / tracker_cfg
    given as paths (src/factory.cpp:31-45) and returns strict JSON text."""
    if isinstance(cfg, dict):
        d = dict(cfg)
    else:
        if "{" not in cfg:
            base_dir = base_dir or os.path.dirname(os.path.abspath(cfg))
            cfg = open(cfg).read()
        d = json.loads(strip_json_comments(cfg))
    for k in ("camera_cfg", "tracker_cfg"):
        if isinstance(d.get(k), str):
            path = d[k] if os.path.isabs(d[k]) or base_dir is None else os.path.join(base_dir, d[k])
            if not os.path.exists(path) and base_dir:
                path = os.path.join(os.path.dirname(base_dir), d[k])
            d[k] = json.loads(strip_json_comments(open(path).read()))
    return json.dumps(d)


def _cfg_text(cfg, overrides=None) -> str:
    """_resolve_cfg, then `overrides` merged in (one level deep for nested objects)."""
    text = _resolve_cfg(cfg)
    if overrides:
        d = json.loads(text)
        for k, v in overrides.items():
            if isinstance(v, dict) and isinstance(d.get(k), dict):
                d[k].update(v)
            else:
                d[k] = v
        text = json.dumps(d)
    return text


class Batch:
    def __init__(self, cfg, n_seq=1, max_groups=15, max_features=30, tracker_only=False, device=0, ctx=None, overrides=None):
        text = _cfg_text(cfg, overrides)
        self.cfg = json.loads(text)
        self._own_ctx = ctx is None
        self.ctx = ctx or capi.Context(device)
        self._h = C.c_void_p()
        L = capi.lib()
        _check(L.xivo_batch_create(self.ctx._h, text.encode(), int(n_seq), int(max_groups), int(max_features), int(bool(tracker_only)),
                                   C.byref(self._h)), "xivo_batch_create")
        self.n = n_seq
        self.G, self.F = max_groups, max_features
        self.N = L.xivo_batch_state_dim(self._h)
        self.lanes = L.xivo_batch_lanes(self._h)  # always 1: kept for callers that record it (include/xivo_b200_estimator.h)
        self._keep = None
        cam = self.cfg.get("camera_cfg") if isinstance(self.cfg.get("camera_cfg"), dict) else None
        self._cam_shape = (int(cam["rows"]), int(cam["cols"])) if cam and "rows" in cam and "cols" in cam else None

    def close(self):
        if self._h:
            capi.lib().xivo_batch_destroy(self._h)
            self._h = C.c_void_p()
        if self._own_ctx and self.ctx:
            self.ctx.close()
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- ingest -------------------------------------------------------------------------
    def inertial_meas(self, ts_ns, gyro, accel):
        ts = np.ascontiguousarray(np.broadcast_to(np.asarray(ts_ns, dtype=np.uint64), (self.n,)))
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(gyro, dtype=np.float64), (self.n, 3)))
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(accel, dtype=np.float64), (self.n, 3)))
        _check(capi.lib().xivo_batch_inertial_meas(self._h, _p(ts), _p(g), _p(a)), "xivo_batch_inertial_meas")

    def _check_images(self, imgs):
        """One image per sequence, all of the same shape (rows x cols [x 1 | 3]), uint8, C-contiguous: the C side reads
        rows * cols * channels bytes behind every pointer."""
        if isinstance(imgs, np.ndarray):
            imgs = [imgs] * self.n
        imgs = list(imgs)
        if len(imgs) != self.n:
            raise XivoError(f"expected {self.n} images (one per sequence), got {len(imgs)}")
        imgs = [np.ascontiguousarray(i, dtype=np.uint8) for i in imgs]
        shp = imgs[0].shape
        if len(shp) not in (2, 3) or (len(shp) == 3 and shp[2] not in (1, 3)):
            raise XivoError(f"image shape {shp}: expected rows x cols or rows x cols x 3")
        for k, i in enumerate(imgs):
            if i.shape != shp:
                raise XivoError(f"image {k} has shape {i.shape}, image 0 has {shp}: all sequences of a batch share one geometry")
        cam = self._cam_shape
        if cam and (shp[0], shp[1]) != cam:
            raise XivoError(f"image is {shp[0]} x {shp[1]} but camera_cfg says {cam[0]} x {cam[1]}")
        return imgs, shp[0], shp[1], (1 if len(shp) == 2 else shp[2])

    def visual_meas(self, ts_ns, imgs, tracker_only=False):
        """imgs: list of n arrays (rows x cols [x 3], uint8, C-contiguous) or one array shared by all."""
        imgs, rows, cols, ch = self._check_images(imgs)
        ts = np.ascontiguousarray(np.broadcast_to(np.asarray(ts_ns, dtype=np.uint64), (self.n,)))
        ptrs = (C.c_void_p * self.n)(*[i.ctypes.data for i in imgs])
        self._keep = imgs
        _check(capi.lib().xivo_batch_visual_meas(self._h, _p(ts), ptrs, rows, cols, ch, int(bool(tracker_only))), "xivo_batch_visual_meas")

    def visual_meas_png(self, ts_ns, blobs, channels=3, tracker_only=False):
        """visual_meas with the frames given as PNG file bytes (one per sequence, or one shared by all), decoded on the device straight
        into the frame ring (xivo_batch_visual_meas_png) as cv2.imread decodes them: channels = 3 is IMREAD_COLOR (BGR), channels = 1 is
        IMREAD_GRAYSCALE of grey / grey + alpha files.  A refused or corrupt file raises XivoError before any sequence's state changes."""
        if isinstance(blobs, (bytes, bytearray, memoryview)):
            blobs = [blobs] * self.n
        blobs = [bytes(x) for x in blobs]
        if len(blobs) != self.n:
            raise XivoError(f"expected {self.n} PNG frames (one per sequence), got {len(blobs)}")
        ts = np.ascontiguousarray(np.broadcast_to(np.asarray(ts_ns, dtype=np.uint64), (self.n,)))
        src = (C.c_char_p * self.n)(*blobs)
        sizes = (C.c_size_t * self.n)(*[len(x) for x in blobs])
        _check(capi.lib().xivo_batch_visual_meas_png(self._h, _p(ts), src, sizes, int(channels), int(bool(tracker_only))), "xivo_batch_visual_meas_png")

    def prefetch_frames(self, imgs):
        """Start uploading the frames of the NEXT visual_meas / step call (same arrays) while the current one is computed."""
        imgs, rows, cols, ch = self._check_images(imgs)
        ptrs = (C.c_void_p * self.n)(*[i.ctypes.data for i in imgs])
        self._keep_next = imgs
        _check(capi.lib().xivo_batch_prefetch_frames(self._h, ptrs, rows, cols, ch), "xivo_batch_prefetch_frames")

    def step(self, imu_ts, gyro, accel, frame_ts, imgs):
        """n_imu InertialMeas + one VisualMeas per sequence in one call (xivo_batch_step).
        imu_ts: (n_imu, n) or (n_imu,), gyro/accel: (n_imu, n, 3) or (n_imu, 3)."""
        imgs, rows, cols, ch = self._check_images(imgs)
        its = np.asarray(imu_ts, dtype=np.uint64)
        n_imu = its.shape[0]
        its = np.ascontiguousarray(np.broadcast_to(its.reshape(n_imu, -1), (n_imu, self.n)))
        g = np.ascontiguousarray(np.broadcast_to(np.asarray(gyro, dtype=np.float64).reshape(n_imu, -1, 3), (n_imu, self.n, 3)))
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(accel, dtype=np.float64).reshape(n_imu, -1, 3), (n_imu, self.n, 3)))
        fts = np.ascontiguousarray(np.broadcast_to(np.asarray(frame_ts, dtype=np.uint64), (self.n,)))
        ptrs = (C.c_void_p * self.n)(*[i.ctypes.data for i in imgs])
        self._keep = imgs
        _check(capi.lib().xivo_batch_step(self._h, n_imu, _p(its), _p(g), _p(a), _p(fts), ptrs, rows, cols, ch, 0), "xivo_batch_step")

    def visual_meas_pointcloud(self, ts_ns, ids, xp_depth, tracker_only=False):
        """ids / xp_depth: lists of per-sequence arrays, or single arrays shared by all."""
        if isinstance(ids, np.ndarray):
            ids, xp_depth = [ids] * self.n, [xp_depth] * self.n
        ids = [np.ascontiguousarray(i, dtype=np.int32).reshape(-1) for i in ids]
        xpd = [np.ascontiguousarray(x, dtype=np.float64).reshape(-1, 3) for x in xp_depth]
        if len(ids) != self.n or len(xpd) != self.n:
            raise XivoError(f"expected {self.n} point lists (one per sequence), got {len(ids)} / {len(xpd)}")
        for k, (i, x) in enumerate(zip(ids, xpd)):
            if len(i) != len(x):  # the C side reads 3 * n_pts doubles behind xp_depth[k]
                raise XivoError(f"sequence {k}: {len(i)} ids but {len(x)} (xp, depth) rows")
        npts = np.array([len(i) for i in ids], dtype=np.int32)
        ts = np.ascontiguousarray(np.broadcast_to(np.asarray(ts_ns, dtype=np.uint64), (self.n,)))
        pi = (C.c_void_p * self.n)(*[i.ctypes.data for i in ids])
        px = (C.c_void_p * self.n)(*[x.ctypes.data for x in xpd])
        _check(capi.lib().xivo_batch_visual_meas_pointcloud(self._h, _p(ts), _p(npts), pi, px, int(bool(tracker_only))),
               "xivo_batch_visual_meas_pointcloud")

    def init_with_sim_depths(self):
        _check(capi.lib().xivo_init_with_sim_depths(self._h), "xivo_init_with_sim_depths")

    def reset_sequence(self, seq, cfg=None, overrides=None):
        """Sequence `seq` starts over as a new estimator (xivo_batch_reset_sequence): with the handle's creation config when cfg and
        overrides are None, else with `cfg` (default: the creation config) plus `overrides`, resolved as in __init__.  The config must
        agree with the handle on the batch-wide settings; a refusal raises XivoError and leaves the handle unchanged."""
        text = None
        if cfg is not None or overrides:
            text = _cfg_text(self.cfg if cfg is None else cfg, overrides).encode()
        _check(capi.lib().xivo_batch_reset_sequence(self._h, int(seq), text), "xivo_batch_reset_sequence")

    # ---- read-back ----------------------------------------------------------------------
    def _g(self, fn, seq):
        out = np.zeros(12)
        _check(getattr(capi.lib(), fn)(self._h, seq, _p(out)), fn)
        return out.reshape(3, 4)

    def gsb(self, seq=0):
        return self._g("xivo_get_gsb", seq)

    def gbc(self, seq=0):
        return self._g("xivo_get_gbc", seq)

    def gsc(self, seq=0):
        return self._g("xivo_get_gsc", seq)

    def motion(self, seq=0):
        V, bg, ba, Rsg = np.zeros(3), np.zeros(3), np.zeros(3), np.zeros(9)
        _check(capi.lib().xivo_get_motion(self._h, seq, _p(V), _p(bg), _p(ba), _p(Rsg)), "xivo_get_motion")
        return V, bg, ba, Rsg.reshape(3, 3)

    def P(self, seq=0):
        out = np.zeros((self.N, self.N))
        _check(capi.lib().xivo_get_P(self._h, seq, _p(out)), "xivo_get_P")
        return out

    def Pstate(self, seq=0):
        out = np.zeros((9, 9))
        _check(capi.lib().xivo_get_Pstate(self._h, seq, _p(out)), "xivo_get_Pstate")
        return out

    COUNTER_NAMES = ("num_instate_features", "num_instate_groups", "gauge_group", "num_mh_rejected", "num_tracker_failed",
                     "num_tracker_new_detections", "vision_counter", "imu_counter", "MeasurementUpdateInitialized",
                     "VisionInitialized", "num_tracked", "error")

    def counters(self, seq=0):
        out = np.zeros(12, np.int32)
        _check(capi.lib().xivo_get_counters(self._h, seq, _p(out)), "xivo_get_counters")
        return dict(zip(self.COUNTER_NAMES, out.tolist()))

    def now(self, seq=0):
        ts = C.c_uint64()
        _check(capi.lib().xivo_get_time_ns(self._h, seq, C.byref(ts)), "xivo_get_time_ns")
        return ts.value

    def tracked_features(self, seq=0, max_n=4096):
        ids, xy, st, n = np.zeros(max_n, np.int32), np.zeros((max_n, 2)), np.zeros(max_n, np.int32), C.c_int()
        _check(capi.lib().xivo_get_tracked_features(self._h, seq, _p(ids), _p(xy), _p(st), max_n, C.byref(n)), "xivo_get_tracked_features")
        k = min(n.value, max_n)
        return ids[:k].copy(), xy[:k].copy(), st[:k].copy()

    def tracked_descriptors(self, seq=0, max_n=4096):
        """BRIEF-32 descriptors of the tracked features (rows of 32 bytes, same order as tracked_features) and which features carry one."""
        d, has, n = np.zeros((max_n, 32), np.uint8), np.zeros(max_n, np.uint8), C.c_int()
        _check(capi.lib().xivo_get_tracked_descriptors(self._h, seq, _p(d), _p(has), max_n, C.byref(n)), "xivo_get_tracked_descriptors")
        k = min(n.value, max_n)
        return d[:k].copy(), has[:k].astype(bool)

    def instate_features(self, seq=0):
        m = self.F
        ids, sinds, refs, Xs, x, n = np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros((m, 3)), np.zeros((m, 3)), C.c_int()
        _check(capi.lib().xivo_get_instate_features(self._h, seq, _p(ids), _p(sinds), _p(refs), _p(Xs), _p(x), m, C.byref(n)),
               "xivo_get_instate_features")
        k = min(n.value, m)
        return dict(ids=ids[:k].copy(), sinds=sinds[:k].copy(), ref_groups=refs[:k].copy(), Xs=Xs[:k].copy(), x=x[:k].copy())

    def instate_feature_table(self, seq=0, n_output=-1):
        """src/estimator_accessors.cpp in one call: n_output < 0 = the no-argument overloads (features of the last update),
        n_output >= 0 = the (int n_output) overloads (sorted by covariance norm, first min(count, n_output) rows)."""
        m = self.F
        i32, f64 = (lambda: np.zeros(m, np.int32)), (lambda w: np.zeros((m, w)))
        t = dict(ids=i32(), sinds=i32(), ref_groups=i32(), Xs=f64(3), Xc=f64(3), xc=f64(3), pred=f64(2), meas=f64(2), cov=f64(6))
        n = C.c_int()
        _check(capi.lib().xivo_get_instate_feature_table(self._h, seq, int(n_output), *[_p(t[k]) for k in ("ids", "sinds", "ref_groups", "Xs", "Xc", "xc", "pred", "meas", "cov")],
                                                         m, C.byref(n)), "xivo_get_instate_feature_table")
        k = min(n.value, m)
        return {key: v[:k].copy() for key, v in t.items()}

    def instate_group_table(self, seq=0):
        """InstateGroup{IDs, Sinds, Poses (qx qy qz qw T), Covs (full 6x6 blocks)} of the groups the last update saw."""
        m = self.G
        ids, sinds, pose, cov, n = np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros((m, 7)), np.zeros((m, 36)), C.c_int()
        _check(capi.lib().xivo_get_instate_group_table(self._h, seq, _p(ids), _p(sinds), _p(pose), _p(cov), m, C.byref(n)), "xivo_get_instate_group_table")
        k = min(n.value, m)
        return dict(ids=ids[:k].copy(), sinds=sinds[:k].copy(), pose=pose[:k].copy(), cov=cov[:k].reshape(k, 6, 6).copy())

    def calibration(self, seq=0):
        Ca, Cg, intr, td, dt = np.zeros(9), np.zeros(9), np.zeros(9), C.c_double(), C.c_int()
        _check(capi.lib().xivo_get_calibration(self._h, seq, _p(Ca), _p(Cg), C.byref(td), _p(intr), C.byref(dt)), "xivo_get_calibration")
        return dict(Ca=Ca.reshape(3, 3), Cg=Cg.reshape(3, 3), td=td.value, intrinsics=intr, distortion_type=dt.value)

    def just_dropped(self, seq=0, max_n=4096):
        ids, n = np.zeros(max_n, np.int32), C.c_int()
        _check(capi.lib().xivo_get_just_dropped(self._h, seq, _p(ids), max_n, C.byref(n)), "xivo_get_just_dropped")
        return ids[: min(n.value, max_n)].copy()

    TRACKER_COUNTER_NAMES = ("num_tracker_outlier_rejected", "num_tracker_failed_to_track", "num_tracker_new_detections", "num_oneptransac_rejected")

    def tracker_counters(self, seq=0):
        out = np.zeros(4, np.int32)
        _check(capi.lib().xivo_get_tracker_counters(self._h, seq, _p(out)), "xivo_get_tracker_counters")
        return dict(zip(self.TRACKER_COUNTER_NAMES, out.tolist()))

    def scale_init_velocity(self, scale, seq=0):
        _check(capi.lib().xivo_scale_init_velocity(self._h, seq, C.c_double(scale)), "xivo_scale_init_velocity")

    def instate_groups(self, seq=0):
        m = self.G
        ids, sinds, g, n = np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros((m, 12)), C.c_int()
        _check(capi.lib().xivo_get_instate_groups(self._h, seq, _p(ids), _p(sinds), _p(g), m, C.byref(n)), "xivo_get_instate_groups")
        k = min(n.value, m)
        return dict(ids=ids[:k].copy(), sinds=sinds[:k].copy(), gsb=g[:k].reshape(k, 3, 4).copy())


def reference_group_cov_layout(cov_blocks):
    """InstateGroupCovs as the reference returns it (src/estimator_accessors.cpp, InstateGroupCovs): n x 21, but the column counter is
    reset inside the row loop (`cnt = 0` per `ii`), so only columns 0..5 are ever written and they end up holding
    cov(5,5), cov(4,5), cov(3,5), cov(2,5), cov(1,5), cov(0,5); columns 6..20 are uninitialised there and zero here."""
    cov_blocks = np.asarray(cov_blocks, dtype=np.float64).reshape(-1, 6, 6)
    out = np.zeros((len(cov_blocks), 21))
    for ii in range(6):
        cnt = 0
        for jj in range(ii, 6):
            out[:, cnt] = cov_blocks[:, ii, jj]
            cnt += 1
    return out


class Estimator:
    """Single-sequence facade with the reference's pyxivo method names
    (pybind11/pyxivo.cpp:332-398): pyxivo.Estimator(cfg_path, viewer_cfg_path, name, tracker_only)."""

    def __init__(self, cfg, viewer_cfg="", name="", tracker_only=False, max_groups=15, max_features=30, device=0):
        self._b = Batch(cfg, 1, max_groups, max_features, tracker_only, device)
        self._tracker_only = tracker_only

    def InertialMeas(self, ts, wx, wy, wz, ax, ay, az):
        self._b.inertial_meas(int(ts), [wx, wy, wz], [ax, ay, az])

    def _visual(self, ts, image, tracker_only):
        if isinstance(image, (str, os.PathLike)):  # cv::imread(path) as the reference's binding does (pybind11/pyxivo.cpp:81-85, :119-123)
            with open(image, "rb") as f:
                self._b.visual_meas_png(int(ts), [f.read()], channels=3, tracker_only=tracker_only)
        else:
            self._b.visual_meas(int(ts), [image], tracker_only=tracker_only)

    def VisualMeas(self, ts, image):
        """image: a decoded uint8 array, or the path of a PNG file (decoded on the device like cv::imread(path))"""
        self._visual(ts, image, False)

    def VisualMeasTrackerOnly(self, ts, image):
        self._visual(ts, image, True)

    def VisualMeasPointCloud(self, ts, feature_ids, xp_and_depths):
        self._b.visual_meas_pointcloud(int(ts), [np.asarray(feature_ids)], [np.asarray(xp_and_depths)], tracker_only=False)

    def VisualMeasPointCloudTrackerOnly(self, ts, feature_ids, xp_and_depths):
        self._b.visual_meas_pointcloud(int(ts), [np.asarray(feature_ids)], [np.asarray(xp_and_depths)], tracker_only=True)

    def InitWithSimDepths(self):
        self._b.init_with_sim_depths()

    def CloseLoop(self):
        return None  # USE_MAPPER is off in the default build (src/CMakeLists.txt:18)

    def gsb(self):
        return self._b.gsb()

    def gsc(self):
        return self._b.gsc()

    def gbc(self):
        return self._b.gbc()

    def Vsb(self):
        return self._b.motion()[0]

    def bg(self):
        return self._b.motion()[1]

    def ba(self):
        return self._b.motion()[2]

    def Rsg(self):
        return self._b.motion()[3]

    def P(self):
        return self._b.P()

    def Pstate(self):
        return self._b.Pstate()

    def now(self):
        return self._b.now()

    def ts(self):
        return self._b.now()

    def gauge_group(self):
        return self._b.counters()["gauge_group"]

    def num_instate_features(self):
        return self._b.counters()["num_instate_features"]

    def num_instate_groups(self):
        return self._b.counters()["num_instate_groups"]

    def num_mh_rejected(self):
        return self._b.counters()["num_mh_rejected"]

    def num_tracker_failed(self):
        return self._b.counters()["num_tracker_failed"]

    def num_tracker_new_detections(self):
        return self._b.counters()["num_tracker_new_detections"]

    def MeasurementUpdateInitialized(self):
        return bool(self._b.counters()["MeasurementUpdateInitialized"])

    def VisionInitialized(self):
        return bool(self._b.counters()["VisionInitialized"])

    def UsingLoopClosure(self):
        return False

    # ---- per-feature accessors, both overloads of src/estimator_accessors.cpp (pybind11/pyxivo.cpp:357-374) -------------
    def _feature_column(self, key, n_output):
        """No argument: the features of the last update.  (int n_output): sorted by covariance norm; the reference returns
        max(count, n_output) rows of which it fills the first min(count, n_output) (the rest is uninitialised memory there, zeros here)."""
        if n_output is None:
            return self._b.instate_feature_table(0, -1)[key]
        n_output = int(n_output)
        col = self._b.instate_feature_table(0, n_output)[key]
        count = len(self._b.instate_feature_table(0, 1 << 20)["ids"])
        out = np.zeros((max(count, n_output),) + col.shape[1:], dtype=col.dtype)
        out[: len(col)] = col
        return out

    def InstateFeatureIDs(self, n_output=None):
        return self._feature_column("ids", n_output)

    def InstateFeatureSinds(self, n_output=None):
        return self._feature_column("sinds", n_output)

    def InstateFeatureRefGroups(self, n_output=None):
        return self._feature_column("ref_groups", n_output)

    def InstateFeaturePositions(self, n_output=None):
        return self._feature_column("Xs", n_output)

    def InstateFeatureXc(self, n_output=None):
        return self._feature_column("Xc", n_output)

    def InstateFeaturexc(self, n_output=None):
        return self._feature_column("xc", n_output)

    def InstateFeaturePreds(self, n_output=None):
        return self._feature_column("pred", n_output)

    def InstateFeatureMeas(self, n_output=None):
        return self._feature_column("meas", n_output)

    def InstateFeatureCovs(self, n_output=None):
        return self._feature_column("cov", n_output)

    def InstateGroupIDs(self):
        return self._b.instate_group_table()["ids"]

    def InstateGroupSinds(self):
        return self._b.instate_group_table()["sinds"]

    def InstateGroupPoses(self):
        """n x 7: qx qy qz qw Tx Ty Tz (MatX7, estimator_accessors.cpp InstateGroupPoses)."""
        return self._b.instate_group_table()["pose"]

    def InstateGroupCovs(self):
        """n x 21, laid out exactly as the reference fills it (see reference_group_cov_layout)."""
        return reference_group_cov_layout(self._b.instate_group_table()["cov"])

    def InstateGroupCovBlocks(self):
        """n x 6 x 6: the groups' full covariance blocks (not in the reference's API; what InstateGroupCovs was meant to expose)."""
        return self._b.instate_group_table()["cov"]

    def JustDroppedFeatureIDs(self):
        return self._b.just_dropped()

    def Rg(self):  # the binding's name for Rsg (pybind11/pyxivo.cpp:353)
        return self._b.motion()[3]

    def td(self):
        return self._b.calibration()["td"]

    def Ca(self):
        return self._b.calibration()["Ca"]

    def Cg(self):
        return self._b.calibration()["Cg"]

    def CameraIntrinsics(self):
        return self._b.calibration()["intrinsics"]

    def CameraDistortionType(self):
        return self._b.calibration()["distortion_type"]

    def ScaleInitVelocity(self, scale):
        self._b.scale_init_velocity(float(scale))

    def num_oneptransac_rejected(self):
        return self._b.tracker_counters()["num_oneptransac_rejected"]

    def num_tracker_outlier_rejected(self):
        return self._b.tracker_counters()["num_tracker_outlier_rejected"]

    def num_tracker_failed_to_track(self):
        return self._b.tracker_counters()["num_tracker_failed_to_track"]

    def Visualize(self):
        return None  # the Pangolin viewer is outside the hot path (SURVEY.md §2); kept so that reference scripts run unchanged

    def tracked_features(self):
        """[(id, pixel, descriptor)] like the reference's binding (pybind11/pyxivo.cpp:377-393: the cv::Mat descriptor converted to a float
        matrix): a 1 x 32 float32 row of the BRIEF bytes, or an empty matrix when the tracker extracts no descriptors."""
        ids, xy, _ = self._b.tracked_features()
        d, has = self._b.tracked_descriptors()
        return [(int(i), p, d[k : k + 1].astype(np.float32) if has[k] else np.zeros((0, 0), np.float32)) for k, (i, p) in enumerate(zip(ids, xy))]

    def tracked_features_no_descriptor(self):
        ids, xy, _ = self._b.tracked_features()
        return [(int(i), p) for i, p in zip(ids, xy)]

    def close(self):
        self._b.close()

"""Restarting one sequence of a batch (xivo_batch_reset_sequence).

From the reset on, the sequence must be bit-identical to sequence 0 of a new one-sequence handle with the same config fed the same
messages, and every other sequence bit-identical to a handle that never reset -- queued heap messages and frames in the ring included.
Every comparison is exact (np.array_equal).  Messages go in per frame as 8 IMU samples, then the frame (the grouping of xivo_batch_step),
so a new stream can start from t = 0 at any frame boundary while the other sequences continue."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from xivo_b200 import capi, pyxivo, sim

pytestmark = pytest.mark.gpu
CFG = os.path.join(os.path.dirname(pyxivo.__file__), "cfg")
G, F = 15, 30
# equidistant (Kannala-Brandt) intrinsics and measurement noise of tests/test_reference_pin.py::CASES "equidistant_203", on the
# handle's frame geometry (rows x cols are batch-wide)
EQUIDISTANT = {"model": "equidistant", "fx": 190.97847715128717, "fy": 190.9733070521226, "cx": 254.93170605935475, "cy": 256.8974428996504,
               "max_iter": 15, "k0123": [0.0034823894022493434, 0.0007150348452162257, -0.0020532361418706202, 0.00020293673591811182]}


def equidistant_cfg(cfg, Vsb=(0.02, -0.01, 0.0)):
    c = dict(cfg)
    cam = dict(EQUIDISTANT, rows=cfg["camera_cfg"]["rows"], cols=cfg["camera_cfg"]["cols"])
    c["camera_cfg"] = cam
    c["visual_meas_std"] = 1.5
    c["X"] = dict(cfg["X"], Vsb=list(Vsb))
    return c


def frames_of(msgs):
    """[(imu chunk of 8 (ts, (gyro, accel))), (frame ts, payload)] per frame."""
    imu = [(ts, p) for k, ts, p in msgs if k == "imu"]
    vis = [(ts, p) for k, ts, p in msgs if k != "imu"]
    n = min(len(vis), len(imu) // 8)
    return [(imu[8 * f : 8 * f + 8], vis[f]) for f in range(n)]


def pc_frames(cfg, seed, duration=3.2):
    return frames_of(sim.pcw_stream(cfg, duration=duration, seed=seed)[0])


def feed_pc(batch, frames):
    """One frame per sequence: its 8 IMU samples, then its point cloud."""
    for k in range(8):
        batch.inertial_meas(np.array([f[0][k][0] for f in frames], np.uint64), np.stack([f[0][k][1][0] for f in frames]),
                            np.stack([f[0][k][1][1] for f in frames]))
    batch.visual_meas_pointcloud(np.array([f[1][0] for f in frames], np.uint64), [f[1][1][0] for f in frames], [f[1][1][1] for f in frames])


def state(b, s):
    return (b.gsb(s), *b.motion(s), np.array([b.now(s)]), b.instate_features(s)["ids"], np.array(list(b.counters(s).values())))


def assert_same(b, s, ref, r, what):
    for a, w in zip(state(b, s), state(ref, r)):
        assert np.array_equal(a, w), what


def assert_fresh(b, s, solo):
    """What a reset sequence reads back before its first message: exactly what a new handle reads."""
    assert_same(b, s, solo, 0, f"sequence {s} right after its reset")
    assert b.now(s) == 0
    assert np.array_equal(b.P(s), solo.P(0))
    c, cs = b.calibration(s), solo.calibration(0)
    for k in ("Ca", "Cg", "intrinsics"):
        assert np.array_equal(c[k], cs[k]), k
    assert c["td"] == cs["td"] and c["distortion_type"] == cs["distortion_type"]
    assert np.array_equal(b.gbc(s), solo.gbc(0))
    assert len(b.tracked_features(s)[0]) == 0 and len(b.instate_features(s)["ids"]) == 0
    assert b.tracker_counters(s) == solo.tracker_counters(0)


MODES = {
    "prince_dormand": {},
    "rk4": {"integration_method": "RK4"},
    "tf32x3": {"covariance_update": "tf32x3"},
    "one_point_ransac": {"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 1.5, "sim_outliers": {"fraction": 0.08, "pixels": 2.5}},
}


@pytest.mark.parametrize("mode", list(MODES))
def test_restart_mid_run_equals_a_new_handle_and_leaves_the_others_alone(ctx, mode):
    B, RESET_AFTER, SAME, OWN = 7, 40, 3, 5
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    cfg.update(MODES[mode])
    own = equidistant_cfg(cfg)
    old = [pc_frames(cfg, 20 + s) for s in range(B)]
    new = {SAME: pc_frames(cfg, 60), OWN: pc_frames(own, 61)}
    n = len(old[0])
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    for b in (batch, ref):
        b.init_with_sim_depths()
    for f in range(RESET_AFTER + 1):
        feed_pc(batch, [old[s][f] for s in range(B)])
        feed_pc(ref, [old[s][f] for s in range(B)])
    assert batch.counters(SAME)["MeasurementUpdateInitialized"] == 1
    batch.reset_sequence(SAME)
    batch.reset_sequence(OWN, own)
    solo = {SAME: pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx), OWN: pyxivo.Batch(own, n_seq=1, max_groups=G, max_features=F, ctx=ctx)}
    for s, b in solo.items():
        b.init_with_sim_depths()
        assert_fresh(batch, s, b)
    assert batch.calibration(OWN)["distortion_type"] == 3 and batch.calibration(SAME)["distortion_type"] == 0
    updated = 0
    for k, f in enumerate(range(RESET_AFTER + 1, n)):
        feed_pc(batch, [new[s][k] if s in new else old[s][f] for s in range(B)])
        feed_pc(ref, [old[s][f] for s in range(B)])
        for s, b in solo.items():
            feed_pc(b, [new[s][k]])
        for s in range(B):
            if s in solo:
                assert_same(batch, s, solo[s], 0, f"{mode}: frame {k} after the reset, reset sequence {s}")
            else:
                assert_same(batch, s, ref, s, f"{mode}: frame {f}, sequence {s}")
        updated += batch.counters(OWN)["MeasurementUpdateInitialized"]
    assert updated > 0
    for s in range(B):
        want = solo[s].P(0) if s in solo else ref.P(s)
        assert np.array_equal(batch.P(s), want), f"{mode}: P of sequence {s}"
        assert batch.counters(s)["error"] == 0
    for b in [batch, ref, *solo.values()]:
        b.close()


def test_same_sequence_reset_three_times(ctx):
    B, SEQ, RESETS = 3, 1, (12, 30, 50)
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    old = [pc_frames(cfg, 30 + s) for s in range(B)]
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    for b in (batch, ref):
        b.init_with_sim_depths()
    solo, seg, k, segments = None, None, 0, 0
    for f in range(len(old[0])):
        if f in RESETS:
            if solo is not None:
                assert np.array_equal(batch.P(SEQ), solo.P(0)), f"segment ending at frame {f}"
                solo.close()
            seg_cfg = cfg if segments != 1 else equidistant_cfg(cfg, Vsb=(0.0, 0.01, 0.0))
            batch.reset_sequence(SEQ, None if segments != 1 else seg_cfg)
            solo = pyxivo.Batch(seg_cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx)
            solo.init_with_sim_depths()
            assert_fresh(batch, SEQ, solo)
            seg, k, segments = pc_frames(seg_cfg, 70 + segments), 0, segments + 1
        cur = [old[s][f] for s in range(B)]
        feed_pc(ref, cur)
        if solo is not None:
            cur[SEQ] = seg[k]
            feed_pc(solo, [seg[k]])
            k += 1
        feed_pc(batch, cur)
        for s in range(B):
            if s == SEQ and solo is not None:
                assert_same(batch, s, solo, 0, f"frame {f}, segment {segments}")
            else:
                assert_same(batch, s, ref, s, f"frame {f}, sequence {s}")
    assert segments == 3
    assert np.array_equal(batch.P(SEQ), solo.P(0))
    for s in range(B):
        if s != SEQ:
            assert np.array_equal(batch.P(s), ref.P(s))
    for b in (batch, ref, solo):
        b.close()


# ---------------------------------------------------------------- image path
def img_frames(cfg, seed, duration):
    return frames_of(sim.image_stream(cfg, duration=duration, seed=seed)[0])


def tracked(b, s):
    ids, xy, st = b.tracked_features(s)
    return ids, xy, st


def assert_same_img(b, s, ref, r, what):
    assert_same(b, s, ref, r, what)
    for a, w in zip(tracked(b, s), tracked(ref, r)):
        assert np.array_equal(a, w), what


def dev_step(batch, frames, dptrs):
    """xivo_batch_step with device-resident frames (one per sequence)."""
    n = len(frames)
    its = np.ascontiguousarray(np.array([[f[0][k][0] for f in frames] for k in range(8)], np.uint64))
    g = np.ascontiguousarray(np.array([[f[0][k][1][0] for f in frames] for k in range(8)], np.float64))
    a = np.ascontiguousarray(np.array([[f[0][k][1][1] for f in frames] for k in range(8)], np.float64))
    fts = np.ascontiguousarray(np.array([f[1][0] for f in frames], np.uint64))
    rows, cols = frames[0][1][1].shape[:2]
    ptrs = (C.c_void_p * n)(*dptrs)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    capi._check(capi.lib().xivo_batch_step(batch._h, 8, p(its), p(g), p(a), p(fts), ptrs, rows, cols, 1, 1), "xivo_batch_step")


def feed_img(batch, frames, how, dptrs=None):
    """visual_meas: 8 inertial_meas calls, then visual_meas with host frames; device_step: one fused xivo_batch_step on device frames."""
    if how == "device_step":
        dev_step(batch, frames, dptrs)
        return
    for k in range(8):
        batch.inertial_meas(np.array([f[0][k][0] for f in frames], np.uint64), np.stack([f[0][k][1][0] for f in frames]),
                            np.stack([f[0][k][1][1] for f in frames]))
    batch.visual_meas(np.array([f[1][0] for f in frames], np.uint64), [f[1][1] for f in frames])


@pytest.mark.parametrize("how", ["visual_meas", "device_step"])
def test_image_path_restart_with_a_prefetch_pending(ctx, how):
    import torch

    B, SEQ, RESET_AFTER, DUR = 3, 1, 12, 1.3
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    old = [img_frames(cfg, 40 + s, DUR) for s in range(B)]
    new = img_frames(cfg, 49, DUR)
    n = len(old[0])
    dev = {}

    def dptr(img):  # device copies of the frames for the device-resident step (kept alive for the whole run)
        key = img.ctypes.data
        if key not in dev:
            dev[key] = torch.from_numpy(img).cuda()
        return dev[key].data_ptr()

    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=4, max_features=14, ctx=ctx)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=4, max_features=14, ctx=ctx)
    solo = None
    k = 0
    for f in range(n):
        cur = [old[s][f] for s in range(B)]
        feed_img(ref, cur, how, [dptr(c[1][1]) for c in cur] if how == "device_step" else None)
        if solo is not None:
            cur[SEQ] = new[k]
            feed_img(solo, [new[k]], how, [dptr(new[k][1][1])] if how == "device_step" else None)
            k += 1
        feed_img(batch, cur, how, [dptr(c[1][1]) for c in cur] if how == "device_step" else None)
        if f == RESET_AFTER:
            # the next frames of the old streams are on their way when the sequence restarts: the prefetch is dropped, nothing else
            batch.prefetch_frames([old[s][f + 1][1][1] for s in range(B)])
            batch.reset_sequence(SEQ)
            solo = pyxivo.Batch(cfg, n_seq=1, max_groups=4, max_features=14, ctx=ctx)
            assert_fresh(batch, SEQ, solo)
            continue
        for s in range(B):
            if s == SEQ and solo is not None:
                assert_same_img(batch, s, solo, 0, f"{how}: frame {k - 1} after the reset")
            else:
                assert_same_img(batch, s, ref, s, f"{how}: frame {f}, sequence {s}")
    assert k > 10 and batch.counters(SEQ)["num_tracked"] > 50
    assert batch.counters(SEQ)["VisionInitialized"] == 1
    assert np.array_equal(batch.P(SEQ), solo.P(0))
    for s in range(B):
        if s != SEQ:
            assert np.array_equal(batch.P(s), ref.P(s))
    for b in (batch, ref, solo):
        b.close()


def test_tracker_only_handle_restart(ctx):
    B, SEQ, RESET_AFTER = 3, 2, 9
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=75, num_features_max=100)
    old = [[p for k, _, p in sim.image_stream(cfg, duration=1.0, seed=50 + s)[0] if k == "img"] for s in range(B)]
    new = [p for k, _, p in sim.image_stream(cfg, duration=1.0, seed=59)[0] if k == "img"]
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=4, max_features=14, tracker_only=True, ctx=ctx)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=4, max_features=14, tracker_only=True, ctx=ctx)
    solo, k = None, 0
    for f in range(len(old[0])):
        ts = 40_000_000 * f
        cur = [old[s][f] for s in range(B)]
        ref.visual_meas(ts, cur, tracker_only=True)
        tsv = np.full(B, ts, np.uint64)
        if solo is not None:
            cur[SEQ] = new[k]
            tsv[SEQ] = 40_000_000 * k
            solo.visual_meas(40_000_000 * k, [new[k]], tracker_only=True)
            k += 1
        batch.visual_meas(tsv, cur, tracker_only=True)
        if f == RESET_AFTER:
            batch.reset_sequence(SEQ)
            solo = pyxivo.Batch(cfg, n_seq=1, max_groups=4, max_features=14, tracker_only=True, ctx=ctx)
            assert len(batch.tracked_features(SEQ)[0]) == 0 and batch.now(SEQ) == 0
            continue
        for s in range(B):
            want = tracked(solo, 0) if (s == SEQ and solo is not None) else tracked(ref, s)
            for a, w in zip(tracked(batch, s), want):
                assert np.array_equal(a, w), f"frame {f}, sequence {s}"
            assert batch.tracker_counters(s) == (solo.tracker_counters(0) if (s == SEQ and solo is not None) else ref.tracker_counters(s))
    assert k > 5 and len(batch.tracked_features(SEQ)[0]) > 50
    for b in (batch, ref, solo):
        b.close()


def test_per_sequence_configs_from_creation(ctx):
    """Create with one config, reset every sequence with its own before the first message: two pinhole intrinsics and one equidistant."""
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    pin2 = dict(cfg, camera_cfg=dict(cfg["camera_cfg"], fx=300.0, fy=298.0, cx=315.0, cy=245.0))
    cfgs = [cfg, pin2, equidistant_cfg(cfg)]
    B = len(cfgs)
    streams = [pc_frames(c, 80 + s, duration=2.4) for s, c in enumerate(cfgs)]
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    batch.init_with_sim_depths()  # before the resets: a handle-level switch the reset sequences inherit
    for s, c in enumerate(cfgs):
        batch.reset_sequence(s, c)
    solo = [pyxivo.Batch(c, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for c in cfgs]
    for s, b in enumerate(solo):
        b.init_with_sim_depths()
        assert_fresh(batch, s, b)
    assert [batch.calibration(s)["distortion_type"] for s in range(B)] == [0, 0, 3]
    assert batch.calibration(1)["intrinsics"][0] == 300.0
    for f in range(len(streams[0])):
        feed_pc(batch, [streams[s][f] for s in range(B)])
        for s in range(B):
            feed_pc(solo[s], [streams[s][f]])
            assert_same(batch, s, solo[s], 0, f"frame {f}, sequence {s}")
    for s in range(B):
        assert batch.counters(s)["MeasurementUpdateInitialized"] == 1
        assert np.array_equal(batch.P(s), solo[s].P(0))
    for b in [batch, *solo]:
        b.close()


# ---------------------------------------------------------------- refusals
REFUSED = [  # batch-wide key, value on a handle configured with REFUSAL_BASE
    ("covariance_update", "tf32x3"), ("use_1pt_RANSAC", True), ("subfilter.visual_meas_std", 2.5), ("subfilter.MH_thresh", 5.991),
    ("camera_cfg.rows", 512), ("camera_cfg.cols", 512), ("message_buffer_size", 6), ("tracker_cfg.tracker_type", "MATCH"),
    ("tracker_cfg.mask_size", 11), ("tracker_cfg.margin", 12), ("tracker_cfg.num_features_min", 100), ("tracker_cfg.num_features_max", 160),
    ("tracker_cfg.max_pixel_displacement", 32), ("tracker_cfg.KLT.win_size", 21), ("tracker_cfg.KLT.max_level", 3), ("tracker_cfg.KLT.max_iter", 10),
    ("tracker_cfg.KLT.eps", 0.03), ("tracker_cfg.FAST.threshold", 10), ("tracker_cfg.FAST.nonmaxSuppression", False),
    ("tracker_cfg.extract_descriptor", False), ("tracker_cfg.differential", False), ("tracker_cfg.match_dropped_tracks", True),
    ("tracker_cfg.descriptor_distance_thresh", 40), ("tracker_cfg.do_outlier_rejection", True), ("tracker_cfg.outlier_rejection.method", "LMEDS"),
    ("tracker_cfg.outlier_rejection.RANSAC_max_iters", 500), ("tracker_cfg.outlier_rejection.RANSAC_reproj_thresh", 2.0),
    ("tracker_cfg.outlier_rejection.confidence", 0.99),
]


def changed(cfg, path, value):
    out = json.loads(json.dumps(cfg))
    d = out
    *head, last = path.split(".")
    for k in head:
        d = d.setdefault(k, {})
    d[last] = value
    return out


def test_refusals_change_nothing(ctx):
    B = 3
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    # point clouds go through the point-cloud tracker whatever tracker_cfg says; an LK tracker with descriptors lets every tracker key be
    # changed alone into a config that parses
    cfg["tracker_cfg"].update(tracker_type="LK", extract_descriptor=True)
    streams = [pc_frames(cfg, 90 + s, duration=2.0) for s in range(B)]
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    for b in (batch, ref):
        b.init_with_sim_depths()
    L = capi.lib()
    for f in range(len(streams[0])):
        feed_pc(batch, [s[f] for s in streams])
        feed_pc(ref, [s[f] for s in streams])
        if f == 20:
            for key, value in REFUSED:
                rc = L.xivo_batch_reset_sequence(batch._h, 1, json.dumps(changed(cfg, key, value)).encode())
                msg = L.xivo_last_error().decode()
                assert rc == -1 and f'"{key}"' in msg, (key, rc, msg)
            for seq in (-1, B):
                assert L.xivo_batch_reset_sequence(batch._h, seq, None) == -1
                assert "out of range" in L.xivo_last_error().decode()
            assert L.xivo_batch_reset_sequence(batch._h, 0, b"{\"camera_cfg\": ") == -1
            assert "parse" in L.xivo_last_error().decode()
            assert L.xivo_batch_reset_sequence(batch._h, 0, json.dumps(changed(cfg, "camera_cfg.model", "fisheye")).encode()) == -1
            assert "fisheye" in L.xivo_last_error().decode()
            with pytest.raises(pyxivo.XivoError, match="tracker_cfg.KLT.win_size"):
                batch.reset_sequence(2, overrides={"tracker_cfg": {"KLT": {"win_size": 21, "max_level": 5, "max_iter": 30, "eps": 0.01}}})
        for s in range(B):
            assert_same(batch, s, ref, s, f"frame {f}, sequence {s}")
    for s in range(B):
        assert np.array_equal(batch.P(s), ref.P(s))
    for b in (batch, ref):
        b.close()


def test_a_failed_handle_cannot_be_reset(ctx):
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14, ctx=ctx, overrides={"message_buffer_size": 0})
    img = np.zeros((480, 640), np.uint8)
    with pytest.raises(pyxivo.XivoError):  # an image on a simulation config: a sticky error of every sequence
        b.visual_meas(0, [img, img])
    assert capi.lib().xivo_batch_reset_sequence(b._h, 0, None) == -3
    assert "earlier call" in capi.lib().xivo_last_error().decode()
    b.close()

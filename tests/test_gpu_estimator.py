"""GPU parity of the full per-frame pipeline (estimator-level C ABI) against the numpy oracle
pipeline on identical synthetic streams.  Tolerances (fp64 device kernels vs fp64 numpy; the update
uses the algebraically identical symmetric standard form instead of Joseph's, DESIGN.md §4):
  pose trajectory   |dT| <= 1e-7 m, |dR| <= 1e-8 after every frame
  covariance        |dP| <= 1e-7 * max|P| at the end
  id / slot tables  exact."""
import os

import numpy as np
import pytest

from oracle.estimator_oracle import EstimatorOracle
from xivo_b200 import pyxivo, sim

pytestmark = pytest.mark.gpu
CFG = os.path.join(os.path.dirname(pyxivo.__file__), "cfg")


def run_oracle_pcw(cfg, msgs, G, F, sim_depths):
    est = EstimatorOracle(cfg, G=G, F=F)
    est.sim_init_depths = sim_depths
    out = []
    for k, ts, p in msgs:
        if k == "imu":
            est.InertialMeas(ts, p[0], p[1])
        else:
            est.VisualMeasPointCloud(ts, p[0], p[1])
            out.append((est.gsb().copy(), sorted(f.id for f in est.instate_features), est.gauge_group))
    return est, out


@pytest.mark.parametrize("G,F,method,sim_depths", [(4, 14, "PrinceDormand", True), (15, 30, "RK4", True), (4, 14, "PrinceDormand", False)])
def test_pcw_trajectory_parity(G, F, method, sim_depths):
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    cfg["integration_method"] = method
    msgs, traj = sim.pcw_stream(cfg, duration=3.0, seed=0)
    ref, ref_out = run_oracle_pcw(cfg, msgs, G, F, sim_depths)
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=G, max_features=F)
    if sim_depths:
        b.init_with_sim_depths()
    k = 0
    for kind, ts, p in msgs:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
        else:
            b.visual_meas_pointcloud(ts, p[0], p[1])
            g_ref, ids_ref, gauge_ref = ref_out[k]
            k += 1
            for s in range(2):
                g = b.gsb(s)
                assert np.abs(g[:, 3] - g_ref[:, 3]).max() <= 1e-7, f"frame {k} seq {s}"
                assert np.abs(g[:, :3] - g_ref[:, :3]).max() <= 1e-8
                assert sorted(b.instate_features(s)["ids"].tolist()) == ids_ref
                assert b.counters(s)["gauge_group"] == gauge_ref
    P = b.P(0)
    assert np.abs(P - ref.P).max() <= 1e-7 * np.abs(ref.P).max()
    assert np.abs(P - P.T).max() <= 1e-12 * np.abs(P).max()  # motion block comes from the host integrator
    assert np.array_equal(b.P(1), P)  # identical inputs -> bit-identical sequences
    V, bg, ba, Rsg = b.motion(0)
    assert np.abs(V - ref.X.Vsb).max() <= 1e-7
    if sim_depths:
        t_end = b.now(0) * 1e-9
        assert np.linalg.norm(b.gsb(0)[:, 3] - traj.pos(t_end)) < 0.05  # and it is actually a working VIO
    b.close()


@pytest.mark.parametrize("case", ["default_203", "small_89", "nodepth_89", "rk4_89", "equidistant_203",
                                  # use_1pt_RANSAC (Estimator::OnePointRANSAC): pass-through, temporary update with every feature rescued, rejections
                                  "ransac_clean_89", "ransac_tight_89", "ransac_outliers_89", "ransac_outliers_203", "ransac_two_groups_89"])
def test_pcw_trajectory_matches_the_reference_estimator(case, tmp_path):
    """The CUDA pipeline against the REFERENCE'S OWN ESTIMATOR (its unmodified sources built into oracle/_ref by oracle/build_ref.py;
    golden arrays tests/golden/reference_pcw.npz where the library is absent) on the point-cloud streams of tests/test_reference_pin.py:
    identical in-state id tables and gauge group after every frame, pose within 1e-7 m / 1e-8, covariance within 1e-7 * max|P|."""
    import test_reference_pin as RP

    name, G, F, duration, seed, sim_depths, over, offset = next(c for c in RP.CASES if c[0] == case)
    cfg = sim.load_cfg(RP.CFG)
    if over:
        cfg.update(over)
    ref, how = RP.reference_result(name, over, G, F, duration, seed, sim_depths, offset, tmp_path)
    msgs, _ = RP.stream(cfg, duration, seed, offset)
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F)
    if sim_depths:
        b.init_with_sim_depths()
    k = 0
    for kind, ts, p in msgs:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
        else:
            b.visual_meas_pointcloud(ts, p[0], p[1])
            g = b.gsb(0)
            assert b.now(0) == int(ref["ts"][k]), f"{how}: frame {k}: a different message executed (heap order)"
            assert sorted(b.instate_features(0)["ids"].tolist()) == [int(x) for x in ref["ids"][k] if x >= 0], f"{how}: frame {k}"
            assert b.counters(0)["gauge_group"] == int(ref["gauge"][k])
            assert np.abs(g[:, 3] - ref["gsb"][k][:, 3]).max() <= 1e-7 and np.abs(g[:, :3] - ref["gsb"][k][:, :3]).max() <= 1e-8, f"{how}: frame {k}"
            k += 1
    assert k == len(ref["gsb"])
    P = b.P(0)
    assert np.abs(P - ref["P"]).max() <= 1e-7 * np.abs(ref["P"]).max()
    if case.startswith("ransac_outliers") or case.startswith("ransac_two"):
        assert b.tracker_counters(0)["num_oneptransac_rejected"] >= 0  # (the last frame's count; rejections over the run are what the id tables pin)
    b.close()


def test_pcw_trajectory_tensor_core_covariance():
    """"covariance_update": "tf32x3" — the downdate of every measurement update runs on wgmma tensor cores with
    fp32-level accuracy (BASELINE configs[2] "fp32 covariance").  Stated tolerance against the fp64 oracle after
    3 s (75 updates): position 1e-4 m, rotation 1e-5, covariance 1e-4 * max|P|; the in-state id tables stay exact."""
    G, F = 15, 30
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    msgs, traj = sim.pcw_stream(cfg, duration=3.0, seed=0)
    ref, ref_out = run_oracle_pcw(cfg, msgs, G, F, True)
    cfg = dict(cfg)
    cfg["covariance_update"] = "tf32x3"
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=G, max_features=F)
    b.init_with_sim_depths()
    k = 0
    for kind, ts, p in msgs:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
        else:
            b.visual_meas_pointcloud(ts, p[0], p[1])
            g_ref, ids_ref, gauge_ref = ref_out[k]
            k += 1
            g = b.gsb(0)
            assert np.abs(g[:, 3] - g_ref[:, 3]).max() <= 1e-4, f"frame {k}"
            assert np.abs(g[:, :3] - g_ref[:, :3]).max() <= 1e-5
            assert sorted(b.instate_features(0)["ids"].tolist()) == ids_ref
    P = b.P(0)
    assert np.abs(P - ref.P).max() <= 1e-4 * np.abs(ref.P).max()
    assert np.abs(P - ref.P).max() > 0  # and it is not the fp64 path
    assert np.array_equal(b.P(1), P)
    assert np.linalg.eigvalsh(0.5 * (P + P.T)).min() > -1e-6 * np.abs(P).max()  # PSD to fp32 accuracy
    b.close()


def test_pcw_single_sequence_pyxivo_facade():
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    msgs, _ = sim.pcw_stream(cfg, duration=1.0, seed=3)
    ref, ref_out = run_oracle_pcw(cfg, msgs, 4, 14, True)
    e = pyxivo.Estimator(cfg, max_groups=4, max_features=14)
    e.InitWithSimDepths()
    for kind, ts, p in msgs:
        if kind == "imu":
            e.InertialMeas(ts, *p[0], *p[1])
        else:
            e.VisualMeasPointCloud(ts, p[0], p[1])
    assert np.abs(e.gsb() - ref.gsb()).max() <= 1e-7
    assert e.num_instate_features() == len(ref.instate_features)
    assert sorted(e.InstateFeatureIDs().tolist()) == sorted(f.id for f in ref.instate_features)
    assert e.MeasurementUpdateInitialized() and e.VisionInitialized()
    e.close()


def test_wrong_mode_is_an_error_not_a_fallback():
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=4, max_features=14, overrides={"message_buffer_size": 0})
    img = np.zeros((480, 640), np.uint8)
    with pytest.raises(pyxivo.XivoError):  # VisualMeas in simulation mode throws in the reference too
        b.visual_meas(0, [img])
        b.visual_meas(40_000_000, [img])
    b.close()


@pytest.mark.parametrize("channels", [1, 3])
def test_image_pipeline_parity(channels):
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    msgs, traj = sim.image_stream(cfg, duration=1.6, channels=channels, seed=1)
    G, F = 4, 14
    ref = EstimatorOracle(cfg, G=G, F=F)
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F)
    nframes = 0
    for kind, ts, p in msgs:
        if kind == "imu":
            ref.InertialMeas(ts, p[0], p[1])
            b.inertial_meas(ts, p[0], p[1])
        else:
            ref.VisualMeas(ts, p)
            b.visual_meas(ts, [p])
            nframes += 1
            ids, xy, st = b.tracked_features(0)
            rid = [f.id for f in ref.tracks]
            # feature-ID / match tables must be identical; positions to float rounding
            assert ids.tolist() == rid, f"frame {nframes}"
            if rid:
                rxy = np.array([f.xp() for f in ref.tracks])
                assert np.abs(xy - rxy).max() <= 1e-3
            g, gr = b.gsb(0), ref.gsb()
            assert np.abs(g - gr).max() <= 1e-5, f"frame {nframes}"
    assert nframes > 25 and len(ref.tracks) >= 30
    c = b.counters(0)
    assert c["num_instate_features"] == len(ref.instate_features) and c["VisionInitialized"] == 1
    b.close()


def _run_image_parity(cfg, G, F, duration, seed, pos_tol=1e-5):
    msgs, _ = sim.image_stream(cfg, duration=duration, seed=seed)
    ref = EstimatorOracle(cfg, G=G, F=F)
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F)
    nframes = 0
    ref.track_counts = []  # tracked features after every frame: workload assertions use run statistics, not the last frame's sawtooth sample
    for kind, ts, p in msgs:
        if kind == "imu":
            ref.InertialMeas(ts, p[0], p[1])
            b.inertial_meas(ts, p[0], p[1])
        else:
            ref.VisualMeas(ts, p)
            b.visual_meas(ts, [p])
            nframes += 1
            ids, xy, _ = b.tracked_features(0)
            rid = [f.id for f in ref.tracks]
            ref.track_counts.append(len(rid))
            assert ids.tolist() == rid, f"frame {nframes}"
            if rid:
                assert np.abs(xy - np.array([f.xp() for f in ref.tracks])).max() <= 1e-3
            assert np.abs(b.gsb(0) - ref.gsb()).max() <= pos_tol, f"frame {nframes}"
            assert sorted(b.instate_features(0)["ids"].tolist()) == sorted(f.id for f in ref.instate_features)
    return ref, b, nframes


def test_config3_tumvi_equidistant_512_parity():
    """BASELINE configs[2]: equidistant 512x512 (cfg/tumvi_cam0.json intrinsics), 200 tracked features, N = 203."""
    cfg = sim.load_cfg(os.path.join(CFG, "tumvi_512_equidistant.json"))
    ref, b, nframes = _run_image_parity(cfg, 15, 30, 1.6, 1)
    tc = np.array(ref.track_counts[5:])  # after the first detections
    print("config3 track counts: mean %.0f min %d max %d, in-state %d" % (tc.mean(), tc.min(), tc.max(), len(ref.instate_features)))
    assert nframes >= 40 and tc.max() == 200 and tc.mean() >= 120 and len(ref.instate_features) >= 15
    P = b.P(0)
    assert P.shape == (203, 203) and np.abs(P - ref.P).max() <= 1e-7 * np.abs(ref.P).max()
    b.close()


def test_config4_stress_1280x1024_800_features_parity():
    """BASELINE configs[3]: 1280x1024, 800 tracked features, G = 15, F = 62 -> N = 299, M up to 124."""
    cfg = sim.load_cfg(os.path.join(CFG, "stress_1280x1024.json"))
    ref, b, nframes = _run_image_parity(cfg, 15, 62, 1.0, 1)
    # the tracked-feature count is a sawtooth (800 right after a re-detection, a few hundred before the next one), and the rendered
    # stream — hence the phase of that sawtooth — may differ between hosts: the workload is asserted on run statistics
    tc = np.array(ref.track_counts[3:])
    print("config4 track counts: mean %.0f min %d max %d" % (tc.mean(), tc.min(), tc.max()))
    assert nframes >= 25 and tc.max() == 800 and tc.mean() >= 350
    assert b.counters(0)["num_instate_features"] == len(ref.instate_features) >= 25
    P = b.P(0)
    assert P.shape == (299, 299) and np.abs(P - ref.P).max() <= 1e-7 * np.abs(ref.P).max()
    b.close()


def test_ate_within_one_percent_of_oracle_through_asl_files(tmp_path):
    """BASELINE north_star: "ATE within 1 % of reference".  The synthetic sequence goes through the formats around the
    path (xivo_b200.dataio): written as an ASL folder, loaded like src/loader.cpp, run, trajectory written like
    src/app/vio.cpp:101-106, evaluated like scripts/tum_rgbd_benchmark_tools/evaluate_ate.py against the ground truth."""
    from xivo_b200 import dataio

    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    msgs, traj = sim.image_stream(cfg, duration=2.4, seed=3)
    cam_dir, imu_dir = dataio.write_asl(str(tmp_path / "seq"), msgs)
    loaded = dataio.load_asl(cam_dir, imu_dir)
    assert sorted((ts, k) for k, ts, _ in loaded) == sorted((ts, k) for k, ts, _ in msgs)
    ref = EstimatorOracle(cfg, G=4, F=14)
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=4, max_features=14)
    st_ours, g_ours, g_ref = [], [], []
    for kind, ts, p in loaded:
        if kind == "imu":
            ref.InertialMeas(ts, p[0], p[1])
            b.inertial_meas(ts, p[0], p[1])
        else:
            img = dataio.read_pnm(p)
            ref.VisualMeas(ts, img)
            b.visual_meas(ts, [img])
            if b.counters(0)["VisionInitialized"]:
                st_ours.append(b.now(0))
                g_ours.append(b.gsb(0))
                g_ref.append(ref.gsb().copy())
    assert len(st_ours) > 30
    out = str(tmp_path / "traj.txt")
    dataio.write_vio_trajectory(out, st_ours, g_ours)
    stamps, poses = dataio.read_vio_trajectory(out)
    t = stamps * 1e-9
    gt = np.array([traj.pos(max(0.0, x - 0.2)) for x in t])  # image_stream keeps the platform at rest for the first 0.2 s
    ate_ours = dataio.ate(t, gt, t, poses[:, :, 3])["rmse"]
    ate_ref = dataio.ate(t, gt, t, np.array(g_ref)[:, :, 3])["rmse"]
    assert abs(ate_ours - ate_ref) <= 0.01 * ate_ref, (ate_ours, ate_ref)
    assert np.abs(poses - np.array(g_ref)).max() <= 1e-5  # the written file carries the oracle's trajectory
    b.close()


def test_ate_on_point_cloud_world_is_small_and_within_one_percent_of_oracle():
    """The same criterion where the filter has metric scale (depths initialised from the simulator, like
    scripts/pyxivo_pcw.py): ATE against the analytic ground truth is centimetres, and ours is within 1 % of the oracle's."""
    from xivo_b200 import dataio

    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    msgs, traj = sim.pcw_stream(cfg, duration=4.0, seed=2)
    ref, _ = run_oracle_pcw(cfg, [], 4, 14, True)
    b = pyxivo.Batch(cfg, n_seq=1, max_groups=4, max_features=14)
    b.init_with_sim_depths()
    t, p_ours, p_ref = [], [], []
    for kind, ts, p in msgs:
        if kind == "imu":
            ref.InertialMeas(ts, p[0], p[1])
            b.inertial_meas(ts, p[0], p[1])
        else:
            ref.VisualMeasPointCloud(ts, p[0], p[1])
            b.visual_meas_pointcloud(ts, p[0], p[1])
            t.append(b.now(0) * 1e-9)
            p_ours.append(b.gsb(0)[:, 3].copy())
            p_ref.append(ref.gsb()[:, 3].copy())
    t = np.array(t)
    keep = t > 0  # the first messages sit in the reorder buffer: the filter clock has not started
    t, p_ours, p_ref = t[keep], np.array(p_ours)[keep], np.array(p_ref)[keep]
    gt = np.array([traj.pos(x) for x in t])
    a_ours, a_ref = dataio.ate(t, gt, t, p_ours), dataio.ate(t, gt, t, p_ref)
    assert a_ref["rmse"] < 0.05 and a_ours["pairs"] > 60
    assert abs(a_ours["rmse"] - a_ref["rmse"]) <= 0.01 * a_ref["rmse"], (a_ours, a_ref)
    b.close()


def test_tracker_only_mode():
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=75, num_features_max=100)
    msgs, _ = sim.image_stream(cfg, duration=1.0, seed=2)
    ref = EstimatorOracle(cfg, G=4, F=14, tracker_only=True)
    b = pyxivo.Batch(cfg, n_seq=3, max_groups=4, max_features=14, tracker_only=True)
    for kind, ts, p in msgs:
        if kind != "img":
            continue
        ref.VisualMeasTrackerOnly(ts, p)
        b.visual_meas(ts, [p, p, p], tracker_only=True)
        for s in range(3):
            ids, xy, _ = b.tracked_features(s)
            assert ids.tolist() == [f.id for f in ref.tracks]
    assert len(ref.tracks) > 50
    b.close()


def test_step_call_equals_message_by_message():
    """xivo_batch_step (8 IMU + 1 frame per call) must be bit-identical to issuing the messages one by one."""
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    msgs, _ = sim.image_stream(cfg, duration=1.2, seed=4)
    a = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14)
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14)
    imu = [m for m in msgs if m[0] == "imu"]
    frames = [m for m in msgs if m[0] == "img"]
    for f, (_, fts, img) in enumerate(frames):
        chunk = imu[8 * f : 8 * f + 8]
        if len(chunk) < 8:
            break
        for _, ts, p in chunk:
            a.inertial_meas(ts, p[0], p[1])
        a.visual_meas(fts, [img, img])
        b.step([ts for _, ts, _ in chunk], [p[0] for _, _, p in chunk], [p[1] for _, _, p in chunk], fts, [img, img])
        for s in range(2):
            assert np.array_equal(a.gsb(s), b.gsb(s))
            assert a.tracked_features(s)[0].tolist() == b.tracked_features(s)[0].tolist()
    assert np.array_equal(a.P(0), b.P(0))
    assert a.counters(0)["num_instate_features"] > 0
    a.close()
    b.close()


def test_prefetched_frames_give_identical_results():
    """xivo_batch_prefetch_frames only moves the upload of the next frame ahead of the current step: the results are bit-identical; a
    prefetch that the next call does not consume (other buffers) is dropped without leaving a trace in the frame ring."""
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    msgs, _ = sim.image_stream(cfg, duration=1.2, seed=5)
    a = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14)
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14)
    imu = [m for m in msgs if m[0] == "imu"]
    frames = [m for m in msgs if m[0] == "img"]
    imgs = [np.ascontiguousarray(f[2]) for f in frames]
    decoy = np.ascontiguousarray(imgs[0][::-1].copy())
    n = min(len(frames), len(imu) // 8)
    pending = []  # what the library holds, oldest first (frame index, or "decoy")
    for f in range(n):
        chunk = imu[8 * f : 8 * f + 8]
        fts = frames[f][1]
        its, g, ac = [ts for _, ts, _ in chunk], [p[0] for _, _, p in chunk], [p[1] for _, _, p in chunk]
        a.step(its, g, ac, fts, [imgs[f], imgs[f]])
        primed = bool(pending) and pending[0] == f
        if primed and len(pending) < 2:
            # streaming order: frame f is on its way already; frame f + 1 (or, now and then, buffers that are never consumed) starts to travel
            if f % 5 == 3:
                b.prefetch_frames([decoy, decoy])
                pending.append("decoy")
            elif f + 1 < n:
                b.prefetch_frames([imgs[f + 1], imgs[f + 1]])
                pending.append(f + 1)
        if len(pending) == 2 and f == 2:
            with pytest.raises(pyxivo.XivoError):
                b.prefetch_frames([decoy, decoy])  # a third pending frame is refused, nothing changes
        b.step(its, g, ac, fts, [imgs[f], imgs[f]])
        pending = pending[1:] if primed else []  # a step with other buffers drops everything that was pending
        if not pending and f + 1 < n:
            b.prefetch_frames([imgs[f + 1], imgs[f + 1]])  # (re)prime after the call
            pending.append(f + 1)
        for s in range(2):
            assert np.array_equal(a.gsb(s), b.gsb(s)), f
            assert a.tracked_features(s)[0].tolist() == b.tracked_features(s)[0].tolist()
    assert np.array_equal(a.P(0), b.P(0))
    assert a.counters(0)["num_instate_features"] > 0
    a.close()
    b.close()

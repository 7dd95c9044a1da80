"""Image-path parity AT THE SIZES BASELINE.json NAMES (round-1 verdict, "no image-path parity at the headline workload"):

* configs[1] = the bench workload: 640x480, 150 tracked features, N = 89 (G=4, F=14), one lock-step batch of 64 sequences
  fed through xivo_batch_step (8 IMU samples + 1 frame per call, like bench.py) from 8 distinct synthetic streams that are
  scattered over the batch, >= 40 frames.  Every sequence must reproduce the oracle of its stream: feature-ID tables exact,
  positions <= 1e-3 px, pose <= 1e-5 per frame, in-state tables exact.
* configs[0] = tracker only at 512x512 with the KLT / FAST parameters of the reference's cfg/tumvi_tracker_only_cam0.json:15-56
  (window 15, 5 levels, 30 iterations, FAST threshold 20 with NMS, mask 15, margin 8), 100 KLT features, grey and BGR input.

The oracles of the distinct streams run in worker processes (they are independent; the GPU box has 16 host CPUs)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
pytestmark = pytest.mark.gpu

N_STREAMS, N_SEQ, DURATION, G, F = 8, 64, 2.0, 4, 14


def _oracle_stream(seed):
    """Renders stream `seed`, runs the pipeline oracle over it, returns the inputs and the per-frame tables."""
    from oracle.estimator_oracle import EstimatorOracle
    from xivo_b200 import sim

    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    msgs, _ = sim.image_stream(cfg, duration=DURATION, seed=seed)
    ref = EstimatorOracle(cfg, G=G, F=F)
    imu_ts, gyro, accel, frames, fts, tables = [], [], [], [], [], []
    for kind, ts, p in msgs:
        if kind == "imu":
            ref.InertialMeas(ts, p[0], p[1])
            imu_ts.append(ts); gyro.append(p[0]); accel.append(p[1])
        else:
            ref.VisualMeas(ts, p)
            frames.append(p); fts.append(ts)
            tables.append(dict(ids=[f.id for f in ref.tracks], xy=np.array([f.xp() for f in ref.tracks]).reshape(-1, 2), gsb=ref.gsb().copy(),
                               instate=sorted(f.id for f in ref.instate_features), n_imu=len(imu_ts)))
    return dict(imu_ts=np.array(imu_ts, np.uint64), gyro=np.array(gyro), accel=np.array(accel), frames=frames, fts=fts, tables=tables)


def _oracle_streams(n, tmp):
    """The oracles of n distinct streams, one worker process each (`python tests/test_gpu_bench_workload.py <seed> <out.pkl>`)."""
    import pickle
    import subprocess

    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(s), os.path.join(tmp, f"stream{s}.pkl")]) for s in range(n)]
    for p in procs:
        assert p.wait() == 0
    return [pickle.load(open(os.path.join(tmp, f"stream{s}.pkl"), "rb")) for s in range(n)]


def test_bench_workload_640x480_150_features_batch_of_64_through_batch_step(tmp_path):
    """One lock-step batch on the shared worker pool, driven as bench.py drives each of its batches."""
    from xivo_b200 import pyxivo, sim

    streams = _oracle_streams(N_STREAMS, str(tmp_path))
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    assert cfg["tracker_cfg"]["num_features_max"] == 150 and cfg["camera_cfg"]["rows"] == 480 and cfg["camera_cfg"]["cols"] == 640
    seq_stream = [(5 * s + 3) % N_STREAMS for s in range(N_SEQ)]  # replicas of a stream are scattered over the batch
    b = pyxivo.Batch(cfg, n_seq=N_SEQ, max_groups=G, max_features=F)
    assert b.N == 89 and b.lanes == 1
    nframes = len(streams[0]["frames"])
    assert nframes >= 40
    k0 = 0
    track_counts = []
    for f in range(nframes):
        # the IMU samples that arrived before frame f (same arrival order as the message list: IMU first on a tie)
        k1 = streams[0]["tables"][f]["n_imu"]
        its = np.stack([streams[t]["imu_ts"][k0:k1] for t in seq_stream], 1)
        g = np.stack([streams[t]["gyro"][k0:k1] for t in seq_stream], 1)
        a = np.stack([streams[t]["accel"][k0:k1] for t in seq_stream], 1)
        fts = np.array([streams[t]["fts"][f] for t in seq_stream], np.uint64)
        b.step(its, g, a, fts, [streams[t]["frames"][f] for t in seq_stream])
        k0 = k1
        for s in range(N_SEQ):
            tab = streams[seq_stream[s]]["tables"][f]
            ids, xy, _ = b.tracked_features(s)
            assert ids.tolist() == tab["ids"], f"frame {f} sequence {s}"
            if tab["ids"]:
                assert np.abs(xy - tab["xy"]).max() <= 1e-3, f"frame {f} sequence {s}"
            assert np.abs(b.gsb(s) - tab["gsb"]).max() <= 1e-5, f"frame {f} sequence {s}"
            if s < N_STREAMS:
                assert sorted(b.instate_features(s)["ids"].tolist()) == tab["instate"], f"frame {f} sequence {s}"
        track_counts.append(np.mean([len(streams[t]["tables"][f]["ids"]) for t in range(N_STREAMS)]))
    tc = np.array(track_counts[6:])
    print("bench workload: tracked features per frame mean %.0f min %.0f max %.0f" % (tc.mean(), tc.min(), tc.max()))
    assert tc.max() >= 140 and tc.mean() >= 100  # "150 tracked features": the cap is reached, the run average stays near it
    c = b.counters(0)
    assert c["MeasurementUpdateInitialized"] == 1 and c["num_instate_features"] >= 8 and c["error"] == 0
    b.close()


def test_config_with_several_lanes_is_refused_at_creation():
    """A handle is one lock-step batch: "lanes" > 1 in the config fails at creation with a message that names the key."""
    from xivo_b200 import pyxivo, sim
    from xivo_b200.capi import XivoError

    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    with pytest.raises(XivoError, match="lanes"):
        pyxivo.Batch(dict(cfg, lanes=3), n_seq=4, max_groups=G, max_features=F)


TRACKER_ONLY_512 = {  # the reference's cfg/tumvi_tracker_only_cam0.json:9-56 with SURVEY.md §8d's overrides for configs[0]
    "simulation": False,
    "camera_cfg": {"model": "equidistant", "rows": 512, "cols": 512},
    "tracker_cfg": {
        "use_prediction": False, "mask_size": 15, "margin": 8, "num_features_min": 75, "num_features_max": 100, "max_pixel_displacement": 64,
        "normalize": False, "match_dropped_tracks": False, "do_outlier_rejection": False,
        "KLT": {"win_size": 15, "max_level": 5, "max_iter": 30, "eps": 0.01},
        "extract_descriptor": False, "descriptor_distance_thresh": -1, "tracker_type": "LK", "detector": "FAST",
        "FAST": {"threshold": 20, "nonmaxSuppression": True},
    },
}


@pytest.mark.parametrize("channels", [1, 3])
def test_config1_tracker_only_512x512_100_klt_features(channels):
    """BASELINE configs[0]: 512x512 frame pair (and the following frames of the same motion), 100 KLT features.  The product is
    created from the reference-shaped tracker-only config (camera geometry + tracker block only, as CreateSystemTrackerOnly is given,
    factory.cpp:84-122); the oracle wants a complete estimator config, so it gets the same two blocks inside the VIO config."""
    from oracle.estimator_oracle import EstimatorOracle
    from xivo_b200 import pyxivo, sim, synth

    canvas = synth.texture_canvas(512, 512, seed=0, pad=64)
    frames = [synth.frame_from_canvas(canvas, 512, 512, (3 * k, 2 * k), noise_seed=10 + k, pad=32) for k in range(8)]
    if channels == 3:
        frames = [synth.to_bgr(f, distinct=True) for f in frames]
    full = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    full["camera_cfg"] = dict(TRACKER_ONLY_512["camera_cfg"], fx=190.98, fy=190.97, cx=254.93, cy=256.90, k0123=[0.0034, 0.0007, -0.0020, 0.0002])
    full["tracker_cfg"] = TRACKER_ONLY_512["tracker_cfg"]
    full["message_buffer_size"] = 0  # no reorder heap: every frame is tracked when it is pushed
    ref = EstimatorOracle(full, G=4, F=14, tracker_only=True)
    b = pyxivo.Batch(TRACKER_ONLY_512, n_seq=2, max_groups=4, max_features=14, tracker_only=True, overrides={"message_buffer_size": 0})
    counts = []
    for k, img in enumerate(frames):
        ts = k * 50_000_000
        ref.VisualMeasTrackerOnly(ts, img)
        b.visual_meas(ts, [img, img], tracker_only=True)
        for s in range(2):
            ids, xy, _ = b.tracked_features(s)
            assert ids.tolist() == [f.id for f in ref.tracks], f"frame {k}"
            assert np.abs(xy - np.array([f.xp() for f in ref.tracks]).reshape(-1, 2)).max() <= 1e-3, f"frame {k}"
        counts.append(len(ref.tracks))
    print("config1 track counts", counts)
    assert counts[0] == 100 and min(counts) >= 75, counts  # 100 detected on the first frame, never below num_features_min afterwards
    b.close()


if __name__ == "__main__":  # oracle worker of _oracle_streams
    import pickle

    with open(sys.argv[2], "wb") as fh:
        pickle.dump(_oracle_stream(int(sys.argv[1])), fh)

"""A sequence's result does not depend on the rest of its batch.

Seven point-cloud sequences that differ from each other run in one pyxivo.Batch and, each alone, in Batch(n_seq=1):
  - different worlds and noise (sim.pcw_stream seeds);
  - a per-sequence deterministic jitter of the IMU stamps (order preserving), so the filters of one propagation launch integrate
    different numbers of Runge-Kutta sub-steps;
  - one sequence with its vision stamps 1000 ns behind the IMU grid (as in test_reference_pin.CASES);
  - one "blind" sequence that receives empty point lists for a stretch of frames, so that it has no measurement while the others update.
Every kernel of the batch sees the other filters' counts, edit lists, staging offsets and operand slabs; a filter that read another
filter's entry would change its own result.  Each sequence must therefore match its solo run bit for bit: pose, motion state, time,
in-state ids and counters after every frame, the covariance at the end.  One jittered stream is also checked against the numpy oracle
(tolerances of test_gpu_estimator.py), since jittered stamps are an input the other pipeline tests never give."""
import os

import numpy as np
import pytest

from oracle.estimator_oracle import EstimatorOracle
from xivo_b200 import pyxivo, sim

pytestmark = pytest.mark.gpu
CFG = os.path.join(os.path.dirname(pyxivo.__file__), "cfg", "pcw_sim.json")
B, G, F, DURATION = 7, 15, 30, 3.0
OFFSET_SEQ, BLIND_SEQ, BLIND_FRAMES = 2, 4, range(30, 46)


def streams(cfg):
    """B message lists with the same kinds in the same order (one Batch call per message index)."""
    out = []
    for s in range(B):
        msgs, _ = sim.pcw_stream(cfg, duration=DURATION, seed=20 + s)
        rng = np.random.default_rng(900 + s)
        amp = 0 if s == 0 else 300_000 * s  # up to 1.8 ms earlier, below the 5 ms IMU period and the 40 ms frame period
        res, frame = [], 0
        for kind, ts, p in msgs:
            if kind == "imu":
                if ts > 0 and amp:
                    ts -= int(rng.integers(0, amp))
            else:
                if s == OFFSET_SEQ:
                    ts += 1000
                if s == BLIND_SEQ and frame in BLIND_FRAMES:
                    p = (np.zeros(0, np.int32), np.zeros((0, 3)))
                frame += 1
            res.append((kind, ts, p))
        assert all(a[1] < b[1] or (a[1] == b[1] and a[0] == "imu" and b[0] == "pc") for a, b in zip(res, res[1:]))  # the arrival order
        out.append(res)
    kinds = [m[0] for m in out[0]]
    assert all([m[0] for m in o] == kinds for o in out)
    return out


def feed(batch, seqs, m):
    kind = seqs[0][m][0]
    ts = np.array([q[m][1] for q in seqs], np.uint64)
    if kind == "imu":
        batch.inertial_meas(ts, np.stack([q[m][2][0] for q in seqs]), np.stack([q[m][2][1] for q in seqs]))
    else:
        batch.visual_meas_pointcloud(ts, [q[m][2][0] for q in seqs], [q[m][2][1] for q in seqs])
    return kind


def state(b, s):
    return (b.gsb(s), *b.motion(s), np.array([b.now(s)]), b.instate_features(s)["ids"], np.array(list(b.counters(s).values())))


MODES = {
    "prince_dormand": ({}, {}),
    "rk4": ({"integration_method": "RK4"}, {}),
    "tf32x3": ({"covariance_update": "tf32x3"}, {}),
    "tf32x3_tc_v1": ({"covariance_update": "tf32x3"}, {"XIVO_TC_V1": "1"}),
    "one_point_ransac": ({"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 1.5, "sim_outliers": {"fraction": 0.08, "pixels": 2.5}}, {}),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_sequence_result_does_not_depend_on_its_batch(ctx, mode, monkeypatch):
    over, env = MODES[mode]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = sim.load_cfg(CFG)
    cfg.update(over)
    seqs = streams(cfg)
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    solo = [pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for _ in range(B)]
    for b in [batch] + solo:
        b.init_with_sim_depths()
    oracle = None
    if mode == "prince_dormand":  # one jittered stream against the numpy oracle
        oracle = EstimatorOracle(cfg, G=G, F=F)
        oracle.sim_init_depths = True
    frame = 0
    updated = np.zeros(B, int)
    for m in range(len(seqs[0])):
        kind = feed(batch, seqs, m)
        for s in range(B):
            feed(solo[s], [seqs[s]], m)
        if oracle is not None:
            _, ts, p = seqs[1][m]
            if kind == "imu":
                oracle.InertialMeas(ts, p[0], p[1])
            else:
                oracle.VisualMeasPointCloud(ts, p[0], p[1])
        if kind == "imu":
            continue
        for s in range(B):
            got, want = state(batch, s), state(solo[s], 0)
            for a, w in zip(got, want):
                assert np.array_equal(a, w), f"{mode}: frame {frame}, sequence {s}"
            updated[s] += batch.counters(s)["MeasurementUpdateInitialized"]
        if oracle is not None:
            g = batch.gsb(1)
            ref = oracle.gsb()
            assert np.abs(g[:, 3] - ref[:, 3]).max() <= 1e-7 and np.abs(g[:, :3] - ref[:, :3]).max() <= 1e-8, f"frame {frame}"
            assert sorted(batch.instate_features(1)["ids"].tolist()) == sorted(f.id for f in oracle.instate_features)
        frame += 1
    assert (updated > 0).all()
    for s in range(B):
        assert np.array_equal(batch.P(s), solo[s].P(0)), f"{mode}: sequence {s}"
    if oracle is not None:
        P = batch.P(1)
        assert np.abs(P - oracle.P).max() <= 1e-7 * np.abs(oracle.P).max()
    # the blind sequence had no measurement during its blind frames while the others had
    assert batch.counters(BLIND_SEQ)["error"] == 0
    for b in [batch] + solo:
        b.close()

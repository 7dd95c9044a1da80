"""Failure isolation (xivo_batch_isolate_failures, pyxivo.Batch(isolate_failures=True), `vio --batch --isolate-failures`).

With isolation on, a sequence that fails leaves the frame and every later call, reports XIVO_SEQ_FAILED once and its status afterwards,
and every other sequence continues bit-identically to a run without it: pose, motion state, time, in-state ids and counters (and the
tracked features on the image path) after every frame, P at the end.  A reset brings the failed sequence back, bit-identical from then on
to a new one-sequence handle.  Failures are provoked only by what a user's config or messages can cause: a memory pool too small for
the features or groups a sequence needs, and a message of the wrong kind.  No test feeds non-finite values."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from xivo_b200 import XivoError, capi, dataio, pyxivo, sim

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "xivo_b200")
CFG = os.path.join(LIBDIR, "cfg")
G, F = 15, 30
SLOTS, STATE = capi.XIVO_ERR_SLOTS, capi.XIVO_ERR_STATE
NO_FEATURES = {"memory": {"max_features": 8}}  # fewer pool slots than the first detection or point cloud asks for
NO_GROUPS = {"memory": {"max_groups": 2}}  # fewer pool slots than the groups a few frames create


def pc_cfg(**kw):
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    cfg.update(kw)
    return cfg


def img_cfg(**tracker):
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80, **tracker)
    return cfg


def with_(cfg, extra):
    out = json.loads(json.dumps(cfg))
    for k, v in extra.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k].update(v)
        else:
            out[k] = v
    return out


def frames_of(msgs):
    """[(imu chunk of 8 (ts, (gyro, accel))), (frame ts, payload)] per frame."""
    imu = [(ts, p) for k, ts, p in msgs if k == "imu"]
    vis = [(ts, p) for k, ts, p in msgs if k != "imu"]
    n = min(len(vis), len(imu) // 8)
    return [(imu[8 * f : 8 * f + 8], vis[f]) for f in range(n)]


def pc_frames(cfg, seed, duration=2.4):
    return frames_of(sim.pcw_stream(cfg, duration=duration, seed=seed)[0])


def img_frames(cfg, seed, duration=1.3):
    return frames_of(sim.image_stream(cfg, duration=duration, seed=seed)[0])


def feed(batch, frames, images):
    """One frame per sequence: its 8 IMU samples, then its point cloud or image."""
    for k in range(8):
        batch.inertial_meas(np.array([f[0][k][0] for f in frames], np.uint64), np.stack([f[0][k][1][0] for f in frames]),
                            np.stack([f[0][k][1][1] for f in frames]))
    ts = np.array([f[1][0] for f in frames], np.uint64)
    if images:
        batch.visual_meas(ts, [f[1][1] for f in frames])
    else:
        batch.visual_meas_pointcloud(ts, [f[1][1][0] for f in frames], [f[1][1][1] for f in frames])


def state(b, s, images):
    out = [b.gsb(s), *b.motion(s), np.array([b.now(s)]), b.instate_features(s)["ids"], np.array(list(b.counters(s).values()))]
    if images:
        out += [*b.tracked_features(s), np.array(list(b.tracker_counters(s).values()))]
    return out


def assert_same(b, s, ref, r, what, images):
    for a, w in zip(state(b, s, images), state(ref, r, images)):
        assert np.array_equal(a, w), what


def spy(batch):
    """Records the return code of every message call of `batch`."""
    rcs = []
    inner = batch._msg

    def rec(rc, what):
        rcs.append(rc)
        return inner(rc, what)

    batch._msg = rec
    return rcs


def assert_refuses(batch, s, code, text):
    got, msg = batch.status(s)
    assert got == code and text in msg, (got, msg)
    assert batch.failed()[s][0] == code
    for get in (batch.gsb, batch.motion, batch.now, batch.counters, batch.P, batch.instate_features, batch.tracked_features):
        with pytest.raises(XivoError, match=f"sequence {s} has failed"):
            get(s)
    out = np.zeros(12)
    assert capi.lib().xivo_get_gsb(batch._h, s, out.ctypes.data_as(C.c_void_p)) == STATE


# ---------------------------------------------------------------- 1. no failure: isolation on is isolation off
CASES = {
    "pcw": (False, lambda: pc_cfg()),
    "pcw_1pt": (False, lambda: pc_cfg(use_1pt_RANSAC=True, **{"1pt_RANSAC_thresh": 1.5, "sim_outliers": {"fraction": 0.08, "pixels": 2.5}})),
    "lk": (True, lambda: img_cfg()),
    "match_brief": (True, lambda: img_cfg(tracker_type="MATCH", extract_descriptor=True, descriptor="BRIEF")),
}


@pytest.mark.parametrize("case", list(CASES))
def test_isolation_without_a_failure_changes_nothing(ctx, case):
    images, make = CASES[case]
    cfg = make()
    B = 3
    streams = [img_frames(cfg, 10 + s) if images else pc_frames(cfg, 10 + s) for s in range(B)]
    on = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx, isolate_failures=True)
    off = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    if not images:
        for b in (on, off):
            b.init_with_sim_depths()
    rcs = spy(on)
    for f in range(len(streams[0])):
        cur = [streams[s][f] for s in range(B)]
        feed(on, cur, images)
        feed(off, cur, images)
        for s in range(B):
            assert_same(on, s, off, s, f"{case}: frame {f}, sequence {s}", images)
    assert set(rcs) == {0} and on.failed() == {}
    for s in range(B):
        assert np.array_equal(on.P(s), off.P(s)), f"{case}: P of sequence {s}"
        assert on.counters(s)["VisionInitialized"] == 1
    for b in (on, off):
        b.close()


# ---------------------------------------------------------------- 2. out of feature slots at the first detection
@pytest.mark.parametrize("images", [True, False], ids=["images", "pointclouds"])
def test_out_of_feature_slots_at_first_detection(ctx, images):
    B, BAD = 4, 2
    cfg = img_cfg() if images else pc_cfg()
    streams = [img_frames(cfg, 20 + s) if images else pc_frames(cfg, 20 + s) for s in range(B)]
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx, isolate_failures=True)
    solo = {s: pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for s in range(B) if s != BAD}
    if not images:
        for b in (batch, *solo.values()):
            b.init_with_sim_depths()
    batch.reset_sequence(BAD, with_(cfg, NO_FEATURES))
    rcs = spy(batch)
    failed_at = None
    for f in range(len(streams[0])):
        n = len(rcs)
        feed(batch, [streams[s][f] for s in range(B)], images)
        if failed_at is None and batch.status(BAD)[0]:
            failed_at = f
            # the message heap may release the frame during one of the IMU calls
            assert rcs[n:].count(capi.XIVO_SEQ_FAILED) == 1 and set(rcs[n:]) == {0, capi.XIVO_SEQ_FAILED}, f"frame {f}: {rcs[n:]}"
        else:
            assert set(rcs[n:]) == {0}, f"frame {f}: {rcs[n:]}"
        for s, b in solo.items():
            feed(b, [streams[s][f]], images)
            assert_same(batch, s, b, 0, f"frame {f}, sequence {s}", images)
    assert failed_at is not None and failed_at < len(streams[0]) - 5
    assert_refuses(batch, BAD, SLOTS, "Out of feature slots in the memory manager")
    for s, b in solo.items():
        assert np.array_equal(batch.P(s), b.P(0)), f"P of sequence {s}"
        assert batch.counters(s)["VisionInitialized"] == 1
    for b in (batch, *solo.values()):
        b.close()


# ---------------------------------------------------------------- 3 + 4. a failure in a later phase, then revival (point clouds)
def test_group_failure_mid_run_then_revival(ctx):
    B, BAD, FAIL_FROM = 3, 1, 10
    cfg = pc_cfg(use_1pt_RANSAC=True, **{"1pt_RANSAC_thresh": 1.5, "sim_outliers": {"fraction": 0.08, "pixels": 2.5}})
    old = [pc_frames(cfg, 30 + s, duration=4.0) for s in range(B)]
    tiny = with_(cfg, NO_GROUPS)
    new_bad, new_good = pc_frames(tiny, 40, duration=4.0), pc_frames(cfg, 41, duration=4.0)
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx, isolate_failures=True)
    ref = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    for b in (batch, ref):
        b.init_with_sim_depths()
    rcs = spy(batch)
    fresh, k, failed_at, revived_at = None, 0, None, None
    for f in range(len(old[0])):
        if f == FAIL_FROM:
            batch.reset_sequence(BAD, tiny)
            k = 0
        if failed_at is not None and revived_at is None and f == failed_at + 3:
            batch.reset_sequence(BAD)  # the failed sequence comes back with the creation config
            fresh = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx)
            fresh.init_with_sim_depths()
            assert batch.status(BAD) == (0, "") and batch.failed() == {}
            revived_at, k = f, 0
        cur = [old[s][f] for s in range(B)]
        feed(ref, cur, False)
        if f >= FAIL_FROM:
            cur[BAD] = (new_good if fresh is not None else new_bad)[k]
            k += 1
        if fresh is not None:
            feed(fresh, [cur[BAD]], False)
        n = len(rcs)
        feed(batch, cur, False)
        if failed_at is None and batch.status(BAD)[0]:
            failed_at = f
            assert rcs[n:].count(capi.XIVO_SEQ_FAILED) == 1 and set(rcs[n:]) == {0, capi.XIVO_SEQ_FAILED}, f"frame {f}: {rcs[n:]}"
            assert_refuses(batch, BAD, SLOTS, "Out of group slots in the memory manager")
        else:
            assert set(rcs[n:]) == {0}, f"frame {f}: {rcs[n:]}"
        for s in range(B):
            if s == BAD:
                if fresh is not None:
                    assert_same(batch, s, fresh, 0, f"frame {f}: revived sequence", False)
                elif f < FAIL_FROM:
                    assert_same(batch, s, ref, s, f"frame {f}, sequence {s}", False)
            else:
                assert_same(batch, s, ref, s, f"frame {f}, sequence {s}", False)
    assert failed_at is not None and revived_at is not None and len(old[0]) - revived_at > 20
    assert batch.counters(BAD)["MeasurementUpdateInitialized"] == 1
    assert np.array_equal(batch.P(BAD), fresh.P(0))
    for s in range(B):
        if s != BAD:
            assert np.array_equal(batch.P(s), ref.P(s))
    for b in (batch, ref, fresh):
        b.close()


# ---------------------------------------------------------------- 4. revival through ragged per-sequence feeding (images)
def pieces(frames, drop=()):
    """feed rounds of one sequence: [(imu (ts, gyro, accel) | None, frame (ts, image) | None)]; frames in `drop` keep only their IMU."""
    out = []
    for f, (imu, (ts, img)) in enumerate(frames):
        im = (np.array([t for t, _ in imu], np.uint64), np.array([p[0] for _, p in imu]), np.array([p[1] for _, p in imu]))
        out.append((im, None if f in drop else (ts, img)))
    return out


def feed_solo(b, piece):
    imu, fr = piece
    if imu is not None:
        for t, g, a in zip(*imu):
            b.inertial_meas(int(t), g, a)
    if fr is not None:
        b.visual_meas(fr[0], [fr[1]])


def test_revival_with_ragged_feed(ctx):
    B, BAD, REVIVE = 3, 1, 10
    cfg = img_cfg()
    drops = [(), (4, 5), tuple(range(6, 9))]
    rounds = [pieces(img_frames(cfg, 50 + s, duration=1.6), drops[s]) for s in range(B)]
    new = pieces(img_frames(cfg, 59, duration=1.0), (3,))
    n = len(rounds[0])
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx, isolate_failures=True)
    solo = {s: pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for s in range(B) if s != BAD}
    batch.reset_sequence(BAD, with_(cfg, NO_FEATURES))
    fresh, k = None, 0
    for r in range(n):
        rnd = [rounds[s][r] for s in range(B)]
        if r == REVIVE:
            batch.reset_sequence(BAD)
            fresh = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx)
        if fresh is not None:
            rnd[BAD] = new[k] if k < len(new) else (None, None)
            feed_solo(fresh, rnd[BAD])
            k += 1
        batch.feed([p[0] for p in rnd], [p[1] for p in rnd])
        for s in range(B):
            if s in solo:
                feed_solo(solo[s], rnd[s])
            ref = solo.get(s, fresh)
            if rnd[s][1] is not None and ref is not None:
                assert_same(batch, s, ref, 0, f"round {r}, sequence {s}", True)
        if r == REVIVE - 1:
            assert_refuses(batch, BAD, SLOTS, "Out of feature slots")
    assert k > 10 and batch.counters(BAD)["VisionInitialized"] == 1 and batch.failed() == {}
    assert np.array_equal(batch.P(BAD), fresh.P(0))
    for s, b in solo.items():
        assert np.array_equal(batch.P(s), b.P(0))
    for b in (batch, fresh, *solo.values()):
        b.close()


# ---------------------------------------------------------------- 5. every sequence fails; the C ABI's refusals
def test_every_sequence_fails(ctx):
    cfg = pc_cfg()
    img = np.zeros((480, 640), np.uint8)
    L = capi.lib()
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14, ctx=ctx, overrides={"message_buffer_size": 0}, isolate_failures=True)
    rcs = spy(b)
    b.visual_meas(0, [img, img])  # an image on a simulation config: a sticky error of every sequence
    assert rcs == [capi.XIVO_SEQ_FAILED]
    for s in range(2):
        assert_refuses(b, s, STATE, "cannot be called in simulation")
    b.visual_meas(1, [img, img])  # both failed: their messages are dropped
    assert rcs[-1] == 0
    assert L.xivo_batch_isolate_failures(b._h, 0) == STATE and "reset it" in L.xivo_last_error().decode()
    code, msg = C.c_int(), C.create_string_buffer(8)
    for seq in (-1, 2):
        assert L.xivo_batch_sequence_status(b._h, seq, C.byref(code), msg, 8) == capi.XIVO_ERR_ARG
    assert L.xivo_batch_sequence_status(b._h, 0, C.byref(code), msg, 8) == 0 and code.value == STATE and len(msg.value) == 7
    assert L.xivo_batch_sequence_status(b._h, 0, None, None, 0) == capi.XIVO_ERR_ARG
    for s in range(2):
        assert L.xivo_batch_reset_sequence(b._h, s, None) == 0
    assert b.failed() == {}
    b.set_isolate_failures(False)  # nothing failed any more
    b.close()
    # without isolation the existing refusals hold
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14, ctx=ctx, overrides={"message_buffer_size": 0})
    with pytest.raises(XivoError):
        b.visual_meas(0, [img, img])
    assert L.xivo_batch_reset_sequence(b._h, 0, None) == STATE and "earlier call" in L.xivo_last_error().decode()
    assert L.xivo_batch_isolate_failures(b._h, 1) == STATE and "earlier call" in L.xivo_last_error().decode()
    assert b.status(0)[0] == STATE and b.status(1)[0] == STATE
    b.close()


# ---------------------------------------------------------------- 6. vio --batch --isolate-failures
def build_vio(tmp_path):
    exe = str(tmp_path / "vio")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "vio.cpp"), "-o", exe,
           "-L", LIBDIR, "-lxivo_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
def test_vio_batch_isolate_failures(tmp_path):
    exe = build_vio(tmp_path)
    cfg = img_cfg()
    paths = {"cfg": str(tmp_path / "cfg.json"), "tiny": str(tmp_path / "tiny.json")}
    json.dump(cfg, open(paths["cfg"], "w"))
    json.dump(with_(cfg, NO_FEATURES), open(paths["tiny"], "w"))
    seqs = {}
    for name, seed, dur in [("a", 131, 1.2), ("bad", 132, 1.0), ("c", 133, 1.4)]:
        msgs, _ = sim.image_stream(cfg, duration=dur, seed=seed)
        cam, imu = dataio.write_asl(str(tmp_path / name), msgs)
        seqs[name] = (cam, imu)
    line = lambda n, out, c=None: f"{seqs[n][0]} {seqs[n][1]} {tmp_path / out}" + (f" {c}" if c else "") + "\n"
    (tmp_path / "three.txt").write_text(line("a", "a3") + line("bad", "bad3", paths["tiny"]) + line("c", "c3"))
    (tmp_path / "two.txt").write_text(line("a", "a2") + line("c", "c2"))
    r = subprocess.run([exe, "--batch", "--isolate-failures", paths["cfg"], str(tmp_path / "three.txt"), "4", "14"], capture_output=True, text=True)
    assert r.returncode == 4, r.stdout + r.stderr
    assert f"sequence 1 ({seqs['bad'][0]}) failed" in r.stderr and "Out of feature slots" in r.stderr, r.stderr
    r2 = subprocess.run([exe, "--batch", paths["cfg"], str(tmp_path / "two.txt"), "4", "14"], capture_output=True, text=True)
    assert r2.returncode == 0, r2.stdout + r2.stderr
    for n in ("a", "c"):
        got, want = open(tmp_path / f"{n}3", "rb").read(), open(tmp_path / f"{n}2", "rb").read()
        assert got == want and len(want.splitlines()) >= 20, n
    n_frames = sum(1 for m in dataio.load_asl(*seqs["bad"]) if m[0] == "img")
    assert len(open(tmp_path / "bad3").read().splitlines()) < n_frames
    # without the flag the first failure ends the run as before
    r3 = subprocess.run([exe, "--batch", paths["cfg"], str(tmp_path / "three.txt"), "4", "14"], capture_output=True, text=True)
    assert r3.returncode == 3 and "Out of feature slots" in r3.stderr, r3.stdout + r3.stderr

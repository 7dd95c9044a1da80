"""Per-sequence feeding (xivo_batch_feed / xivo_batch_feed_png, pyxivo.Batch.feed / feed_png, `vio --batch`).

Image sequences whose message patterns differ -- IMU at 200 or 400 Hz, frames at 20, 25 or 30 Hz, staggered start times, different
lengths, one sequence starting several rounds late, one dropping a stretch of frames -- run in one handle, scheduled by
dataio.feed_rounds.  Each must match a one-sequence handle fed the same messages one at a time, bit for bit: pose, motion state, time,
in-state ids, counters and tracked features after each of its frames, P at the end."""
import ctypes as C
import functools
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import png_oracle as O
from xivo_b200 import XivoError, capi, dataio, pyxivo, sim

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "xivo_b200")
G, F = 4, 14


def small_cfg():
    cfg = sim.load_cfg(os.path.join(LIBDIR, "cfg", "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    return cfg


# seed, IMU period [s], frame period [s], start [ns], duration [s], rounds of delay, dropped frame indices
RAGGED = [
    (71, 0.005, 0.040, 0, 2.0, 0, ()),
    (72, 0.0025, 0.050, 13_000_000, 2.0, 0, ()),
    (73, 0.005, 0.033, 7_000_000, 1.8, 6, ()),  # starts six rounds late
    (74, 0.0025, 0.040, 21_000_000, 0.9, 0, ()),  # ends early
    (75, 0.005, 0.050, 3_000_000, 2.0, 0, tuple(range(12, 20))),  # drops a stretch of frames
    (76, 0.0025, 0.033, 0, 1.6, 0, ()),
]


@functools.lru_cache(maxsize=None)
def stream(seed, imu_dt, vision_dt, t0, duration, dropped=(), channels=1):
    msgs, _ = sim.image_stream(small_cfg(), duration=duration, imu_dt=imu_dt, vision_dt=vision_dt, seed=seed, channels=channels)
    out, k = [], 0
    for kind, ts, p in msgs:
        if kind == "img":
            k += 1
            if k - 1 in dropped:
                continue
        out.append((kind, ts + t0, p))
    return out


def schedule(streams, delays):
    """dataio.feed_rounds, with sequence s's pieces starting delays[s] rounds late."""
    per = [[r[0] for r in dataio.feed_rounds([m])] for m in streams]
    per = [[[]] * d + p for p, d in zip(per, delays)]
    n = max(len(p) for p in per)
    return [[p[r] if r < len(p) else [] for p in per] for r in range(n)]


def ragged(specs=RAGGED, channels=1):
    streams = [stream(seed, idt, vdt, t0, dur, drop, channels) for seed, idt, vdt, t0, dur, _, drop in specs]
    return streams, schedule(streams, [s[5] for s in specs])


def feed_args(rnd, frame=lambda s, img: img):
    """pyxivo.Batch.feed arguments of one round."""
    imu, frames = [], []
    for s, piece in enumerate(rnd):
        im = [m for m in piece if m[0] == "imu"]
        imu.append((np.array([m[1] for m in im], np.uint64), np.array([m[2][0] for m in im]).reshape(-1, 3),
                    np.array([m[2][1] for m in im]).reshape(-1, 3)) if im else None)
        fr = piece[-1] if piece and piece[-1][0] != "imu" else None
        frames.append((fr[1], frame(s, fr[2])) if fr else None)
    return imu, frames


def feed_solo(b, piece):
    for kind, ts, p in piece:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
        else:
            b.visual_meas(ts, [p])


def state(b, s):
    ids, xy, st = b.tracked_features(s)
    return (b.gsb(s), *b.motion(s), np.array([b.now(s)]), b.instate_features(s)["ids"], np.array(list(b.counters(s).values())),
            np.array(list(b.tracker_counters(s).values())), ids, xy, st)


def assert_same(b, s, ref, r, what):
    for a, w in zip(state(b, s), state(ref, r)):
        assert np.array_equal(a, w), what


def run_against_solo(ctx, cfg, rounds, feed, what, on_round=None):
    """Feeds `rounds` through feed(batch, round) and every sequence's pieces one message at a time into its own one-sequence handle;
    compares after every round each sequence that received a frame, and P at the end."""
    B = len(rounds[0])
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    solo = [pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for _ in range(B)]
    frames = np.zeros(B, int)
    partial = 0
    for r, rnd in enumerate(rounds):
        if on_round:
            on_round(r, batch, solo)
        feed(batch, rnd)
        got = [bool(p) and p[-1][0] != "imu" for p in rnd]
        partial += 0 < sum(got) < B
        for s in range(B):
            feed_solo(solo[s], rnd[s])
            if got[s]:
                assert_same(batch, s, solo[s], 0, f"{what}: round {r}, sequence {s}")
                frames[s] += 1
    for s in range(B):
        assert np.array_equal(batch.P(s), solo[s].P(0)), f"{what}: P of sequence {s}"
        assert batch.counters(s)["error"] == 0
    assert partial > 0 and (frames > 0).all()
    return batch, solo


MODES = {
    "prince_dormand": {},
    "rk4": {"integration_method": "RK4"},
    "tf32x3": {"covariance_update": "tf32x3"},
    "one_point_ransac": {"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 1.5},
    "brief_rescue": {"tracker_cfg": {"extract_descriptor": True, "match_dropped_tracks": True, "differential": False, "descriptor_distance_thresh": -1,
                                     "descriptor": "BRIEF"}},
}


@pytest.mark.parametrize("mode", list(MODES))
def test_ragged_image_sequences_match_solo_runs(ctx, mode):
    cfg = small_cfg()
    for k, v in MODES[mode].items():
        if isinstance(v, dict):
            cfg[k] = dict(cfg[k], **v)
        else:
            cfg[k] = v
    _, rounds = ragged()
    batch, solo = run_against_solo(ctx, cfg, rounds, lambda b, rnd: b.feed(*feed_args(rnd)), mode)
    assert sum(batch.counters(s)["MeasurementUpdateInitialized"] for s in range(batch.n)) >= 4
    # the late sequence received nothing during its first rounds, the early one nothing during the last
    assert all(not r[2] for r in rounds[:6]) and not rounds[-1][3]
    for b in [batch, *solo]:
        b.close()


@pytest.mark.parametrize("how", ["copy_engine", "zero_copy", "device"])
def test_ingest_modes(ctx, how):
    import torch

    cfg = small_cfg()
    specs = [(81, 0.005, 0.040, 0, 1.0, 0, ()), (82, 0.0025, 0.050, 5_000_000, 1.0, 1, ()), (83, 0.005, 0.033, 9_000_000, 0.8, 0, ()),
             (84, 0.005, 0.040, 2_000_000, 1.0, 0, (5, 6, 7))]
    _, rounds = ragged(specs)
    B = len(specs)
    pool = torch.empty((B, 240, 320), dtype=torch.uint8).pin_memory()  # evenly spaced pinned sources: pitched runs and the gather path
    pool_np = pool.numpy()

    def frame(s, img):
        if how == "device":
            return torch.from_numpy(img).cuda()
        pool_np[s] = img
        return pool_np[s]

    mode = capi.lib().xivo_set_frame_ingest(0 if how == "zero_copy" else 1)
    try:
        batch, solo = run_against_solo(ctx, cfg, rounds, lambda b, rnd: b.feed(*feed_args(rnd, frame)), how)
    finally:
        capi.lib().xivo_set_frame_ingest(mode)
    for b in [batch, *solo]:
        b.close()


def test_lock_step_feed_equals_step(ctx):
    cfg = small_cfg()
    B = 4
    streams = [stream(90 + s, 0.005, 0.040, 0, 1.2) for s in range(B)]
    rounds = dataio.feed_rounds(streams)
    a = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    b = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    steps = 0
    for r, rnd in enumerate(rounds):
        assert len({len(p) for p in rnd}) == 1  # lock-step: the same pattern for every sequence
        if rnd[0][-1][0] == "imu":  # the trailing IMU samples
            for i in range(len(rnd[0])):
                a.inertial_meas(np.array([p[i][1] for p in rnd], np.uint64), np.stack([p[i][2][0] for p in rnd]), np.stack([p[i][2][1] for p in rnd]))
            b.feed(*feed_args(rnd))
            continue
        k = len(rnd[0]) - 1
        its = np.array([[p[i][1] for p in rnd] for i in range(k)], np.uint64).reshape(k, B)
        g = np.array([[p[i][2][0] for p in rnd] for i in range(k)]).reshape(k, B, 3)
        acc = np.array([[p[i][2][1] for p in rnd] for i in range(k)]).reshape(k, B, 3)
        a.step(its, g, acc, np.array([p[-1][1] for p in rnd], np.uint64), [p[-1][2] for p in rnd])
        b.feed(*feed_args(rnd))
        steps += 1
        for s in range(B):
            assert_same(b, s, a, s, f"round {r}, sequence {s}")
    assert steps >= 25
    for s in range(B):
        assert np.array_equal(a.P(s), b.P(s))
    a.close()
    b.close()


def encode(img, s, k):
    """sequence-specific PNG form of a 3-channel cv2.imread result of a grey frame: 8-bit colour (even s) or 16-bit grey (odd s)"""
    if s % 2 == 0:
        return O.encode(img[..., ::-1], 2, 8, level=[1, 6, 9][k % 3], seed=k)
    rng = np.random.default_rng(100 * s + k)
    return O.encode(img[..., 0].astype(np.uint16) << 8 | rng.integers(0, 256, img.shape[:2]).astype(np.uint16), 0, 16, seed=k)


def test_feed_png_on_subsets_equals_feed_with_decoded_arrays(ctx):
    cfg = small_cfg()
    specs = [(101, 0.005, 0.040, 0, 1.2, 0, ()), (102, 0.0025, 0.050, 4_000_000, 1.2, 0, ()), (103, 0.005, 0.033, 0, 1.0, 2, ()),
             (104, 0.005, 0.050, 8_000_000, 1.2, 0, (3, 4))]
    _, rounds = ragged(specs, channels=3)
    B = len(specs)
    a = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    b = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    partial = 0
    for r, rnd in enumerate(rounds):
        pngs = {}

        def as_png(s, img):
            pngs[s] = encode(img, s, r)
            return pngs[s]

        imu, png_frames = feed_args(rnd, as_png)
        decoded = [None if f is None else (f[0], O.imread(f[1], 3)) for f in png_frames]
        for s, f in enumerate(decoded):
            if f is not None:
                assert np.array_equal(f[1], rnd[s][-1][2])
        a.feed(imu, decoded)
        b.feed_png(imu, png_frames, channels=3)
        partial += 0 < len(pngs) < B
        for s in range(B):
            assert_same(b, s, a, s, f"round {r}, sequence {s}")
    assert partial > 0
    for s in range(B):
        assert np.array_equal(a.P(s), b.P(s))
    a.close()
    b.close()


def test_refusals_change_nothing(ctx):
    cfg = small_cfg()
    specs = RAGGED[:4]
    _, rounds = ragged(specs)
    L = capi.lib()
    B = len(specs)
    refused = []

    def refuse(r, batch, solo):
        if r not in (3, 10, 17, 24):
            return
        before = [state(batch, s) for s in range(B)]
        n_imu = np.array([2, 0, 1, 0], np.int32)
        its = np.arange(1, 4, dtype=np.uint64) * 10**12  # far in the future: pushed, they would change every later result
        g, acc = np.zeros((3, 3)), np.zeros((3, 3))
        fts = np.zeros(B, np.uint64)
        p = lambda x: x.ctypes.data_as(C.c_void_p)
        img = np.zeros((240, 320), np.uint8)
        if r == 3:  # a negative n_imu
            bad = n_imu.copy()
            bad[2] = -1
            rc = L.xivo_batch_feed(batch._h, p(bad), p(its), p(g), p(acc), p(fts), None, 0, 0, 0, 0, 0)
            assert rc == -1 and "sequence 2" in L.xivo_last_error().decode()
        elif r == 10:  # NULL IMU arrays while some n_imu > 0
            rc = L.xivo_batch_feed(batch._h, p(n_imu), None, None, None, p(fts), None, 0, 0, 0, 0, 0)
            assert rc == -1 and "sequence 0" in L.xivo_last_error().decode()
        elif r == 17:  # a frame geometry other than the handle's, for a subset
            ptrs = (C.c_void_p * B)(None, img.ctypes.data, None, img.ctypes.data)
            rc = L.xivo_batch_feed(batch._h, p(n_imu), p(its), p(g), p(acc), p(fts), ptrs, 200, 320, 1, 0, 0)
            assert rc == -1 and "sequence 1" in L.xivo_last_error().decode()
        else:  # a corrupt PNG in one sequence of a subset: found on the device, after the other frame was decoded into its slot
            good = O.encode(img, 0, 8)
            z = O.zstream(good)
            bad = O.with_zstream(good, z[: len(z) // 2])
            with pytest.raises(XivoError, match="png frame 2: truncated deflate"):
                batch.feed_png([(its[:2], g[:2], acc[:2]), None, None, None], [None, (5, good), (6, bad), None], channels=1)
        refused.append(r)
        for s in range(B):
            for x, y in zip(state(batch, s), before[s]):
                assert np.array_equal(x, y), f"refusal at round {r} changed sequence {s}"

    batch, solo = run_against_solo(ctx, cfg, rounds, lambda b, rnd: b.feed(*feed_args(rnd)), "refusals", refuse)
    assert refused == [3, 10, 17, 24]
    for b in [batch, *solo]:
        b.close()


def test_a_failed_handle_refuses_feed(ctx):
    cfg = sim.load_cfg(os.path.join(LIBDIR, "cfg", "pcw_sim.json"))
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=4, max_features=14, ctx=ctx, overrides={"message_buffer_size": 0})
    img = np.zeros((480, 640), np.uint8)
    with pytest.raises(XivoError):  # an image on a simulation config: a sticky error of every sequence
        b.visual_meas(0, [img, img])
    n_imu = np.zeros(2, np.int32)
    assert capi.lib().xivo_batch_feed(b._h, n_imu.ctypes.data_as(C.c_void_p), None, None, None, None, None, 0, 0, 0, 0, 0) == -3
    assert "earlier call" in capi.lib().xivo_last_error().decode()
    b.close()


def test_reset_mid_run_then_feed_matches_a_new_handle(ctx):
    cfg = small_cfg()
    specs = RAGGED[:3]
    streams, rounds = ragged(specs)
    B, SEQ, RESET_AT = 3, 1, 14
    new = dataio.feed_rounds([stream(111, 0.005, 0.040, 0, 1.2)])
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=G, max_features=F, ctx=ctx)
    solo = [pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx) for _ in range(B)]
    fresh = None
    k = 0
    for r, rnd in enumerate(rounds):
        rnd = list(rnd)
        if r == RESET_AT:
            batch.reset_sequence(SEQ)
            fresh = pyxivo.Batch(cfg, n_seq=1, max_groups=G, max_features=F, ctx=ctx)
        if fresh is not None:
            rnd[SEQ] = new[k][0] if k < len(new) else []
            feed_solo(fresh, rnd[SEQ])
            k += 1
        batch.feed(*feed_args(rnd))
        for s in range(B):
            ref = fresh if (s == SEQ and fresh is not None) else solo[s]
            if not (s == SEQ and fresh is not None):
                feed_solo(solo[s], rnd[s])
            if rnd[s] and rnd[s][-1][0] != "imu":
                assert_same(batch, s, ref, 0, f"round {r}, sequence {s}")
    assert k > 20 and batch.counters(SEQ)["VisionInitialized"] == 1
    assert np.array_equal(batch.P(SEQ), fresh.P(0))
    for s in range(B):
        if s != SEQ:
            assert np.array_equal(batch.P(s), solo[s].P(0))
    for b in [batch, fresh, *solo]:
        b.close()


# ---------------------------------------------------------------- vio --batch
def build_vio(tmp_path):
    exe = str(tmp_path / "vio")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "vio.cpp"), "-o", exe,
           "-L", LIBDIR, "-lxivo_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def png_folder(cam, bits):
    """cam0/data as PNG files: 8-bit colour, or 16-bit grey of a grey frame"""
    data = os.path.join(cam, "data")
    for k, f in enumerate(sorted(os.listdir(data))):
        stem, _ = os.path.splitext(f)
        img = dataio.read_pnm(os.path.join(data, f))
        os.remove(os.path.join(data, f))
        png = encode(img, 0 if bits == 8 else 1, k)
        with open(os.path.join(data, stem + ".png"), "wb") as fh:
            fh.write(png)
    csv = os.path.join(cam, "data.csv")
    text = open(csv).read().replace(".ppm", ".png")
    open(csv, "w").write(text)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
def test_vio_batch_equals_solo_vio_runs(tmp_path):
    exe = build_vio(tmp_path)
    cfg = small_cfg()
    own = json.loads(json.dumps(cfg))
    own["visual_meas_std"] = 1.5
    own["X"]["Vsb"] = [0.01, 0.0, -0.01]
    paths = {"cfg": str(tmp_path / "cfg.json"), "own": str(tmp_path / "own.json"), "bad": str(tmp_path / "bad.json")}
    json.dump(cfg, open(paths["cfg"], "w"))
    json.dump(own, open(paths["own"], "w"))
    bad = json.loads(json.dumps(cfg))
    bad["tracker_cfg"]["num_features_max"] = 90
    json.dump(bad, open(paths["bad"], "w"))
    seqs = []
    for name, seed, idt, vdt, t0, dur, kind, c in [("pnm", 121, 0.005, 0.040, 0, 1.2, None, None), ("png8", 122, 0.0025, 0.050, 6_000_000, 1.0, 8, None),
                                                   ("png16", 123, 0.005, 0.033, 3_000_000, 1.4, 16, paths["own"])]:
        msgs = stream(seed, idt, vdt, t0, dur, (), 3)
        cam, imu = dataio.write_asl(str(tmp_path / name), msgs)
        if kind:
            png_folder(cam, kind)
        seqs.append((cam, imu, str(tmp_path / (name + ".batch")), c))
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{cam} {imu} {out}" + (f" {c}" if c else "") + "\n" for cam, imu, out, c in seqs))
    r = subprocess.run([exe, "--batch", paths["cfg"], str(lst), "4", "14"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    for cam, imu, out, c in seqs:
        solo_out = out + ".solo"
        r = subprocess.run([exe, c or paths["cfg"], cam, imu, solo_out, "4", "14"], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        lines = open(solo_out).read().splitlines()
        at_frames = [line for line, m in zip(lines, dataio.load_asl(cam, imu)) if m[0] == "img"]
        got = open(out).read().splitlines()
        assert len(at_frames) >= 20 and got == at_frames, cam
    # a line whose config differs in a batch-wide setting fails with that key
    lst.write_text(lst.read_text() + f"{seqs[0][0]} {seqs[0][1]} {tmp_path}/x.batch {paths['bad']}\n")
    r = subprocess.run([exe, "--batch", paths["cfg"], str(lst), "4", "14"], capture_output=True, text=True)
    assert r.returncode == 3 and '"tracker_cfg.num_features_max"' in r.stderr, r.stderr

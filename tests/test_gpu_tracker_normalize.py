"""tracker_cfg.normalize on the device: cv::normalize(NORM_MINMAX) of every frame before the tracker reads it (src/tracker.cpp:343-344,
:463-467).

Kernel level: xivo_normalize_minmax is bit-identical to the numpy restatement (tests/normalize_oracle.py, pinned on cv2 by
tests/test_normalize_logic.py) over every (min, max) pair, on seeded and constant frames, and on frames that start off the 16-byte grid.
End to end, by equivalence: a handle with normalize on, fed raw low-contrast frames, must end every frame bit-identical to a handle with
normalize off fed the oracle-normalised frames -- pose, P, tracked features and descriptors, in-state feature and group tables, counters --
while a handle with normalize off fed the raw frames must not (so that the comparison is not vacuous)."""
import hashlib
import json
import os

import numpy as np
import pytest

import normalize_oracle as O
import png_oracle as PO
from xivo_b200 import XivoError, capi, dataio, pyxivo, sim

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
GOLDEN = os.path.join(ROOT, "tests", "golden", "normalize_cv2.npz")
G, F = 4, 14


# ---------------------------------------------------------------- kernel level
def test_every_min_max_pair_matches_the_oracle(ctx):
    pairs = [(lo, hi) for lo in range(256) for hi in range(lo, 256)]
    assert len(pairs) == 32_896
    lo, hi = np.array(pairs, np.int64).T
    frames = np.clip(np.arange(256)[None, :], lo[:, None], hi[:, None]).astype(np.uint8).reshape(-1, 16, 16)
    got = ctx.normalize_minmax(frames)
    want = np.stack([O.lut(a, b) for a, b in pairs])[np.arange(len(pairs))[:, None], frames.reshape(len(pairs), -1)].reshape(frames.shape)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("rows,cols,cn", [(480, 640, 1), (480, 640, 3), (481, 643, 1), (481, 643, 3), (1024, 1280, 1)])
def test_seeded_frames_match_the_oracle(ctx, rows, cols, cn):
    rng = np.random.default_rng(rows + cols + cn)
    shape = (rows, cols) if cn == 1 else (rows, cols, 3)
    frames = np.stack([rng.integers(lo, hi + 1, shape).astype(np.uint8) for lo, hi in [(0, 255), (40, 170), (90, 91), (7, 250), (200, 255)]])
    frames[3, 0, 0] = 7  # the extremes sit in the first and the last byte of a frame
    frames[3, -1, -1] = 250
    got = ctx.normalize_minmax(frames, channels=cn)
    for k in range(len(frames)):
        assert np.array_equal(got[k], O.normalize_minmax(frames[k])), (rows, cols, cn, k)


def test_constant_frames_become_zeros(ctx):
    frames = np.stack([np.full((481, 643, 3), v, np.uint8) for v in (0, 1, 77, 254, 255)])
    assert not ctx.normalize_minmax(frames, channels=3).any()


def test_golden_frames_match_cv2(ctx):
    """The frames of tests/golden/normalize_cv2.npz, as cv2 4.13 normalised them, through the kernels."""
    g = np.load(GOLDEN)
    for k, case in enumerate(O.GOLDEN_CASES):
        img = O.golden_frame(*case)
        got = ctx.normalize_minmax(img[None], channels=case[2])[0]
        assert hashlib.sha256(got.tobytes()).digest() == g["out_sha"][k].tobytes(), case


@pytest.mark.parametrize("rows,cols,cn,n", [(1, 1, 1, 7), (1, 15, 1, 5), (1, 17, 1, 9), (3, 5, 3, 11), (2, 8, 1, 3), (7, 9, 3, 33), (33, 31, 1, 17)])
def test_frames_off_the_16_byte_grid(ctx, rows, cols, cn, n):
    """Frames lie back to back, so with an odd size frame k starts at k * size bytes: every head / body / tail split of the kernels."""
    rng = np.random.default_rng(rows * cols * cn + n)
    shape = (n, rows, cols) if cn == 1 else (n, rows, cols, 3)
    frames = rng.integers(0, 256, shape).astype(np.uint8)
    for k in range(n):  # each frame its own extremes, placed anywhere
        f = frames[k].reshape(-1)
        lo, hi = sorted(rng.integers(0, 256, 2))
        f[:] = np.clip(f, lo, hi)
        f[rng.integers(0, f.size)] = lo
        f[rng.integers(0, f.size)] = hi
    got = ctx.normalize_minmax(frames, channels=cn)
    for k in range(n):
        assert np.array_equal(got[k], O.normalize_minmax(frames[k])), (rows, cols, cn, k)


def test_wrapper_refuses_bad_shapes(ctx):
    with pytest.raises(ValueError):
        ctx.normalize_minmax(np.zeros((2, 4, 4, 3), np.uint8), channels=1)
    with pytest.raises(ValueError):
        ctx.normalize_minmax(np.zeros((2, 4, 4, 2), np.uint8), channels=3)
    assert ctx.normalize_minmax(np.zeros((0, 4, 4), np.uint8)).shape == (0, 4, 4)


# ---------------------------------------------------------------- end to end, by equivalence
def small_cfg(normalize, **tracker):
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80, normalize=normalize, **tracker)
    return cfg


BRIEF = dict(extract_descriptor=True, descriptor="BRIEF", differential=False, descriptor_distance_thresh=-1)
MODES = {
    "lk": {},
    "match_brief": dict(BRIEF, tracker_type="MATCH"),
    "rescue_homography": dict(BRIEF, match_dropped_tracks=True, do_outlier_rejection=True),
}


def squeeze(img):
    """Low-contrast version of a rendered frame: the texture in [40, 150], a colour frame's channels shifted apart by 10 (so the extremes of
    the frame are not those of any one channel)."""
    out = 40 + img.astype(np.int32) * 110 // 255
    if img.ndim == 3:
        out = out + np.array([0, 10, 20])
    return out.astype(np.uint8)


def stream(seed, imu_dt, vision_dt, t0, duration, channels=1):
    msgs, _ = sim.image_stream(small_cfg(False), duration=duration, imu_dt=imu_dt, vision_dt=vision_dt, seed=seed, channels=channels)
    return [(k, ts + t0, squeeze(p) if k == "img" else p) for k, ts, p in msgs]


RAGGED = [(131, 0.005, 0.040, 0, 1.6), (132, 0.0025, 0.050, 11_000_000, 1.6), (133, 0.005, 0.033, 5_000_000, 1.2), (134, 0.005, 0.040, 0, 1.6)]


def ragged_rounds(channels=1, specs=RAGGED):
    return dataio.feed_rounds([stream(*s, channels=channels) for s in specs])


def feed_args(rnd, frame=lambda s, img: img):
    imu, frames = [], []
    for s, piece in enumerate(rnd):
        im = [m for m in piece if m[0] == "imu"]
        imu.append((np.array([m[1] for m in im], np.uint64), np.array([m[2][0] for m in im]).reshape(-1, 3),
                    np.array([m[2][1] for m in im]).reshape(-1, 3)) if im else None)
        fr = piece[-1] if piece and piece[-1][0] != "imu" else None
        frames.append((fr[1], frame(s, fr[2])) if fr else None)
    return imu, frames


def normalised(s, img):
    return O.normalize_minmax(img)


def state(b, s, desc, tracker_only):
    out = [*b.tracked_features(s), np.array(list(b.tracker_counters(s).values()))]
    if desc:
        out += list(b.tracked_descriptors(s))
    if not tracker_only:
        out += [b.gsb(s), *b.motion(s), b.P(s), np.array(list(b.counters(s).values()))]
        out += list(b.instate_feature_table(s).values()) + list(b.instate_group_table(s).values())
    return out


def same(x, y):
    return len(x) == len(y) and all(a.shape == b.shape and np.array_equal(a, b) for a, b in zip(x, y))


class Trio:
    """on: normalize on, fed the raw frames; ref: normalize off, fed the oracle-normalised frames; raw: normalize off, fed the raw frames."""

    def __init__(self, ctx, tracker=None, n_seq=4, tracker_only=False):
        tracker = tracker or {}
        self.cfgs = {k: small_cfg(k == "on", **tracker) for k in ("on", "ref", "raw")}
        self.h = {k: pyxivo.Batch(c, n_seq=n_seq, max_groups=G, max_features=F, tracker_only=tracker_only, ctx=ctx) for k, c in self.cfgs.items()}
        self.tracker_only = tracker_only
        self.desc = bool(tracker.get("extract_descriptor"))
        self.differs = False
        self.checked = 0

    def check(self, seqs, what):
        on, ref, raw = self.h["on"], self.h["ref"], self.h["raw"]
        for s in seqs:
            a = state(on, s, self.desc, self.tracker_only)
            assert same(a, state(ref, s, self.desc, self.tracker_only)), f"{what}, sequence {s}"
            self.differs |= not same(a, state(raw, s, self.desc, self.tracker_only))
            self.checked += 1

    def close(self):
        assert self.checked >= 20 and self.differs, "normalize on and off gave the same results on the raw frames: the comparison is vacuous"
        for b in self.h.values():
            assert self.tracker_only or all(b.counters(s)["error"] == 0 for s in range(b.n))
            b.close()


def json_copy(d):
    return json.loads(json.dumps(d))


def with_frames(rnd):
    return [s for s, p in enumerate(rnd) if p and p[-1][0] != "imu"]


def run_feed(trio, rounds, on_frame=lambda s, img: img, on_round=None):
    for r, rnd in enumerate(rounds):
        if on_round:
            on_round(r)
        trio.h["on"].feed(*feed_args(rnd, on_frame))
        trio.h["ref"].feed(*feed_args(rnd, normalised))
        trio.h["raw"].feed(*feed_args(rnd))
        trio.check(with_frames(rnd), f"round {r}")


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("channels", [1, 3])
def test_ragged_feed_equals_normalised_frames(ctx, mode, channels):
    if mode != "lk" and channels == 3:
        pytest.skip("the colour case is the LK tracker's; the descriptor paths read the same level-0 image")
    trio = Trio(ctx, MODES[mode])
    run_feed(trio, ragged_rounds(channels))
    trio.close()


def test_host_tracker_decisions(ctx, monkeypatch):
    monkeypatch.setenv("XIVO_HOST_TRACKER_DECISIONS", "1")  # read when a handle sees its first frame
    trio = Trio(ctx)
    run_feed(trio, ragged_rounds())
    trio.close()


def test_tracker_only_handle(ctx):
    frames = [[p for k, _, p in stream(150 + s, 0.005, 0.040, 0, 1.2) if k == "img"] for s in range(4)]
    trio = Trio(ctx, n_seq=4, tracker_only=True)
    for k in range(len(frames[0])):
        cur = [frames[s][k] for s in range(4)]
        trio.h["on"].visual_meas(k * 40_000_000, cur, tracker_only=True)
        trio.h["ref"].visual_meas(k * 40_000_000, [O.normalize_minmax(f) for f in cur], tracker_only=True)
        trio.h["raw"].visual_meas(k * 40_000_000, cur, tracker_only=True)
        trio.check(range(4), f"frame {k}")
    trio.close()


@pytest.mark.parametrize("how", ["copy_engine", "zero_copy", "device"])
def test_ingest_modes_leave_the_callers_frames_alone(ctx, how):
    import torch

    rounds = ragged_rounds()
    pool = torch.empty((4, 240, 320), dtype=torch.uint8).pin_memory()
    pool_np = pool.numpy()
    given = []

    def frame(s, img):
        if how == "device":
            t = torch.from_numpy(img).cuda()
            given.append((t, img.copy()))
            return t
        pool_np[s] = img
        given.append((pool_np[s], img.copy()))
        return pool_np[s]

    mode = capi.lib().xivo_set_frame_ingest(0 if how == "zero_copy" else 1)
    try:
        trio = Trio(ctx)

        def after_round(r):
            for buf, was in given:  # the frames of the previous round, as the caller still holds them
                now = buf.cpu().numpy() if how == "device" else buf
                assert np.array_equal(now, was), f"{how}: the caller's frame was written (round {r})"
            given.clear()

        run_feed(trio, rounds, frame, on_round=after_round)
        after_round(len(rounds))
        trio.close()
    finally:
        capi.lib().xivo_set_frame_ingest(mode)


@pytest.mark.parametrize("channels", [1, 3])
def test_feed_png_on_subsets(ctx, channels):
    rounds = ragged_rounds(channels)
    trio = Trio(ctx)
    partial = 0
    for r, rnd in enumerate(rounds):
        def as_png(s, img):
            return PO.encode(img if channels == 1 else img[..., ::-1], 0 if channels == 1 else 2, 8, level=1, seed=r)

        trio.h["on"].feed_png(*feed_args(rnd, as_png), channels=channels)
        trio.h["ref"].feed(*feed_args(rnd, normalised))
        trio.h["raw"].feed(*feed_args(rnd))
        seqs = with_frames(rnd)
        partial += 0 < len(seqs) < 4
        trio.check(seqs, f"round {r}")
    assert partial > 0
    trio.close()


def test_ragged_feed_with_a_reset_in_the_middle(ctx):
    rounds = ragged_rounds()
    SEQ, RESET_AT = 1, 12
    trio = Trio(ctx)
    new = dataio.feed_rounds([stream(139, 0.005, 0.040, 0, 1.0)])
    k = 0
    for r, rnd in enumerate(rounds):
        rnd = list(rnd)
        if r == RESET_AT:
            off = json_copy(trio.h["on"].cfg)
            off["tracker_cfg"]["normalize"] = False
            with pytest.raises(XivoError, match="tracker_cfg.normalize"):  # batch-wide: a sequence cannot switch it alone
                trio.h["on"].reset_sequence(SEQ, cfg=off)
            for b in trio.h.values():
                b.reset_sequence(SEQ)
        if r >= RESET_AT:
            rnd[SEQ] = new[k][0] if k < len(new) else []
            k += 1
        trio.h["on"].feed(*feed_args(rnd))
        trio.h["ref"].feed(*feed_args(rnd, normalised))
        trio.h["raw"].feed(*feed_args(rnd))
        trio.check(with_frames(rnd), f"round {r}")
    assert k > 10 and trio.h["on"].counters(SEQ)["VisionInitialized"] == 1
    trio.close()


# ---------------------------------------------------------------- launch count
@pytest.mark.parametrize("mode", ["lk", "match_brief"])
def test_normalize_adds_two_launches_per_frame_batch(ctx, mode):
    """With no message buffering every visual_meas call is one frame-batch through the tracker.  The normalize-on handle fed the raw frames
    and the normalize-off handle fed the normalised frames track identically, so their launches differ by the two normalisation kernels
    per frame-batch exactly."""
    cfg = small_cfg(False, **MODES[mode])
    cfg["message_buffer_size"] = 0
    frames = [[squeeze(p) for k, _, p in sim.image_stream(cfg, duration=0.8, seed=140 + s)[0] if k == "img"] for s in range(3)]
    counts = {}
    for name, normalize, transform in (("on", True, lambda f: f), ("off", False, O.normalize_minmax)):
        c = json_copy(cfg)
        c["tracker_cfg"]["normalize"] = normalize
        b = pyxivo.Batch(c, n_seq=3, max_groups=G, max_features=F, tracker_only=True, ctx=ctx)
        n0 = capi.launch_count()
        for k in range(len(frames[0])):
            b.visual_meas(k * 40_000_000, [transform(frames[s][k]) for s in range(3)], tracker_only=True)
        counts[name] = capi.launch_count() - n0
        counts[name + "_features"] = [b.tracked_features(s)[0].tolist() for s in range(3)]
        b.close()
    assert counts["on_features"] == counts["off_features"]
    assert counts["on"] - counts["off"] == 2 * len(frames[0])

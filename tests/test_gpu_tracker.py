"""GPU parity: tracker kernels through the C ABI vs the committed cv2 golden vectors and the C
oracle.  Integer stages are bit-exact; LK positions agree to float rounding."""
import os

import numpy as np
import pytest

from oracle import tracker_oracle as T
from xivo_b200 import synth

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "tracker_cv2.npz"))


def test_pyramid_golden(ctx):
    lv = ctx.build_pyramid(G["a"], 15, 5)
    assert len(lv) == 3
    for i, l in enumerate(lv):
        assert np.array_equal(l, G[f"pyr{i}"])
    lv3 = ctx.build_pyramid(G["pyr3_0"], 15, 5)
    for i, l in enumerate(lv3):
        assert np.array_equal(l, G[f"pyr3_{i}"])


@pytest.mark.parametrize("shape,cn", [((480, 640), 1), ((512, 512), 3), ((477, 635), 1), ((1024, 1280), 1), ((33, 47), 3)])
def test_pyramid_vs_oracle(ctx, shape, cn):
    a, _ = synth.frame_pair(shape[0], shape[1], seed=1)
    img = a if cn == 1 else synth.to_bgr(a, True)
    got, ref = ctx.build_pyramid(img, 15, 5), T.pyramid(img, 15, 5)
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)


@pytest.mark.parametrize("thr", [10, 20])
def test_fast_golden(ctx, thr):
    xy, sc, n = ctx.fast_detect(G["a"], thr)
    g = G[f"fast{thr}"]
    assert n == len(g) and np.array_equal(xy, g[:, :2]) and np.array_equal(sc, g[:, 2])


def test_fast_bgr_golden(ctx):
    xy, sc, n = ctx.fast_detect(G["pyr3_0"], 20)
    g = G["fast20_bgr"]
    assert n == len(g) and np.array_equal(xy, g[:, :2]) and np.array_equal(sc, g[:, 2])


@pytest.mark.parametrize("shape,thr,nonmax", [((480, 640), 20, True), ((512, 512), 5, True), ((1024, 1280), 20, True),
                                              ((61, 67), 10, True), ((240, 320), 20, False), ((7, 9), 5, True)])
def test_fast_vs_oracle(ctx, shape, thr, nonmax):
    a, _ = synth.frame_pair(shape[0], shape[1], seed=2)
    xy, sc, n = ctx.fast_detect(a, thr, nonmax, max_kp=1 << 17)
    rxy, rsc, rn = T.fast_detect(a, thr, nonmax)
    assert n == rn
    assert np.array_equal(xy, rxy) and np.array_equal(sc, rsc)


def test_fast_constant_image_has_no_corners(ctx):
    xy, sc, n = ctx.fast_detect(np.full((64, 64), 127, np.uint8), 5)
    assert n == 0 and len(xy) == 0


def test_fast_truncation_reports_total(ctx):
    a, _ = synth.frame_pair(240, 320, seed=4)
    xy_all, _, n_all = ctx.fast_detect(a, 5)
    xy, sc, n = ctx.fast_detect(a, 5, max_kp=10)
    assert n == n_all and len(xy) == 10 and np.array_equal(xy, xy_all[:10])


@pytest.mark.parametrize("name", ["gray", "bgr"])
def test_lk_golden(ctx, name):
    a, b = (G["a"], G["b"]) if name == "gray" else (synth.to_bgr(G["a"], True), synth.to_bgr(G["b"], True))
    p1, st, er = ctx.lk_track(a, b, G["lk_p0"], G["lk_init"])
    assert np.array_equal(st, G[f"lk_{name}_st"])
    ok = st == 1
    assert np.abs(p1[ok] - G[f"lk_{name}_p1"][ok]).max() < 5e-3  # OpenCV's own float-lane rounding
    assert np.abs(er[ok] - G[f"lk_{name}_err"][ok]).max() < 5e-3


@pytest.mark.parametrize("shape,cn,npts,init_off", [((480, 640), 1, 150, (0, 0)), ((480, 640), 3, 150, (-2.5, -1.5)),
                                                    ((512, 512), 3, 200, (0, 0)), ((1024, 1280), 1, 800, (1.0, 1.0))])
def test_lk_vs_oracle(ctx, shape, cn, npts, init_off):
    a, b = synth.frame_pair(shape[0], shape[1], seed=0)
    xy, sc, _ = T.fast_detect(a, 20)
    order = np.lexsort((xy[:, 0], xy[:, 1], -sc))[:npts]
    p0 = xy[order].astype(np.float32)
    if cn == 3:
        a, b = synth.to_bgr(a), synth.to_bgr(b)
    init = p0 + np.float32(init_off)
    p1, st, er = ctx.lk_track(a, b, p0, init)
    r1, rst, rer = T.lk_track(a, b, p0, init)
    # status table is an index table -> must match exactly; positions to float rounding
    assert np.array_equal(st, rst)
    ok = st == 1
    assert ok.sum() > 0.9 * len(p0)
    assert np.abs(p1[ok] - r1[ok]).max() < 1e-4
    assert np.abs(er[ok] - rer[ok]).max() < 1e-4
    assert np.abs((p1[ok] - p0[ok]).mean(0) - np.array([-3.0, -2.0])).max() < 0.1


def test_lk_edge_cases(ctx):
    a, b = synth.frame_pair(240, 320, seed=6)
    # points outside the image, on the border, on a flat patch; plus an empty call
    p0 = np.float32([[-40, -40], [0, 0], [319, 239], [400, 100], [160, 120]])
    flat = a.copy()
    flat[80:160, 100:220] = 128
    p1, st, er = ctx.lk_track(flat, b, p0, p0)
    r1, rst, rer = T.lk_track(flat, b, p0, p0)
    assert np.array_equal(st, rst)
    assert st[0] == 0 and st[3] == 0 and st[4] == 0  # out of bounds / minEig rejections
    ok = st == 1
    if ok.any():
        assert np.abs(p1[ok] - r1[ok]).max() < 1e-4
    p1, st, er = ctx.lk_track(a, b, np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32))
    assert len(p1) == 0


def test_lk_no_initial_flow_and_params(ctx):
    a, b = synth.frame_pair(240, 320, seed=7, shift=(1, 0))
    xy, sc, _ = T.fast_detect(a, 20)
    p0 = xy[np.lexsort((xy[:, 0], xy[:, 1], -sc))[:64]].astype(np.float32)
    for kw in (dict(use_initial_flow=False), dict(win=11, max_level=3), dict(max_iter=5, eps=0.1), dict(win=21, max_level=2)):
        p1, st, _ = ctx.lk_track(a, b, p0, p0 + 3.0, **kw)
        r1, rst, _ = T.lk_track(a, b, p0, p0 + 3.0, **kw)
        assert np.array_equal(st, rst)
        ok = st == 1
        assert np.abs(p1[ok] - r1[ok]).max() < 1e-4


@pytest.mark.parametrize("win", [3, 7, 13, 15])
def test_lk_fast_path_equals_generic_kernel(ctx, win, monkeypatch):
    """Single-channel frames with win <= 15 take lk_kernel_fast (register template, shuffled neighbours);
    XIVO_LK_GENERIC=1 routes the same call through lk_kernel<1>.  Both evaluate the same exact integer
    window sums, so every output is bit-identical — including points whose windows cross the border."""
    a, b = synth.frame_pair(240, 320, seed=11, shift=(2, -1))
    xy, sc, _ = T.fast_detect(a, 20)
    p0 = xy[np.lexsort((xy[:, 0], xy[:, 1], -sc))[:100]].astype(np.float32)
    border = np.float32([[1, 1], [318, 2], [3, 237], [317, 238], [0.5, 120.25], [319, 100], [160.5, 0], [100, 239]])
    p0 = np.concatenate([p0, border])
    init = p0 + np.float32([1.5, -0.75])
    max_level = 3 if win >= 7 else 4
    monkeypatch.delenv("XIVO_LK_GENERIC", raising=False)
    p1, st, er = ctx.lk_track(a, b, p0, init, win=win, max_level=max_level)
    monkeypatch.setenv("XIVO_LK_GENERIC", "1")
    g1, gst, ger = ctx.lk_track(a, b, p0, init, win=win, max_level=max_level)
    monkeypatch.delenv("XIVO_LK_GENERIC", raising=False)
    assert np.array_equal(st, gst)
    assert np.array_equal(p1, g1)
    assert np.array_equal(er, ger)
    r1, rst, rer = T.lk_track(a, b, p0, init, win=win, max_level=max_level)
    assert np.array_equal(st, rst)
    ok = st == 1
    assert np.abs(p1[ok] - r1[ok]).max() < 1e-4
    assert np.abs(er[ok] - rer[ok]).max() < 1e-4


@pytest.mark.parametrize("shape", [(480, 640), (240, 320), (96, 132), (67, 44), (1024, 1280)])
def test_pyramid_vector_path_equals_bytewise_kernel(ctx, shape, monkeypatch):
    """Single-channel levels whose width is a multiple of 4 take pyrdown_vec_kernel (word staging, dp4a);
    XIVO_PYRDOWN_GENERIC=1 forces the byte-wise kernel.  Same integers, so every level is identical —
    and equal to the C oracle (cv2.pyrDown restated)."""
    a, _ = synth.frame_pair(shape[0], shape[1], seed=21)
    monkeypatch.delenv("XIVO_PYRDOWN_GENERIC", raising=False)
    fast = ctx.build_pyramid(a, 15, 4)
    monkeypatch.setenv("XIVO_PYRDOWN_GENERIC", "1")
    slow = ctx.build_pyramid(a, 15, 4)
    monkeypatch.delenv("XIVO_PYRDOWN_GENERIC", raising=False)
    ref = T.pyramid(a, 15, 4)
    assert len(fast) == len(slow) == len(ref)
    for f, s_, r in zip(fast, slow, ref):
        assert np.array_equal(f, s_)
        assert np.array_equal(f, r)


@pytest.mark.parametrize("shape,thr,cn", [((480, 640), 5, 1), ((480, 640), 20, 1), ((241, 323), 10, 1), ((96, 70), 5, 3), ((480, 640), 40, 3)])
def test_fast_pair_kernel_equals_oracle(ctx, shape, thr, cn):
    """fast_pair_kernel (two pixels per thread, s16x2 min/max, decision 'cornerScore > thr') against the C oracle
    (cv2's FAST-9/16 restated), grey and BGR: identical keypoint sets and scores."""
    a, _ = synth.frame_pair(shape[0], shape[1], seed=31)
    img = a if cn == 1 else synth.to_bgr(a, True)
    xy, sc, n = ctx.fast_detect(img, thr, max_kp=1 << 17)
    rxy, rsc, rn = T.fast_detect(img, thr)
    key = lambda xy_, sc_: sorted(zip(xy_[:, 1].tolist(), xy_[:, 0].tolist(), sc_.tolist()))
    assert n == rn and n > 0
    assert key(xy, sc) == key(rxy, rsc)
    # without non-max suppression every corner is reported: checks the decision itself
    xy, sc, n = ctx.fast_detect(img, thr, nonmax=False, max_kp=1 << 18)
    rxy, rsc, rn = T.fast_detect(img, thr, nonmax=False, max_kp=1 << 18)
    assert n == rn and key(xy, sc) == key(rxy, rsc)


@pytest.mark.parametrize("shape", [(480, 640), (240, 320), (512, 512), (1024, 1280), (67, 48), (176, 208), (35, 16)])
def test_pyramid_tma_kernel_equals_thread_staged_kernel(ctx, shape, monkeypatch):
    """Levels whose rows are multiples of 16 bytes take pyrdown_tma_kernel by default (one cp.async.bulk.tensor box per CTA, zero fill
    outside the image, REFLECT_101 patched on the rim CTAs); XIVO_PYRDOWN_TMA=0 keeps pyrdown_vec_kernel.  Same integers, every level
    identical and equal to the C oracle.  Shapes: the bench frame, a quarter of it, BASELINE configs[0] / [2] (512 x 512, six levels), the
    stress frame, widths whose coarser levels stop being 16-byte multiples (TMA and thread-staged passes inside one pyramid), a frame
    narrower than one box."""
    a, _ = synth.frame_pair(shape[0], shape[1], seed=23)
    monkeypatch.delenv("XIVO_PYRDOWN_TMA", raising=False)
    tma = ctx.build_pyramid(a, 15, 5)
    monkeypatch.setenv("XIVO_PYRDOWN_TMA", "0")
    staged = ctx.build_pyramid(a, 15, 5)
    monkeypatch.delenv("XIVO_PYRDOWN_TMA", raising=False)
    ref = T.pyramid(a, 15, 5)
    assert len(tma) == len(staged) == len(ref)
    for lvl, (f, s_, r) in enumerate(zip(tma, staged, ref)):
        assert np.array_equal(f, s_), f"level {lvl}: TMA pass differs from the thread-staged pass"
        assert np.array_equal(f, r), f"level {lvl}: differs from the oracle"


@pytest.mark.parametrize("shape,thr", [((480, 640), 5), ((480, 640), 20), ((512, 512), 20), ((1024, 1280), 20), ((240, 320), 40), ((70, 96), 5), ((33, 16), 5)])
def test_fast_tma_kernel_equals_thread_staged_kernel(ctx, shape, thr, monkeypatch):
    """Single-channel images with 16-byte rows take fast_pair_tma_kernel by default (the tile arrives as one cp.async.bulk.tensor box,
    zero-filled outside the image); XIVO_FAST_TMA=0 keeps the thread-staged tile load.  Identical keypoints and scores, equal to the C oracle,
    with and without non-max suppression."""
    a, _ = synth.frame_pair(shape[0], shape[1], seed=37)
    key = lambda xy_, sc_: sorted(zip(xy_[:, 1].tolist(), xy_[:, 0].tolist(), sc_.tolist()))
    for nonmax in (True, False):
        monkeypatch.delenv("XIVO_FAST_TMA", raising=False)
        xy, sc, n = ctx.fast_detect(a, thr, nonmax=nonmax, max_kp=1 << 18)
        monkeypatch.setenv("XIVO_FAST_TMA", "0")
        xy2, sc2, n2 = ctx.fast_detect(a, thr, nonmax=nonmax, max_kp=1 << 18)
        monkeypatch.delenv("XIVO_FAST_TMA", raising=False)
        rxy, rsc, rn = T.fast_detect(a, thr, nonmax=nonmax, max_kp=1 << 18)
        assert n == n2 == rn
        assert key(xy, sc) == key(xy2, sc2) == key(rxy, rsc)


@pytest.mark.parametrize("shape,cn", [((480, 640), 1), ((240, 320), 3), ((512, 512), 1), ((120, 97), 1)])
def test_brief_descriptors_equal_the_oracle(ctx, shape, cn):
    """brief_kernel (warp per keypoint, separable 9 x 9 box sums of the 56 x 56 neighbourhood in shared memory, lane = descriptor byte) against
    oracle/tracker_oracle.c (direct 81-pixel sums): identical bytes and identical border drops, for keypoints on a grid that includes the
    28-pixel border band, sub-pixel positions on both sides of the .5 rounding, and BGR input (grey conversion fused)."""
    a, _ = synth.frame_pair(shape[0], shape[1], seed=41)
    img = a if cn == 1 else synth.to_bgr(a, True)
    rng = np.random.default_rng(5)
    kp = np.concatenate([rng.uniform(0, [shape[1], shape[0]], (400, 2)),
                         np.array([[28.0, 28.0], [27.99, 40.0], [shape[1] - 28.0, 50.0], [shape[1] - 28.01, 50.0], [60.5, 70.5], [60.49, 70.51]])]).astype(np.float32)
    d, v = ctx.brief_describe(img, kp)
    rd, rv = T.brief(img, kp)
    assert np.array_equal(v, rv) and v.sum() > 50 and (~v).sum() > 5
    assert np.array_equal(d, rd)
    assert len({bytes(x) for x in d[v]}) > 0.9 * v.sum()  # the descriptors are informative, not constant


def test_hamming_matcher_equals_the_oracle_and_cv2(ctx):
    """hamming_nearest_kernel x 2 + cross-check against the C restatement, which tests/test_oracle_tracker.py pins on cv2.BFMatcher: random
    descriptors, descriptors with few distinct values (many ties: first index wins), more queries than trains and the reverse."""
    rng = np.random.default_rng(9)
    for nq, nt, mask in [(40, 300, 0xFF), (300, 40, 0xFF), (64, 64, 0x03), (1, 500, 0xFF), (200, 1, 0x0F), (150, 2500, 0xFF)]:
        q = rng.integers(0, 256, (nq, 32), dtype=np.uint8) & mask
        t = rng.integers(0, 256, (nt, 32), dtype=np.uint8) & mask
        if mask != 0xFF:
            q[:, 2:] = 0
            t[:, 2:] = 0
        assert ctx.hamming_match(q, t) == T.bf_match_crosscheck(q, t)

"""The measurement update as Batch runs it, through xivo_filter_update_batch: several filters per launch, each with its own measurement
count, feature tables, R and pre-gate / post-gate covariance edit lists, three passes on the same device buffers (the TF32 operand buffers
of the tensor-core downdate are zeroed once, so a pass whose M shrinks runs on words an earlier, larger update left behind).

Reference: numpy fp64 per filter and pass, from the device's own prior of that pass (so errors do not accumulate over passes):
oracle/ekf_oracle.py's feature_jacobian, mh_distance, fill_jacobian_block (or the raw rows of J for the 1-point RANSAC update) and
update_joseph, plus the edit-op interpreter below.  Tolerances, with d_i = P_ii of the prior (after the post-gate edits):
  fp64       |dP_ij| <= 1e-9 sqrt(d_i d_j); rows / columns that are zero in the prior stay exactly 0; P exactly symmetric;
             |derr_i| <= 1e-9 sqrt(d_i) |inn|_S (|inn|_S^2 = inn' S^-1 inn bounds |err_i| / sqrt(d_i)); mh within 1e-8 relative;
             diag(P) after the pre-gate edits exact
  tf32x3     |dP_ij| <= 1e-5 sqrt(d_i d_j) against the fp64 reference (both tensor-core kernels); err, mh, diag identical to the fp64
             run on the first pass (same prior), within the fp64 bounds of their own reference afterwards
A filter whose S is not positive definite gets an all-NaN err and keeps its post-gate covariance bit for bit.

Also here: the IMU covariance kernel at the edges of its loops (no strips, strips that wrap the thread count, a full staging queue,
a single sub-step), both formulations."""
import numpy as np
import pytest

from oracle import ekf_oracle as E
from xivo_b200 import synth

SHAPES = [(1, 1), (2, 3), (4, 14), (15, 30), (15, 62)]  # N = 32 (one-warp gate CTA), 44, 89, 203, 299
M_VALUES = (0, 2, 8, 30, 32, 34, 64)  # plus 2F; those a layout can hold


# ---------------------------------------------------------------------------------------------------------------------------------
# covariance slot surgery as edit ops (include/xivo_b200.h, xivo_cov_edit) and an interpreter of them
# ---------------------------------------------------------------------------------------------------------------------------------
def surgery_ops(lay, act):
    """The edit ops Estimator queues for one slot-surgery action."""
    kind, s = act[0], act[1]
    if kind == "add_group":  # AddGroupToState: rows then columns of Wsb / Tsb into the group slot
        return [(1, lay.goff(s), E.WSB, 3), (1, lay.goff(s) + 3, E.TSB, 3)]
    if kind == "remove_group":
        return [(0, lay.goff(s), 0, 6)]
    if kind == "add_feature":  # AddFeatureToState + FillCovarianceBlock
        return [(0, lay.foff(s), 0, 3), (2, lay.foff(s), 0, 3, act[2])]
    if kind == "remove_feature":
        return [(0, lay.foff(s), 0, 3)]
    if kind == "fix_xy":
        return [(0, lay.foff(s), 0, 2)]
    if kind == "switch_ref":
        return [(0, lay.goff(s) + 2, 0, 4)] if act[2] == 4 else [(0, lay.goff(s), 0, 6)]
    raise ValueError(kind)


def surgery_oracle(lay, P, act):
    """The same action through oracle/ekf_oracle.py's restatement of the reference."""
    err = np.zeros(lay.N)
    kind, s = act[0], act[1]
    if kind == "add_group":
        E.add_group_to_state(lay, P, err, s)
    elif kind == "remove_group":
        E.remove_group_from_state(lay, P, err, s)
    elif kind == "add_feature":
        E.add_feature_to_state(lay, P, s, np.reshape(act[2], (3, 3)))
    elif kind == "remove_feature":
        E.remove_feature_from_state(lay, P, err, s)
    elif kind == "fix_xy":
        E.fix_feature_xy(lay, P, s)
    elif kind == "switch_ref":
        E.switch_ref_group_cov(lay, P, s, act[2])


def apply_ops(P, ops):
    """Edit-op interpreter (apply_edits of ekf_kernels.cu): 0 = zero rows + columns [a, a+n), 1 = copy rows then columns b -> a (n wide),
    2 = set the 3 x 3 block at (a, a)."""
    for op in ops:
        t, a, b, n = op[:4]
        if t == 0:
            P[a : a + n, :] = 0.0
            P[:, a : a + n] = 0.0
        elif t == 1:
            P[a : a + n, :] = P[b : b + n, :]
            P[:, a : a + n] = P[:, b : b + n]
        else:
            P[a : a + 3, a : a + 3] = np.reshape(op[4], (3, 3))
    return P


def to_ops(lay, acts):
    return [op for act in acts for op in surgery_ops(lay, act)]


# ---------------------------------------------------------------------------------------------------------------------------------
# problems
# ---------------------------------------------------------------------------------------------------------------------------------
# standard deviations of the motion state (Wsb Tsb Vsb bg ba Wbc Tbc Wsg): the bias and extrinsics blocks are where a tensor-core
# downdate that is accurate only relative to max|P| would go wrong
_MOTION_STD = np.array([1e-2] * 3 + [3e-2] * 3 + [5e-2] * 3 + [1e-4] * 3 + [1e-3] * 3 + [1e-4] * 6 + [1e-3] * 2)


def realistic_cov(lay, live, rng):
    """SPD on the live slots with a running filter's spread of variances (1e-8 ... 1), zero elsewhere."""
    std = np.zeros(lay.N)
    std[:23] = _MOTION_STD * rng.uniform(0.5, 2.0, 23)
    for i in live[live >= 23]:
        if i < lay.feature_begin:
            std[i] = rng.uniform(1e-3, 3e-2)
        else:
            std[i] = rng.uniform(1e-1, 1.0) if (i - lay.feature_begin) % 3 == 2 else rng.uniform(1e-2, 5e-2)
    A = rng.normal(size=(len(live), len(live)))
    C = A @ A.T / len(live) + 0.3 * np.eye(len(live))
    c = np.sqrt(np.diag(C))
    C = C / np.outer(c, c)
    P = np.zeros((lay.N, lay.N))
    P[np.ix_(live, live)] = C * np.outer(std[live], std[live])
    return 0.5 * (P + P.T)


def make_filter(G, F, n, seed, model):
    prob = synth.random_filter_problem(G, F, n, seed=seed, model=model)
    synth.set_measurements_near_prediction(prob, E, 1.0, seed=seed)
    lay = E.Layout(G, F)
    ng = min(G, max(2, n // 3))
    live = list(range(23)) + [lay.goff(g) + k for g in range(ng) for k in range(6)] + [lay.foff(s) + k for s in prob["feat_sind"] for k in range(3)]
    rng = np.random.default_rng(seed + 1000)
    prob["P"] = realistic_cov(lay, np.array(sorted(live)), rng)
    prob["R"] = float(rng.uniform(0.5, 3.0))
    cam = synth.camera_from_array(E, prob["camera"])
    X = prob["X24"]
    Js, inns = [], []
    for i in range(n):
        g = prob["groups"][prob["feat_ref"][i]]
        J, r, _ = E.feature_jacobian(lay, cam, X[:9].reshape(3, 3), X[9:12], X[12:21].reshape(3, 3), X[21:24], g[:9].reshape(3, 3), g[9:12],
                                     prob["feat_x"][i], prob["feat_xp"][i], int(prob["feat_ref"][i]), int(prob["feat_sind"][i]))
        Js.append(J)
        inns.append(r)
    prob["J"], prob["inn"] = Js, inns
    return prob


def spd_block(rng):
    A = rng.normal(size=(3, 3)) * 0.02
    B = A @ A.T + np.diag(rng.uniform(1e-4, 1e-2, 3))
    return 0.5 * (B + B.T)


def schedule(G, F, B, seed):
    """Per filter: measurement counts of three passes (grows, then shrinks to a count that is not a multiple of 8, so the downdate's
    last K step reads operand rows an earlier pass wrote), selections and edit lists of every kind, some touching the slots of
    selected features, some ending at N, some empty."""
    rng = np.random.default_rng(seed)
    cand = sorted({m for m in M_VALUES + (2 * F,) if m <= 2 * F})
    L = len(cand)
    Ms = []
    for b in range(B):
        i = b % L
        m0 = cand[i]
        m1 = cand[min(i + 2, L - 1)]
        small = [m for m in cand if m < m1 and m % 8]
        m2 = small[-1 - (b % len(small))] if small else 0
        Ms.append((m0, m1, m2))
    lay = E.Layout(G, F)
    filters = []
    for b in range(B):
        n = max(1, max(Ms[b]) // 2)
        n = int(min(F, n + rng.integers(0, F - n + 1)))
        filters.append(make_filter(G, F, n, seed * 100 + b, model=b % 2 * 3))
    passes, acts = [], []  # acts: the surgery actions behind every list (for the interpreter's CPU check)
    for p in range(3):
        row = []
        for b in range(B):
            f = filters[b]
            n = len(f["feat_x"])
            sel = rng.permutation(n)[: Ms[b][p] // 2]
            s_sel = int(f["feat_sind"][sel[0]]) if len(sel) else int(f["feat_sind"][0])
            s_sel2 = int(f["feat_sind"][sel[-1]]) if len(sel) else s_sel
            ref = int(f["feat_ref"][sel[0]]) if len(sel) else 0
            g_other = (ref + 1) % G
            pre = [[],
                   [("remove_feature", s_sel), ("add_feature", s_sel, spd_block(rng))],
                   [("add_group", g_other), ("fix_xy", s_sel2), ("switch_ref", ref, 4)],
                   [("remove_feature", F - 1), ("add_feature", F - 1, spd_block(rng))]][(b + p) % 4]
            post = [[],
                    [("remove_feature", s_sel2), ("add_feature", s_sel2, spd_block(rng))],
                    [("remove_group", g_other), ("add_group", g_other), ("switch_ref", g_other, 6)],
                    [("add_group", ref), ("add_feature", F - 1, spd_block(rng))]][(b + 2 * p + 1) % 4]
            row.append(dict(pre=to_ops(lay, pre), sel=sel, post=to_ops(lay, post)))
            acts += [pre, post]
        passes.append(row)
    return filters, passes, acts


# ---------------------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------------------
def reference_pass(lay, f, Pin, ps, full_j, R=None):
    """One gate + update phase of one filter from the prior Pin: (diag after the pre-gate edits, mh, prior after the post-gate
    edits, P after the update, err, |inn|_S)."""
    R = f["R"] if R is None else R
    P1 = apply_ops(Pin.copy(), ps["pre"])
    diag = np.diag(P1).copy()
    mh = np.array([E.mh_distance(f["J"][i], P1, f["inn"][i], R) for i in range(len(f["J"]))])
    P2 = apply_ops(P1, ps["post"])
    sel = ps["sel"]
    M = 2 * len(sel)
    if M == 0:
        return diag, mh, P2, P2.copy(), np.zeros(lay.N), 0.0
    H = np.zeros((M, lay.N))
    inn = np.zeros(M)
    for r, i in enumerate(sel):
        if full_j:
            H[2 * r : 2 * r + 2] = f["J"][i]
        else:
            E.fill_jacobian_block(lay, H, 2 * r, f["J"][i], int(f["feat_ref"][i]), int(f["feat_sind"][i]))
        inn[2 * r : 2 * r + 2] = f["inn"][i]
    Pn, er, _, S = E.update_joseph(H, P2, inn, np.full(M, R))
    return diag, mh, P2, Pn, er, float(np.sqrt(inn @ np.linalg.solve(S, inn)))


def check_against_reference(lay, filters, passes, P0, out, full_j, ptol, what):
    """Every filter and pass of one device run against the reference from the device's own prior; returns the worst
    |dP_ij| / sqrt(d_i d_j) seen."""
    Po, err, mh, diag = out
    worst = 0.0
    for p in range(len(passes)):
        for b, f in enumerate(filters):
            Pin = P0[b] if p == 0 else Po[p - 1, b]
            rd, rmh, P2, Pn, er, inn_s = reference_pass(lay, f, Pin, passes[p][b], full_j)
            tag = f"{what}: pass {p} filter {b} (M = {2 * len(passes[p][b]['sel'])})"
            n = len(f["J"])
            assert np.array_equal(diag[p, b], rd), tag
            assert np.all(np.abs(mh[p, b, :n] - rmh) <= 1e-8 * np.maximum(1.0, rmh)), tag
            assert np.all(mh[p, b, n:] == 0), tag
            P = Po[p, b]
            assert np.array_equal(P, P.T), tag
            dead = ~np.any(P2 != 0, axis=0)
            assert np.all(P[dead] == 0) and np.all(P[:, dead] == 0), tag
            d = np.sqrt(np.diag(P2))
            scale = np.outer(d, d)
            live = scale > 0
            rel = np.abs(P - Pn)[live] / scale[live]
            worst = max(worst, float(rel.max()))
            assert rel.max() <= ptol, f"{tag}: max |dP_ij| / sqrt(P_ii P_jj) = {rel.max():.3e}"
            assert np.all(np.abs(err[p, b] - er) <= 1e-9 * d * inn_s), tag
            if not passes[p][b]["sel"].size:
                assert np.array_equal(P, P2) and np.all(err[p, b] == 0), tag
    return worst


def run_modes(ctx, G, F, filters, passes, full_j, monkeypatch):
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    r64 = ctx.filter_update_batch(G, F, filters, passes, full_j=full_j)
    r2 = ctx.filter_update_batch(G, F, filters, passes, tf32x3=True, full_j=full_j)
    monkeypatch.setenv("XIVO_TC_V1", "1")
    r1 = ctx.filter_update_batch(G, F, filters, passes, tf32x3=True, full_j=full_j)
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    return r64, r2, r1


# ---------------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------------
def test_edit_interpreter_matches_slot_surgery():
    """CPU only: the interpreter the GPU references use reproduces oracle/ekf_oracle.py's slot-surgery functions exactly, on every
    edit list of the GPU cases."""
    for (G, F) in SHAPES:
        lay = E.Layout(G, F)
        _, _, acts = schedule(G, F, 7, seed=G * 100 + F)
        rng = np.random.default_rng(F)
        kinds = set()
        for lst in acts:
            A = rng.normal(size=(lay.N, lay.N))
            P = A @ A.T
            got, want = apply_ops(P.copy(), to_ops(lay, lst)), P.copy()
            for act in lst:
                surgery_oracle(lay, want, act)
                kinds.add(act[0])
            assert np.array_equal(got, want), (G, F, lst)
        assert kinds >= {"add_group", "remove_group", "add_feature", "remove_feature", "fix_xy", "switch_ref"}


@pytest.mark.gpu
@pytest.mark.parametrize("G,F,full_j", [(G, F, False) for G, F in SHAPES] + [(4, 14, True), (15, 62, True)])
def test_batched_update_phases_match_reference(ctx, G, F, full_j, monkeypatch):
    """fp64 and both tensor-core downdates on 6-7 heterogeneous filters per launch, three passes with M growing then shrinking."""
    B = 7 if F >= 14 else 6
    filters, passes, _ = schedule(G, F, B, seed=G * 100 + F + (7 if full_j else 0))
    lay = E.Layout(G, F)
    Ms = {2 * len(ps["sel"]) for row in passes for ps in row}
    assert Ms >= {m for m in M_VALUES + (2 * F,) if m <= 2 * F}
    P0 = np.stack([f["P"] for f in filters])
    r64, r2, r1 = run_modes(ctx, G, F, filters, passes, full_j, monkeypatch)
    check_against_reference(lay, filters, passes, P0, r64, full_j, 1e-9, "fp64")
    for name, r in (("tc2", r2), ("tc1", r1)):
        worst = check_against_reference(lay, filters, passes, P0, r, full_j, 1e-5, name)
        assert worst > 0  # the tensor cores did the downdate
        # first pass: the same prior as the fp64 run
        assert np.array_equal(r[1][0], r64[1][0]) and np.array_equal(r[2][0], r64[2][0]) and np.array_equal(r[3][0], r64[3][0]), name


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp64", "tc2", "tc1"])
def test_non_positive_definite_innovation_covariance(ctx, mode, monkeypatch):
    """A filter whose R makes S indefinite publishes NaN err and a zero gain: its covariance stays what the post-gate edits left, bit
    for bit, on every pass; the other filters of the launch are updated as usual."""
    G, F, B, bad = 4, 14, 5, 2
    filters, passes, _ = schedule(G, F, B, seed=77)
    filters[bad]["R"] = -1e6
    for row in passes:
        if not row[bad]["sel"].size:
            row[bad]["sel"] = np.array([0, 1][: len(filters[bad]["feat_x"])])
    monkeypatch.setenv("XIVO_TC_V1", "1" if mode == "tc1" else "0")
    out = ctx.filter_update_batch(G, F, filters, passes, tf32x3=mode != "fp64")
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    Po, err, mh, diag = out
    lay = E.Layout(G, F)
    P0 = np.stack([f["P"] for f in filters])
    for p in range(3):
        Pin = P0[bad] if p == 0 else Po[p - 1, bad]
        rd, rmh, P2, _, _, _ = reference_pass(lay, filters[bad], Pin, passes[p][bad], False)
        assert np.all(np.isnan(err[p, bad])), p
        assert np.array_equal(Po[p, bad], P2), p
        assert np.array_equal(diag[p, bad], rd)
    good = [b for b in range(B) if b != bad]
    sub = ([filters[b] for b in good], [[row[b] for b in good] for row in passes])
    Pg = np.stack([P0[b] for b in good])
    check_against_reference(lay, sub[0], sub[1], Pg, tuple(a[:, good] for a in out), False, 1e-9 if mode == "fp64" else 1e-5, mode)


def _imu_problem(N, method, nsub, seed):
    """P (N x N), per-stage records of exactly nsub Runge-Kutta sub-steps from a mix of Propagate calls, and the oracle's result."""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(N, N))
    scale = np.exp(rng.uniform(-4, 0, N))
    P = (A @ A.T / N + np.eye(N)) * np.outer(scale, scale)
    P = 0.5 * (P + P.T)
    X = E.MotionState(synth.random_rotation(rng, 0.3), rng.normal(0, 1, 3), rng.normal(0, 0.5, 3), rng.normal(0, 0.01, 3), rng.normal(0, 0.05, 3),
                      np.eye(3), np.zeros(3), synth.random_rotation(rng, 0.02))
    Cg = np.eye(3) + 0.01 * rng.normal(size=(3, 3))
    Ca = np.eye(3) + 0.01 * rng.normal(size=(3, 3))
    g = np.array([0.0, 0.0, -9.8])
    qimu = np.array([2.5e-5] * 3 + [2.5e-3] * 3 + [1e-8] * 3 + [1e-7] * 3)
    qmodel = np.zeros(23)
    qmodel[0:3], qmodel[15:18], qmodel[21:23] = 1e-4, 1e-6, 1e-7
    nst = 7 if method == "PrinceDormand" else 4
    rec = []
    Pr = P.copy()
    while len(rec) < nsub * nst:
        gyro0, accel0 = rng.normal(0, 0.2, 3), np.array([0.0, 0.0, 9.8]) + rng.normal(0, 0.5, 3)
        sg, sa = rng.normal(0, 2.0, 3), rng.normal(0, 5.0, 3)
        # whole Propagate calls of several sub-steps (at most 4 for 5 ms at h = 2 ms) while they fit, single sub-steps to fill
        h0 = 0.002 if len(rec) + 4 * nst <= nsub * nst else -1.0
        Phi, Pmm = E.integrate(method, X, Pr[:23, :23].copy(), gyro0, accel0, sg, sa, [0.005, 0.0043, 0.0031][len(rec) % 3], Cg, Ca, g,
                               np.diag(qimu), h0, rec)
        E.apply_propagation(Pr, Phi, Pmm, np.diag(qmodel))
    assert len(rec) == nsub * nst
    return P, np.array(rec), g, qimu, qmodel, nst, Pr


@pytest.mark.gpu
@pytest.mark.parametrize("N", [23, 299])
@pytest.mark.parametrize("method,nsub", [("PrinceDormand", 1), ("RK4", 1), ("PrinceDormand", 146), ("RK4", 256)])
def test_imu_cov_propagate_edges(ctx, N, method, nsub):
    """N = 23 (no strips) and N = 299 (the strip loop over 276 columns wraps past 256 threads); one sub-step, and a queue at capacity
    (1022 Prince-Dormand / 1024 RK4 stages, several chunks of the kernel's stage loader)."""
    P, rec, g, qimu, qmodel, nst, Pr = _imu_problem(N, method, nsub, seed=N + nsub)
    d = np.sqrt(np.outer(np.diag(Pr), np.diag(Pr)))
    Pg = ctx.imu_cov_propagate(P, rec, g, qimu, qmodel, nst)
    assert np.abs(Pg - Pr).max() <= 1e-10 * np.abs(Pr).max()
    assert (np.abs(Pg - Pr) / d).max() <= 1e-10
    assert np.abs(Pg - Pg.T).max() <= 1e-13 * np.abs(Pg).max()

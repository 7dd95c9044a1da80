"""GPU parity: EKF kernels through the C ABI vs the numpy fp64 oracle.
Tolerances: fp64 kernels vs fp64 oracle -> relative 1e-9 on Jacobians/distances, 1e-9 * max|P|
absolute on covariances (different but algebraically identical update form, see DESIGN.md)."""
import numpy as np
import pytest

from oracle import ekf_oracle as E
from xivo_b200 import synth

pytestmark = pytest.mark.gpu

CONFIGS = [(4, 14, 12, 0), (15, 30, 30, 0), (15, 30, 17, 3), (15, 62, 62, 0), (2, 3, 1, 0)]


def oracle_all(prob):
    lay = E.Layout(prob["G"], prob["F"])
    cam = synth.camera_from_array(E, prob["camera"])
    X = prob["X24"]
    Js, inns = [], []
    for i in range(prob["n"]):
        g = prob["groups"][prob["feat_ref"][i]]
        J, r, _ = E.feature_jacobian(lay, cam, X[:9].reshape(3, 3), X[9:12], X[12:21].reshape(3, 3), X[21:24], g[:9].reshape(3, 3),
                                     g[9:12], prob["feat_x"][i], prob["feat_xp"][i], int(prob["feat_ref"][i]), int(prob["feat_sind"][i]))
        Js.append(J)
        inns.append(r)
    return lay, cam, np.array(Js), np.array(inns)


@pytest.mark.parametrize("G_,F_,n,model", CONFIGS)
def test_jacobian_and_gate(ctx, G_, F_, n, model):
    prob = synth.random_filter_problem(G_, F_, n, seed=G_ + F_, model=model)
    synth.set_measurements_near_prediction(prob, E, 2.0)
    lay, cam, Js, inns = oracle_all(prob)
    R = 1.5
    J, inn, mh = ctx.jacobian_batch(G_, F_, prob["camera"], prob["X24"], prob["groups"], prob["feat_x"], prob["feat_xp"],
                                    prob["feat_ref"], prob["feat_sind"], prob["P"], R)
    assert np.abs(J - Js).max() <= 1e-9 * np.abs(Js).max()
    assert np.abs(inn - inns).max() <= 1e-9 * max(1.0, np.abs(inns).max())
    ref_mh = np.array([E.mh_distance(Js[i], prob["P"], inns[i], R) for i in range(n)])
    assert np.abs(mh - ref_mh).max() <= 1e-8 * max(1.0, ref_mh.max())
    mh2 = ctx.mh_gate(G_, F_, prob["camera"], prob["X24"], prob["groups"], prob["feat_x"], prob["feat_xp"], prob["feat_ref"],
                      prob["feat_sind"], prob["P"], R)
    assert np.array_equal(mh, mh2)


def test_jacobian_empty(ctx):
    prob = synth.random_filter_problem(4, 14, 0, seed=0)
    J, inn, mh = ctx.jacobian_batch(4, 14, prob["camera"], prob["X24"], prob["groups"], prob["feat_x"], prob["feat_xp"],
                                    prob["feat_ref"], prob["feat_sind"], prob["P"], 1.0)
    assert J.shape[0] == 0


@pytest.mark.parametrize("N,M", [(89, 24), (203, 60), (299, 124), (23, 2), (50, 1)])
def test_dense_update_matches_joseph(ctx, N, M):
    rng = np.random.default_rng(N + M)
    A = rng.normal(size=(N, N))
    scale = np.exp(rng.uniform(-5, 1, N))
    P = (A @ A.T / N + np.eye(N)) * np.outer(scale, scale)
    P = 0.5 * (P + P.T)
    H = rng.normal(size=(M, N)) * (rng.uniform(size=(M, N)) < 0.15)
    inn = rng.normal(size=M)
    diagR = rng.uniform(0.5, 2.0, M)
    Pg, err = ctx.ekf_update(H, P, inn, diagR)
    Pr, er, K, S = E.update_joseph(H, P, inn, diagR)
    assert np.abs(Pg - Pr).max() <= 1e-9 * np.abs(P).max()
    assert np.abs(err - er).max() <= 1e-9 * max(1.0, np.abs(er).max())
    assert np.array_equal(Pg, Pg.T)  # mirrored write -> exactly symmetric
    assert np.linalg.eigvalsh(Pg).min() > -1e-12 * np.abs(P).max()


@pytest.mark.parametrize("N,M", [(89, 24), (203, 60), (299, 124), (23, 2), (130, 33)])
def test_dense_update_tensor_core_tf32x3(ctx, N, M):
    """XIVO_UPDATE_TF32X3: the downdate P -= K (HP) on wgmma tensor cores (3xTF32, fp32 accumulate in registers).
    Tolerance (stated in include/xivo_b200.h): fp32-level, |dP_ij| <= 1e-5 sqrt(P_ii P_jj) elementwise and
    1e-5 max|P|; gain / err are the fp64 kernels, hence identical."""
    rng = np.random.default_rng(N + M)
    A = rng.normal(size=(N, N))
    scale = np.exp(rng.uniform(-5, 1, N))
    P = (A @ A.T / N + np.eye(N)) * np.outer(scale, scale)
    P = 0.5 * (P + P.T)
    H = rng.normal(size=(M, N)) * (rng.uniform(size=(M, N)) < 0.15)
    inn = rng.normal(size=M)
    diagR = rng.uniform(0.5, 2.0, M)
    P64, e64 = ctx.ekf_update(H, P, inn, diagR)
    P32, e32 = ctx.ekf_update(H, P, inn, diagR, tf32x3=True)
    d = np.sqrt(np.outer(np.diag(P), np.diag(P)))
    assert np.abs(P64 - P).max() > 1e-3 * np.abs(P).max()  # the update is not a no-op
    assert (np.abs(P32 - P64) / d).max() <= 1e-5
    assert np.abs(P32 - P64).max() <= 1e-5 * np.abs(P).max()
    assert np.array_equal(e32, e64)
    assert np.array_equal(P32, P32.T)
    Pr, _, _, _ = E.update_joseph(H, P, inn, diagR)
    assert np.abs(P32 - Pr).max() <= 1e-5 * np.abs(P).max()


@pytest.mark.parametrize("N,M,B", [(89, 28, 7), (203, 60, 5), (299, 124, 3), (299, 40, 3), (130, 33, 4)])
def test_batched_update_both_tensor_core_kernels_and_fp64(ctx, N, M, B, monkeypatch):
    """xivo_ekf_update_batch: B filters in one launch pair.  fp64 path against the Joseph oracle per filter; the tensor-core downdate in
    both formulations -- ekf_cov_tc2_kernel (default: TF32 hi / lo operands written by the gain kernel, TMA-staged, several column chunks
    per CTA, MMAs of the next chunk overlapping the epilogue) and the first kernel (XIVO_TC_V1=1) -- at the stated fp32 tolerance, exactly symmetric,
    and equal to each other to fp32 rounding.  Sizes: the three BASELINE state dimensions with their maximal measurement counts, a
    measurement count that is not a multiple of the 32-row K block, and a state dimension that crosses one 128-row tile by 2 rows."""
    rng = np.random.default_rng(N * 7 + M + B)
    Ps, Hs, inns, Rs = [], [], [], []
    for _ in range(B):
        A = rng.normal(size=(N, N))
        scale = np.exp(rng.uniform(-5, 1, N))
        P = (A @ A.T / N + np.eye(N)) * np.outer(scale, scale)
        Ps.append(0.5 * (P + P.T))
        Hs.append(rng.normal(size=(M, N)) * (rng.uniform(size=(M, N)) < 0.15))
        inns.append(rng.normal(size=M))
        Rs.append(rng.uniform(0.5, 2.0, M))
    Ps, Hs, inns, Rs = np.stack(Ps), np.stack(Hs), np.stack(inns), np.stack(Rs)
    P64, e64 = ctx.ekf_update_batch(Hs, Ps, inns, Rs)
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    P2, e2 = ctx.ekf_update_batch(Hs, Ps, inns, Rs, tf32x3=True)
    P2r, _ = ctx.ekf_update_batch(Hs, Ps, inns, Rs, tf32x3=True, repeat=3)  # re-applied to the original P: same result
    monkeypatch.setenv("XIVO_TC_V1", "1")
    P1, e1 = ctx.ekf_update_batch(Hs, Ps, inns, Rs, tf32x3=True)
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    for b in range(B):
        Pr, er, _, _ = E.update_joseph(Hs[b], Ps[b], inns[b], Rs[b])
        pmax = np.abs(Ps[b]).max()
        d = np.sqrt(np.outer(np.diag(Ps[b]), np.diag(Ps[b])))
        assert np.abs(P64[b] - Pr).max() <= 1e-9 * pmax and np.abs(e64[b] - er).max() <= 1e-9 * max(1.0, np.abs(er).max())
        assert np.abs(P64[b] - Ps[b]).max() > 1e-3 * pmax
        for Pt, et in ((P2[b], e2[b]), (P1[b], e1[b])):
            assert (np.abs(Pt - P64[b]) / d).max() <= 1e-5 and np.abs(Pt - P64[b]).max() <= 1e-5 * pmax
            assert np.array_equal(Pt, Pt.T) and np.array_equal(et, e64[b])
        assert np.array_equal(P2[b], P2r[b])
        assert (np.abs(P2[b] - P1[b]) / d).max() <= 2e-6


def test_dense_update_zero_measurements(ctx):
    P = np.eye(23)
    Pg, err = ctx.ekf_update(np.zeros((0, 23)), P, np.zeros(0), np.zeros(0))
    assert np.array_equal(Pg, P) and np.all(err == 0)


@pytest.mark.parametrize("G_,F_,n,model", CONFIGS)
def test_filter_update_production_path(ctx, G_, F_, n, model):
    """Jacobian -> FillJacobianBlock stacking (incl. the reference's quirk) -> update, on device."""
    prob = synth.random_filter_problem(G_, F_, n, seed=7 + n, model=model)
    synth.set_measurements_near_prediction(prob, E, 1.0)
    lay, cam, Js, inns = oracle_all(prob)
    rng = np.random.default_rng(n)
    sel = rng.permutation(n)[: max(1, (3 * n) // 4)].astype(np.int32)
    R = 1.0
    H = np.zeros((2 * len(sel), lay.N))
    inn = np.zeros(2 * len(sel))
    for r, i in enumerate(sel):
        E.fill_jacobian_block(lay, H, 2 * r, Js[i], int(prob["feat_ref"][i]), int(prob["feat_sind"][i]))
        inn[2 * r : 2 * r + 2] = inns[i]
    Pr, er, _, _ = E.update_joseph(H, prob["P"], inn, np.full(2 * len(sel), R))
    Pg, err, Hg = ctx.filter_update(G_, F_, prob["camera"], prob["X24"], prob["groups"], prob["feat_x"], prob["feat_xp"],
                                    prob["feat_ref"], prob["feat_sind"], sel, R, prob["P"])
    assert np.abs(Hg - H).max() <= 1e-9 * np.abs(H).max()
    assert np.abs(Pg - Pr).max() <= 1e-9 * np.abs(prob["P"]).max()
    assert np.abs(err - er).max() <= 1e-9 * max(1.0, np.abs(er).max())
    # empty slots keep exactly zero rows/cols (SURVEY Appendix B)
    dead = np.abs(prob["P"]).sum(0) == 0
    assert np.all(Pg[dead] == 0) and np.all(Pg[:, dead] == 0)


@pytest.mark.parametrize("model", [0, 3])
def test_subfilter(ctx, model):
    prob = synth.random_filter_problem(15, 30, 30, seed=11, model=model)
    cam = synth.camera_from_array(E, prob["camera"])
    rng = np.random.default_rng(3)
    n = 200
    X = prob["X24"]
    gsb, gbc = (X[:9].reshape(3, 3), X[9:12]), (X[12:21].reshape(3, 3), X[21:24])
    x = np.column_stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.4, 0.4, n), np.log(rng.uniform(0.5, 4, n))])
    Ps = np.array([np.diag(rng.uniform(1e-4, 1e-1, 3)) + 1e-5 for _ in range(n)])
    ref = prob["groups"][rng.integers(0, 15, n)]
    oc = rng.uniform(0, 2, n)
    xp = np.zeros((n, 2))
    for i in range(n):
        xp[i] = E.predict_pixel(cam, x[i], (ref[i][:9].reshape(3, 3), ref[i][9:]), gsb, gbc) + rng.normal(0, 6 if i % 3 == 0 else 1, 2)
    xo, Po, oo = ctx.subfilter_batch(prob["camera"], X, x, Ps, xp, ref, oc, 3.5**2, 8.991)
    for i in range(n):
        xr, Pr, orr = E.subfilter_update(cam, x[i], Ps[i], xp[i], gsb, gbc, (ref[i][:9].reshape(3, 3), ref[i][9:]), 3.5**2, 8.991, oc[i])
        assert np.abs(xo[i] - xr).max() <= 1e-9 * max(1.0, np.abs(xr).max())
        assert np.abs(Po[i] - Pr).max() <= 1e-9 * np.abs(Ps[i]).max()
        assert abs(oo[i] - orr) <= 1e-9 * max(1.0, orr)


def test_cov_edit_and_propagate(ctx):
    lay = E.Layout(4, 14)
    rng = np.random.default_rng(5)
    A = rng.normal(size=(lay.N, lay.N))
    P = A @ A.T
    ref = P.copy()
    err = np.zeros(lay.N)
    blk = np.diag([1.0, 2.0, 3.0]) + 0.1
    E.add_group_to_state(lay, ref, err, 1)
    E.add_feature_to_state(lay, ref, 4, blk)
    E.fix_feature_xy(lay, ref, 4)
    E.remove_feature_from_state(lay, ref, err, 2)
    E.remove_group_from_state(lay, ref, err, 3)
    E.switch_ref_group_cov(lay, ref, 0, 4)
    ops = [[1, lay.goff(1), 0, 3], [1, lay.goff(1) + 3, 3, 3], [0, lay.foff(4), 0, 3], [2, lay.foff(4), 0, 3], [0, lay.foff(4), 0, 2],
           [0, lay.foff(2), 0, 3], [0, lay.goff(3), 0, 6], [0, lay.goff(0) + 2, 0, 4]]
    blks = np.zeros((len(ops), 9))
    blks[3] = blk.ravel()
    got = ctx.cov_edit(P, ops, blks)
    assert np.array_equal(got, ref)
    Phi = np.eye(23) + 0.01 * rng.normal(size=(23, 23))
    Pmm = ref[:23, :23] * 1.1
    ref2 = ref.copy()
    E.apply_propagation(ref2, Phi, Pmm, np.zeros((23, 23)))
    got2 = ctx.cov_propagate(ref, Phi, Pmm)
    assert np.abs(got2 - ref2).max() <= 1e-12 * np.abs(ref2).max()


@pytest.mark.parametrize("k", [5, 15])
def test_oos_projection_invariants(ctx, k):
    """The reference's nullspace basis is arbitrary (FullPivLU::kernel), so parity is on the
    blocks (exact) and on the invariants of the projection."""
    G_, F_ = 15, 30
    prob = synth.random_filter_problem(G_, F_, 10, seed=21)
    lay = E.Layout(G_, F_)
    cam = synth.camera_from_array(E, prob["camera"])
    rng = np.random.default_rng(k)
    X = prob["X24"]
    Rbc, Tbc = X[12:21].reshape(3, 3), X[21:24]
    nf = 6
    Xs = np.zeros((nf, 3))
    poses = np.zeros((nf, k, 12))
    sinds = np.zeros((nf, k), np.int32)
    xps = np.zeros((nf, k, 2))
    for f in range(nf):
        sinds[f] = rng.permutation(G_)[:k]
        for j in range(k):
            poses[f, j] = prob["groups"][sinds[f, j]]
        g0 = poses[f, 0]
        Xc = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0]) * rng.uniform(1.5, 4)
        Xs[f] = g0[:9].reshape(3, 3) @ (Rbc @ Xc + Tbc) + g0[9:]
        xps[f] = rng.uniform(100, 400, (k, 2))
    Hf, Hx, inn, Hp, ip = ctx.oos_project(G_, F_, prob["camera"], np.concatenate([Rbc.ravel(), Tbc]), Xs, poses, sinds, xps)
    for f in range(nf):
        obs = [(poses[f, j][:9].reshape(3, 3), poses[f, j][9:], int(sinds[f, j]), xps[f, j]) for j in range(k)]
        rHf, rHx, rinn = E.oos_jacobian(lay, cam, Xs[f], obs, Rbc, Tbc)
        assert np.abs(Hf[f] - rHf).max() <= 1e-9 * np.abs(rHf).max()
        assert np.abs(Hx[f] - rHx).max() <= 1e-9 * np.abs(rHx).max()
        assert np.abs(inn[f] - rinn).max() <= 1e-9 * np.abs(rinn).max()
        A, rHp, rip = E.left_nullspace_project(rHf, rHx, rinn)
        # same row space and same Gram matrices (orthonormal bases differ by a rotation Q)
        assert np.abs(Hp[f].T @ Hp[f] - rHp.T @ rHp).max() <= 1e-8 * np.abs(rHp.T @ rHp).max()
        assert np.abs(Hp[f].T @ ip[f] - rHp.T @ rip).max() <= 1e-8 * max(1.0, np.abs(rHp.T @ rip).max())
        assert abs(ip[f] @ ip[f] - rip @ rip) <= 1e-8 * (rip @ rip)


@pytest.mark.parametrize("method", ["PrinceDormand", "RK4"])
def test_imu_cov_propagate_matches_oracle(ctx, method):
    """Device covariance propagation (from per-stage records) vs the numpy restatement of
    Propagate + PrinceDormand/RK4 (fp64, 1e-10)."""
    rng = np.random.default_rng(7)
    lay = E.Layout(4, 14)
    N = lay.N
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
    rec = []
    Pr, Xr = P.copy(), X.copy()
    for k in range(9):
        gyro0, accel0 = rng.normal(0, 0.2, 3), np.array([0.0, 0.0, 9.8]) + rng.normal(0, 0.5, 3)
        sg, sa = rng.normal(0, 2.0, 3), rng.normal(0, 5.0, 3)
        dt = [0.005, 0.0025, 0.0071, 0.04][k % 4]
        Phi, Pmm = E.integrate(method, Xr, Pr[:23, :23].copy(), gyro0, accel0, sg, sa, dt, Cg, Ca, g, np.diag(qimu), 0.002, rec)
        E.apply_propagation(Pr, Phi, Pmm, np.diag(qmodel))
    nst = 7 if method == "PrinceDormand" else 4
    assert len(rec) % nst == 0 and len(rec) > 9 * nst
    Pg = ctx.imu_cov_propagate(P, np.array(rec), g, qimu, qmodel, nst)
    assert np.abs(Pg - Pr).max() <= 1e-10 * np.abs(Pr).max()
    assert np.abs(Pg - Pg.T).max() <= 1e-13 * np.abs(Pg).max()

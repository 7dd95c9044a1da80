"""The measurement update at the edges of its layout: state dimensions on the tile boundaries of the covariance downdates, measurement
counts up to what the shared-memory working sets of the update kernels hold, and the refusal of a larger layout when a batch handle is
created.

Limits (kernels.h; Hopper's 227 KB of opt-in shared memory per block):
  gain kernel, sparse H (the estimator)   8 Mmax^2 + 260 Mmax bytes     -> Mmax <= 154, max_features <= 77
  gain kernel, dense H                    8 M^2 + 8 M bytes             -> M <= 169
  ekf_cov_tc2_kernel ("tf32x3")           49152 ceil(Mmax / 32) + 16896 -> Mmax <= 128, max_features <= 64
  ekf_cov_tc_kernel (XIVO_TC_V1=1)        streams K in blocks: no bound of its own
Tile boundaries: the fp64 downdate tiles by 32, both tensor-core kernels by 128 rows and 32 columns, and the K loop of the tensor-core
kernels runs in blocks of 32 (M = 128 fills the four K blocks tc2 keeps resident).

Tolerances are those of tests/test_gpu_ekf_batch.py, with d_i = P_ii of the prior: fp64 |dP_ij| <= 1e-9 sqrt(d_i d_j), tf32x3
1e-5 sqrt(d_i d_j); P exactly symmetric; rows and columns that are zero in the prior stay exactly zero.  The dense update is checked
against an extended-precision (np.longdouble) Joseph update, so that at N ~ 385, M ~ 169 the reference's own rounding takes no part of
the 1e-9 sqrt(d_i d_j) bound on the small-variance entries."""
import os
import types

import numpy as np
import pytest

import test_gpu_ekf_batch as EB
import test_gpu_estimator as GE
from oracle import ekf_oracle as E
from xivo_b200 import pyxivo, sim
from xivo_b200.capi import XivoError

SMEM_OPTIN = 227 * 1024


def _largest(fits):
    m = 0
    while fits(m + 1):
        m += 1
    return m


GAIN_SPARSE_ROWS = _largest(lambda m: 8 * m * m + 260 * m <= SMEM_OPTIN)
GAIN_DENSE_ROWS = _largest(lambda m: 8 * m * m + 8 * m <= SMEM_OPTIN)
TC2_ROWS = _largest(lambda m: 49152 * -(-m // 32) + 16896 <= SMEM_OPTIN)
F_MAX, F_TC2 = GAIN_SPARSE_ROWS // 2, TC2_ROWS // 2

DENSE_N = (128, 129, 256, 257, 384, 385, E.Layout(15, 64).N)  # one tile, one past it, two tiles, ..., and the largest tc2 layout
DENSE_M = (1, 32, 126, 128, GAIN_DENSE_ROWS)


# ---------------------------------------------------------------------------------------------------------------------------------
# extended-precision reference
# ---------------------------------------------------------------------------------------------------------------------------------
def _cholesky(S):
    L = np.zeros_like(S)
    for k in range(len(S)):
        d = S[k, k] - L[k, :k] @ L[k, :k]
        assert d > 0
        L[k, k] = np.sqrt(d)
        L[k + 1 :, k] = (S[k + 1 :, k] - L[k + 1 :, :k] @ L[k, :k]) / L[k, k]
    return L


def _cho_solve(L, B):
    Y = np.zeros_like(B)
    for r in range(len(L)):
        Y[r] = (B[r] - L[r, :r] @ Y[:r]) / L[r, r]
    X = np.zeros_like(B)
    for r in reversed(range(len(L))):
        X[r] = (Y[r] - L[r + 1 :, r] @ X[r + 1 :]) / L[r, r]
    return X


def joseph_longdouble(H, P, inn, diagR):
    """UpdateJosephForm (E.update_joseph) in np.longdouble: S = H P H' + R, K' = S^-1 H P, err = K inn, P' = A P A' + K R K' with
    A = I - K H, expanded as P - K HP - (K HP)' + K S K' so that every product is N x M x N.  Returns (P', err, |inn|_S) in fp64."""
    ld = np.longdouble
    H, P, inn, R = (np.asarray(a, dtype=ld) for a in (H, P, inn, diagR))
    HP = H @ P
    S = HP @ H.T + np.diag(R)
    L = _cholesky(S)
    Kt = _cho_solve(L, HP)
    KHP = Kt.T @ HP
    Pn = P - KHP - KHP.T + Kt.T @ (S @ Kt)
    inn_s = np.sqrt(inn @ _cho_solve(L, inn[:, None])[:, 0])
    return (0.5 * (Pn + Pn.T)).astype(np.float64), (Kt.T @ inn).astype(np.float64), float(inn_s)


def dense_problem(N, M, B, seed):
    """B filters of state dimension N: the spread-variance P of realistic_cov on a random live set (the last state always live, some
    others dead), a dense H whose columns are scaled by 1 / sqrt(P_jj) with 30 % of the entries nonzero, and R of the size of H P H'."""
    rng = np.random.default_rng(seed)
    lay = types.SimpleNamespace(N=N, feature_begin=23 + 6 * min(15, (N - 23) // 9))
    H, P, inn, R = np.zeros((B, M, N)), np.zeros((B, N, N)), np.zeros((B, M)), np.zeros((B, M))
    for b in range(B):
        dead = rng.choice(np.arange(23, N - 1), size=(N - 24) // 10, replace=False)
        live = np.setdiff1d(np.arange(N), dead)
        P[b] = EB.realistic_cov(lay, live, rng)
        s = np.sqrt(np.diag(P[b]))
        H[b] = rng.normal(size=(M, N)) * (rng.random((M, N)) < 0.3) / np.where(s > 0, s, 1.0)
        R[b] = 0.03 * len(live) * rng.uniform(0.2, 2.0, M)
        inn[b] = rng.normal(size=M) * np.sqrt(R[b])
    return H, P, inn, R


def check_dense(P0, H, inn, R, out, ptol, what):
    """The device's result of every filter against joseph_longdouble; returns the worst |dP_ij| / sqrt(d_i d_j)."""
    Pg, errg = out
    worst = 0.0
    for b in range(len(P0)):
        Pn, er, inn_s = joseph_longdouble(H[b], P0[b], inn[b], R[b])
        tag = f"{what}: filter {b}"
        P = Pg[b]
        assert np.array_equal(P, P.T), tag
        dead = ~np.any(P0[b] != 0, axis=0)
        assert dead.any() and np.all(P[dead] == 0) and np.all(P[:, dead] == 0), tag
        d = np.sqrt(np.diag(P0[b]))
        scale = np.outer(d, d)
        rel = np.abs(P - Pn) / np.where(scale > 0, scale, np.inf)
        i, j = np.unravel_index(np.argmax(rel), rel.shape)
        worst = max(worst, float(rel[i, j]))
        assert rel[i, j] <= ptol, f"{tag}: max |dP_ij| / sqrt(P_ii P_jj) = {rel[i, j]:.3e} at ({i}, {j})"
        assert np.all(np.abs(errg[b] - er) <= 1e-9 * d * inn_s), tag
    return worst


# ---------------------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------------------
def test_longdouble_joseph_matches_the_oracle():
    """CPU only: the extended-precision reference agrees with oracle/ekf_oracle.py's update_joseph on small problems, one of them with
    more measurement rows than states."""
    for N, M, seed in ((40, 10, 1), (62, 21, 2), (29, 33, 3)):
        H, P, inn, R = dense_problem(N, M, 1, seed)
        Pl, el, inn_s = joseph_longdouble(H[0], P[0], inn[0], R[0])
        Pr, er, _, S = E.update_joseph(H[0], P[0], inn[0], R[0])
        d = np.sqrt(np.diag(P[0]))
        scale = np.outer(d, d)
        live = scale > 0
        assert (np.abs(Pl - Pr)[live] / scale[live]).max() <= 1e-11
        assert np.all(Pl[~live] == 0)
        assert np.all(np.abs(el - er) <= 1e-11 * d * inn_s)
        assert abs(inn_s - np.sqrt(inn[0] @ np.linalg.solve(S, inn[0]))) <= 1e-12 * inn_s


def test_shared_memory_limits():
    """CPU only: the limits the formulas above give, as include/xivo_b200_estimator.h states them."""
    assert (GAIN_SPARSE_ROWS, GAIN_DENSE_ROWS, TC2_ROWS) == (154, 169, 128)
    assert (F_MAX, F_TC2) == (77, 64)


# ---------------------------------------------------------------------------------------------------------------------------------
# a. dense update at tile-boundary sizes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("M", DENSE_M)
@pytest.mark.parametrize("N", DENSE_N)
def test_dense_update_at_tile_boundaries(ctx, N, M, monkeypatch):
    """xivo_ekf_update_batch, two filters per launch: fp64 and the first tensor-core kernel at every M up to the gain kernel's limit,
    the second tensor-core kernel up to its own (M = 128: all four resident K blocks)."""
    H, P0, inn, R = dense_problem(N, M, 2, seed=N * 1000 + M)
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    worst = {"fp64": check_dense(P0, H, inn, R, ctx.ekf_update_batch(H, P0, inn, R), 1e-9, "fp64")}
    if M <= TC2_ROWS:
        worst["tc2"] = check_dense(P0, H, inn, R, ctx.ekf_update_batch(H, P0, inn, R, tf32x3=True), 1e-5, "tc2")
    monkeypatch.setenv("XIVO_TC_V1", "1")
    worst["tc1"] = check_dense(P0, H, inn, R, ctx.ekf_update_batch(H, P0, inn, R, tf32x3=True), 1e-5, "tc1")
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    assert worst["tc1"] > 0 and worst.get("tc2", 1.0) > 0  # the tensor cores did the downdate
    print(f"dense N = {N} M = {M}: worst |dP_ij| / sqrt(d_i d_j) " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---------------------------------------------------------------------------------------------------------------------------------
# b. the estimator's sparse update at the largest layouts
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("G,F,full_j", [(5, 25, False), (15, 48, False), (15, F_TC2, False), (15, F_TC2, True), (15, F_MAX, False)])
def test_batched_update_at_the_largest_layouts(ctx, G, F, full_j, monkeypatch):
    """xivo_filter_update_batch as in test_batched_update_phases_match_reference, three passes with M growing then shrinking, on
    N = 128 (one tile), 257 (one row into a third), 305 (the largest tc2 layout, M up to 128) and the largest layout of the gain kernel
    (M up to 154), where tc2 must be refused and fp64 and the first tensor-core kernel run."""
    B = 7
    filters, passes, _ = EB.schedule(G, F, B, seed=G * 100 + F + (7 if full_j else 0) + 5000)
    lay = E.Layout(G, F)
    Ms = [2 * len(ps["sel"]) for row in passes for ps in row]
    assert max(Ms) == 2 * F and Ms.count(2 * F) >= 1
    P0 = np.stack([f["P"] for f in filters])
    if F <= F_TC2:
        r64, r2, r1 = EB.run_modes(ctx, G, F, filters, passes, full_j, monkeypatch)
        runs = (("tc2", r2), ("tc1", r1))
    else:
        monkeypatch.delenv("XIVO_TC_V1", raising=False)
        r64 = ctx.filter_update_batch(G, F, filters, passes, full_j=full_j)
        with pytest.raises(XivoError, match=r"code -1\).*resident A operand"):
            ctx.filter_update_batch(G, F, filters, passes, tf32x3=True, full_j=full_j)
        monkeypatch.setenv("XIVO_TC_V1", "1")
        r1 = ctx.filter_update_batch(G, F, filters, passes, tf32x3=True, full_j=full_j)
        monkeypatch.delenv("XIVO_TC_V1", raising=False)
        runs = (("tc1", r1),)
    worst = {"fp64": EB.check_against_reference(lay, filters, passes, P0, r64, full_j, 1e-9, "fp64")}
    for name, r in runs:
        worst[name] = EB.check_against_reference(lay, filters, passes, P0, r, full_j, 1e-5, name)
        assert worst[name] > 0
        assert np.array_equal(r[1][0], r64[1][0]) and np.array_equal(r[2][0], r64[2][0]) and np.array_equal(r[3][0], r64[3][0]), name
    print(f"sparse G = {G} F = {F} full_j = {full_j} (N = {lay.N}, M up to {max(Ms)}): worst |dP_ij| / sqrt(d_i d_j) "
          + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ---------------------------------------------------------------------------------------------------------------------------------
# c. refusals leave the context usable
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refused_update_leaves_the_context_usable(ctx, monkeypatch):
    """A dense update one row past the gain kernel's limit, and a tf32x3 update past tc2's, return XIVO_ERR_ARG with the reason;
    the same context then runs a valid update of the same kind correctly."""
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    N = 257
    H, P0, inn, R = dense_problem(N, GAIN_DENSE_ROWS + 1, 2, seed=11)
    with pytest.raises(XivoError, match=r"code -1\).*M too large for the shared-memory Cholesky"):
        ctx.ekf_update_batch(H, P0, inn, R)
    m = GAIN_DENSE_ROWS
    check_dense(P0, H[:, :m], inn[:, :m], R[:, :m], ctx.ekf_update_batch(H[:, :m], P0, inn[:, :m], R[:, :m]), 1e-9, "fp64 after the refusal")
    H, P0, inn, R = dense_problem(N, TC2_ROWS + 2, 2, seed=12)
    with pytest.raises(XivoError, match=r"code -1\).*resident A operand"):
        ctx.ekf_update_batch(H, P0, inn, R, tf32x3=True)
    m = TC2_ROWS
    out = ctx.ekf_update_batch(H[:, :m], P0, inn[:, :m], R[:, :m], tf32x3=True)
    assert check_dense(P0, H[:, :m], inn[:, :m], R[:, :m], out, 1e-5, "tc2 after the refusal") > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# d. the estimator at the largest layouts; e. creation-time refusal
# ---------------------------------------------------------------------------------------------------------------------------------
def _pcw_cfg(cov):
    cfg = sim.load_cfg(os.path.join(GE.CFG, "pcw_sim.json"))
    cfg["covariance_update"] = cov
    return cfg


def run_pcw_against_oracle(b, cfg, G, F, pos_tol, rot_tol, ptol):
    """The 3 s point-cloud stream of pcw_sim.json through the (two-sequence) handle b against EstimatorOracle: pose after every frame,
    in-state id tables exact, P at the end.  Returns the largest in-state feature count reached."""
    msgs, _ = sim.pcw_stream(cfg, duration=3.0, seed=0)
    ref, ref_out = GE.run_oracle_pcw(cfg, msgs, G, F, True)
    b.init_with_sim_depths()
    k, most = 0, 0
    for kind, ts, p in msgs:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
        else:
            b.visual_meas_pointcloud(ts, p[0], p[1])
            g_ref, ids_ref, _ = ref_out[k]
            k += 1
            g = b.gsb(0)
            assert np.abs(g[:, 3] - g_ref[:, 3]).max() <= pos_tol, f"frame {k}"
            assert np.abs(g[:, :3] - g_ref[:, :3]).max() <= rot_tol, f"frame {k}"
            assert sorted(b.instate_features(0)["ids"].tolist()) == ids_ref, f"frame {k}"
            most = max(most, b.counters(0)["num_instate_features"])
    P = b.P(0)
    assert P.shape == (E.Layout(G, F).N,) * 2
    assert np.abs(P - ref.P).max() <= ptol * np.abs(ref.P).max()
    assert np.array_equal(b.P(1), P)
    return most


@pytest.mark.gpu
@pytest.mark.parametrize("cov,F", [("tf32x3", F_TC2), ("fp64", F_MAX)])
def test_pcw_stream_at_the_largest_layouts(cov, F):
    """(G = 15, F = 64) with tf32x3 and (G = 15, F = 77) with fp64: pose within 1e-7 m / 1e-8 (fp64) or 1e-4 m / 1e-5 (tf32x3) of
    the oracle, covariance within 1e-7 / 1e-4 of max|P|.  The point-cloud world may not fill F; tests a and b cover full M."""
    cfg = _pcw_cfg(cov)
    b = pyxivo.Batch(cfg, n_seq=2, max_groups=15, max_features=F)
    tol = (1e-7, 1e-8, 1e-7) if cov == "fp64" else (1e-4, 1e-5, 1e-4)
    most = run_pcw_against_oracle(b, cfg, 15, F, *tol)
    b.close()
    print(f"pcw {cov} G = 15 F = {F}: at most {most} features in state")
    assert most > 0


def _creates(cfg, F, tracker_only=False):
    try:
        b = pyxivo.Batch(cfg, n_seq=1, max_groups=15, max_features=F, tracker_only=tracker_only)
    except XivoError as e:
        assert "max_features" in str(e) and "code -1)" in str(e), str(e)
        return False
    b.close()
    return True


def _largest_creatable(cfg):
    lo, hi = 1, 1024
    assert _creates(cfg, lo) and not _creates(cfg, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _creates(cfg, mid) else (lo, mid)
    return lo


@pytest.mark.gpu
def test_batch_create_refuses_layouts_the_update_cannot_run(monkeypatch):
    """xivo_batch_create refuses max_features beyond what the selected update path holds, with XIVO_ERR_ARG naming max_features, instead
    of failing at the first measurement update; the largest F that creates is the limit of the shared-memory formulas.  The first
    tensor-core kernel (XIVO_TC_V1=1, chosen at creation) has no bound of its own, and a tracker-only handle runs no update.  A reset
    cannot change max_features or covariance_update (batch_incompatibility refuses either), so only creation needs the check."""
    monkeypatch.delenv("XIVO_TC_V1", raising=False)
    f64, tf32 = _pcw_cfg("fp64"), _pcw_cfg("tf32x3")
    f_max, f_tc2 = _largest_creatable(f64), _largest_creatable(tf32)
    print(f"largest max_features that creates: fp64 {f_max}, tf32x3 {f_tc2}")
    assert (f_max, f_tc2) == (F_MAX, F_TC2)
    with pytest.raises(XivoError, match="max_features = 78"):
        pyxivo.Batch(f64, n_seq=1, max_groups=15, max_features=F_MAX + 1)
    with pytest.raises(XivoError, match="max_features = 65"):
        pyxivo.Batch(tf32, n_seq=1, max_groups=15, max_features=F_TC2 + 1)
    assert _creates(f64, 300, tracker_only=True) and _creates(tf32, 300, tracker_only=True)
    monkeypatch.setenv("XIVO_TC_V1", "1")
    assert _largest_creatable(tf32) == F_MAX  # the gain kernel's bound still holds
    b = pyxivo.Batch(tf32, n_seq=2, max_groups=15, max_features=F_TC2 + 1)
    monkeypatch.delenv("XIVO_TC_V1", raising=False)  # the path was chosen at creation; updates follow it
    most = run_pcw_against_oracle(b, tf32, 15, F_TC2 + 1, 1e-4, 1e-5, 1e-4)
    b.close()
    print(f"pcw tf32x3 (first tensor-core kernel) G = 15 F = {F_TC2 + 1}: at most {most} features in state")

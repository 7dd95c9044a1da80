"""The product's host state machine (C++, compiled by g++ into tests/cpp/host_harness.cpp) run through WHOLE point-cloud
sequences on the CPU, with every device phase (depth sub-filter, Mahalanobis distances, EKF update) replaced by the values the numpy
oracle computed for the same frame; the image tracker's host decisions likewise through whole tracker-only image sequences, with the C
oracle (oracle/tracker_oracle.c) in place of the LK, FAST, BRIEF and matcher kernels.  Each frame the host's decisions — track list, feature/group slots, in-state and gauge sets, the
features that enter the update, the absorbed pose — must equal the oracle's, and the oracle itself is pinned on the reference's own
estimator (tests/test_reference_pin.py).  This covers the selection / gating / management logic incl. the libstdc++-defined orders
(std::unordered_map iteration, unstable std::sort, heap ties) without a GPU; the kernels are covered by the GPU parity tests."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import estimator_oracle as EO
from oracle import tracker_oracle as T
from xivo_b200 import sim, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
pytestmark = pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="needs g++ and the CUDA headers (host-only compile)")


@pytest.fixture(scope="module")
def hh(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("twin") / "libhost_harness.so")
    cmd = ["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-I", CUDA_INC, "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", "host_harness.cpp"), "-o", so]
    if os.environ.get("XIVO_HH_SO"):  # a pre-built harness, e.g. one compiled with -fsanitize=address,undefined (run under LD_PRELOAD=libasan.so)
        so = os.environ["XIVO_HH_SO"]
    else:
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.hh_create.restype = C.c_void_p
    lib.hh_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int]
    lib.hh_error.restype = C.c_char_p
    lib.hh_error_msg.restype = C.c_char_p
    lib.hh_error_msg.argtypes = [C.c_void_p]
    lib.hh_curr_time.restype = C.c_ulonglong
    for n in ("hh_destroy", "hh_init_with_sim_depths", "hh_curr_time", "hh_sticky_error"):
        getattr(lib, n).argtypes = [C.c_void_p]
    lib.hh_motion.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_inertial.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p]
    lib.hh_push.argtypes = [C.c_void_p, C.c_ulonglong, C.c_int]
    lib.hh_pop.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hh_pcw_begin.argtypes = [C.c_void_p, C.c_ulonglong, C.c_int, C.c_void_p, C.c_void_p]
    lib.hh_subfilter_ids.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_subfilter_inputs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hh_triangulation_counts.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_feature_states.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.hh_depth_refine_counts.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_feature_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    lib.hh_group_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.hh_just_dropped.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.hh_after_subfilter.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_after_gate.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_after_gate_diag.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hh_ransac_info.argtypes = [C.c_void_p] + [C.c_void_p] * 7
    lib.hh_ransac_temp.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_ransac_finish.argtypes = [C.c_void_p, C.c_void_p]
    lib.hh_ransac_rejected.argtypes = [C.c_void_p]
    lib.hh_after_update.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.hh_features.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    lib.hh_groups.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return lib


def feats(lib, h, which):
    buf = np.zeros((4096, 5), np.int32)
    n = lib.hh_features(h, which, buf.ctypes.data, 4096)
    return buf[:n].copy()


class Recorder:
    """Captures, per visual frame of the oracle, what the device computes in the product."""

    def __init__(self, est, monkeypatch):
        self.est, self.sub, self.sub_in, self.mh, self.err, self.P = est, [], [], [], None, None
        E = EO.E
        sub0, mh0, absorb0, adapt0 = E.subfilter_update, E.mh_distance, est.absorb, est.adapt_initial_depth

        def sub(*a, **k):
            self.sub_in.append(np.asarray(a[1], float).copy())  # the state the sub-filter starts from (after Feature::Triangulate)
            r = sub0(*a, **k)
            self.sub.append(np.concatenate([np.asarray(r[0], float).ravel(), np.asarray(r[1], float).ravel(), [float(r[2])]]))
            return r

        self.in_ransac = False
        ransac0 = est.one_point_ransac

        def mh(*a, **k):
            d = mh0(*a, **k)
            if not self.in_ransac:  # (the distances and the temporary correction of the 1-point RANSAC are read from est.ransac_trace)
                self.mh.append(float(d))
            return d

        def absorb(err, *a, **k):
            if not self.in_ransac:
                self.err = np.array(err, float).copy()
            return absorb0(err, *a, **k)

        def ransac(*a, **k):
            self.in_ransac = True
            try:
                return ransac0(*a, **k)
            finally:
                self.in_ransac = False

        est.one_point_ransac = ransac

        def adapt(*a, **k):
            self.P = est.P.copy()  # P after the update (or after this frame's slot edits when nothing was updated)
            return adapt0(*a, **k)

        monkeypatch.setattr(E, "subfilter_update", sub)
        monkeypatch.setattr(E, "mh_distance", mh)
        est.absorb, est.adapt_initial_depth = absorb, adapt

    def reset(self):
        self.sub, self.sub_in, self.mh, self.err, self.P = [], [], [], None, None


def _tri(method, zmax=60.0, theta=0.1):  # depth triangulation before the sub-filter (manager.cpp:229-231, :585-586), as in cfg/tumvi_cam0.json:119-158
    return {"triangulate_pre_subfilter": True, "initial_std_x_badtri": 1.0, "initial_std_y_badtri": 1.0, "initial_std_z_badtri": 1.0,
            "triangulation": {"method": method, "zmin": 0.05, "zmax": zmax, "max_theta_thresh": theta, "beta_thesh": 0.25}}


def _close(a, b, tol, scale=None):
    """|a - b| <= tol * max(1, |b|) element-wise; non-finite entries (a diverged depth refinement leaves inf / NaN states in the reference
    too, and the gate throws those features out) must be non-finite on both sides."""
    a, b = np.asarray(a, float), np.asarray(b, float)
    fin = np.isfinite(a) & np.isfinite(b)
    if not np.array_equal(np.isfinite(a), np.isfinite(b)):
        return False
    s = np.maximum(1.0, np.abs(b[fin])) if scale is None else scale
    return bool(np.all(np.abs(a[fin] - b[fin]) <= tol * s))


def _dopt(two_view, use_hessian):  # depth_opt block as in cfg/tumvi_cam1.json:162-169
    return {"use_depth_opt": True, "depth_opt": {"two_view": two_view, "use_hessian": use_hessian, "max_iters": 5, "eps": 1e-3, "damping": 1e-3, "max_res_norm": 2.5}}


TWIN_CASES = [(4, 14, 4.0, 1, True, "PrinceDormand", None), (15, 30, 3.0, 0, True, "RK4", None), (4, 14, 3.0, 6, False, "PrinceDormand", None),
              (15, 30, 6.0, 2, True, "PrinceDormand", None), (15, 30, 4.0, 0, True, "PrinceDormand", None),
              (4, 14, 4.0, 11, False, "PrinceDormand", _tri("l1_angular")), (15, 30, 3.0, 12, True, "PrinceDormand", _tri("l1_angular", zmax=5.0)),
              (4, 14, 3.0, 13, False, "PrinceDormand", _tri("l2_angular")), (4, 14, 3.0, 14, False, "RK4", _tri("linf_angular")),
              (4, 14, 3.0, 15, False, "PrinceDormand", _tri("direct_linear_transform_svd")), (4, 14, 3.0, 16, False, "PrinceDormand", _tri("direct_linear_transform_avg")),
              # use_depth_opt (Feature::RefineDepth on in-state candidates), all-views and two-view, Hessian as covariance on / off
              (4, 14, 4.0, 21, True, "PrinceDormand", _dopt(False, True)), (15, 30, 4.0, 22, True, "PrinceDormand", _dopt(True, True)),
              (4, 14, 3.0, 23, True, "RK4", _dopt(True, False)),
              # all views without the Hessian covariance: diverged candidates reach the gate with NaN Jacobians and are rejected there
              (4, 14, 4.0, 21, True, "PrinceDormand", _dopt(False, False)),
              # filter-level 1-point RANSAC (update.cpp:213-393): pass-through, every high-innovation feature rescued, rejections (two groups affected at once)
              (4, 14, 4.0, 31, True, "PrinceDormand", {"use_1pt_RANSAC": True}),
              (4, 14, 4.0, 32, True, "PrinceDormand", {"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 0.8}),
              (15, 30, 4.0, 34, True, "PrinceDormand", {"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 1.5, "sim_outliers": {"fraction": 0.08, "pixels": 2.5}}),
              (4, 14, 4.0, 35, True, "RK4", {"use_1pt_RANSAC": True, "1pt_RANSAC_thresh": 2.0, "1pt_RANSAC_Chi2": 3.0, "sim_outliers": {"fraction": 0.1, "pixels": 3.5}})]
# XIVO_TWIN_SWEEP=n adds n more seeds x both state sizes x with/without simulated depths (a wider offline sweep; 48 extra sequences passed at n = 12)
for _s in range(int(os.environ.get("XIVO_TWIN_SWEEP", "0"))):
    for _g, _f in ((4, 14), (15, 30)):
        for _d in (True, False):
            TWIN_CASES.append((_g, _f, 4.0, 100 + _s, _d, "PrinceDormand", _tri("l1_angular") if _s % 2 else None))


# (all-view depth refinement carries inf / NaN feature states through the oracle exactly as the reference carries them)
@pytest.mark.filterwarnings("ignore::RuntimeWarning")
@pytest.mark.parametrize("G,F,duration,seed,sim_depths,method,over", TWIN_CASES)
def test_host_state_machine_follows_the_oracle_frame_by_frame(hh, monkeypatch, tmp_path, G, F, duration, seed, sim_depths, method, over):
    cfg = sim.load_cfg(os.path.join(CFG, "pcw_sim.json"))
    cfg["integration_method"] = method
    cfg.update(over or {})
    msgs, _ = sim.pcw_stream(cfg, duration=duration, seed=seed)  # IMU and vision share timestamps: heap ties are exercised
    N = 23 + 6 * G + 3 * F
    est = EO.EstimatorOracle(cfg, G=G, F=F)
    est.sim_init_depths = sim_depths
    rec = Recorder(est, monkeypatch)
    h = hh.hh_create(json.dumps(cfg).encode(), G, F, 0)
    assert h, hh.hh_error()
    if sim_depths:
        hh.hh_init_with_sim_depths(h)
    # the oracle executes a message inside InertialMeas / VisualMeasPointCloud once its heap releases one; mirror that with the
    # product's own heap (hh_push / hh_pop) so that both execute the same message at the same step
    payload = {}
    n_vis = n_upd = n_ransac = n_ransac_rejected = 0
    for k, (kind, ts, p) in enumerate(msgs):
        payload[k] = (kind, ts, p)
        # ---- oracle
        rec.reset()
        vc0 = est.vision_counter
        if kind == "imu":
            est.InertialMeas(ts, p[0], p[1])
        else:
            est.VisualMeasPointCloud(ts, p[0], p[1])
        # ---- product host: push, pop, execute
        hh.hh_push(h, ts, k)  # the message type field carries the payload key
        t, key = C.c_ulonglong(), C.c_int()
        if not hh.hh_pop(h, C.byref(t), C.byref(key)):
            assert est.vision_counter == vc0 and rec.P is None
            continue
        mk, mts, mp = payload.pop(key.value)
        assert mts == t.value
        if mk == "imu":
            g, a = np.ascontiguousarray(mp[0], dtype=np.float64), np.ascontiguousarray(mp[1], dtype=np.float64)
            hh.hh_inertial(h, mts, g.ctypes.data, a.ctypes.data)
            assert est.vision_counter == vc0, "the oracle executed a visual message where the product executed an IMU one"
        else:
            assert est.vision_counter == vc0 + 1, "the product executed a visual message where the oracle did not"
            ids = np.ascontiguousarray(mp[0], dtype=np.int32)
            xpd = np.ascontiguousarray(mp[1], dtype=np.float64)
            nsub = hh.hh_pcw_begin(h, mts, len(ids), ids.ctypes.data, xpd.ctypes.data)
            assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
            if nsub < 0:
                assert rec.P is None  # neither side got past the clock / initialisation checks
                continue
            n_vis += 1
            assert nsub == len(rec.sub), f"frame {n_vis}: sub-filter batch {nsub} vs oracle {len(rec.sub)}"
            if nsub:  # what the product uploads to the sub-filter kernel: the feature states, triangulated where the oracle triangulated
                xin, tri_ok = np.zeros((nsub, 3)), np.zeros(nsub, np.int32)
                hh.hh_subfilter_inputs(h, xin.ctypes.data, tri_ok.ctypes.data)
                # the DLT forms solve a system whose conditioning is ~ 1 / sin^2(parallax of two consecutive frames): the rounding-level
                # difference of the two nominal states is amplified accordingly
                tol = 1e-6 if over and over.get("triangulation", {}).get("method", "").startswith("direct") else 1e-9
                # all-view depth refinement: Gauss-Newton along the nearly flat depth direction (pseudo-inverse entries up to 1e7,
                # feature.cpp:382) amplifies the 1e-10 difference between the two nominal states; refined-but-not-added candidates
                # come back through the sub-filter
                if over and over.get("use_depth_opt") and not over["depth_opt"]["two_view"]:
                    tol = 1e-3
                assert _close(xin, np.array(rec.sub_in), tol), f"frame {n_vis}: sub-filter input states"
            sub = np.ascontiguousarray(np.array(rec.sub).reshape(nsub, 13)) if nsub else np.zeros((1, 13))
            ninst = hh.hh_after_subfilter(h, sub.ctypes.data)
            assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
            # the gate batch: one Mahalanobis distance per in-state feature, in the product's (slot) order
            gated = len(rec.mh) > 0
            if gated:
                assert ninst == len(rec.mh), f"frame {n_vis}: {ninst} in-state features vs {len(rec.mh)} gated by the oracle"
            mh = np.ascontiguousarray(rec.mh if gated else np.zeros(max(1, ninst)), dtype=np.float64)
            if cfg.get("use_1pt_RANSAC"):
                tr_ = est.ransac_trace
                diag0 = np.ascontiguousarray(tr_["diag"] if tr_ else np.diag(est.P))  # the diagonal only matters when the RANSAC phases run
                nupd = hh.hh_after_gate_diag(h, mh.ctypes.data, diag0.ctypes.data)
                assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
                assert (nupd == -1) == (tr_ is not None), f"frame {n_vis}: the product {'runs' if nupd == -1 else 'skips'} the RANSAC phases, the oracle does not agree"
                if nupd == -1:
                    n_ransac += 1
                    tab, lo, hi, zp = np.zeros(64, np.int32), np.zeros(64, np.int32), np.zeros(64, np.int32), np.zeros(128, np.int32)
                    nl, nh, nz = C.c_int(), C.c_int(), C.c_int()
                    nt = hh.hh_ransac_info(h, tab.ctypes.data, lo.ctypes.data, C.addressof(nl), hi.ctypes.data, C.addressof(nh), zp.ctypes.data, C.addressof(nz))
                    assert lo[: nl.value].tolist() == tr_["low"] and hi[: nh.value].tolist() == tr_["high"], f"frame {n_vis}: low / high innovation sets"
                    e_tmp = np.ascontiguousarray(tr_["err"] if tr_["err"] is not None else np.zeros(N))
                    hh.hh_ransac_temp(h, e_tmp.ctypes.data)
                    mh_tab = np.ascontiguousarray([tr_["mh"].get(int(i), 0.0) for i in tab[:nt]] + [0.0])
                    nupd = hh.hh_ransac_finish(h, mh_tab.ctypes.data)
                    n_ransac_rejected += hh.hh_ransac_rejected(h)
                    assert hh.hh_ransac_rejected(h) == est.num_oneptransac_rejected
            else:
                nupd = hh.hh_after_gate(h, mh.ctypes.data)
            assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
            had = rec.err is not None
            assert (nupd > 0) == had, f"frame {n_vis}"
            n_upd += had
            P = rec.P if rec.P is not None else est.P
            err = np.ascontiguousarray(rec.err if had else np.zeros(N))
            Pmm, diag = np.ascontiguousarray(P[:23, :23]), np.ascontiguousarray(np.diag(P))
            hh.hh_after_update(h, err.ctypes.data, Pmm.ctypes.data, diag.ctypes.data, int(had))
            assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
            # ---- decisions must be identical
            tr = feats(hh, h, 2)
            assert tr[:, 0].tolist() == [f.id for f in est.tracks], f"frame {n_vis}: track list"
            assert tr[:, 3].tolist() == [int(f.status) for f in est.tracks], f"frame {n_vis}: feature status"
            inst = feats(hh, h, 0)
            o_inst = sorted(est.instate_features, key=lambda f: f.slot)
            assert sorted(map(tuple, inst[:, :3].tolist())) == sorted((f.id, f.sind, f.ref.sind) for f in o_inst), f"frame {n_vis}: in-state slots"
            assert sorted(inst[inst[:, 3] == 7, 0].tolist()) == sorted(f.id for f in o_inst if f.status == EO.F_GAUGE), f"frame {n_vis}: gauge features"
            if over and over.get("use_depth_opt"):  # the refined local states / Hessian covariances of the features now in the state
                fid, fx, fP = np.zeros(64, np.int32), np.zeros((64, 3)), np.zeros((64, 9))
                nf = hh.hh_feature_states(h, 1, fid.ctypes.data, fx.ctypes.data, fP.ctypes.data, 64)
                want = {f.id: f for f in est.instate_features}
                for i in range(nf):
                    o = want[int(fid[i])]
                    rt = 1e-8 if over["depth_opt"]["two_view"] else 1e-3
                    assert _close(fx[i], o.x, rt), f"frame {n_vis}: refined state of feature {fid[i]}"
                    assert _close(fP[i].reshape(3, 3), o.P, 100 * rt, scale=max(1e-12, float(np.nanmax(np.abs(o.P))))), f"frame {n_vis}: covariance of feature {fid[i]}"
            gb, gauge = np.zeros((64, 3), np.int32), C.c_int()
            ng = hh.hh_groups(h, gb.ctypes.data, 64, C.byref(gauge))
            assert sorted(map(tuple, gb[:ng, :2].tolist())) == sorted((g.id, g.sind) for g in est.groups.values() if g.instate())
            assert gauge.value == est.gauge_group
        m = np.zeros(42)
        hh.hh_motion(h, m.ctypes.data)
        # nominal state: the host integrates / absorbs with AVX2-FMA C++, the oracle with numpy: rounding-level drift over 150 updates
        assert np.abs(m[:9].reshape(3, 3) - est.X.Rsb).max() <= 1e-10 and np.abs(m[9:12] - est.X.Tsb).max() <= 1e-10, f"message {k}"
        assert np.abs(m[12:15] - est.X.Vsb).max() <= 1e-10 and hh.hh_curr_time(h) == est.curr_time
    assert n_vis >= 60 and n_upd >= 50 and len(est.instate_features) >= min(F, 10)
    if over and over.get("sim_outliers"):
        assert n_ransac >= 10 and n_ransac_rejected >= 3, "the RANSAC cases must exercise the temporary update and rejections"
    elif over and over.get("use_1pt_RANSAC") and over.get("1pt_RANSAC_thresh", 5) < 1:
        assert n_ransac >= 10
    gb2 = (C.c_int * 2)()
    hh.hh_triangulation_counts(h, gb2)
    assert (gb2[0], gb2[1]) == (est.num_good_tri, est.num_bad_tri)
    if over and over.get("triangulate_pre_subfilter"):
        assert gb2[0] >= 20 and gb2[1] >= 5, "the triangulation case must exercise both outcomes"
    if over and over.get("use_depth_opt"):
        hh.hh_depth_refine_counts(h, gb2)
        assert (gb2[0], gb2[1]) == (est.num_refined, est.num_refine_failed) and gb2[0] >= 100
    check_read_back_against_the_reference(hh, h, est, G, F, duration, seed, sim_depths, method, over, tmp_path)
    hh.hh_destroy(h)


# twin cases that are also pinned sequences of tests/test_reference_pin.py: (G, F, duration, seed, sim_depths, method) -> case name
PINNED = {(4, 14, 4.0, 1, True, "PrinceDormand"): "small_89", (15, 30, 4.0, 0, True, "PrinceDormand"): "default_203"}


def check_read_back_against_the_reference(hh, h, est, G, F, duration, seed, sim_depths, method, over, tmp_path):
    """Drop-in boundary: the host's read-back tables (csrc/estimator_host.cpp.inc: instate_feature_rows / instate_group_rows, what the
    C ABI's xivo_get_instate_feature_table / xivo_get_instate_group_table return) against what the REFERENCE'S OWN accessors
    (src/estimator_accessors.cpp through oracle/ref_wrap.cpp; golden copy in tests/golden/reference_pcw.npz) return at the end of
    the same sequence: InstateFeature{IDs,Sinds,RefGroups,Positions,Xc,xc,Preds,Meas,Covs} in both overloads (as-updated order, and
    sorted by covariance norm for n = 5 and n = 50), InstateGroup{IDs,Sinds,Poses,Covs}, JustDroppedFeatureIDs."""
    name = PINNED.get((G, F, duration, seed, sim_depths, method)) if not over else None
    if name is None:
        return
    import test_reference_pin as RP

    ref, how = RP.reference_result(name, None, G, F, duration, seed, sim_depths, 0, tmp_path)
    assert "acc.all.ids" in ref, f"{how}: no accessor dump (rebuild oracle/_ref or regenerate the golden file)"
    P = np.ascontiguousarray(est.P)
    buf = np.zeros((64, 22))
    for tag, n in (("all", -1), ("top5", 5), ("top50", 50)):
        k = hh.hh_feature_rows(h, P.ctypes.data, n, buf.ctypes.data, 64)
        want_ids = ref[f"acc.{tag}.ids"]
        assert k == len(want_ids)
        if n < 0:
            # `instate_features_` order: the reference sorts raw POINTERS (MakePtrVectorUnique, helpers.h:36-39) of separately
            # allocated pool objects, so its order changes from run to run of the same binary (observed); ours is slot order.
            # Same rows, matched by id.
            assert sorted(buf[:k, 0].astype(int).tolist()) == sorted(want_ids.tolist()), f"{how} {tag}: rows of the feature table"
            perm = [want_ids.tolist().index(i) for i in buf[:k, 0].astype(int)]
        else:
            assert buf[:k, 0].astype(int).tolist() == want_ids.tolist(), f"{how} {tag}: order of the feature table (sorted by covariance norm)"
            perm = list(range(k))
        assert buf[:k, 1].astype(int).tolist() == ref[f"acc.{tag}.sinds"][perm].tolist() and buf[:k, 2].astype(int).tolist() == ref[f"acc.{tag}.refs"][perm].tolist()
        for col, key, w in ((3, "Xs", 3), (6, "Xc", 3), (9, "xc", 3), (12, "pred", 2), (14, "meas", 2), (16, "cov", 6)):
            assert np.abs(buf[:k, col:col + w] - ref[f"acc.{tag}.{key}"][perm]).max() <= 1e-9, f"{how} {tag}.{key}"
    gbuf = np.zeros((32, 45))
    ng = hh.hh_group_rows(h, P.ctypes.data, gbuf.ctypes.data, 32)
    assert gbuf[:ng, 0].astype(int).tolist() == ref["acc.groups.ids"].tolist() and gbuf[:ng, 1].astype(int).tolist() == ref["acc.groups.sinds"].tolist()
    assert np.abs(gbuf[:ng, 2:9] - ref["acc.groups.pose"]).max() <= 1e-9
    cov = gbuf[:ng, 9:].reshape(ng, 6, 6)
    # the reference's InstateGroupCovs resets its column counter inside the row loop: only columns 0..5 are written, ending as
    # cov(5,5), cov(4,5), cov(3,5), cov(2,5), cov(1,5), cov(0,5) (pyxivo.Estimator.InstateGroupCovs reproduces exactly that)
    assert np.abs(cov[:, ::-1, 5] - ref["acc.groups.cov6"]).max() <= 1e-12
    tr = feats(hh, h, 2)  # tracked_features_no_descriptor(): Tracker::features_ order
    assert tr[:, 0].tolist() == ref["acc.tracked.ids"].tolist(), f"{how}: tracker list order"
    jd = (C.c_int * 512)()
    nj = hh.hh_just_dropped(h, jd, 512)
    assert sorted(jd[:nj]) == sorted(ref["acc.just_dropped"].tolist())


# ---- the image tracker (csrc/tracker_host.cpp.inc) against the oracle's Tracker, with the C oracle in place of the kernels ----
def _tracker_cfg(nmin=60, nmax=80, **tracker):  # as tests/test_gpu_widen_5_descriptors.py: 240 x 320 frames
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["message_buffer_size"] = 0
    cfg["tracker_cfg"].update(num_features_min=nmin, num_features_max=nmax)
    for k, v in tracker.items():  # (a block given here replaces only the keys it names)
        cfg["tracker_cfg"][k] = {**cfg["tracker_cfg"].get(k, {}), **v} if isinstance(v, dict) else v
    return cfg


def _frames(seed, n, step=(2, 1), bgr=False, mover=False, jumps=None):
    pad = 96 if jumps else 64
    canvas = synth.texture_canvas(240, 320, seed=seed, pad=pad)
    pos = np.cumsum([(0, 0)] + [(jumps or {}).get(k, step) for k in range(1, n)], axis=0)  # jumps: frame -> its shift from the previous frame
    out = [synth.frame_from_canvas(canvas, 240, 320, (int(pos[k][0]), int(pos[k][1])), noise_seed=10 * seed + k, pad=pad) for k in range(n)]
    if mover:  # a block moving against the background: its tracks are the homography's outliers
        for k, f in enumerate(out):
            f[60:180, 90:250] = synth.frame_from_canvas(canvas, 240, 320, (-step[0] * k, step[1] * k), noise_seed=10 * seed + k, pad=64)[60:180, 90:250]
    return [synth.to_bgr(f, distinct=True) for f in out] if bgr else out


def _orf(method):
    return {"method": method, "RANSAC_reproj_thresh": 3.0, "RANSAC_max_iters": 2000, "confidence": 0.995}


_DESC = dict(extract_descriptor=True, match_dropped_tracks=True)
# two sudden camera jumps that LK with few pyramid levels cannot follow: it converges to wrong places, where the descriptor check or the
# mask drops the tracks while the true keypoints are in view, so the rescue matches them
_JUMPS = dict(seed=7, n=12, jumps={4: (28, 12), 8: (-24, 10)})
TRACKER_CASES = {
    # low FAST threshold and a small mask: thousands of keypoints in a narrow score band (ties resolved by (y, x)); on the second of two
    # blank frames every track is lost and nothing is detected, the next frame finds an empty list and the one after re-initialises
    "lk_ties_blank": (_tracker_cfg(300, 400, mask_size=5, margin=4, FAST={"threshold": 5, "nonmaxSuppression": True}), dict(seed=3, n=10, blank=4)),
    "lk_bgr": (_tracker_cfg(75, 100, FAST={"threshold": 20, "nonmaxSuppression": True}), dict(seed=4, n=8, bgr=True)),
    "lk_outliers_lmeds": (_tracker_cfg(do_outlier_rejection=True, outlier_rejection=_orf("LMEDS")), dict(seed=5, n=10, step=(3, 2), mover=True)),
    "lk_outliers_ransac": (_tracker_cfg(do_outlier_rejection=True, outlier_rejection=_orf("RANSAC")), dict(seed=6, n=10, step=(3, 2), mover=True)),
    # (num_features_min = max: a detection every frame with a small budget, which a rescue can use up)
    "rescue_like_tumvi_cam0": (_tracker_cfg(80, 80, **_DESC, differential=False, descriptor_distance_thresh=-1, KLT={"max_level": 2}), dict(_JUMPS, seed=12)),
    "distance_check_differential": (_tracker_cfg(**_DESC, differential=True, descriptor_distance_thresh=70, KLT={"max_level": 0}), _JUMPS),
    "rescue_with_outlier_rejection": (_tracker_cfg(**_DESC, differential=True, do_outlier_rejection=True, outlier_rejection=_orf("LMEDS"),
                                                   KLT={"max_level": 1}), dict(_JUMPS, mover=True)),
    "match": (_tracker_cfg(tracker_type="MATCH", extract_descriptor=True, differential=True, descriptor_distance_thresh=-1), dict(seed=10, n=12, step=(3, 2))),
    "match_outliers_lmeds": (_tracker_cfg(tracker_type="MATCH", extract_descriptor=True, differential=True, descriptor_distance_thresh=-1, do_outlier_rejection=True,
                                          outlier_rejection=_orf("LMEDS")), dict(seed=11, n=10, step=(3, 2), mover=True)),
}


def _pack(xy, sc):  # launch_fast_detect's keypoint format: y << 20 | x << 8 | score
    assert len(sc) == 0 or sc.max() <= 255
    return np.ascontiguousarray((xy[:, 1].astype(np.uint32) << 20) | (xy[:, 0].astype(np.uint32) << 8) | sc.astype(np.uint32))


def _ptr(a):
    return a.ctypes.data if a is not None else None


@pytest.mark.parametrize("case", list(TRACKER_CASES))
def test_image_tracker_follows_the_oracle_frame_by_frame(hh, case):
    cfg, fr = TRACKER_CASES[case]
    frames = _frames(fr["seed"], fr["n"], fr.get("step", (2, 1)), fr.get("bgr", False), fr.get("mover", False), fr.get("jumps"))
    if "blank" in fr:
        frames[fr["blank"]:fr["blank"]] = [np.full((240, 320), 128, np.uint8)] * 2
    for n, t in (("hh_tracker_lk_begin", [C.c_void_p] * 3 + [C.c_int]), ("hh_tracker_lk_accept", [C.c_void_p] * 6),
                 ("hh_tracker_detect_select", [C.c_void_p] * 2 + [C.c_int]), ("hh_tracker_order_keypoints", [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p]),
                 ("hh_tracker_queries", [C.c_void_p] * 2 + [C.c_int]), ("hh_tracker_detect_select_desc", [C.c_void_p] * 3 + [C.c_int]),
                 ("hh_tracker_match_begin", [C.c_void_p] * 2 + [C.c_int, C.c_void_p]), ("hh_tracker_match_finish", [C.c_void_p] * 3 + [C.c_int]),
                 ("hh_tracks", [C.c_void_p] * 4 + [C.c_int]), ("hh_track_descriptors", [C.c_void_p] * 2 + [C.c_int]), ("hh_tracker_counts", [C.c_void_p] * 2), ("hh_tracker_geometry", [C.c_void_p, C.c_int, C.c_int]),
                 ("hh_visual_begin", [C.c_void_p, C.c_ulonglong, C.c_int])):
        getattr(hh, n).argtypes = t
    for n in ("hh_tracker_detect_budget", "hh_tracker_lk_finish", "hh_tracker_only_finish"):
        getattr(hh, n).argtypes = [C.c_void_p]
    est = EO.EstimatorOracle(cfg, G=4, F=14, tracker_only=True)
    h = hh.hh_create(json.dumps(cfg).encode(), 4, 14, 1)
    assert h, hh.hh_error()
    hh.hh_tracker_geometry(h, 240, 320)
    max_pts = est.t_max + 8
    p0, p1 = np.zeros((max_pts, 2), np.float32), np.zeros((max_pts, 2), np.float32)
    qd = np.zeros((max_pts, 32), np.uint8)
    ids, st, xy, tdesc = np.zeros(4096, np.int32), np.zeros(4096, np.int32), np.zeros((4096, 2)), np.zeros((4096, 32), np.uint8)
    cnt = np.zeros(3, np.int32)

    def detect(img):
        kxy, sc, _ = T.fast_detect(img, est.fast_thr, est.fast_nms)
        return _pack(kxy, sc)

    def describe_and_match(img, nk, kpxy):
        D = np.ascontiguousarray(T.brief(img, kpxy[:nk])[0]) if nk else np.zeros((1, 32), np.uint8)
        nq = hh.hh_tracker_queries(h, _ptr(qd), max_pts)
        m = np.ascontiguousarray(T.bf_match_crosscheck(qd[:nq], D[:nk]) if nq and nk else np.zeros((0, 3)), np.int32).reshape(-1, 3)
        return D, m

    # DetectLK's outcome before UpdateLK marks the newly dropped tracks DROPPED again (what a rescue did to a track is visible only here):
    # the oracle's track list right after detect_lk
    snap, n_rescued, n_dist_drops, n_candidates = [], 0, 0, 0
    detect0 = est.detect_lk

    def detect_lk(img, num_to_add, newly_dropped=(), check_homography=False):
        nonlocal n_rescued
        seen = {f.id: len(f.track) for f in newly_dropped}
        detect0(img, num_to_add, newly_dropped, check_homography)
        # the product marks a newly dropped track DROPPED before DetectLK, the oracle after it; a rescued one is TRACKED in both
        rescued = {f.id for f in newly_dropped if len(f.track) > seen[f.id]}
        n_rescued += len(rescued)
        status = lambda f: int(EO.TRACKED if f.id in rescued else EO.DROPPED) if f.id in seen else int(f.tstatus)
        snap.append([(f.id, status(f), float(f.xp()[0]), float(f.xp()[1]), bytes(np.asarray(f.descriptor, np.uint8).tobytes()) if est.extract_descriptor else b"")
                     for f in est.tracks])

    est.detect_lk = detect_lk

    def snapshot():
        n = hh.hh_tracks(h, _ptr(ids), _ptr(st), _ptr(xy), len(ids))
        hh.hh_track_descriptors(h, _ptr(tdesc), len(tdesc))
        return [(int(ids[i]), int(st[i]), float(xy[i, 0]), float(xy[i, 1]), tdesc[i].tobytes() if est.extract_descriptor else b"") for i in range(n)]

    prev, tracks_seen, rejected = None, [], []
    for k, img in enumerate(frames):
        ts = (k + 1) * 40_000_000
        vc = est.vision_counter
        est.VisualMeasTrackerOnly(ts, img)
        assert est.vision_counter == vc + 1
        assert hh.hh_visual_begin(h, ts, 2) == 1
        if est.tracker_type == "MATCH":
            kps = detect(img)
            kpxy = np.zeros((max(1, len(kps)), 2), np.float32)
            nk = hh.hh_tracker_match_begin(h, _ptr(kps), len(kps), _ptr(kpxy))
            D, m = describe_and_match(img, nk, kpxy)
            hh.hh_tracker_match_finish(h, _ptr(D), _ptr(m), len(m))
        else:
            ntr = hh.hh_tracks(h, _ptr(ids), _ptr(st), _ptr(xy), len(ids))
            kind = hh.hh_tracker_lk_begin(h, _ptr(p0), _ptr(p1), max_pts)
            assert kind in (1, 2, 3), f"frame {k}: kind {kind}"
            if kind == 2:  # the LK kernel on the points the host staged
                r1, lkst, _ = T.lk_track(prev, img, p0[:ntr], p1[:ntr], **est.klt)
                r1, lkst = np.ascontiguousarray(r1, np.float32), np.ascontiguousarray(lkst, np.uint8)
                d = v = None
                if est.extract_descriptor:
                    d, v = T.brief(img, r1)
                    d, v = np.ascontiguousarray(d), np.ascontiguousarray(v, np.uint8)
                lkst0 = lkst.copy()
                hh.hh_tracker_lk_accept(h, _ptr(p0), _ptr(r1), _ptr(lkst), _ptr(d), _ptr(v))
                n_dist_drops += int((lkst0 > lkst).sum())  # tracks the descriptor-distance check dropped
            if kind != 3:
                if hh.hh_tracker_detect_budget(h) > 0:
                    kps = detect(img)
                    if not est.extract_descriptor:
                        hh.hh_tracker_detect_select(h, _ptr(kps), len(kps))
                    else:
                        kpxy = np.zeros((max(1, len(kps)), 2), np.float32)
                        nk = hh.hh_tracker_order_keypoints(h, _ptr(kps), len(kps), 1, _ptr(kpxy))
                        D, m = describe_and_match(img, nk, kpxy)
                        hh.hh_tracker_detect_select_desc(h, _ptr(D), _ptr(m), len(m))
                        n_candidates += len(m)
                    assert snapshot() == snap.pop(0), f"frame {k}: track list after DetectLK"
                prev = img
            hh.hh_tracker_lk_finish(h)
        hh.hh_tracker_only_finish(h)
        assert hh.hh_sticky_error(h) == 0, hh.hh_error_msg(h)
        assert not snap, f"frame {k}: the oracle detected, the product did not"
        n = hh.hh_tracks(h, _ptr(ids), _ptr(st), _ptr(xy), len(ids))
        assert ids[:n].tolist() == [f.id for f in est.tracks], f"frame {k}: track ids / order"
        assert st[:n].tolist() == [int(f.tstatus) for f in est.tracks], f"frame {k}: TrackStatus"
        assert np.array_equal(xy[:n], np.array([f.xp() for f in est.tracks]).reshape(-1, 2)), f"frame {k}: positions"
        hh.hh_tracker_counts(h, _ptr(cnt))
        assert (cnt[0], cnt[1]) == (est.num_failed_to_track, est.num_outliers_rejected), f"frame {k}: failed / outlier counts"
        if est.tracker_type == "MATCH":
            assert cnt[2] == est.num_new_detections, f"frame {k}: new detections"
        tracks_seen.append(n)
        rejected.append(int(cnt[1]))
    hh.hh_destroy(h)
    print(case, "frames", len(frames), "tracks per frame", tracks_seen, "outliers rejected", rejected, "rescued", n_rescued, "of", n_candidates, "candidates", "distance-check drops", n_dist_drops)
    assert max(tracks_seen) >= 0.9 * est.t_max
    if "blank" in fr:
        b = fr["blank"]
        assert tracks_seen[b + 1] == tracks_seen[b + 2] == 0 and tracks_seen[b + 3] == est.t_max, "the blank frames force a re-initialisation"
    if est.do_outlier_rejection:
        assert sum(rejected) >= 50, "the homography rejection must reject tracks"
    if est.match_dropped and not est.do_outlier_rejection:
        assert n_rescued >= 5, "the rescue of newly dropped tracks must be exercised"
    if est.match_dropped and est.do_outlier_rejection:  # CheckHomography compares the creation keypoint: under camera motion it rejects them all
        assert n_candidates >= 5, "cross-checked matches must reach the homography check of the rescue"
    if est.desc_thresh > 0 and est.tracker_type == "LK":
        assert n_dist_drops >= 5, "the descriptor-distance check must drop tracks"

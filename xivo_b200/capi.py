"""ctypes binding of include/xivo_b200.h (kernel-level entry points) with numpy in/out.

This is plumbing only: every function forwards to the C ABI of libxivo_b200.so, which runs the
CUDA kernels.  There is no Python/CPU implementation behind any of these calls; if the shared
library is missing or no CUDA device is present the call raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libxivo_b200.so")


class XivoError(RuntimeError):
    pass


XIVO_ERR_ARG, XIVO_ERR_CUDA, XIVO_ERR_STATE, XIVO_ERR_SLOTS = -1, -2, -3, -4
XIVO_SEQ_FAILED = 1  # a message call of a failure-isolating batch handle: sequences failed during it, the others finished it normally


_lib = None


def lib() -> C.CDLL:
    """Load libxivo_b200.so (built in-tree by xivo_b200/build.py). Fails loudly when absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise XivoError(
                f"{LIB_PATH} not found: build it with `python -m xivo_b200.build` "
                "(xivo_b200 has no CPU fallback)"
            )
        _lib = C.CDLL(LIB_PATH)
        _lib.xivo_last_error.restype = C.c_char_p
        _lib.xivo_launch_count.restype = C.c_ulonglong
        _lib.xivo_pyramid_layout.restype = C.c_ulonglong
        _lib.xivo_batch_isolate_failures.argtypes = [C.c_void_p, C.c_int]
        _lib.xivo_batch_sequence_status.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_int]
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        raise XivoError(f"{what} failed (code {rc}): {lib().xivo_last_error().decode()}")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def launch_count() -> int:
    return int(lib().xivo_launch_count())


def png_info(data: bytes):
    """xivo_png_info: (rows, cols, channels, bit_depth) of a PNG file's bytes; XivoError names the reason for a refused file."""
    data = bytes(data)
    r, c, ch, bd = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    _check(lib().xivo_png_info(C.c_char_p(data), C.c_size_t(len(data)), C.byref(r), C.byref(c), C.byref(ch), C.byref(bd)), "xivo_png_info")
    return r.value, c.value, ch.value, bd.value


class Context:
    """xivo_ctx: one CUDA device + stream."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        _check(lib().xivo_ctx_create(C.c_int(device), C.byref(self._h)), "xivo_ctx_create")

    def close(self):
        if self._h:
            lib().xivo_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ tracker
    @staticmethod
    def pyramid_layout(rows, cols, cn, win, max_level):
        n = C.c_int()
        r = (C.c_int * 8)()
        c = (C.c_int * 8)()
        o = (C.c_ulonglong * 8)()
        total = lib().xivo_pyramid_layout(rows, cols, cn, win, max_level, C.byref(n), r, c, o)
        L = n.value
        return int(total), [(r[i], c[i], int(o[i])) for i in range(L)]

    def build_pyramid(self, img: np.ndarray, win: int, max_level: int):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        rows, cols = img.shape[:2]
        cn = 1 if img.ndim == 2 else img.shape[2]
        total, levels = self.pyramid_layout(rows, cols, cn, win, max_level)
        out = np.zeros(total, np.uint8)
        _check(lib().xivo_build_pyramid(self._h, _p(img), rows, cols, cn, win, max_level, _p(out)), "xivo_build_pyramid")
        res = []
        for (r, c, off) in levels:
            a = out[off : off + r * c * cn]
            res.append(a.reshape(r, c) if cn == 1 else a.reshape(r, c, cn))
        return res

    def fast_detect(self, img: np.ndarray, threshold: int, nonmax: bool = True, max_kp: int = 1 << 16):
        img = np.ascontiguousarray(img, dtype=np.uint8)
        rows, cols = img.shape[:2]
        cn = 1 if img.ndim == 2 else img.shape[2]
        xy = np.zeros((max_kp, 2), np.int32)
        sc = np.zeros(max_kp, np.int32)
        n = C.c_int()
        _check(
            lib().xivo_fast_detect(self._h, _p(img), rows, cols, cn, int(threshold), int(bool(nonmax)), _p(xy), _p(sc), max_kp, C.byref(n)),
            "xivo_fast_detect",
        )
        k = min(n.value, max_kp)
        return xy[:k].copy(), sc[:k].copy(), n.value

    def normalize_minmax(self, frames: np.ndarray, channels: int = 1):
        """xivo_normalize_minmax: cv2.normalize(f, None, 0, 255, cv2.NORM_MINMAX) of each frame of an (n, rows, cols) (channels = 1) or
        (n, rows, cols, 3) (channels = 3) uint8 array; returns a new array of the same shape."""
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        if frames.ndim != (3 if channels == 1 else 4) or (channels == 3 and frames.shape[3] != 3):
            raise ValueError(f"normalize_minmax: expected (n, rows, cols{'' if channels == 1 else ', 3'}) frames, got {frames.shape}")
        n, rows, cols = frames.shape[:3]
        out = np.empty_like(frames)
        _check(lib().xivo_normalize_minmax(self._h, n, rows, cols, int(channels), _p(frames), _p(out)), "xivo_normalize_minmax")
        return out

    def lk_track(self, prev, nxt, prev_pts, init_pts, win=15, max_level=5, max_iter=30, eps=0.01, use_initial_flow=True, min_eig=1e-4):
        prev = np.ascontiguousarray(prev, dtype=np.uint8)
        nxt = np.ascontiguousarray(nxt, dtype=np.uint8)
        assert prev.shape == nxt.shape
        rows, cols = prev.shape[:2]
        cn = 1 if prev.ndim == 2 else prev.shape[2]
        p0 = np.ascontiguousarray(prev_pts, dtype=np.float32).reshape(-1, 2)
        p1 = np.array(init_pts, dtype=np.float32).reshape(-1, 2).copy()
        n = len(p0)
        st = np.zeros(n, np.uint8)
        er = np.zeros(n, np.float32)
        _check(
            lib().xivo_lk_track(
                self._h, _p(prev), _p(nxt), rows, cols, cn, _p(p0), _p(p1), _p(st), _p(er), n, win, max_level, max_iter,
                C.c_double(eps), int(bool(use_initial_flow)), C.c_double(min_eig),
            ),
            "xivo_lk_track",
        )
        return p1, st, er

    def decode_png(self, blobs, channels=3):
        """xivo_decode_png: PNG files' bytes (any geometry) -> list of rows x cols x 3 (BGR, cv2.imread) or rows x cols (grey) uint8."""
        blobs = [bytes(b) for b in blobs]
        n = len(blobs)
        outs = []
        for i, b in enumerate(blobs):
            try:
                r, c, _, _ = png_info(b)  # the output geometry; xivo_decode_png walks the same chunks again
            except XivoError as e:
                raise XivoError(f"png frame {i}: {e}") from None
            outs.append(np.zeros((r, c, channels) if channels == 3 else (r, c), np.uint8))
        src = (C.c_char_p * max(n, 1))(*blobs)
        sizes = (C.c_size_t * max(n, 1))(*[len(b) for b in blobs])
        dst = (C.c_void_p * max(n, 1))(*[o.ctypes.data for o in outs])
        _check(lib().xivo_decode_png(self._h, n, src, sizes, int(channels), dst), "xivo_decode_png")
        return outs

    # ------------------------------------------------------------------ EKF
    def jacobian_batch(self, G, F, camera, X24, groups, feat_x, feat_xp, feat_ref, feat_sind, P=None, R=1.0, dense=True):
        camera, X24, groups = _f64(camera), _f64(X24), _f64(groups)
        fx, fxp = _f64(feat_x).reshape(-1, 3), _f64(feat_xp).reshape(-1, 2)
        fr, fs = _i32(feat_ref), _i32(feat_sind)
        n = len(fx)
        N = 23 + 6 * G + 3 * F
        J = np.zeros((n, 2, N)) if dense else None
        inn = np.zeros((n, 2))
        mh = np.zeros(n)
        Pd = None if P is None else _f64(P)
        _check(
            lib().xivo_jacobian_batch(self._h, G, F, _p(camera), _p(X24), _p(groups), n, _p(fx), _p(fxp), _p(fr), _p(fs), _p(Pd),
                                      C.c_double(R), _p(J), _p(inn), _p(mh)),
            "xivo_jacobian_batch",
        )
        return J, inn, mh

    def mh_gate(self, G, F, camera, X24, groups, feat_x, feat_xp, feat_ref, feat_sind, P, R):
        camera, X24, groups = _f64(camera), _f64(X24), _f64(groups)
        fx, fxp = _f64(feat_x).reshape(-1, 3), _f64(feat_xp).reshape(-1, 2)
        fr, fs = _i32(feat_ref), _i32(feat_sind)
        n = len(fx)
        mh = np.zeros(n)
        _check(
            lib().xivo_mh_gate(self._h, G, F, _p(camera), _p(X24), _p(groups), n, _p(fx), _p(fxp), _p(fr), _p(fs), _p(_f64(P)),
                               C.c_double(R), _p(mh)),
            "xivo_mh_gate",
        )
        return mh

    def brief_describe(self, img, kp_xy):
        """BRIEF-32 at the keypoints (n x 2) -> (descriptors n x 32 uint8, valid n bool)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        rows, cols = img.shape[:2]
        cn = 1 if img.ndim == 2 else img.shape[2]
        kp = np.ascontiguousarray(kp_xy, dtype=np.float32).reshape(-1, 2)
        n = len(kp)
        desc, valid = np.zeros((max(n, 1), 32), np.uint8), np.zeros(max(n, 1), np.uint8)
        _check(lib().xivo_brief_describe(self._h, _p(img), rows, cols, cn, _p(kp), n, _p(desc), _p(valid)), "xivo_brief_describe")
        return desc[:n], valid[:n].astype(bool)

    def hamming_match(self, query, train):
        """Cross-checked 1-NN Hamming matches of 32-byte descriptors -> [(queryIdx, trainIdx, distance)] in query order."""
        q, t = np.ascontiguousarray(query, np.uint8).reshape(-1, 32), np.ascontiguousarray(train, np.uint8).reshape(-1, 32)
        out, n = np.zeros((max(len(q), 1), 3), np.int32), C.c_int()
        _check(lib().xivo_hamming_match(self._h, _p(q), len(q), _p(t), len(t), _p(out), C.byref(n)), "xivo_hamming_match")
        return [tuple(int(v) for v in r) for r in out[: n.value]]

    def ekf_update(self, H, P, inn, diagR, tf32x3=False):
        """UpdateJosephForm; tf32x3=True runs the covariance downdate on the tensor cores (XIVO_UPDATE_TF32X3)."""
        H, inn, diagR = _f64(H), _f64(inn), _f64(diagR)
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        M, N = H.shape if H.size else (0, P.shape[0])
        err = np.zeros(N)
        _check(lib().xivo_ekf_update_ex(self._h, N, M, _p(H), _p(P), _p(inn), _p(diagR), _p(err), C.c_uint(1 if tf32x3 else 0)),
               "xivo_ekf_update_ex")
        return P, err

    def ekf_update_batch(self, H, P, inn, diagR, tf32x3=False, repeat=1):
        """`batch` filters of one (N, M) in one launch pair: H (B, M, N), P (B, N, N), inn / diagR (B, M) -> (P, err).  repeat > 1 re-applies
        the update to the original P on the device (kernel timing through the in-library profiler)."""
        H, inn, diagR = _f64(H), _f64(inn), _f64(diagR)
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        B, M, N = H.shape
        assert P.shape == (B, N, N) and inn.shape == (B, M) and diagR.shape == (B, M)
        err = np.zeros((B, N))
        _check(lib().xivo_ekf_update_batch(self._h, N, M, B, _p(H), _p(P), _p(inn), _p(diagR), _p(err), C.c_uint(1 if tf32x3 else 0), int(repeat)),
               "xivo_ekf_update_batch")
        return P, err

    def filter_update(self, G, F, camera, X24, groups, feat_x, feat_xp, feat_ref, feat_sind, sel, R, P, want_H=True):
        camera, X24, groups = _f64(camera), _f64(X24), _f64(groups)
        fx, fxp = _f64(feat_x).reshape(-1, 3), _f64(feat_xp).reshape(-1, 2)
        fr, fs, sel = _i32(feat_ref), _i32(feat_sind), _i32(sel)
        n, ns = len(fx), len(sel)
        N = 23 + 6 * G + 3 * F
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        err = np.zeros(N)
        Hd = np.zeros((2 * ns, N)) if want_H else None
        _check(
            lib().xivo_filter_update(self._h, G, F, _p(camera), _p(X24), _p(groups), n, _p(fx), _p(fxp), _p(fr), _p(fs), _p(sel), ns,
                                     C.c_double(R), _p(P), _p(err), _p(Hd)),
            "xivo_filter_update",
        )
        return P, err, Hd

    def filter_update_batch(self, G, F, filters, passes, tf32x3=False, full_j=False):
        """The estimator's gate + update phases for B filters of one layout, len(passes) times on the same device buffers.
        filters: B dicts with camera, X24, groups (G x 12), feat_x (n x 3), feat_xp (n x 2), feat_ref, feat_sind (n), R, P (N x N).
        passes: per pass, B dicts with "pre" / "post" edit lists of (type, a, b, n[, blk9]) ops and "sel" (indices into the features).
        Returns P (npass, B, N, N), err (npass, B, N), mh (npass, B, F), diag (npass, B, N) after every pass."""
        B, npass, N = len(filters), len(passes), 23 + 6 * G + 3 * F
        cam = np.zeros((B, 11)); X = np.zeros((B, 24)); grp = np.zeros((B, G, 12)); R = np.zeros(B); P0 = np.zeros((B, N, N))
        fx = np.zeros((B, F, 3)); fxp = np.zeros((B, F, 2)); fr = np.zeros((B, F), np.int32); fs = np.zeros((B, F), np.int32)
        nfeat = np.zeros(B, np.int32)
        for b, f in enumerate(filters):
            n = len(f["feat_x"])
            cam[b], X[b], grp[b], R[b], P0[b], nfeat[b] = f["camera"], f["X24"], f["groups"], f["R"], f["P"], n
            fx[b, :n], fxp[b, :n], fr[b, :n], fs[b, :n] = f["feat_x"], f["feat_xp"], f["feat_ref"], f["feat_sind"]

        def pack(key):
            counts, ops, blks = np.zeros((npass, B), np.int32), [], []
            for p, ps in enumerate(passes):
                assert len(ps) == B
                for b, d in enumerate(ps):
                    lst = d.get(key, [])
                    counts[p, b] = len(lst)
                    for op in lst:
                        ops.append(op[:4])
                        blks.append(np.ravel(op[4]) if len(op) > 4 else np.zeros(9))
            return counts, _i32(np.reshape(ops, (-1, 4))), _f64(np.reshape(blks, (-1, 9)))

        pre_n, pre_ops, pre_blk = pack("pre")
        post_n, post_ops, post_blk = pack("post")
        nsel, sel = np.zeros((npass, B), np.int32), np.zeros((npass, B, F), np.int32)
        for p, ps in enumerate(passes):
            for b, d in enumerate(ps):
                s = np.asarray(d.get("sel", []), np.int32)
                nsel[p, b] = len(s)
                sel[p, b, : len(s)] = s
        Po, err, mh, diag = np.zeros((npass, B, N, N)), np.zeros((npass, B, N)), np.zeros((npass, B, F)), np.zeros((npass, B, N))
        flags = (1 if tf32x3 else 0) | (2 if full_j else 0)
        _check(
            lib().xivo_filter_update_batch(self._h, G, F, B, npass, _p(cam), _p(X), _p(grp), _p(nfeat), _p(fx), _p(fxp), _p(fr), _p(fs), _p(R),
                                           _p(P0), _p(pre_n), _p(pre_ops), _p(pre_blk), _p(nsel), _p(sel), _p(post_n), _p(post_ops), _p(post_blk),
                                           C.c_uint(flags), _p(Po), _p(err), _p(mh), _p(diag)),
            "xivo_filter_update_batch",
        )
        return Po, err, mh, diag

    def subfilter_batch(self, camera, X24, x, P33, xp, ref, outlier, Rtri, mh_thresh):
        camera, X24 = _f64(camera), _f64(X24)
        x, P33, xp, ref, outlier = _f64(x).reshape(-1, 3), _f64(P33).reshape(-1, 9), _f64(xp).reshape(-1, 2), _f64(ref).reshape(-1, 12), _f64(outlier)
        n = len(x)
        xo, Po, oo = np.zeros((n, 3)), np.zeros((n, 9)), np.zeros(n)
        _check(
            lib().xivo_subfilter_batch(self._h, _p(camera), _p(X24), n, _p(x), _p(P33), _p(xp), _p(ref), _p(outlier), C.c_double(Rtri),
                                       C.c_double(mh_thresh), _p(xo), _p(Po), _p(oo)),
            "xivo_subfilter_batch",
        )
        return xo, Po.reshape(n, 3, 3), oo

    def oos_project(self, G, F, camera, gbc12, Xs, obs_pose, obs_sind, obs_xp):
        camera, gbc12 = _f64(camera), _f64(gbc12)
        Xs = _f64(Xs).reshape(-1, 3)
        nf = len(Xs)
        obs_pose = _f64(obs_pose).reshape(nf, -1, 12)
        k = obs_pose.shape[1]
        obs_sind, obs_xp = _i32(obs_sind).reshape(nf, k), _f64(obs_xp).reshape(nf, k, 2)
        N = 23 + 6 * G + 3 * F
        Hf, Hx, inn = np.zeros((nf, 2 * k, 3)), np.zeros((nf, 2 * k, N)), np.zeros((nf, 2 * k))
        Hp, ip = np.zeros((nf, 2 * k, N)), np.zeros((nf, 2 * k))
        _check(
            lib().xivo_oos_project(self._h, G, F, _p(camera), _p(gbc12), nf, k, _p(Xs), _p(obs_pose), _p(obs_sind), _p(obs_xp), _p(Hf),
                                   _p(Hx), _p(inn), _p(Hp), _p(ip)),
            "xivo_oos_project",
        )
        return Hf, Hx, inn, Hp[:, : 2 * k - 3], ip[:, : 2 * k - 3]

    def cov_edit(self, P, ops, blk=None):
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        ops = _i32(ops).reshape(-1, 4)
        blk = np.zeros((len(ops), 9)) if blk is None else _f64(blk).reshape(len(ops), 9)
        _check(lib().xivo_cov_edit(self._h, P.shape[0], _p(P), _p(ops), _p(blk), len(ops)), "xivo_cov_edit")
        return P

    def cov_propagate(self, P, Phi, Pmm):
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        _check(lib().xivo_cov_propagate(self._h, P.shape[0], _p(P), _p(_f64(Phi)), _p(_f64(Pmm))), "xivo_cov_propagate")
        return P

    def imu_cov_propagate(self, P, stages, g, qimu, qmodel, stages_per_step):
        P = np.array(P, dtype=np.float64, order="C", copy=True)
        stages = _f64(stages).reshape(-1, 16)
        _check(lib().xivo_imu_cov_propagate(self._h, P.shape[0], _p(P), len(stages), _p(stages), _p(_f64(g)), _p(_f64(qimu)), _p(_f64(qmodel)),
                                            int(stages_per_step)), "xivo_imu_cov_propagate")
        return P

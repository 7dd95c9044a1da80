"""Data formats either side of the hot path (SURVEY.md §8f row 4):

* ASL / EuRoC / TUM-VI sequence folders — `cam0/data.csv` + `imu0/data.csv` — merged into one time-ordered message
  list like DataLoader (src/loader.cpp:14-60): header line skipped, `#` lines skipped, image rows `ts,filename`, IMU rows
  `ts,wx,wy,wz,ax,ay,az`, stable ascending sort on the timestamp.
* the trajectory text the reference's `vio` app writes (src/app/vio.cpp:101-106: `ts_ns Tsb(3) Wsb(3)`, rotation as a
  rotation vector) and the TUM format its evaluation scripts read (`ts tx ty tz qx qy qz qw`, scripts/savers.py,
  scripts/tum_rgbd_benchmark_tools/).
* ATE / RPE of the TUM RGB-D benchmark tools (closed-form rigid alignment by SVD, RMSE of the translational residual;
  relative pose error over a fixed frame delta), the quantities behind "ATE within 1 % of the reference".

numpy only; host-side utilities, nothing here touches the GPU."""
from __future__ import annotations

import math
import os

import numpy as np


# ---------------------------------------------------------------- ASL loader
def _rows(csv_path):
    if not os.path.exists(csv_path):
        raise FileNotFoundError(f"failed to open data.csv @ {csv_path}")  # reference: LOG(FATAL)
    with open(csv_path) as f:
        f.readline()  # header
        for tok in f.read().split():  # `is >> line`: whitespace-separated tokens
            if tok and tok[0] != "#":
                yield tok.split(",")


def load_asl(image_dir: str, imu_dir: str | None = None):
    """[(kind, ts_ns, payload)] with kind 'img' -> image path, 'imu' -> (gyro[3], accel[3]); images are listed first and
    the sort is stable, so an image and an IMU sample with the same stamp keep that order (std::sort is not stable in
    the reference; ties are then implementation-defined)."""
    out = []
    for c in _rows(os.path.join(image_dir, "data.csv")):
        out.append(("img", int(c[0]), os.path.join(image_dir, "data", c[1])))
    if imu_dir is not None:
        for c in _rows(os.path.join(imu_dir, "data.csv")):
            v = [float(x) for x in c[1:7]]
            out.append(("imu", int(c[0]), (np.array(v[:3]), np.array(v[3:6]))))
    out.sort(key=lambda m: m[1])
    return out


def feed_rounds(msg_lists):
    """Schedules B message lists (the load_asl format) for pyxivo.Batch.feed / xivo_batch_feed: round r holds, per sequence, the r-th
    piece of its list, where a piece is the IMU messages up to and including the next frame (any kind other than 'imu'), and IMU
    messages after the last frame form a last piece.  So every round gives a sequence at most one frame, as the last message, and a
    sequence whose list is exhausted gets an empty piece.  -> [round][sequence] lists of messages; no rounds when every list is empty."""
    pieces = []
    for msgs in msg_lists:
        cur, out = [], []
        for m in msgs:
            cur.append(m)
            if m[0] != "imu":
                out.append(cur)
                cur = []
        if cur:
            out.append(cur)
        pieces.append(out)
    n = max((len(p) for p in pieces), default=0)
    return [[p[r] if r < len(p) else [] for p in pieces] for r in range(n)]


def write_asl(root: str, msgs, image_writer=None):
    """Writes a message list as an ASL folder (cam0/data.csv, cam0/data/<ts>.pgm|.ppm, imu0/data.csv).  Images are stored
    as binary PGM/PPM unless `image_writer(path, array)` is given."""
    cam, imu = os.path.join(root, "cam0"), os.path.join(root, "imu0")
    os.makedirs(os.path.join(cam, "data"), exist_ok=True)
    os.makedirs(imu, exist_ok=True)
    with open(os.path.join(cam, "data.csv"), "w") as fc, open(os.path.join(imu, "data.csv"), "w") as fi:
        fc.write("#timestamp [ns],filename\n")
        fi.write("#timestamp [ns],w_RS_S_x [rad s^-1],w_RS_S_y [rad s^-1],w_RS_S_z [rad s^-1],a_RS_S_x [m s^-2],a_RS_S_y [m s^-2],a_RS_S_z [m s^-2]\n")
        for kind, ts, p in msgs:
            if kind == "imu":
                fi.write("%d,%s\n" % (ts, ",".join(repr(float(x)) for x in (*p[0], *p[1]))))
            elif kind == "img":
                ext = "ppm" if p.ndim == 3 else "pgm"
                name = "%d.%s" % (ts, ext)
                path = os.path.join(cam, "data", name)
                if image_writer:
                    image_writer(path, p)
                else:
                    write_pnm(path, p)
                fc.write("%d,%s\n" % (ts, name))
    return cam, imu


def write_pnm(path, img):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    with open(path, "wb") as f:
        if img.ndim == 2:
            f.write(b"P5\n%d %d\n255\n" % (img.shape[1], img.shape[0]))
            f.write(img.tobytes())
        else:
            f.write(b"P6\n%d %d\n255\n" % (img.shape[1], img.shape[0]))
            f.write(img[:, :, ::-1].tobytes())  # stored RGB, handed out BGR like cv::imread


def read_pnm(path):
    """Binary PGM (-> H x W) / PPM (-> H x W x 3 in BGR order, like cv::imread)."""
    with open(path, "rb") as f:
        data = f.read()
    toks, pos = [], 0
    while len(toks) < 4:
        while data[pos : pos + 1].isspace():
            pos += 1
        if data[pos : pos + 1] == b"#":
            pos = data.index(b"\n", pos) + 1
            continue
        end = pos
        while not data[end : end + 1].isspace():
            end += 1
        toks.append(data[pos:end])
        pos = end
    pos += 1
    magic, w, h, mx = toks[0], int(toks[1]), int(toks[2]), int(toks[3])
    if mx != 255 or magic not in (b"P5", b"P6"):
        raise ValueError(f"unsupported PNM {magic!r} maxval {mx}")
    if magic == b"P5":
        return np.frombuffer(data, np.uint8, w * h, pos).reshape(h, w).copy()
    return np.frombuffer(data, np.uint8, w * h * 3, pos).reshape(h, w, 3)[:, :, ::-1].copy()


# ---------------------------------------------------------------- rotations
def so3_log(R):
    """Rotation vector of a rotation matrix (Sophus SO3::log as used at src/app/vio.cpp:103)."""
    c = max(-1.0, min(1.0, 0.5 * (np.trace(R) - 1.0)))
    th = math.acos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    if th < 1e-9:
        return 0.5 * w
    if math.pi - th < 1e-6:  # near pi: axis from the symmetric part
        A = 0.5 * (R + np.eye(3))
        k = int(np.argmax(np.diag(A)))
        ax = A[:, k] / math.sqrt(max(A[k, k], 1e-300))
        if np.dot(ax, w) < 0:
            ax = -ax
        return th * ax
    return th / (2.0 * math.sin(th)) * w


def so3_exp(w):
    th = float(np.linalg.norm(w))
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=float)
    if th < 1e-9:
        return np.eye(3) + K
    return np.eye(3) + math.sin(th) / th * K + (1 - math.cos(th)) / (th * th) * K @ K


def rot_to_quat_xyzw(R):
    """(qx, qy, qz, qw), qw >= 0 — the order of the TUM format."""
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        q = [(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s]
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(max(R[i, i] - R[j, j] - R[k, k] + 1.0, 0.0)) * 2
        q = [0.0, 0.0, 0.0, (R[k, j] - R[j, k]) / s]
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
    q = np.array(q)
    return -q if q[3] < 0 else q


def quat_xyzw_to_rot(q):
    x, y, z, w = np.asarray(q, dtype=float) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# ---------------------------------------------------------------- trajectory files
def write_vio_trajectory(path, stamps_ns, poses34):
    """The `vio` app's output (src/app/vio.cpp:101-106): `ts_ns Tx Ty Tz Wx Wy Wz` per processed message."""
    with open(path, "w") as f:
        for ts, g in zip(stamps_ns, poses34):
            g = np.asarray(g)
            w = so3_log(g[:, :3])
            f.write("%d %s %s\n" % (ts, " ".join("%.9g" % v for v in g[:, 3]), " ".join("%.9g" % v for v in w)))


def read_vio_trajectory(path):
    stamps, poses = [], []
    with open(path) as f:
        for line in f:
            v = line.split()
            if len(v) < 7:
                continue
            g = np.zeros((3, 4))
            g[:, :3] = so3_exp(np.array([float(x) for x in v[4:7]]))
            g[:, 3] = [float(x) for x in v[1:4]]
            stamps.append(int(v[0]))  # nanosecond stamps do not fit a double exactly
            poses.append(g)
    return np.array(stamps, dtype=np.int64), np.array(poses)


def write_tum_trajectory(path, stamps_s, poses34):
    """TUM RGB-D format: `timestamp tx ty tz qx qy qz qw` (seconds)."""
    with open(path, "w") as f:
        for ts, g in zip(stamps_s, poses34):
            g = np.asarray(g)
            q = rot_to_quat_xyzw(g[:, :3])
            f.write("%.9f %s %s\n" % (ts, " ".join("%.9g" % v for v in g[:, 3]), " ".join("%.9g" % v for v in q)))


def read_tum_trajectory(path):
    """-> (stamps [s], poses n x 3 x 4); `#` comment lines and ',' separators are accepted like associate.py does."""
    stamps, poses = [], []
    with open(path) as f:
        for line in f:
            line = line.replace(",", " ").strip()
            if not line or line[0] == "#":
                continue
            v = [float(x) for x in line.split()]
            if len(v) < 8:
                continue
            g = np.zeros((3, 4))
            g[:, :3] = quat_xyzw_to_rot(v[4:8])
            g[:, 3] = v[1:4]
            stamps.append(v[0])
            poses.append(g)
    return np.array(stamps), np.array(poses)


# ---------------------------------------------------------------- evaluation
def associate(stamps_a, stamps_b, max_difference=0.02, offset=0.0):
    """Greedy best-first matching of two stamp lists (associate.py): pairs (i, j) with |a_i - (b_j + offset)| < max."""
    a, b = np.asarray(stamps_a, dtype=float), np.asarray(stamps_b, dtype=float) + offset
    order = np.argsort(b, kind="stable")  # the stamp lists need not be sorted
    bs = b[order]
    cand = []
    for i, ta in enumerate(a):
        lo, hi = np.searchsorted(bs, ta - max_difference, "left"), np.searchsorted(bs, ta + max_difference, "right")
        for k in range(lo, hi):
            d = abs(ta - bs[k])
            if d < max_difference:
                cand.append((d, ta, bs[k], i, int(order[k])))
    cand.sort()
    cand = [(d, i, j) for d, _, _, i, j in cand]
    used_a, used_b, out = set(), set(), []
    for _, i, j in cand:
        if i not in used_a and j not in used_b:
            used_a.add(i)
            used_b.add(j)
            out.append((i, j))
    out.sort()
    return out


def align_rigid(model, data):
    """Closed-form rotation + translation (Horn / Kabsch by SVD, evaluate_ate.py:51-83) mapping `model` (3 x n) onto
    `data` (3 x n).  Returns R, t and the per-point translational residual."""
    model, data = np.asarray(model, dtype=float), np.asarray(data, dtype=float)
    mc, dc = model.mean(1, keepdims=True), data.mean(1, keepdims=True)
    W = (model - mc) @ (data - dc).T
    U, _, Vt = np.linalg.svd(W.T)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    t = dc - R @ mc
    err = np.linalg.norm(R @ model + t - data, axis=0)
    return R, t, err


def ate(stamps_gt, pos_gt, stamps_est, pos_est, max_difference=0.02, offset=0.0, scale=1.0):
    """Absolute trajectory error: RMSE [m] of the translational residual after rigid alignment of the estimate onto the
    ground truth (evaluate_ate.py).  pos_*: n x 3.  Returns dict(rmse, mean, median, max, pairs)."""
    m = associate(stamps_gt, stamps_est, max_difference, offset)
    if len(m) < 3:
        raise ValueError("Couldn't find matching timestamp pairs between groundtruth and estimated trajectory")
    gt = np.asarray(pos_gt, dtype=float)[[i for i, _ in m]].T
    est = np.asarray(pos_est, dtype=float)[[j for _, j in m]].T * scale
    _, _, err = align_rigid(est, gt)
    return dict(rmse=float(np.sqrt(np.mean(err * err))), mean=float(err.mean()), median=float(np.median(err)), max=float(err.max()), pairs=len(m))


def _h(g):
    T = np.eye(4)
    T[:3, :4] = g
    return T


def rpe(stamps_gt, poses_gt, stamps_est, poses_est, delta=1.0, max_difference=0.02):
    """Relative pose error over a time delta [s] (evaluate_rpe.py with --fixed_delta, delta_unit 's'): for every estimated
    pose and the one `delta` later, compare the relative motion with the ground truth's.  Returns RMSE of the translational
    [m] and rotational [rad] parts."""
    m = associate(stamps_est, stamps_gt, max_difference)
    if len(m) < 2:
        raise ValueError("not enough associated poses")
    se = np.asarray(stamps_est, dtype=float)
    idx_e = [i for i, _ in m]
    gt_of = {i: j for i, j in m}
    te, re_ = [], []
    for i in idx_e:
        k = int(np.searchsorted(se, se[i] + delta - 1e-9))
        while k < len(se) and k not in gt_of:
            k += 1
        if k >= len(se) or abs(se[k] - se[i] - delta) > max_difference + 0.5 * delta:
            continue
        dE = np.linalg.inv(_h(poses_est[i])) @ _h(poses_est[k])
        dG = np.linalg.inv(_h(poses_gt[gt_of[i]])) @ _h(poses_gt[gt_of[k]])
        E = np.linalg.inv(dG) @ dE
        te.append(np.linalg.norm(E[:3, 3]))
        re_.append(math.acos(max(-1.0, min(1.0, 0.5 * (np.trace(E[:3, :3]) - 1.0)))))
    if not te:
        raise ValueError("no pose pairs at the requested delta")
    te, re_ = np.array(te), np.array(re_)
    return dict(trans_rmse=float(np.sqrt(np.mean(te * te))), rot_rmse=float(np.sqrt(np.mean(re_ * re_))), pairs=len(te))

"""numpy restatement of cv::normalize(image, img_, 0, 255, cv::NORM_MINMAX) on an 8-bit frame, which the reference's tracker runs on
every frame when tracker_cfg.normalize is set (src/tracker.cpp:343-344 in UpdateMatch, :465-467 in UpdateLK).

OpenCV takes the minimum and maximum over all channels together and then calls convertTo with
    scale = 255 * (max - min > DBL_EPSILON ? 1 / (max - min) : 0),  shift = 0 - min * scale      (double)
rounded to float, and out = saturate_u8(rint(fmaf(v, scale, shift))): one rounding of the fused multiply-add in float32, then round half
to even.  Here the fused form is float64(v) * float64(scale) + float64(shift), which is exact in double for 8-bit v, rounded once to
float32.  tests/test_normalize_logic.py checks this against cv2 over every (min, max, v)."""
import numpy as np


def scale_shift(lo, hi):
    """(scale, shift) as the float32 pair convertTo applies for a frame whose extremes are lo <= hi."""
    lo, hi = float(lo), float(hi)
    scale = 255.0 * (1.0 / (hi - lo) if hi - lo > np.finfo(np.float64).eps else 0.0)
    shift = 0.0 - lo * scale
    return np.float32(scale), np.float32(shift)


def lut(lo, hi):
    """The 256-entry output table of a frame whose extremes are lo <= hi."""
    scale, shift = scale_shift(lo, hi)
    v = np.arange(256, dtype=np.float64)
    fused = (v * np.float64(scale) + np.float64(shift)).astype(np.float32)
    return np.clip(np.rint(fused), 0, 255).astype(np.uint8)


def normalize_minmax(img):
    """cv2.normalize(img, None, 0, 255, cv2.NORM_MINMAX) of a uint8 frame of any shape (grey or interleaved channels)."""
    img = np.asarray(img, dtype=np.uint8)
    return lut(int(img.min()), int(img.max()))[img]


# The frames of tests/golden/normalize_cv2.npz: both channel counts at a 16-byte-multiple and an odd geometry, each as a low-contrast
# texture, a full-range frame, a frame of two adjacent values and a constant frame.
GOLDEN_CASES = [(rows, cols, cn, kind) for rows, cols in ((480, 640), (481, 643)) for cn in (1, 3) for kind in ("low", "full", "two", "const")]


def golden_frame(rows, cols, cn, kind):
    seed = rows * 7 + cols * 3 + cn * 11 + ("low", "full", "two", "const").index(kind)
    rng = np.random.default_rng(seed)
    shape = (rows, cols) if cn == 1 else (rows, cols, cn)
    if kind == "low":
        y, x = np.mgrid[0:rows, 0:cols]
        base = 55 + (x * 37 + y * 61) % 101  # integer arithmetic only: the frame is the same on every machine
        img = (base if cn == 1 else base[..., None]) + rng.integers(-15, 16, shape)
        return np.clip(img, 40, 170).astype(np.uint8)
    if kind == "full":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == "two":
        return (100 + rng.integers(0, 2, shape)).astype(np.uint8)
    return np.full(shape, 77, np.uint8)

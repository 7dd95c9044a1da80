"""Generates tests/golden/normalize_cv2.npz: what cv2.normalize(f, None, 0, 255, cv2.NORM_MINMAX) returns for the seeded frames of
tests/normalize_oracle.py (GOLDEN_CASES).  Needs cv2 (written with OpenCV 4.13); the tests only read the npz.  The frames are not
stored: each case keeps the SHA-256 of its input (so that a change in how the frames are generated is told apart from a change in
the arithmetic), of cv2's output, and cv2's extremes of the input.

usage: python tests/golden/make_golden_normalize.py"""
import hashlib
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import normalize_oracle as O  # noqa: E402


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def main():
    names, ins, outs, ext = [], [], [], []
    for case in O.GOLDEN_CASES:
        img = O.golden_frame(*case)
        out = cv2.normalize(img, None, 0, 255, cv2.NORM_MINMAX)
        assert out.dtype == np.uint8 and out.shape == img.shape
        lo, hi, _, _ = cv2.minMaxLoc(img.reshape(img.shape[0], -1))
        names.append("%dx%dx%d_%s" % case)
        ins.append(sha(img))
        outs.append(sha(out))
        ext.append((int(lo), int(hi)))
    np.savez_compressed(os.path.join(HERE, "normalize_cv2.npz"), names=np.array(names), in_sha=np.stack(ins), out_sha=np.stack(outs),
                        extremes=np.array(ext, np.int32), cv2_version=np.array(cv2.__version__))


if __name__ == "__main__":
    main()

"""Generates tests/golden/png_imread.npz: small PNG files and what cv2.imread returns for them (IMREAD_COLOR for every file,
IMREAD_GRAYSCALE for the grey and grey + alpha ones).  Needs cv2 (written with OpenCV 4.13); the tests only read the npz.

Files: every accepted colour type (grey, RGB, grey + alpha, RGBA) at 8 and 16 bits written by cv2.imencode, every filter type forced
on every row by the stdlib encoder of tests/png_oracle.py, zlib levels / strategies, a split IDAT and one file with gAMA and tRNS chunks.

usage: python tests/golden/make_golden_png.py"""
import os
import sys
import tempfile
import zlib

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import png_oracle as O  # noqa: E402


def textured(rows, cols, ch, bits, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:rows, 0:cols]
    top = (1 << bits) - 1
    base = (np.sin(x / 3.0 + seed) * np.cos(y / 5.0) * 0.4 + 0.5) * top
    img = np.stack([base * (0.6 + 0.2 * c) + rng.integers(0, top // 8 + 1, (rows, cols)) for c in range(ch)], axis=2)
    return np.clip(img, 0, top).astype(np.uint16 if bits == 16 else np.uint8)


def main():
    files = []  # (name, png bytes)
    # cv2.imencode: cv2 writes grey, BGR and BGRA (stored as grey, RGB, RGBA) at 8 and 16 bits
    for bits in (8, 16):
        for ch, name in ((1, "grey"), (3, "rgb"), (4, "rgba")):
            img = textured(40 + ch, 52 - ch, ch, bits, seed=bits + ch)
            ok, buf = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, 2 * ch + 1])
            assert ok
            files.append((f"cv2_{name}{bits}", bytes(buf)))
    # the stdlib encoder: grey + alpha (cv2 does not write it), every filter type on every row, levels and strategies
    for bits in (8, 16):
        files.append((f"stdlib_greyalpha{bits}", O.encode(textured(33, 29, 2, bits, 7), 4, bits, filters=None, seed=bits)))
    for ft in range(5):
        ct, bits = [(0, 8), (2, 8), (6, 16), (4, 8), (0, 16)][ft]
        img = textured(24 + ft, 31, O.CHANNELS[ct], bits, 20 + ft)
        files.append((f"stdlib_filter{ft}_ct{ct}_{bits}", O.encode(img, ct, bits, filters=ft, level=[9, 1, 6, 0, 9][ft])))
    files.append(("stdlib_rle_split", O.encode(textured(64, 64, 1, 8, 30), 0, 8, level=6, strategy=zlib.Z_RLE, idat_size=97)))
    files.append(("stdlib_fixed_rgb16", O.encode(textured(17, 33, 3, 16, 31), 2, 16, level=6, strategy=zlib.Z_FIXED)))
    files.append(("stdlib_gama_trns", O.encode(textured(20, 20, 3, 8, 32), 2, 8, ancillary=[(b"gAMA", (45455).to_bytes(4, "big")),
                                                                                        (b"tRNS", bytes([0, 10, 0, 20, 0, 30]))])))
    out = {"names": np.array([n for n, _ in files])}
    with tempfile.TemporaryDirectory() as td:
        for i, (name, data) in enumerate(files):
            path = os.path.join(td, name + ".png")
            with open(path, "wb") as f:
                f.write(data)
            out[f"png_{i}"] = np.frombuffer(data, np.uint8)
            out[f"color_{i}"] = cv2.imread(path)
            if O.CHANNELS[O.info(data)[2]] <= 2:
                out[f"gray_{i}"] = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
    dst = os.path.join(HERE, "png_imread.npz")
    np.savez_compressed(dst, **out)
    print(dst, len(files), "files", os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()

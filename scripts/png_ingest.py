"""PNG ingest measurements on the GPU (DESIGN §6, "PNG ingest"); prints one JSON line (and writes it to --out when given).

  (a) device time of png_inflate_kernel and png_unfilter_kernel from the in-library profiler, for 1024 EuRoC-size (752 x 480 grey8) and
      1024 TUM-VI-size (512 x 512 grey16) frames per xivo_decode_png call: frames/s and GB/s of decoded output
  (b) host µs per sequence-frame inside xivo_batch_visual_meas_png, from its host profile scopes (chunk walk, packing, issue, wait for
      the decode status, whole call), and the host time per frame of the kernel-level xivo_decode_png outside its kernels
  (c) end-to-end frames/s of one 128-sequence Batch on 752 x 480 grey frames: Batch.visual_meas_png (decode into the frame ring)
      against Batch.visual_meas (arrays), alternated, 3 repeats each
  (d) single-thread cv2.imdecode per frame on the same host, if cv2 is importable
The card's name and power limit are read in the same call.

usage: python scripts/png_ingest.py [--frames 1024] [--seqs 128] [--steps 30] [--out result.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import png_oracle as O  # noqa: E402
from xivo_b200 import capi, pyxivo, sim  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def frames(n, rows, cols, bits, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:rows, 0:cols]
    top = (1 << bits) - 1
    out = []
    for k in range(8):  # 8 distinct textured frames, repeated: the compressed size is that of a camera frame, not of noise
        base = (np.sin(x / (5.0 + k) + k) * np.cos(y / 7.0) * 0.4 + 0.5) * top + rng.normal(0, top / 40, (rows, cols))
        img = np.clip(base, 0, top).astype(np.uint16 if bits == 16 else np.uint8)
        out.append(O.encode(img, 0, bits, level=6, seed=k))
    return [out[i % 8] for i in range(n)]


def report(L):
    buf = C.create_string_buffer(1 << 16)
    L.xivo_profile_report(buf, len(buf))
    return json.loads(buf.value.decode())


def device_time(ctx, L, pngs, reps=5):
    ctx.decode_png(pngs[:8])  # warm-up
    L.xivo_profile_reset()
    L.xivo_profile_enable(1)
    for _ in range(reps):
        ctx.decode_png(pngs)
    L.xivo_profile_enable(0)
    r = report(L)
    ms = {k: r[k]["ms"] / r[k]["calls"] for k in ("png_inflate_kernel", "png_unfilter_kernel")}
    t0 = time.perf_counter()
    for _ in range(reps):
        ctx.decode_png(pngs)
    call_ms = (time.perf_counter() - t0) / reps * 1e3
    return ms, call_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = capi.lib()
    ctx = capi.Context(0)
    res = {"card": card()}
    for name, (rows, cols, bits) in {"euroc_752x480_grey8": (480, 752, 8), "tumvi_512x512_grey16": (512, 512, 16)}.items():
        pngs = frames(a.frames, rows, cols, bits, 1)
        ms, call_ms = device_time(ctx, L, pngs)
        dev = ms["png_inflate_kernel"] + ms["png_unfilter_kernel"]
        out_bytes = a.frames * rows * cols * 3
        res[name] = {
            "frames": a.frames, "png_bytes_per_frame": int(np.mean([len(p) for p in pngs])),
            "inflate_ms": round(ms["png_inflate_kernel"], 3), "unfilter_ms": round(ms["png_unfilter_kernel"], 3),
            "device_frames_per_s": round(a.frames / dev * 1e3), "device_GBps_decoded_bgr": round(out_bytes / dev / 1e6, 2),
            "call_ms": round(call_ms, 2), "host_us_per_frame_outside_kernels": round((call_ms - dev) / a.frames * 1e3, 2),
        }
        try:
            import cv2

            t0 = time.perf_counter()
            for p in pngs[:64]:
                cv2.imdecode(np.frombuffer(p, np.uint8), cv2.IMREAD_COLOR)
            res[name]["cv2_imdecode_ms_per_frame_1_thread"] = round((time.perf_counter() - t0) / 64 * 1e3, 3)
        except ImportError:
            res[name]["cv2_imdecode_ms_per_frame_1_thread"] = "not measured (no cv2)"
    # (c) end to end: one 128-sequence batch, PNG ingest vs arrays, alternated
    cfg = sim.load_cfg(os.path.join(ROOT, "xivo_b200", "cfg", "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=480, cols=752, cx=376, cy=240)
    msgs, _ = sim.image_stream(cfg, duration=a.steps * 0.04 + 0.05, seed=2, fast=True)
    n = a.seqs
    runs = {"arrays": [], "png": []}
    for rep in range(3):
        for mode in ("arrays", "png"):
            b = pyxivo.Batch(cfg, n_seq=n, max_groups=15, max_features=30, ctx=ctx)
            cache = {}
            nf, el = 0, 0.0
            for kind, ts, p in msgs:
                if kind == "imu":
                    b.inertial_meas(ts, p[0], p[1])
                    continue
                if mode == "png" and ts not in cache:
                    cache[ts] = O.encode(p, 0, 8, level=6)
                t0 = time.perf_counter()
                if mode == "png":
                    b.visual_meas_png(ts, [cache[ts]] * n, channels=1)
                else:
                    b.visual_meas(ts, [p] * n)
                b.now(0)
                el += time.perf_counter() - t0
                nf += 1
            b.close()
            runs[mode].append(round(nf * n / el))
    res["batch128_e2e_frames_per_s"] = runs
    # (b) host scopes of the batch PNG call, in a separate run (profiling slows the host)
    b = pyxivo.Batch(cfg, n_seq=n, max_groups=15, max_features=30, ctx=ctx)
    nf = 0
    for kind, ts, p in msgs:
        if kind == "imu":
            b.inertial_meas(ts, p[0], p[1])
            continue
        if nf == 3:
            L.xivo_profile_reset()
            L.xivo_profile_enable(3)
        b.visual_meas_png(ts, [cache.get(ts) or O.encode(p, 0, 8, level=6)] * n, channels=1)
        nf += 1
    L.xivo_profile_enable(0)
    b.close()
    r = report(L)
    calls = max(nf - 3, 1)
    res["batch_png_host_us_per_seq_frame"] = {k[5:]: round(r[k]["ms"] / calls / n * 1e3, 3) for k in r
                                              if k.startswith("host:") and (k[5:].startswith("png_") or k[5:] in ("wait_png", "visual_meas_png_total"))}
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

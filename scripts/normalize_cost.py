#!/usr/bin/env python
"""Cost of tracker_cfg.normalize (cv::normalize NORM_MINMAX of every frame in its ring slot, launch_normalize_minmax).

  1. Device time of the two normalisation kernels for one frame-batch of --seqs frames at 640x480 grey, 640x480 BGR and 1280x1024 grey:
     the in-library profiler's CUDA-event pair around the two launches (scope "normalize_minmax") over --reps calls of
     xivo_normalize_minmax, whose frames lie back to back in device memory as in the frame ring.  Bytes moved per frame-batch: the
     minimum / maximum pass reads every frame once, the remap reads and writes it once (3 x frame bytes; the partials are 8 bytes per CTA).
     Achieved bandwidth = bytes / time, and its share of the H100 SXM data-sheet 3.35 TB/s.
  2. frames/s of two handles of bench.py's workload (--config 1: 640x480 grey, frames resident in device memory, one xivo_batch_step of
     8 IMU samples + 1 frame per step), one with normalize on and one with it off, driven with the same frames in alternating blocks
     of --steps steps.
Prints one JSON line with the card name and its power limit.

  python scripts/normalize_cost.py [--seqs 128] [--reps 200] [--steps 30] [--rounds 4]
"""
from __future__ import annotations

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

import bench  # noqa: E402  (the workload constants and stream tables of the benchmark)

HBM_TBS = 3.35  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, plim, clk = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=plim, sm_clock_max=clk)
    except Exception as e:  # noqa: BLE001
        return dict(name=None, error=str(e))


def profile_report(L):
    buf = C.create_string_buffer(1 << 20)
    n = L.xivo_profile_report(buf, len(buf))
    if n < 0:
        raise RuntimeError(L.xivo_last_error().decode())
    return json.loads(buf.value.decode())


def kernel_times(ctx, L, seqs, reps):
    out = {}
    rng = np.random.default_rng(0)
    for name, shape in (("640x480x1", (480, 640)), ("640x480x3", (480, 640, 3)), ("1280x1024x1", (1024, 1280))):
        frames = np.ascontiguousarray(rng.integers(30, 200, (seqs,) + shape).astype(np.uint8))
        cn = 1 if len(shape) == 2 else 3
        for _ in range(5):  # warm-up: module load, allocations
            ctx.normalize_minmax(frames, channels=cn)
        L.xivo_profile_reset()
        L.xivo_profile_enable(1)
        for _ in range(reps):
            ctx.normalize_minmax(frames, channels=cn)
        L.xivo_profile_enable(0)
        e = profile_report(L)["normalize_minmax"]
        us = 1e3 * e["ms"] / e["calls"]
        moved = 3 * frames.nbytes
        out[name] = dict(calls=int(e["calls"]), us_per_frame_batch=round(us, 2), bytes_per_frame_batch=int(moved),
                         achieved_TBs=round(moved / (us * 1e-6) / 1e12, 3), share_of_hbm_peak=round(moved / (us * 1e-6) / 1e12 / HBM_TBS, 3))
    return out


def throughput(args):
    import torch

    from xivo_b200 import capi, pyxivo

    bench.select_config(1)
    cfg = bench.load_cfg()
    B, S0 = args.seqs, min(args.streams, args.seqs)
    bases = bench.make_base_streams(cfg, S0, 1, max(1, min(S0, os.cpu_count() or 1)))
    NFB = bench.REST_FRAMES + bench.PERIOD_FRAMES
    dev = torch.from_numpy(np.stack([b[0][:NFB] for b in bases])).cuda()
    fbytes = bench.ROWS * bench.COLS
    base_g, base_a = np.stack([b[1] for b in bases]), np.stack([b[2] for b in bases])
    n_frames = args.preroll + 2 * args.rounds * args.steps + 8
    fidx, iidx, base = bench.stream_tables(B, S0, n_frames)
    L = capi.lib()
    cols = np.arange(B)
    VP = C.c_void_p
    handles = {}
    for arm, on in (("normalize_off", False), ("normalize_on", True)):
        c = json.loads(json.dumps(cfg))
        c["tracker_cfg"]["normalize"] = on
        handles[arm] = [pyxivo.Batch(c, n_seq=B, max_groups=bench.G, max_features=bench.F), 0]

    def step(arm):
        h = handles[arm]
        g = h[1]
        j = 8 * g + np.arange(8)[:, None] + np.zeros(B, np.int64)[None, :]
        its = np.ascontiguousarray(j.astype(np.uint64) * np.uint64(bench.FRAME_NS // 8))
        gy = np.ascontiguousarray(base_g[base[None, :], iidx[j, cols[None, :]]])
        ac = np.ascontiguousarray(base_a[base[None, :], iidx[j, cols[None, :]]])
        fts = np.full(B, np.uint64(g) * np.uint64(bench.FRAME_NS), np.uint64)
        ptr = np.ascontiguousarray(np.uint64(dev.data_ptr()) + (base.astype(np.uint64) * np.uint64(NFB) + fidx[g, cols].astype(np.uint64)) * np.uint64(fbytes))
        rc = L.xivo_batch_step(h[0]._h, 8, VP(its.ctypes.data), VP(gy.ctypes.data), VP(ac.ctypes.data), VP(fts.ctypes.data), VP(ptr.ctypes.data),
                               bench.ROWS, bench.COLS, 1, 1)
        if rc != 0:
            raise RuntimeError(L.xivo_last_error().decode())
        h[1] = g + 1

    for arm in handles:
        for _ in range(args.preroll):
            step(arm)
    torch.cuda.synchronize()
    fps = {arm: [] for arm in handles}
    for rnd in range(args.rounds):
        for arm in (handles if rnd % 2 == 0 else list(handles)[::-1]):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step(arm)
            torch.cuda.synchronize()
            fps[arm].append(round(B * args.steps / (time.perf_counter() - t0), 1))
    errors = {arm: int(sum(h[0].counters(s)["error"] != 0 for s in range(B))) for arm, h in handles.items()}
    for h in handles.values():
        h[0].close()
    return dict(fps=fps, fps_ratio_median=round(float(np.median(fps["normalize_on"]) / np.median(fps["normalize_off"])), 4),
                sequences_with_error=errors)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--reps", type=int, default=200, help="timed xivo_normalize_minmax calls per geometry")
    ap.add_argument("--streams", type=int, default=8, help="rendered base streams the sequences replay")
    ap.add_argument("--preroll", type=int, default=40)
    ap.add_argument("--steps", type=int, default=30, help="steps per throughput block")
    ap.add_argument("--rounds", type=int, default=4, help="alternating (off, on) block pairs")
    args = ap.parse_args()
    from xivo_b200 import capi

    L = capi.lib()
    ctx = capi.Context(0)
    out = dict(what="cost of tracker_cfg.normalize", card=card(), seqs=args.seqs, kernels=kernel_times(ctx, L, args.seqs, args.reps))
    ctx.close()
    out["throughput_bench_config_1"] = throughput(args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Cost of restarting one sequence of a batch handle (xivo_batch_reset_sequence) on the benchmark workload.

One handle of --seqs sequences of bench.py's workload (--config 1: 640x480, 150 features, G=4, F=14, frames resident in device memory,
one xivo_batch_step of 8 IMU samples + 1 frame per step).  After a pre-roll that brings every sequence to its steady state it measures
  1. the time of one reset_sequence call: a host clock around the call (`call_us`) and around the call followed by a synchronise of the
     device (`call_sync_us`), one reset between two steps, over the sequences in turn;
  2. frames/s of the handle with one reset every step against no resets, in alternating blocks of --steps steps.
A reset sequence replays its base stream from the start (rest phase, t = 0), as a new stream would.  Prints one JSON line with the card
name and its power limit.

  python scripts/reset_cost.py [--seqs 128] [--steps 30] [--rounds 3] [--resets 64]
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, plim, clk = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=plim, sm_clock_max=clk)
    except Exception as e:  # noqa: BLE001
        return dict(name=None, error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=1, choices=sorted(bench.CONFIGS))
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--streams", type=int, default=8, help="rendered base streams the sequences replay")
    ap.add_argument("--preroll", type=int, default=60)
    ap.add_argument("--steps", type=int, default=30, help="steps per throughput block")
    ap.add_argument("--rounds", type=int, default=3, help="alternating (no reset, reset every step) block pairs")
    ap.add_argument("--resets", type=int, default=64, help="timed single reset calls")
    args = ap.parse_args()
    bench.select_config(args.config)
    cfg = bench.load_cfg()
    B, S0 = args.seqs, min(args.streams, args.seqs)
    bases = bench.make_base_streams(cfg, S0, 1, max(1, min(S0, os.cpu_count() or 1)))

    import torch

    from xivo_b200 import capi, pyxivo

    NFB = bench.REST_FRAMES + bench.PERIOD_FRAMES
    dev = torch.from_numpy(np.stack([b[0][:NFB] for b in bases])).cuda()  # (S0, NFB, rows, cols)
    fbytes = bench.ROWS * bench.COLS
    base_g = np.stack([b[1] for b in bases])
    base_a = np.stack([b[2] for b in bases])
    n_local = args.preroll + args.resets + 2 * args.rounds * args.steps + 8  # no sequence gets further than this many frames from its start
    fidx, iidx, base = bench.stream_tables(B, S0, n_local)
    batch = pyxivo.Batch(cfg, n_seq=B, max_groups=bench.G, max_features=bench.F)
    L = capi.lib()
    start = np.zeros(B, np.int64)  # global step at which each sequence (re)started its stream
    cols = np.arange(B)
    VP = C.c_void_p

    def step(g):
        loc = g - start  # per-sequence frame index since its (re)start
        j = 8 * loc[None, :] + np.arange(8)[:, None]  # (8, B)
        its = np.ascontiguousarray(j.astype(np.uint64) * np.uint64(bench.FRAME_NS // 8))
        gy = np.ascontiguousarray(base_g[base[None, :], iidx[j, cols[None, :]]])
        ac = np.ascontiguousarray(base_a[base[None, :], iidx[j, cols[None, :]]])
        fts = np.ascontiguousarray(loc.astype(np.uint64) * np.uint64(bench.FRAME_NS))
        ptr = np.ascontiguousarray(np.uint64(dev.data_ptr()) + (base.astype(np.uint64) * np.uint64(NFB) + fidx[loc, cols].astype(np.uint64)) * np.uint64(fbytes))
        rc = L.xivo_batch_step(batch._h, 8, VP(its.ctypes.data), VP(gy.ctypes.data), VP(ac.ctypes.data), VP(fts.ctypes.data), VP(ptr.ctypes.data),
                               bench.ROWS, bench.COLS, 1, 1)
        if rc != 0:
            raise RuntimeError(L.xivo_last_error().decode())

    def reset(seq, g):
        batch.reset_sequence(seq)
        start[seq] = g

    g = 0
    for _ in range(args.preroll):
        step(g)
        g += 1
    torch.cuda.synchronize()
    # ---- 1. one reset call
    call_us, sync_us = [], []
    for r in range(args.resets):
        step(g)
        g += 1
        torch.cuda.synchronize()
        seq = (r * 37) % B
        t0 = time.perf_counter()
        reset(seq, g)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        call_us.append((t1 - t0) * 1e6)
        sync_us.append((t2 - t0) * 1e6)
    # ---- 2. throughput with one reset every step against none, alternating blocks
    fps = {"none": [], "every_step": []}
    for rnd in range(args.rounds):
        for arm in ("none", "every_step"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for k in range(args.steps):
                if arm == "every_step":
                    reset((rnd * args.steps + k) * 53 % B, g)
                step(g)
                g += 1
            torch.cuda.synchronize()
            fps[arm].append(B * args.steps / (time.perf_counter() - t0))
    errors = sum(batch.counters(s)["error"] != 0 for s in range(B))
    q = lambda v, p: float(np.percentile(v, p))
    out = dict(
        what="xivo_batch_reset_sequence cost on bench --config %d" % args.config,
        card=card(), seqs=B, steps_per_block=args.steps, rounds=args.rounds, resets_timed=args.resets,
        call_us=dict(median=q(call_us, 50), p90=q(call_us, 90), min=min(call_us), max=max(call_us)),
        call_sync_us=dict(median=q(sync_us, 50), p90=q(sync_us, 90), min=min(sync_us), max=max(sync_us)),
        fps_no_reset=[round(x, 1) for x in fps["none"]], fps_reset_every_step=[round(x, 1) for x in fps["every_step"]],
        fps_ratio_median=float(np.median(fps["every_step"]) / np.median(fps["none"])),
        sequences_with_error=int(errors),
    )
    print(json.dumps(out))
    batch.close()


if __name__ == "__main__":
    main()

"""Throughput of per-sequence feeding (xivo_batch_feed) on recorded-like sequences whose rates differ, against the same frames fed
lock-step (xivo_batch_step).

128 synthetic 640x480 image sequences run in one handle: IMU at 200 or 400 Hz, frames at 20, 25 or 30 Hz, start times staggered.
They are replayed by time: call c gives every sequence its messages stamped in (c * tick, (c + 1) * tick], so with a tick no longer
than the shortest frame period a call carries at most one frame per sequence and only the sequences with a frame in that window take
part in the frame-batch.  A frame-batch is one pass of the visual pipeline over the frames the message heaps release together
(the "visual_begin" host scope); raggedness splits the frames of a call into more, smaller frame-batches.  The same frames then go
through xivo_batch_step lock-step (8 IMU samples at 200 Hz and one frame per sequence per call).
Prints one JSON line per schedule.  Needs a GPU.

    python scripts/feed_bench.py [--seqs 128] [--seconds 10] [--tick-ms 33] [--warmup-s 1.5]
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

IMU_DT = (0.005, 0.0025)
FRAME_DT = (0.05, 0.04, 1 / 30)
N_BASE = 12  # rendered base streams: every (IMU rate, frame rate) pair, two seeds each


def _render(args):
    cfg, seed, seconds, imu_dt, frame_dt = args
    from xivo_b200 import sim

    traj = sim.periodic_trajectory(4.0, amp_scale=0.85 + 0.1 * (seed % 4))
    msgs, _ = sim.image_stream(cfg, duration=seconds, imu_dt=imu_dt, vision_dt=frame_dt, seed=seed, fast=True, traj=traj, rest_accel_is_gravity=True)
    return msgs


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the number is still reported, with what is known about the card
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqs", type=int, default=128)
    ap.add_argument("--seconds", type=float, default=10.0, help="length of the longest sequence [s]")
    ap.add_argument("--tick-ms", type=float, default=33.0, help="replay window per call; at most the shortest frame period")
    ap.add_argument("--stagger-ms", type=float, default=37.0, help="start offset between sequences of one base stream")
    ap.add_argument("--warmup-s", type=float, default=1.5, help="replay time excluded from the timed window")
    ap.add_argument("--groups", type=int, default=15)
    ap.add_argument("--features", type=int, default=30)
    args = ap.parse_args()
    from xivo_b200 import sim

    cfg = sim.load_cfg(os.path.join(ROOT, "xivo_b200", "cfg", "vio_640x480.json"))
    B = args.seqs
    t0 = time.time()
    import multiprocessing as mp

    jobs = [(cfg, 200 + b, args.seconds, IMU_DT[b % 2], FRAME_DT[(b // 2) % 3]) for b in range(N_BASE)]
    with mp.get_context("fork").Pool(min(N_BASE, os.cpu_count() or 1)) as pool:
        bases = pool.map(_render, jobs, chunksize=1)
    print(f"rendered {N_BASE} base streams in {time.time() - t0:.1f}s", file=sys.stderr)

    import torch

    from xivo_b200 import capi, pyxivo

    # every frame once, in a pinned pool that all calls read from
    frames = [[p for k, _, p in m if k == "img"] for m in bases]
    nf = sum(len(f) for f in frames)
    pool = torch.empty((nf, 480, 640), dtype=torch.uint8).pin_memory()
    pool_np = pool.numpy()
    fptr, o = [], 0
    for f in frames:
        fptr.append([])
        for img in f:
            pool_np[o] = img
            fptr[-1].append(pool_np[o].ctypes.data)
            o += 1

    # sequence s replays base s % N_BASE, shifted by its start offset, and stops at args.seconds
    end_ns = int(args.seconds * 1e9)
    tick = int(args.tick_ms * 1e6)
    seq_msgs = []
    for s in range(B):
        b = s % N_BASE
        off = int((s // N_BASE) * args.stagger_ms * 1e6)
        fi, out = 0, []
        for kind, ts, p in bases[b]:
            if kind == "img":
                fi += 1
            if ts + off < end_ns:
                out.append((kind, ts + off, p if kind == "imu" else (b, fi - 1)))
        seq_msgs.append(out)
    n_calls = -(-end_ns // tick)
    calls = []  # per call: n_imu, imu_ts, gyro, accel, frame_ts, frame pointers, frames in the call
    pos = [0] * B
    for c in range(n_calls):
        hi = (c + 1) * tick
        n_imu = np.zeros(B, np.int32)
        its, g, a = [], [], []
        fts = np.zeros(B, np.uint64)
        ptrs = (C.c_void_p * B)()
        nfr = 0
        for s in range(B):
            m = seq_msgs[s]
            while pos[s] < len(m) and m[pos[s]][1] <= hi:
                kind, ts, p = m[pos[s]]
                pos[s] += 1
                if kind == "imu":
                    n_imu[s] += 1
                    its.append(ts)
                    g.append(p[0])
                    a.append(p[1])
                else:
                    assert not ptrs[s], "two frames of one sequence in one call: use a shorter --tick-ms"
                    fts[s] = ts
                    ptrs[s] = fptr[p[0]][p[1]]
                    nfr += 1
        calls.append((n_imu, np.array(its, np.uint64), np.array(g, np.float64).reshape(-1, 3), np.array(a, np.float64).reshape(-1, 3), fts, ptrs, nfr))
    warm = int(args.warmup_s * 1e9) // tick
    L = capi.lib()
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    info = gpu_info()

    def run_feed(profile):
        b = pyxivo.Batch(cfg, n_seq=B, max_groups=args.groups, max_features=args.features)
        if profile:
            L.xivo_profile_reset()
            L.xivo_profile_enable(3)  # host scopes only: counts the frame-batches
        t = None
        for c, (n_imu, its, g, a, fts, ptrs, _) in enumerate(calls):
            if c == warm:
                torch.cuda.synchronize()
                t = time.perf_counter()
            capi._check(L.xivo_batch_feed(b._h, P(n_imu), P(its), P(g), P(a), P(fts), ptrs, 480, 640, 1, 0, 0), "xivo_batch_feed")
        torch.cuda.synchronize()
        dt = time.perf_counter() - t
        rep = None
        if profile:
            buf = C.create_string_buffer(1 << 20)
            L.xivo_profile_report(buf, len(buf))
            L.xivo_profile_enable(0)
            rep = json.loads(buf.value.decode())
        b.close()
        return dt, rep

    dt, _ = run_feed(False)
    _, rep = run_feed(True)
    timed = calls[warm:]
    fr_timed = sum(c[6] for c in timed)
    fb = rep.get("host:visual_begin", rep.get("visual_begin", {})).get("calls", 0)
    with_frames = sum(1 for c in calls if c[6])
    print(json.dumps(dict(schedule="feed", seqs=B, tick_ms=args.tick_ms, calls=len(calls), calls_with_frames=with_frames,
                          frames=sum(c[6] for c in calls), frames_per_call=round(sum(c[6] for c in calls) / max(1, with_frames), 2),
                          frame_batches=fb, frame_batches_per_call=round(fb / max(1, with_frames), 3), timed_calls=len(timed), timed_frames=fr_timed,
                          timed_s=round(dt, 4), frames_per_s=round(fr_timed / dt, 1), gpu=info)), flush=True)

    # the same frames lock-step: step k gives sequence s its k-th frame, with 8 IMU samples at 200 Hz before it
    n_step = min(len(frames[s % N_BASE]) for s in range(B))
    b = pyxivo.Batch(cfg, n_seq=B, max_groups=args.groups, max_features=args.features)
    rng = np.random.default_rng(0)
    g8 = np.ascontiguousarray(rng.normal(0, 1e-3, (8, B, 3)))
    a8 = np.ascontiguousarray(np.broadcast_to(np.array([0.0, 9.8, 0.0]), (8, B, 3)) + rng.normal(0, 1e-2, (8, B, 3)))
    warm_s = min(n_step // 4, int(args.warmup_s / 0.04))
    t = None
    for k in range(n_step):
        if k == warm_s:
            torch.cuda.synchronize()
            t = time.perf_counter()
        its = np.ascontiguousarray(np.broadcast_to((np.arange(8, dtype=np.uint64) + np.uint64(8 * k + 1)) * np.uint64(5_000_000), (B, 8)).T)
        fts = np.full(B, (k + 1) * 40_000_000, np.uint64)
        ptrs = (C.c_void_p * B)(*[fptr[s % N_BASE][k] for s in range(B)])
        capi._check(L.xivo_batch_step(b._h, 8, P(its), P(g8), P(a8), P(fts), ptrs, 480, 640, 1, 0), "xivo_batch_step")
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    fr = (n_step - warm_s) * B
    b.close()
    print(json.dumps(dict(schedule="step", seqs=B, calls=n_step, frames_per_call=B, timed_calls=n_step - warm_s, timed_frames=fr, timed_s=round(dt, 4),
                          frames_per_s=round(fr / dt, 1), gpu=info)), flush=True)


if __name__ == "__main__":
    main()

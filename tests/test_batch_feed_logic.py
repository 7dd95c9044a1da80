"""The schedule of per-sequence feeding (no GPU): dataio.feed_rounds, and `vio --batch --plan`, which must schedule loaded ASL folders
by the same rule (xivo::FeedPieces in include/xivo_b200_io.hpp)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from xivo_b200 import dataio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "xivo_b200")


def random_lists(rng, b):
    out = []
    for _ in range(b):
        kinds = rng.choice(["imu", "imu", "imu", "img"], size=int(rng.integers(0, 40)))
        out.append([(str(k), 1000 * i, i) for i, k in enumerate(kinds)])
    return out


def test_feed_rounds_properties():
    rng = np.random.default_rng(3)
    for trial in range(200):
        lists = random_lists(rng, int(rng.integers(1, 6)))
        rounds = dataio.feed_rounds(lists)
        assert all(len(r) == len(lists) for r in rounds)
        for s, msgs in enumerate(lists):
            pieces = [r[s] for r in rounds]
            assert [m for p in pieces for m in p] == msgs, trial  # concatenating a sequence's rounds gives back its list
            for k, p in enumerate(pieces):
                frames = [i for i, m in enumerate(p) if m[0] != "imu"]
                assert len(frames) <= 1 and (not frames or frames[0] == len(p) - 1), trial  # at most one frame, and it is last
                if not frames and p:  # a piece without a frame is the trailing IMU: nothing follows it
                    assert all(not q for q in pieces[k + 1 :]), trial
            # a sequence's pieces are not delayed: the non-empty ones come first
            n = sum(1 for p in pieces if p)
            assert all(pieces[:n]) and not any(pieces[n:])
        assert not rounds or any(r[s] for r in rounds[-1:] for s in range(len(lists)))


def test_feed_rounds_empty():
    assert dataio.feed_rounds([]) == []
    assert dataio.feed_rounds([[], []]) == []
    assert dataio.feed_rounds([[("imu", 1, None)], []]) == [[[("imu", 1, None)], []]]


def test_feed_rounds_example():
    a = [("imu", 1, 0), ("img", 2, 0), ("imu", 3, 0), ("imu", 4, 0), ("img", 5, 0), ("imu", 6, 0)]
    b = [("img", 1, 1)]
    r = dataio.feed_rounds([a, b])
    assert r == [[a[0:2], b], [a[2:5], []], [a[5:6], []]]


def make_folder(root, seed, n_imu, imu_step, every, shape, t0):
    """An ASL folder: n_imu samples imu_step ns apart from t0, a frame with every `every`-th one, and a dropped stretch."""
    rng = np.random.default_rng(seed)
    msgs = []
    for k in range(n_imu):
        ts = t0 + k * imu_step
        msgs.append(("imu", ts, (rng.normal(size=3), rng.normal(size=3))))
        if k % every == 3 and not (10 <= k // every < 12):
            msgs.append(("img", ts + 1, rng.integers(0, 256, shape, dtype=np.uint8)))
    return dataio.write_asl(root, msgs)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
def test_vio_batch_plan_matches_feed_rounds(tmp_path):
    exe = str(tmp_path / "vio")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "vio.cpp"), "-o", exe,
           "-L", LIBDIR, "-lxivo_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    folders = [make_folder(str(tmp_path / "a"), 1, 120, 5_000_000, 8, (12, 16), 1_000_000_000),
               make_folder(str(tmp_path / "b"), 2, 70, 2_500_000, 13, (12, 16), 1_030_000_000),
               make_folder(str(tmp_path / "c"), 3, 200, 5_000_000, 6, (12, 16), 990_000_000)]
    lst = tmp_path / "list.txt"
    lst.write_text("# image_dir imu_dir out_state\n\n" + "".join(f"{cam} {imu} {tmp_path}/out{s}.txt\n" for s, (cam, imu) in enumerate(folders)))
    r = subprocess.run([exe, "--batch", "--plan", str(lst)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [tuple(line.split()) for line in r.stdout.strip().splitlines()]
    want = []
    for k, rnd in enumerate(dataio.feed_rounds([dataio.load_asl(cam, imu) for cam, imu in folders])):
        for s, piece in enumerate(rnd):
            if not piece:
                continue
            frame = piece[-1] if piece[-1][0] != "imu" else None
            want.append((str(k), str(s), str(len(piece) - (frame is not None)), str(frame[1]) if frame else "-"))
    assert got == want
    assert any(w[3] == "-" for w in want) and len({w[1] for w in want if w[0] == want[-1][0]}) < 3  # trailing IMU; a sequence ended early
    bad = tmp_path / "bad.txt"
    bad.write_text(f"{folders[0][0]}\n")
    assert subprocess.run([exe, "--batch", "--plan", str(bad)], capture_output=True).returncode == 2

"""examples/vio.cpp on ASL folders whose data.csv lists PNG frames: `--list` prints the geometry (xivo_png_info) and file size of a
PNG frame (CPU), and on a GPU box the app writes the same trajectory file from a PNG folder as from the PNM folder of the same frames."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import png_oracle as O
from xivo_b200 import dataio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "xivo_b200")
pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")


def build(tmp_path):
    exe = str(tmp_path / "vio")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "vio.cpp"), "-o", exe,
           "-L", LIBDIR, "-lxivo_b200", "-Wl,-rpath," + LIBDIR]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def to_png_folder(src_cam, dst_cam, bits=16):
    """the same frames as PNG files (grey or RGB, 8 or 16 bits) in a copy of the cam0 folder whose data.csv lists them"""
    shutil.copytree(src_cam, dst_cam)
    rng = np.random.default_rng(0)
    data = os.path.join(dst_cam, "data")
    for f in sorted(os.listdir(data)):
        stem, ext = os.path.splitext(f)
        img = dataio.read_pnm(os.path.join(data, f))
        os.remove(os.path.join(data, f))
        s = img if img.ndim == 2 else img[..., ::-1]
        if bits == 16:
            s = s.astype(np.uint16) << 8 | rng.integers(0, 256, s.shape).astype(np.uint16)
        with open(os.path.join(data, stem + ".png"), "wb") as fh:
            fh.write(O.encode(s, 0 if img.ndim == 2 else 2, bits))
    csv = os.path.join(dst_cam, "data.csv")
    text = open(csv).read().replace(".pgm", ".png").replace(".ppm", ".png")
    open(csv, "w").write(text)
    return dst_cam


def test_vio_list_prints_png_geometry_and_size(tmp_path):
    exe = build(tmp_path)
    rng = np.random.default_rng(5)
    msgs = [("imu", 100, (np.zeros(3), np.zeros(3))), ("img", 200, rng.integers(0, 256, (6, 9), dtype=np.uint8)),
            ("img", 300, rng.integers(0, 256, (6, 9, 3), dtype=np.uint8))]
    cam, imu = dataio.write_asl(str(tmp_path / "seq"), msgs)
    pcam = to_png_folder(cam, str(tmp_path / "png_cam"))
    r = subprocess.run([exe, "--list", pcam, imu], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lines = [ln.split() for ln in r.stdout.strip().splitlines()]
    assert [ln[0] for ln in lines] == ["imu", "img", "img"]
    assert lines[1][2] == "6x9x1" and int(lines[1][3]) == os.path.getsize(os.path.join(pcam, "data", "200.png"))
    assert lines[2][2] == "6x9x3" and int(lines[2][3]) == os.path.getsize(os.path.join(pcam, "data", "300.png"))
    # PNM lines are unchanged by PNG support
    r = subprocess.run([exe, "--list", cam, imu], capture_output=True, text=True)
    assert r.stdout.splitlines()[1].split()[2] == "6x9x1"


@pytest.mark.gpu
def test_vio_app_png_folder_gives_the_pnm_folder_trajectory(tmp_path):
    import json

    from xivo_b200 import sim

    exe = build(tmp_path)
    cfg = sim.load_cfg(os.path.join(LIBDIR, "cfg", "vio_640x480.json"))
    cfg["camera_cfg"].update(rows=240, cols=320, fx=137.5, fy=137.5, cx=160, cy=120)
    cfg["tracker_cfg"].update(num_features_min=60, num_features_max=80)
    small = str(tmp_path / "cfg.json")
    json.dump(cfg, open(small, "w"))
    msgs, _ = sim.image_stream(cfg, duration=1.2, seed=6, channels=3)  # PPM frames: the 3-channel cv::imread result of the PNG ones
    cam, imu = dataio.write_asl(str(tmp_path / "seq"), msgs)
    pcam = to_png_folder(cam, str(tmp_path / "png_cam"))
    out_pnm, out_png = str(tmp_path / "pnm_state"), str(tmp_path / "png_state")
    r = subprocess.run([exe, small, cam, imu, out_pnm, "4", "14"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([exe, small, pcam, imu, out_png, "4", "14"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    a, b = open(out_pnm).read(), open(out_png).read()
    assert len(a.splitlines()) == len(msgs)
    assert a == b

"""tracker_cfg.normalize on CPU (no GPU): the numpy restatement of cv::normalize(NORM_MINMAX) (tests/normalize_oracle.py) against cv2
and against the cv2 golden, the config parser's acceptance of the key, and the key's place among the batch-wide settings.  The
device kernels are checked against the same oracle in tests/test_gpu_tracker_normalize.py."""
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

import normalize_oracle as O
from xivo_b200 import capi, sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
GOLDEN = os.path.join(ROOT, "tests", "golden", "normalize_cv2.npz")
REFERENCE_CFGS = os.path.join(ROOT, "tests", "golden", "reference_cfgs.json")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                               reason="needs g++ and the CUDA headers (host-only compile)")


def test_oracle_equals_cv2_on_every_min_max_value_triple():
    cv2 = pytest.importorskip("cv2")
    n = 0
    for lo in range(256):
        for hi in range(lo, 256):
            frame = np.arange(lo, hi + 1, dtype=np.uint8)  # holds every v with lo <= v <= hi, and its extremes are lo and hi
            want = cv2.normalize(frame, None, 0, 255, cv2.NORM_MINMAX).ravel()
            assert np.array_equal(O.lut(lo, hi)[lo : hi + 1], want), (lo, hi)
            n += hi - lo + 1
    assert n == 2_829_056


def test_oracle_equals_cv2_on_frames_across_channels():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for shape in [(31, 17), (31, 17, 3), (480, 640), (481, 643, 3)]:
        for lo, hi in [(0, 255), (40, 170), (90, 91), (13, 13)]:
            img = rng.integers(lo, hi + 1, shape).astype(np.uint8)
            assert np.array_equal(O.normalize_minmax(img), cv2.normalize(img, None, 0, 255, cv2.NORM_MINMAX)), (shape, lo, hi)
    # one array, not channel by channel: a channel that spans less than the frame is not stretched to the full range
    img = np.zeros((4, 4, 3), np.uint8)
    img[..., 0], img[..., 1], img[..., 2] = 50, 100, 150
    out = O.normalize_minmax(img)
    assert out[0, 0].tolist() == [0, 127, 255] and np.array_equal(out, cv2.normalize(img, None, 0, 255, cv2.NORM_MINMAX))


def test_constant_frame_maps_to_zeros():
    for v in (0, 77, 255):
        assert not O.normalize_minmax(np.full((5, 7, 3), v, np.uint8)).any()


def test_oracle_equals_the_cv2_golden():
    g = np.load(GOLDEN)
    assert len(g["names"]) == len(O.GOLDEN_CASES) == 16
    for k, case in enumerate(O.GOLDEN_CASES):
        img = O.golden_frame(*case)
        assert str(g["names"][k]) == "%dx%dx%d_%s" % case
        assert hashlib.sha256(img.tobytes()).digest() == g["in_sha"][k].tobytes(), f"{case}: the seeded frame is not the one the golden was made from"
        assert [int(img.min()), int(img.max())] == g["extremes"][k].tolist(), case
        assert hashlib.sha256(O.normalize_minmax(img).tobytes()).digest() == g["out_sha"][k].tobytes(), case


def test_c_abi_refuses_bad_arguments_before_touching_a_device():
    lib = capi.lib()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data_as(C.c_void_p)
    for n, rows, cols, cn, src, dst in [(1, 0, 4, 1, p, p), (1, 4, -1, 1, p, p), (1, 4, 4, 2, p, p), (1, 4, 4, 4, p, p), (-1, 4, 4, 1, p, p),
                                        (65536, 1, 1, 1, p, p), (1, 4, 4, 1, None, p), (1, 4, 4, 1, p, None), (2, 1 << 20, 1 << 20, 1, p, p)]:
        assert lib.xivo_normalize_minmax(C.c_void_p(), n, rows, cols, cn, src, dst) == -1, (n, rows, cols, cn)
        assert b"normalize_minmax" in lib.xivo_last_error()
    # well-formed arguments get as far as the context check
    assert lib.xivo_normalize_minmax(C.c_void_p(), 1, 4, 4, 1, p, p) == -1 and b"null ctx" in lib.xivo_last_error()


# ---------------------------------------------------------------- the config parser (tests/cpp/host_harness.cpp, reset_harness.cpp)
def _compile(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    cmd = ["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-I", CUDA_INC, "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", f"{name}.cpp"), "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(so)


@pytest.fixture(scope="module")
def hh(tmp_path_factory):
    lib = _compile(tmp_path_factory, "host_harness")
    lib.hh_create.restype = C.c_void_p
    lib.hh_create.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int]
    lib.hh_error.restype = C.c_char_p
    lib.hh_destroy.argtypes = [C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def rh(tmp_path_factory):
    lib = _compile(tmp_path_factory, "reset_harness")
    lib.rh_error.restype = C.c_char_p
    lib.rh_incompatibility.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
    return lib


def _creates(hh, cfg, tracker_only=False):
    h = hh.hh_create(json.dumps(cfg).encode(), 15, 30, int(tracker_only))
    if h:
        hh.hh_destroy(h)
    return bool(h), hh.hh_error().decode()


@needs_gxx
@pytest.mark.parametrize("name", ["vio_640x480.json", "stress_1280x1024.json", "tumvi_512_equidistant.json", "pcw_sim.json"])
def test_parser_accepts_normalize_in_the_package_configs(hh, name):
    cfg = sim.load_cfg(os.path.join(CFG, name))
    cfg["tracker_cfg"]["normalize"] = True
    ok, err = _creates(hh, cfg)
    assert ok, err


@needs_gxx
def test_parser_accepts_normalize_in_every_shipped_reference_config_that_loads(hh):
    """Every config shipped with the reference that the parser accepts as it is also loads with normalize switched on (the point-cloud
    tracker configs among them: Tracker::UpdatePointCloud never normalises, the key is accepted and has no effect there)."""
    with open(REFERENCE_CFGS) as f:
        cfgs = json.load(f)
    loaded = []
    for name, cfg in sorted(cfgs.items()):
        tracker_only = "tracker_only" in name
        if not _creates(hh, cfg, tracker_only)[0]:
            continue
        cfg.setdefault("tracker_cfg", {})["normalize"] = True
        ok, err = _creates(hh, cfg, tracker_only)
        assert ok, f"{name}: {err}"
        loaded.append(name)
    assert loaded == ["pcw.json", "pcw_loops.json", "phab.json", "tumvi_cam0.json", "tumvi_cam1.json", "tumvi_tracker_only_cam0.json",
                      "tumvi_tracker_only_cam1.json"]


@needs_gxx
def test_normalize_is_a_batch_wide_key(rh):
    a = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    b = json.loads(json.dumps(a))
    b["tracker_cfg"]["normalize"] = True
    key = C.create_string_buffer(256)

    def incompatibility(x, y):
        rc = rh.rh_incompatibility(json.dumps(x).encode(), 4, 14, 0, json.dumps(y).encode(), 4, 14, 0, key, 256)
        assert rc >= 0, rh.rh_error().decode()
        return key.value.decode() if rc == 0 else None

    assert incompatibility(a, a) is None and incompatibility(b, b) is None
    assert incompatibility(a, b) == "tracker_cfg.normalize"
    assert incompatibility(b, a) == "tracker_cfg.normalize"

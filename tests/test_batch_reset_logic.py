"""Host side of xivo_batch_reset_sequence on CPU (no GPU): which config keys one batch handle shares across its sequences.

tests/cpp/reset_harness.cpp compiles the product's config parser and batch_incompatibility (xivo_b200/csrc/estimator_host.cpp.inc) with
g++; every batch-wide key changed alone must be named, every per-sequence key changed alone must be accepted.  The entry point itself
must be declared in the public header and exported by the built library."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import pytest

from xivo_b200 import capi, sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "xivo_b200", "cfg")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
needs_gxx = pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                               reason="needs g++ and the CUDA headers (host-only compile)")
G, F = 4, 14


@pytest.fixture(scope="module")
def rh(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rh") / "libreset_harness.so")
    cmd = ["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-I", CUDA_INC, "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", "reset_harness.cpp"), "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.rh_error.restype = C.c_char_p
    lib.rh_incompatibility.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
    return lib


def base(**tracker):
    cfg = sim.load_cfg(os.path.join(CFG, "vio_640x480.json"))
    cfg["tracker_cfg"].update(tracker)
    return cfg


def incompatibility(lib, a, b, lay_a=(G, F, 0), lay_b=(G, F, 0)):
    key = C.create_string_buffer(256)
    rc = lib.rh_incompatibility(json.dumps(a).encode(), *lay_a, json.dumps(b).encode(), *lay_b, key, 256)
    assert rc >= 0, lib.rh_error().decode()
    return key.value.decode() if rc == 0 else None


def changed(cfg, path, value):
    out = json.loads(json.dumps(cfg))
    d = out
    *head, last = path.split(".")
    for k in head:
        d = d.setdefault(k, {})
    d[last] = value
    return out


DESC = dict(extract_descriptor=True)  # base of the descriptor keys: they are only accepted with descriptors on
BATCH_WIDE = [  # (key named, base tracker overrides, value)
    ("covariance_update", {}, "tf32x3"),
    ("use_1pt_RANSAC", {}, True),
    ("subfilter.visual_meas_std", {}, 2.5),
    ("subfilter.MH_thresh", {}, 5.991),
    ("camera_cfg.rows", {}, 512),
    ("camera_cfg.cols", {}, 512),
    ("message_buffer_size", {}, 6),
    ("tracker_cfg.tracker_type", DESC, "MATCH"),
    ("tracker_cfg.mask_size", {}, 11),
    ("tracker_cfg.margin", {}, 12),
    ("tracker_cfg.num_features_min", {}, 100),
    ("tracker_cfg.num_features_max", {}, 160),
    ("tracker_cfg.max_pixel_displacement", {}, 32),
    ("tracker_cfg.KLT.win_size", {}, 21),
    ("tracker_cfg.KLT.max_level", {}, 3),
    ("tracker_cfg.KLT.max_iter", {}, 10),
    ("tracker_cfg.KLT.eps", {}, 0.03),
    ("tracker_cfg.FAST.threshold", {}, 10),
    ("tracker_cfg.FAST.nonmaxSuppression", {}, False),
    ("tracker_cfg.extract_descriptor", {}, True),
    ("tracker_cfg.differential", DESC, False),
    ("tracker_cfg.match_dropped_tracks", DESC, True),
    ("tracker_cfg.descriptor_distance_thresh", DESC, 40),
    ("tracker_cfg.do_outlier_rejection", {}, True),
    ("tracker_cfg.outlier_rejection.method", {}, "LMEDS"),
    ("tracker_cfg.outlier_rejection.RANSAC_max_iters", {}, 500),
    ("tracker_cfg.outlier_rejection.RANSAC_reproj_thresh", {}, 2.0),
    ("tracker_cfg.outlier_rejection.confidence", {}, 0.99),
]

EQUIDISTANT = {"model": "equidistant", "rows": 480, "cols": 640, "fx": 190.97847715128717, "fy": 190.9733070521226, "cx": 254.93170605935475,
               "cy": 256.8974428996504, "k0123": [0.0034823894022493434, 0.0007150348452162257, -0.0020532361418706202, 0.00020293673591811182]}
PER_SEQUENCE = [  # (key, value): may differ between the sequences of one handle
    ("camera_cfg", EQUIDISTANT),
    ("camera_cfg.fx", 300.0),
    ("camera_cfg.cy", 250.0),
    ("X.Wbc", [-1.5, 0.02, 0.0]),
    ("X.Tbc", [0.01, 0.0, -0.02]),
    ("X.Vsb", [0.1, 0.0, 0.0]),
    ("P.Vsb", 0.3),
    ("Qimu.gyro", [1e-3, 1e-3, 1e-3]),
    ("Qmodel.Wsb", 0.02),
    ("visual_meas_std", 1.5),
    ("integration_method", "RK4"),
    ("gravity", [0, 0, -9.81]),
    ("initial_z", 2.0),
    ("MH_thresh", 8.0),
    ("min_inliers", 7),
    ("max_group_lifetime", 30),
    ("subfilter.ready_steps", 4),
    ("gravity_init_counter", 10),
    ("simulation", True),
]


@needs_gxx
@pytest.mark.parametrize("key,tracker,value", BATCH_WIDE, ids=[k for k, _, _ in BATCH_WIDE])
def test_every_batch_wide_key_changed_alone_is_named(rh, key, tracker, value):
    a = base(**tracker)
    b = changed(a, key, value)
    assert incompatibility(rh, a, a) is None
    assert incompatibility(rh, a, b) == key


@needs_gxx
@pytest.mark.parametrize("lay_b,key", [((G + 1, F, 0), "max_groups"), ((G, F + 2, 0), "max_features"), ((G, F, 1), "tracker_only")])
def test_layout_and_mode_are_batch_wide(rh, lay_b, key):
    a = base()
    assert incompatibility(rh, a, a, (G, F, 0), lay_b) == key


@needs_gxx
@pytest.mark.parametrize("key,value", PER_SEQUENCE, ids=[k for k, _ in PER_SEQUENCE])
def test_every_per_sequence_key_changed_alone_is_accepted(rh, key, value):
    a = base()
    assert incompatibility(rh, a, changed(a, key, value)) is None


@needs_gxx
def test_first_differing_key_is_named_when_several_differ(rh):
    a = base()
    b = changed(changed(a, "tracker_cfg.KLT.win_size", 21), "covariance_update", "tf32x3")
    assert incompatibility(rh, a, b) == "covariance_update"


def test_reset_entry_point_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "xivo_b200_estimator.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    assert re.search(r"int\s+xivo_batch_reset_sequence\s*\(\s*xivo_batch\s*\*\s*b\s*,\s*int\s+seq\s*,\s*const\s+char\s*\*\s*cfg_json\s*\)\s*;", code)
    assert os.path.exists(capi.LIB_PATH), "build libxivo_b200.so first (python -m xivo_b200.build)"
    lib = C.CDLL(capi.LIB_PATH)
    assert hasattr(lib, "xivo_batch_reset_sequence")


def test_reset_rejects_a_null_handle_without_touching_a_device():
    lib = capi.lib()
    assert lib.xivo_batch_reset_sequence(C.c_void_p(), 0, None) == -1
    assert b"null batch" in lib.xivo_last_error()

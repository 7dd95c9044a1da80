"""Compact Runge-Kutta records on CPU (no GPU, no nvcc).  Batch switches its estimators to one record per sub-step (kernels.h: ImuStep)
and imu_cov_propagate rebuilds every stage from it with imu_stage_from_step.  tests/cpp/compact_records.cpp compiles the host state
machine with g++; here the same IMU stream runs through an estimator that writes one record per stage and one that writes one per
sub-step: the nominal states must be identical bit for bit, the rebuilt stages must match the per-stage records to rounding, and the
queue must fill (needs_state_now) at the same points."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from xivo_b200 import sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"
pytestmark = pytest.mark.skipif(shutil.which("g++") is None or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")),
                                reason="needs g++ and the CUDA headers (host-only compile)")


@pytest.fixture(scope="module")
def cr(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cr") / "libcompact_records.so")
    cmd = ["g++", "-std=c++17", "-O2", "-march=x86-64-v3", "-I", CUDA_INC, "-shared", "-fPIC", os.path.join(ROOT, "tests", "cpp", "compact_records.cpp"), "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(so)
    lib.cr_create.restype = C.c_void_p
    lib.cr_create.argtypes = [C.c_char_p, C.c_int]
    for name in ("cr_destroy", "cr_pending_stages", "cr_needs_state_now"):
        getattr(lib, name).argtypes = [C.c_void_p]
    lib.cr_inertial.argtypes = [C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p]
    lib.cr_visual_begin.argtypes = [C.c_void_p, C.c_ulonglong]
    lib.cr_motion.argtypes = [C.c_void_p, C.c_void_p]
    lib.cr_take_stages.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    return lib


def motion(lib, h):
    a = np.zeros(15)
    lib.cr_motion(h, a.ctypes.data)
    return a


def take(lib, h):
    buf = np.zeros((4096, 16))
    n = lib.cr_take_stages(h, buf.ctypes.data, 4096)
    assert n >= 0
    return buf[:n].copy()


@pytest.mark.parametrize("method,stepsize", [("PrinceDormand", 0.002), ("RK4", 0.002), ("PrinceDormand", -1.0), ("RK4", -1.0)])
def test_compact_records_rebuild_the_per_stage_records(cr, method, stepsize):
    cfg = sim.load_cfg(os.path.join(ROOT, "xivo_b200", "cfg", "pcw_sim.json"))
    cfg["integration_method"] = method
    cfg[method]["stepsize"] = stepsize
    msgs, _ = sim.pcw_stream(cfg, duration=1.5, seed=5)
    text = json.dumps(cfg).encode()
    full, comp = cr.cr_create(text, 0), cr.cr_create(text, 1)
    assert full and comp
    nst = 7 if method == "PrinceDormand" else 4
    checked = 0
    for i, (kind, ts, p) in enumerate(msgs):
        if kind == "imu":
            g, a = np.ascontiguousarray(p[0]), np.ascontiguousarray(p[1])
            cr.cr_inertial(full, ts, g.ctypes.data, a.ctypes.data)
            cr.cr_inertial(comp, ts, g.ctypes.data, a.ctypes.data)
        else:
            assert cr.cr_visual_begin(full, ts) == cr.cr_visual_begin(comp, ts)
        assert np.array_equal(motion(cr, full), motion(cr, comp))  # the nominal state does not depend on the record form
        assert cr.cr_pending_stages(full) == cr.cr_pending_stages(comp)
        assert cr.cr_needs_state_now(full) == cr.cr_needs_state_now(comp)
        if i % 3:  # let the queues grow over several messages
            continue
        want, got = take(cr, full), take(cr, comp)
        assert len(got) == len(want) and len(got) % nst == 0
        if len(want):
            assert np.array_equal(got[:, 15], want[:, 15])  # sub-step lengths and the sign that closes a Propagate call
            assert np.abs(got[:, :9] - want[:, :9]).max() <= 1e-14
            assert np.abs(got[:, 9:15] - want[:, 9:15]).max() <= 1e-13 * max(1.0, np.abs(want[:, 9:15]).max())
            checked += len(want)
    assert checked > 50 * nst
    cr.cr_destroy(full)
    cr.cr_destroy(comp)

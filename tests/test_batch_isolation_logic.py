"""Failure isolation of a batch handle without a GPU: the entry points are declared and exported, NULL handles are refused before any
device call, XIVO_SEQ_FAILED is distinct from every error code, and the facades carry the new surface."""
import ctypes as C
import inspect
import os
import re
import shutil
import subprocess

import pytest

from xivo_b200 import capi, pyxivo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")


def header_code(name):
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(INC, name)).read(), flags=re.S)


def defines():
    out = {}
    for m in re.finditer(r"#define\s+(XIVO_(?:OK|ERR_\w+|SEQ_FAILED))\s+\(?(-?\d+)\)?", header_code("xivo_b200.h")):
        out[m.group(1)] = int(m.group(2))
    return out


def test_entry_points_are_declared_and_exported():
    code = header_code("xivo_b200_estimator.h")
    assert re.search(r"int\s+xivo_batch_isolate_failures\s*\(\s*xivo_batch\s*\*\s*b\s*,\s*int\s+on\s*\)\s*;", code)
    assert re.search(r"int\s+xivo_batch_sequence_status\s*\(\s*const\s+xivo_batch\s*\*\s*b\s*,\s*int\s+seq\s*,\s*int\s*\*\s*code\s*,\s*char\s*\*\s*msg\s*,"
                     r"\s*int\s+msg_cap\s*\)\s*;", code)
    assert os.path.exists(capi.LIB_PATH), "build libxivo_b200.so first (python -m xivo_b200.build)"
    lib = C.CDLL(capi.LIB_PATH)
    assert hasattr(lib, "xivo_batch_isolate_failures") and hasattr(lib, "xivo_batch_sequence_status")


def test_null_handles_are_refused_before_any_device_call():
    lib = capi.lib()
    for on in (0, 1):
        assert lib.xivo_batch_isolate_failures(None, on) == capi.XIVO_ERR_ARG
        assert b"null batch" in lib.xivo_last_error()
    code, msg = C.c_int(7), C.create_string_buffer(16)
    for seq in (-1, 0, 1):
        assert lib.xivo_batch_sequence_status(None, seq, C.byref(code), msg, 16) == capi.XIVO_ERR_ARG
    assert code.value == 7 and msg.value == b""


def test_seq_failed_is_one_and_no_error_code():
    d = defines()
    assert d["XIVO_SEQ_FAILED"] == 1 == capi.XIVO_SEQ_FAILED
    errors = {k: v for k, v in d.items() if k.startswith("XIVO_ERR_")}
    assert d["XIVO_OK"] == 0 and all(v < 0 for v in errors.values()) and len(set(errors.values())) == len(errors)
    assert 1 not in errors.values()
    for k, v in errors.items():
        assert getattr(capi, k) == v, k


def test_python_facade_surface():
    sig = inspect.signature(pyxivo.Batch.__init__)
    assert sig.parameters["isolate_failures"].default is False
    for name in ("failed", "status", "set_isolate_failures"):
        assert callable(getattr(pyxivo.Batch, name))


def test_message_calls_pass_seq_failed_only_when_isolating():
    b = pyxivo.Batch.__new__(pyxivo.Batch)  # no handle: _msg only interprets a return code
    b.isolate_failures = True
    b._msg(capi.XIVO_SEQ_FAILED, "call")
    b._msg(0, "call")
    with pytest.raises(capi.XivoError):
        b._msg(capi.XIVO_ERR_STATE, "call")
    b.isolate_failures = False
    with pytest.raises(capi.XivoError):
        b._msg(capi.XIVO_SEQ_FAILED, "call")


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
def test_cpp_facade_and_vio_compile(tmp_path):
    exe = str(tmp_path / "vio")
    cmd = ["g++", "-std=c++17", "-O0", "-Wall", "-Wextra", "-Werror", "-I", INC, os.path.join(ROOT, "examples", "vio.cpp"), "-o", exe,
           "-L", os.path.dirname(capi.LIB_PATH), "-lxivo_b200", "-Wl,-rpath," + os.path.dirname(capi.LIB_PATH)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    hpp = open(os.path.join(INC, "xivo_b200.hpp")).read()
    for name in ("IsolateFailures", "SequenceStatus", "Failed"):
        assert re.search(rf"\b{name}\s*\(", hpp), name
    r = subprocess.run([exe, "--batch"], capture_output=True, text=True)
    assert r.returncode == 1 and "--isolate-failures" in r.stderr

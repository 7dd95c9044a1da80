"""Builds libxivo_b200.so in-tree with nvcc for sm_90a (no torch dependency in the library)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libxivo_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-pthread", "-Xptxas", "-v"]

# (source, extra flags).  The tracker is compiled without FMA contraction so its float math
# rounds exactly like the scalar CPU arithmetic of OpenCV's LK (see tracker_kernels.cu).
SOURCES = [
    ("tracker_kernels.cu", ["-fmad=false"]),
    ("ekf_kernels.cu", []),
    ("ekf_tc_kernels.cu", []),
    ("capi.cu", []),
    # host state machine: AVX2/FMA for the 23x23 integrator loops (results within 1e-16 relative)
    ("estimator.cu", ["-Xcompiler", "-march=x86-64-v3"]),
]


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def build(force: bool = False, verbose: bool = False) -> str:
    # every header-like file any source may include: csrc/*.{h,cuh,inc} (estimator.cu includes estimator_host.cpp.inc) and the public C headers
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh", ".inc"))]
    inc = os.path.join(HERE, "..", "include")
    hdrs += [os.path.join(inc, f) for f in os.listdir(inc) if f.endswith(".h")]
    objs = []
    os.makedirs(os.path.join(HERE, "_obj"), exist_ok=True)
    for src, extra in SOURCES:
        s = os.path.join(CSRC, src)
        if not os.path.exists(s):
            continue
        o = os.path.join(HERE, "_obj", src + ".o")
        if force or _newer([s] + hdrs, o):
            cmd = [NVCC] + ARCH + COMMON + extra + ["-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or r.returncode:
                sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
            if r.returncode:
                raise RuntimeError(f"nvcc failed on {src}")
            with open(o + ".ptxas.txt", "w") as f:
                f.write(r.stderr)
        objs.append(o)
    if force or _newer(objs, LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))

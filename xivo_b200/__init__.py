"""xivo_b200 — CUDA-native implementation of XIVO's per-frame visual-inertial inner loop.

The product is libxivo_b200.so (hand-written sm_90a CUDA behind the C ABI of
include/xivo_b200.h).  This package only binds it (ctypes) and mirrors the reference's
pyxivo surface; it contains no CPU implementation of the hot path.
"""
from .capi import Context, XivoError, launch_count, lib, LIB_PATH  # noqa: F401

__all__ = ["Context", "XivoError", "launch_count", "lib", "LIB_PATH"]

"""Kernel-level timing through the C ABI's in-library CUDA-event profiler (diagnostic; not a bench line).
usage: python scripts/kbench.py"""
import ctypes as C, json, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xivo_b200 import capi, synth

L = capi.lib()
ctx = capi.Context(0)

def report():
    buf = C.create_string_buffer(1 << 16)
    L.xivo_profile_report(buf, len(buf))
    return {k: v for k, v in json.loads(buf.value.decode()).items() if not k.startswith("_") and not k.startswith("host:")}

a, b = synth.frame_pair(960, 1280, seed=3, shift=(3, 2))
xy, sc, n = ctx.fast_detect(a, 10, max_kp=1 << 17)
p0 = xy[np.lexsort((xy[:, 0], xy[:, 1], -sc))[:20000]].astype(np.float32)
print("points", len(p0))
for env in ({"XIVO_LK_GENERIC": "1"}, {}):
    os.environ.pop("XIVO_LK_GENERIC", None)
    os.environ.update(env)
    for _ in range(3):
        ctx.lk_track(a, b, p0, p0 + 1.0)
    L.xivo_profile_reset(); L.xivo_profile_enable(1)
    for _ in range(10):
        ctx.lk_track(a, b, p0, p0 + 1.0)
    L.xivo_profile_enable(0)
    r = report()
    print(env, {k: round(v["ms"] / v["calls"] * 1000, 1) for k, v in r.items()})

for _ in range(3):
    ctx.fast_detect(a, 5, max_kp=1 << 18)
L.xivo_profile_reset(); L.xivo_profile_enable(1)
for _ in range(10):
    ctx.fast_detect(a, 5, max_kp=1 << 18)
L.xivo_profile_enable(0)
r = report()
print("fast", {k: round(v["ms"] / v["calls"] * 1000, 1) for k, v in r.items()})

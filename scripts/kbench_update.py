"""EKF measurement update at the BASELINE state sizes, B filters per launch, through xivo_ekf_update_batch and the in-library CUDA-event
profiler: ms per launch of the gain kernel and of the covariance downdate (fp64 CUDA cores / wgmma 3xTF32), Joseph-equivalent and
executed flop rates, and the fp64 traffic of P that bounds the downdate.  usage: python scripts/kbench_update.py [B]"""
import ctypes as C, json, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from xivo_b200 import capi

L = capi.lib()
ctx = capi.Context(0)
B = int(sys.argv[1]) if len(sys.argv) > 1 else 512
peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) if os.path.exists("MEASURED_PEAKS.json") else {}
hbm, tf = peaks.get("hbm_gbs", 3350.0), peaks.get("bf16_tflops_sustained", 989.0)  # fallback: H100 SXM data sheet

def report():
    buf = C.create_string_buffer(1 << 16)
    L.xivo_profile_report(buf, len(buf))
    return {k: v for k, v in json.loads(buf.value.decode()).items() if not k.startswith("_") and not k.startswith("host:")}

rng = np.random.default_rng(0)
out = []
for N, M in ((89, 28), (203, 60), (299, 124)):
    A = rng.normal(size=(N, N))
    P1 = A @ A.T / N + np.eye(N)
    P = np.broadcast_to(P1, (B, N, N)).copy()
    H = rng.normal(size=(B, M, N)) * (rng.uniform(size=(B, M, N)) < 0.09)
    inn = rng.normal(size=(B, M))
    R = np.ones((B, M))
    for mode, env in (("fp64", {}), ("tf32x3 (wgmma, TMA-staged operands)", {}), ("tf32x3 first kernel", {"XIVO_TC_V1": "1"})):
        os.environ.pop("XIVO_TC_V1", None)
        os.environ.update(env)
        tc = mode != "fp64"
        ctx.ekf_update_batch(H, P, inn, R, tf32x3=tc, repeat=2)
        L.xivo_profile_reset(); L.xivo_profile_enable(1)
        ctx.ekf_update_batch(H, P, inn, R, tf32x3=tc, repeat=10)
        L.xivo_profile_enable(0)
        r = report()
        g, c = r["ekf_gain"]["ms"] / r["ekf_gain"]["calls"], r["ekf_cov"]["ms"] / r["ekf_cov"]["calls"]
        joseph = 4 * N**3 + 6 * M * N**2 + 4 * M * M * N + M**3 / 3
        exec_cov = 2.0 * N * N * M * (3 if tc else 0.5)  # tensor: three full TF32 passes; fp64: upper triangle only
        p_bytes = 2.0 * N * N * 8                        # P read + written once (fp64)
        row = dict(N=N, M=M, B=B, mode=mode, gain_us=round(g * 1e3, 1), cov_us=round(c * 1e3, 1), update_us_per_filter=round((g + c) * 1e3 / B, 3),
                   joseph_equiv_tflops=round(joseph * B / ((g + c) * 1e-3) / 1e12, 2), joseph_frac_of_bf16_peak=round(joseph * B / ((g + c) * 1e-3) / 1e12 / tf, 4),
                   cov_executed_tflops=round(exec_cov * B / (c * 1e-3) / 1e12, 2), cov_P_traffic_gbs=round(p_bytes * B / (c * 1e-3) / 1e9, 1),
                   cov_P_traffic_frac_of_hbm=round(p_bytes * B / (c * 1e-3) / 1e9 / hbm, 4))
        out.append(row)
        print(json.dumps(row), flush=True)
os.environ.pop("XIVO_TC_V1", None)

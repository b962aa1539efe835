"""Own-kernel TF32 GEMM throughput, measured the way MEASURED_PEAKS.json measures bf16 (8192^3, best of 10 = burst;
back to back for 4 s = sustained), so that the TF32 roofline denominator `bf16_tflops_sustained / 2` (an assumption, not a
measured TF32 peak) can be put beside a measured figure of THIS repo's generic wgmma kernel
(k_tc_gemm<128, GENERIC>, CTA = 128x128 tiles, tf32 wgmma).  An own kernel is a lower bound of the hardware peak, not the
peak itself; bench.py keeps the assumed value as `peak` and quotes this one next to it.

usage (on the GPU):  python tools/measure_tf32_peak.py > tf32_peak.json"""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import small_params  # noqa: E402
from visdial_b200 import VD_MATH_TF32, Engine  # noqa: E402
from visdial_b200._lib import check  # noqa: E402


def main():
    n = int(os.environ.get("PEAK_N", "8192"))
    eng = Engine(small_params("lf-ques", "disc"))
    eng.set_math_mode(VD_MATH_TF32)
    bufs = []
    for _ in range(3):
        p = C.c_void_p()
        check(eng.lib.vd_device_alloc(eng.h, C.byref(p), n * n * 4))
        bufs.append(p)
    rng = np.random.default_rng(0)
    a = rng.standard_normal((n, n), dtype=np.float32)
    for p in bufs[:2]:
        check(eng.lib.vd_memcpy_h2d(eng.h, p, a.ctypes.data, a.nbytes))
    A, B, Cm = bufs
    flop = 2.0 * n * n * n

    def run(k):
        eng.synchronize()
        eng.timer_start()
        for _ in range(k):
            check(eng.lib.vd_gemm_tn(eng.h, n, n, n, A, n, B, n, Cm, n, 0.0, None, 0))
        return eng.timer_stop() / k

    run(3)
    burst = min(run(1) for _ in range(10))
    t0, ms, reps = time.time(), [], 0
    while time.time() - t0 < 4.0:
        ms.append(run(20))
        reps += 20
    sustained = float(np.mean(ms[len(ms) // 2:]))          # second half of the loop: clocks settled under the power cap
    out = {"what": "k_tc_gemm<128,GENERIC> (this repo, tf32 wgmma, 128x128 tiles, one CTA per SM) C = A B^T, %d^3" % n,
           "tf32_tflops_burst": flop / (burst * 1e-3) / 1e12, "tf32_tflops_sustained": flop / (sustained * 1e-3) / 1e12,
           "ms_burst": burst, "ms_sustained": sustained, "launches_sustained": reps}
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks):
        d = json.load(open(peaks))
        out["assumed_tf32_peak_sustained"] = d["bf16_tflops_sustained"] / 2
        out["assumed_tf32_peak_burst"] = d["bf16_tflops"] / 2
        out["own_kernel_over_assumed_sustained"] = out["tf32_tflops_sustained"] / out["assumed_tf32_peak_sustained"]
    print(json.dumps(out, indent=1))
    eng.close()


if __name__ == "__main__":
    main()

"""Time of one cone projection for the spectral cones of libscs_b200_spectral.so, next to the PSD cone of the same
order. Prints the card's name and power limit first. Each figure is the wall time of one scs_b200_proj_dual_cone
call (host -> device copy of x, the projection, device -> host copy, synchronised), the median of --reps calls after
--warmup calls; the in-solve cone_time per iteration is this minus the two copies.

usage: python scripts/bench_spectral.py [--reps 20] [--warmup 3]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi  # noqa: E402

CASES = [
    ("200 sum-of-largest cones, order 100, k = 10", {"sl_n": [100] * 200, "sl_k": [10] * 200}),
    ("200 PSD cones, order 100", {"s": [100] * 200}),
    ("100 nuclear-norm cones, 100 x 60", {"nuc_m": [100] * 100, "nuc_n": [60] * 100}),
    ("one l1 cone of 10^6 entries", {"ell1": [1000000]}),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    lib = capi.load(spectral=True)
    if not lib.scs_b200_device_ok():
        raise SystemExit("no usable sm_90 device")
    rng = np.random.default_rng(0)
    for label, cone in CASES:
        m = capi.cone_rows(cone)
        k, keep = capi.make_cone(cone, spectral=True)
        cw = lib.scs_b200_init_cone(C.byref(k), m, None)
        assert cw
        x0 = rng.standard_normal(m)
        r_y = np.full(m, 10.0)
        times = []
        for it in range(a.warmup + a.reps):
            x = x0.copy()
            t0 = time.perf_counter()
            assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(x), capi.dptr(r_y)) == 0
            if it >= a.warmup:
                times.append(time.perf_counter() - t0)
        lib.scs_b200_finish_cone(cw)
        print(f"{label:48s} m = {m:9d}  {1e3 * np.median(times):9.3f} ms per projection "
              f"(min {1e3 * min(times):.3f})")


if __name__ == "__main__":
    main()

"""Times of the log-det cone of libscs_b200_spectral.so. Prints the card's name and power limit first.

* one scs_b200_proj_dual_cone call (host -> device copy of x, the projection, device -> host copy, synchronised) on
  200 log-det cones of order 100, next to the same call on 200 PSD cones of order 100: the median of --reps calls after
  --warmup calls, from one seeded x (the log-det cones keep their warm starts between calls, as in a solve);
* the wall time of a full solve, to eps 1e-6, of the seeded D-optimal design problem of oracle/make_golden_logdet.py
  scaled up (order 48, 800 candidate points), with its iteration count.

usage: python scripts/bench_logdet.py [--reps 20] [--warmup 3] [--order 48] [--points 800]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi  # noqa: E402

CASES = [
    ("200 log-det cones, order 100", {"d": [100] * 200}),
    ("200 PSD cones, order 100", {"s": [100] * 200}),
]


def dopt(order, points, seed=24):
    """maximise log det(sum_i lam_i a_i a_i') over the simplex: x = (lam, t), minimise t with
    (t, 1, sum_i lam_i a_i a_i') in the log-det cone (as oracle/make_golden_logdet.py)"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((points, order))
    # the packed lower triangle, column by column: (row i >= column j)
    il = np.concatenate([np.arange(j, order) for j in range(order)])
    jl = np.concatenate([np.full(order - j, j) for j in range(order)])
    svec = a[:, il] * a[:, jl] * np.where(il == jl, 1.0, np.sqrt(2.0))
    nt = svec.shape[1]
    top = sp.vstack([sp.csr_matrix(np.ones((1, points))), -sp.eye(points), sp.csr_matrix((2, points)),
                     sp.csr_matrix(-svec.T)])
    tcol = sp.csr_matrix(([-1.0], ([1 + points], [0])), shape=(3 + points + nt, 1))
    A = sp.hstack([top, tcol]).tocsc()
    b = np.zeros(A.shape[0])
    b[0] = 1.0
    b[2 + points] = 1.0
    c = np.zeros(points + 1)
    c[points] = 1.0
    return A, b, c, {"z": 1, "l": points, "d": [order]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--order", type=int, default=48)
    ap.add_argument("--points", type=int, default=800)
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
        print(f"{label:36s} m = {m:9d}  {1e3 * np.median(times):9.3f} ms per projection "
              f"(min {1e3 * min(times):.3f})")
    A, b, c, cone = dopt(a.order, a.points)
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, {"z": 1, "l": a.points})
    k, keep = capi.make_cone(cone, spectral=True)
    st = capi.default_settings(lib, verbose=0, eps_abs=1e-6, eps_rel=1e-6, max_iters=100000)
    m, n = A.shape
    x, y, s = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    t0 = time.perf_counter()
    flag = lib.scs(C.pointer(hp.data), C.byref(k), C.byref(st), C.byref(sol), C.byref(info))
    dt = time.perf_counter() - t0
    print(f"D-optimal design, order {a.order}, {a.points} points (m = {m}, n = {n}, nnz(A) = {A.nnz}): "
          f"status {info.status.decode()} ({flag}), {info.iter} iterations, {dt:.3f} s to eps 1e-6 "
          f"(solve {info.solve_time / 1e3:.3f} s), objective {info.pobj:.10g}")


if __name__ == "__main__":
    main()

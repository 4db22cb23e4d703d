"""Lean driver for ncu / timing of the CG loop's kernels AS THEY RUN IN A SOLVE: builds the C2 operator, creates the
linsys workspace and runs genuine CG iterations on a real right-hand side (K1 = spmv_flag_kernel<1>, K2 =
spmv_flag_kernel<2>, K3 = k_cg_update, K4 = k_cg_pupdate; up to n = 2 SMs x 4096, K3 / K4 = the two phases of the
fused k_cg_update_p).  REPS (default 20) iterations with per-kernel CUDA events, then REPS iterations timed as a whole
(no events inside: programmatic dependent launch overlap intact)."""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scs_b200 import capi, problems

scale = float(os.environ.get("SCALE", "1.0"))
rng = np.random.default_rng(1234)
n = int(1_000_000 * scale)
m = 3 * n
A = problems.random_sparse_csc(m, n, 10, rng)
hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
lib = capi.load()
dr = np.empty(n + m + 1)
dr[:n] = 1e-6
dr[n:n + m // 10] = 1.0 / 100.0
dr[n + m // 10:] = 10.0
w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
assert w
reps = int(os.environ.get("REPS", "20"))
rhs = rng.standard_normal(n + m)
ms = (C.c_double * 5)()
by = (C.c_double * 5)()
assert lib.scs_b200_time_cg_kernels(w, capi.dptr(rhs), reps, ms, by) == 0
for k, nm in enumerate(("K1 A p /R_y", "K2 A' tmp + R_x p, dot", "K3 update", "K4 p update", "iteration (events inside)")):
    print(f"{nm:28s}: {ms[k]*1e3:7.1f} us  {by[k]/ms[k]/1e6:6.0f} GB/s")
ab = C.c_double()
t = lib.scs_b200_time_cg_iter(w, reps, C.byref(ab))
print(f"{'iteration (no events inside)':28s}: {t*1e3:7.1f} us  {ab.value/t/1e6:6.0f} GB/s")
lib.scs_free_lin_sys_work(w)

"""Phases of the CG loop's batch kernel (kernels/cg.cu k_cg_batch) on the C2 operator, beside the three kernels per
iteration it replaces: one launch of REPS (default 200) genuine CG iterations after a genuine start, block 0's
%globaltimer after every grid barrier or wait (K1 phase, K2 phase, update up to the beta wait, p update, each with the
barrier or wait that ends it) and CUDA events around the launch; then scs_b200_time_cg_iter (three launches per iteration,
no events inside) on the same workspace."""
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
reps = int(os.environ.get("REPS", "200"))
rhs = rng.standard_normal(n + m)
ms = (C.c_double * 5)()
assert lib.scs_b200_time_cg_batch(w, capi.dptr(rhs), reps, ms) == 0, "the workspace cannot run the batch kernel"
for k, nm in enumerate(("K1 phase + barrier", "K2 phase + alpha wait", "update to beta + wait",
                        "p update + barrier", "iteration (events around the launch)")):
    print(f"batch {nm:36s}: {ms[k] * 1e3:7.1f} us")
ab = C.c_double()
t = lib.scs_b200_time_cg_iter(w, reps, C.byref(ab))
print(f"three kernels: iteration (no events inside)  : {t * 1e3:7.1f} us")
lib.scs_free_lin_sys_work(w)

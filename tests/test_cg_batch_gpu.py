"""The CG loop's batch kernel (kernels/cg.cu k_cg_batch: K1, K2 and the fused update of up to a whole batch of CG
iterations in one cooperative launch) against the three kernels per iteration it replaces
(scs_b200_set_cg_batch_kernel(0), as SCS_B200_CG_BATCH_KERNEL=0): the same bits of x, y and the same CG counts for cold
and warm KKT solves, a 1e-12 solve, a first batch far longer than the solve needs, odd n and n at the fused limit; the
same x, y, s and ScsInfo after 200 ADMM iterations; and two host threads at once, one of which holds the token."""
import ctypes as C
import threading

import numpy as np
import pytest

from scs_b200 import capi, problems
from test_cg_fused_gpu import fused_limit, linsys
from test_device_data_gpu import host_solve

pytestmark = pytest.mark.gpu


def batch_kernel(lib, on):
    lib.scs_b200_set_cg_batch_kernel(1 if on else 0)


def kkt_sequence(lib, n, col_nnz, seed):
    """on one workspace (m = 3 n): a cold 1e-10 solve, a cold 1e-12 solve, a warm 1e-12 solve and a warm 1e-3 solve
    whose first batch is sized by the previous one's count (most of it after `done`); (bytes of every answer, CG
    counts, batch-kernel solves)"""
    m = 3 * n
    w, _, _, _ = linsys(lib, n, m, col_nnz, seed)
    rng = np.random.default_rng(seed + 1)
    rhs = [rng.standard_normal(n + m) for _ in range(4)]
    s = rng.standard_normal(n)
    out, its = [], []
    try:
        for k, (tol, warm) in enumerate(((1e-10, False), (1e-12, False), (1e-12, True), (1e-3, True))):
            sol = rhs[k].copy()
            assert lib.scs_solve_lin_sys(w, capi.dptr(sol), capi.dptr(s) if warm else None, tol) == 0
            out.append(sol.tobytes())
            its.append(lib.scs_b200_linsys_last_cg_its(w))
        return out, its, lib.scs_b200_linsys_cg_batch_solves(w)
    finally:
        lib.scs_free_lin_sys_work(w)


@pytest.mark.parametrize("where", ["small-odd", "limit"])
def test_kkt_solves_bit_for_bit(lib, where):
    n, col_nnz = {"small-odd": (20_001, 8), "limit": (fused_limit(), 3)}[where]
    try:
        batch_kernel(lib, True)
        got = kkt_sequence(lib, n, col_nnz, 17)
        batch_kernel(lib, False)
        ref = kkt_sequence(lib, n, col_nnz, 17)
    finally:
        batch_kernel(lib, True)
    assert got[2] == 4 and ref[2] == 0, (got[2], ref[2])
    assert got[1] == ref[1], (got[1], ref[1])
    assert min(got[1]) > 1, got[1]
    for k in range(4):
        assert got[0][k] == ref[0][k], k


def c2(scale):
    import scipy.sparse as sp
    prob = problems.config("C2", scale=scale, seed=1234)
    A = sp.csc_matrix((prob["A"][0], prob["A"][1], prob["A"][2]), shape=prob["A"][3])
    return A, None, prob["b"], prob["c"], prob["cone"]


def admm(prob):
    x, y, s, info = host_solve(*prob, max_iters=200, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)[0]
    return x.tobytes(), y.tobytes(), s.tobytes(), info


def test_admm_200_iterations_bit_for_bit(lib):
    prob = c2(0.1)
    try:
        batch_kernel(lib, False)
        ref = admm(prob)
        batch_kernel(lib, True)
        got = admm(prob)
    finally:
        batch_kernel(lib, True)
    assert got[3]["iter"] == 200
    assert got == ref


def test_two_threads_one_token(lib):
    """two solves at once: at most one holds the token and runs the batch kernel; both give the serial bits"""
    seeds = (3, 4)
    serial = {sd: kkt_sequence(lib, 50_001, 6, sd) for sd in seeds}
    out = {}

    def worker(sd):
        out[sd] = kkt_sequence(lib, 50_001, 6, sd)

    threads = [threading.Thread(target=worker, args=(sd,)) for sd in seeds]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for sd in seeds:
        assert out[sd][0] == serial[sd][0] and out[sd][1] == serial[sd][1], sd
    assert serial[3][2] == 4 and serial[4][2] == 4

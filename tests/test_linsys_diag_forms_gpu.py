"""The CG loop reads R_y^-1 and R_x from tables when diag_r has SCS's own form (R_y two-valued, R_x uniform) and from
the vectors otherwise (kernels/cg.cu b200_cg_classify_diag). Every combination of the two forms, and the switch between
them at scs_update_lin_sys_diag_r, must solve the KKT system as the reference does."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi, problems
from reference_replay import rel

pytestmark = pytest.mark.gpu


def scs_diag_r(n, m, z, scale):
    d = np.empty(n + m + 1)
    d[:n] = 1e-6
    d[n:n + z] = 1.0 / (1000.0 * scale)
    d[n + z:n + m] = 1.0 / scale
    d[n + m] = 10.0
    return d


def diag_r_kind(kind, n, m, z, rng):
    """'ry3': R_y takes three values, R_x uniform; 'rxvec': R_y two-valued, R_x not uniform; 'free': both arbitrary"""
    d = scs_diag_r(n, m, z, 0.1)
    if kind in ("ry3", "free"):
        d[n + m - 1] = 3.7  # one third value is enough to leave the table
    if kind == "free":
        d[n:n + m] = 10.0 ** rng.uniform(-3.0, 1.0, m)
    if kind in ("rxvec", "free"):
        d[:n] = 10.0 ** rng.uniform(-7.0, -5.0, n)
    return d


@pytest.mark.parametrize("kind", ["ry3", "rxvec", "free"])
@pytest.mark.parametrize("m,n,col_nnz,z,seed", [(4000, 1000, 32, 400, 2), (30000, 10000, 10, 3000, 3)])
def test_solve_lin_sys_any_diag_r_matches_reference(lib, reflib, m, n, col_nnz, z, seed, kind):
    rng = np.random.default_rng(300 + seed)
    A = problems.random_sparse_csc(m, n, col_nnz, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_kind(kind, n, m, z, rng)
    dr2 = scs_diag_r(n, m, z, 0.37)  # back to SCS's form: the tables
    rhs = rng.standard_normal(n + m)
    s = 0.01 * rng.standard_normal(n)
    tol = 1e-12
    # the reference first: its answers can be recorded on a host without a GPU
    wr = reflib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert wr
    ref, ref2 = rhs.copy(), rhs.copy()
    try:
        assert reflib.scs_solve_lin_sys(wr, capi.dptr(ref), capi.dptr(s), tol) == 0
        assert reflib.scs_update_lin_sys_diag_r(wr, capi.dptr(dr2)) == 0
        assert reflib.scs_solve_lin_sys(wr, capi.dptr(ref2), None, tol) == 0
    finally:
        reflib.scs_free_lin_sys_work(wr)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    try:
        mine = rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), capi.dptr(s), tol) == 0
        assert lib.scs_b200_linsys_last_cg_its(w) > 0
        err = rel(mine, ref, 0.0)
        assert err <= 1e-10, err
        assert lib.scs_update_lin_sys_diag_r(w, capi.dptr(dr2)) == 0
        mine = rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), None, tol) == 0
        err = rel(mine, ref2, 0.0)
        assert err <= 1e-10, err
        # and back to the vectors
        assert lib.scs_update_lin_sys_diag_r(w, capi.dptr(dr)) == 0
        mine = rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), capi.dptr(s), tol) == 0
        err = rel(mine, ref, 0.0)
        assert err <= 1e-10, err
    finally:
        lib.scs_free_lin_sys_work(w)

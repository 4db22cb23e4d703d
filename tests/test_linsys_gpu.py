"""GPU parity of the linear-system plugin (SpMV + device PCG) against the
UNMODIFIED reference CPU-indirect backend (its answers recorded under tests/golden/reference/),
called through the same five-symbol C ABI (reference include/linsys.h:25-71)."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi, problems
from reference_replay import rel

pytestmark = pytest.mark.gpu


def diag_r_for(n, m, z, scale=0.1, rho_x=1e-6):
    """reference src/scs.c:971-980 + src/cones.c:349-363"""
    d = np.empty(n + m + 1)
    d[:n] = rho_x
    d[n:n + z] = 1.0 / (1000.0 * scale)
    d[n + z:n + m] = 1.0 / scale
    d[n + m] = 10.0
    return d


def kkt_reduced_residual(A, diag_r, rhs, sol):
    """|| (R_x + A' R_y^-1 A) x - (r_x + A' R_y^-1 r_y) ||_inf  and  || y - R_y^-1 (A x - r_y) ||_inf"""
    m, n = A[3]
    rx, ry = diag_r[:n], diag_r[n:n + m]
    x, y = sol[:n], sol[n:]
    Ax = problems.csc_matvec(A, x)
    lhs = rx * x + problems.csc_rmatvec(A, Ax / ry)
    red_rhs = rhs[:n] + problems.csc_rmatvec(A, rhs[n:] / ry)
    return np.abs(lhs - red_rhs).max(), np.abs(y - (Ax - rhs[n:]) / ry).max()


CASES = [
    # (m, n, col_nnz, z, seed)
    (40, 10, 3, 4, 1),
    (4000, 1000, 32, 400, 2),       # C1 shape
    (30000, 10000, 10, 3000, 3),    # C2 shape / 100
    (3000, 50, 700, 10, 4),         # long rows of A' (700 nnz per column): multi-lane rows
    (64, 5000, 40, 0, 5),           # very long rows of A: chunked rows (> tile)
]


@pytest.mark.parametrize("m,n,col_nnz,z,seed", CASES)
def test_spmv_matches_reference(lib, reflib, m, n, col_nnz, z, seed):
    rng = np.random.default_rng(seed)
    A = problems.random_sparse_csc(m, n, col_nnz, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, z)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w, "scs_init_lin_sys_work failed (no sm_90 device?)"
    try:
        x = rng.standard_normal(n)
        yv = rng.standard_normal(m)
        for acc in (0, 1):
            # A x
            y0 = rng.standard_normal(m) if acc else np.zeros(m)
            mine = y0.copy()
            assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(mine), acc) == 0
            ref = y0.copy()
            reflib._scs_accum_by_a(C.byref(hp.A), capi.dptr(x), capi.dptr(ref))
            assert rel(mine, ref, 1e-300) <= 1e-13
            # A' y
            x0 = rng.standard_normal(n) if acc else np.zeros(n)
            mine = x0.copy()
            assert lib.scs_b200_accum_by_atrans(w, capi.dptr(yv), capi.dptr(mine), acc) == 0
            ref = x0.copy()
            reflib._scs_accum_by_atrans(C.byref(hp.A), capi.dptr(yv), capi.dptr(ref))
            assert rel(mine, ref, 1e-300) <= 1e-13
    finally:
        lib.scs_free_lin_sys_work(w)


def ragged_csc(m, n, rng, mean_nnz, p_empty_col=0.1, max_col=120):
    """CSC with ragged columns (some empty, some long) and, for small mean_nnz, many empty rows."""
    lens = np.minimum(rng.poisson(mean_nnz, n), min(m, max_col))
    lens[rng.random(n) < p_empty_col] = 0
    lens[rng.random(n) < 0.02] = min(m, max_col)
    cols = np.repeat(np.arange(n, dtype=np.int64), lens)
    keys = np.unique(cols * m + rng.integers(0, m, size=cols.size))  # sorted (col, row), duplicates dropped
    cols, rows = keys // m, keys % m
    indptr = np.zeros(n + 1, dtype=np.int32)
    indptr[1:] = np.cumsum(np.bincount(cols, minlength=n))
    data = rng.uniform(-1.0, 1.0, size=rows.size)
    return data, rows.astype(np.int32), indptr, (m, n)


@pytest.mark.parametrize("grid_cap", [None, 1, 3])
@pytest.mark.parametrize("m,n,mean_nnz,seed", [(5000, 3000, 2.0, 11), (200000, 30000, 12.0, 12), (300, 4000, 1.0, 13)])
def test_spmv_flagged_stream_ragged(lib, reflib, m, n, mean_nnz, seed, grid_cap, monkeypatch):
    """v3 kernel on ragged operators (empty rows -> explicit zeros, rows ending inside / across lanes),
    also with the grid forced to 1 / 3 CTAs so that every CTA walks many groups (ring wrap-around)."""
    if grid_cap is not None:
        monkeypatch.setenv("SCS_B200_SPMV_GRID", str(grid_cap))
    rng = np.random.default_rng(seed)
    A = ragged_csc(m, n, rng, mean_nnz)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, 0)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    try:
        for rep in range(3):
            x = rng.standard_normal(n)
            yv = rng.standard_normal(m)
            for acc in (0, 1):
                y0 = rng.standard_normal(m) if acc else np.zeros(m)
                mine, ref = y0.copy(), y0.copy()
                assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(mine), acc) == 0
                reflib._scs_accum_by_a(C.byref(hp.A), capi.dptr(x), capi.dptr(ref))
                assert rel(mine, ref, 1e-300) <= 1e-13
                x0 = rng.standard_normal(n) if acc else np.zeros(n)
                mine, ref = x0.copy(), x0.copy()
                assert lib.scs_b200_accum_by_atrans(w, capi.dptr(yv), capi.dptr(mine), acc) == 0
                reflib._scs_accum_by_atrans(C.byref(hp.A), capi.dptr(yv), capi.dptr(ref))
                assert rel(mine, ref, 1e-300) <= 1e-13
        # and a full KKT solve through the same operators (POST_DIV / POST_FMA_DOT epilogues, init chains)
        rhs = rng.standard_normal(n + m)
        wr = reflib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
        mine, ref = rhs.copy(), rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), None, 1e-12) == 0
        assert reflib.scs_solve_lin_sys(wr, capi.dptr(ref), None, 1e-12) == 0
        reflib.scs_free_lin_sys_work(wr)
        assert rel(mine, ref, 0.0) <= 1e-10
    finally:
        lib.scs_free_lin_sys_work(w)


def test_operator_without_rows(lib):
    """A rank's row block is empty when there are more ranks than rows: its operator still exists, with row pointers
    {0} (the equilibration kernels read them), and a product with it launches nothing."""
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    lib.b200_spmv_create.restype = C.c_void_p
    lib.b200_spmv_create.argtypes = [C.c_int, C.c_int, ip, ip, dp]
    lib.b200_spmv.restype = C.c_int
    lib.b200_spmv.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200_spmv_rowptr.restype = C.c_void_p
    lib.b200_spmv_rowptr.argtypes = [C.c_void_p]
    lib.b200_spmv_destroy.argtypes = [C.c_void_p]
    lib.b200_d2h.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    rp, ci, va = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1)
    M = lib.b200_spmv_create(0, 7, rp.ctypes.data_as(ip), ci.ctypes.data_as(ip), va.ctypes.data_as(dp))
    assert M
    try:
        got = np.full(9, -1, np.int32)  # {0} and its padding
        assert lib.b200_d2h(got.ctypes.data, lib.b200_spmv_rowptr(M), got.nbytes) == 0 and lib.b200_sync() == 0
        assert (got == 0).all()
        args = C.create_string_buffer(256)  # a zeroed B200SpmvArgs: nothing of it is read
        launches = lib.scs_b200_launch_count()
        assert lib.b200_spmv(M, args) == 0
        assert lib.scs_b200_launch_count() == launches
    finally:
        lib.b200_spmv_destroy(M)


@pytest.mark.parametrize("m,n,col_nnz,seed", [(3000, 50, 700, 4), (64, 5000, 40, 5), (30000, 10000, 10, 3)])
def test_device_built_operators_equal_host_built(lib, m, n, col_nnz, seed, monkeypatch):
    """scs_init_lin_sys_work builds both flagged streams on the device (kernels/setup.cu; rows longer than a warp-tile
    are cut into the same balanced pieces as the host plan builder cuts them) -- the result must be BIT-identical to
    the host builders' (SCS_B200_HOST_SETUP=1): same stream, same warp-tiles, same summation order."""
    rng = np.random.default_rng(seed)
    A = problems.random_sparse_csc(m, n, col_nnz, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, 0)
    x, yv, rhs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(n + m)
    outs = []
    for host in (0, 1):
        if host:
            monkeypatch.setenv("SCS_B200_HOST_SETUP", "1")
        else:
            monkeypatch.delenv("SCS_B200_HOST_SETUP", raising=False)
        w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
        assert w
        try:
            ax, aty, sol = np.zeros(m), np.zeros(n), rhs.copy()
            assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(ax), 0) == 0
            assert lib.scs_b200_accum_by_atrans(w, capi.dptr(yv), capi.dptr(aty), 0) == 0
            assert lib.scs_solve_lin_sys(w, capi.dptr(sol), None, 1e-12) == 0
            outs.append((ax, aty, sol))
        finally:
            lib.scs_free_lin_sys_work(w)
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_spmv_full_size_c2_properties(lib):
    """BASELINE configs[1] size (n=1e6, m=3e6, nnz=1e7): parity of both operators against numpy in fp64,
    linearity, the adjoint identity <A x, y> = <x, A'y>, and run-to-run bit reproducibility."""
    rng = np.random.default_rng(1234)
    n, m = 1_000_000, 3_000_000
    A = problems.random_sparse_csc(m, n, 10, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, 0)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    try:
        def Ax(x):
            out = np.zeros(m)
            assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(out), 0) == 0
            return out

        def Aty(y):
            out = np.zeros(n)
            assert lib.scs_b200_accum_by_atrans(w, capi.dptr(y), capi.dptr(out), 0) == 0
            return out

        x1, x2 = rng.standard_normal(n), rng.standard_normal(n)
        y1 = rng.standard_normal(m)
        ax1, aty1 = Ax(x1), Aty(y1)
        ref = problems.csc_matvec(A, x1)
        assert np.abs(ax1 - ref).max() / np.abs(ref).max() <= 1e-13
        ref = problems.csc_rmatvec(A, y1)
        assert np.abs(aty1 - ref).max() / np.abs(ref).max() <= 1e-12   # numpy's own cumsum-difference error
        assert np.array_equal(ax1, Ax(x1)) and np.array_equal(aty1, Aty(y1))      # bit-reproducible
        lin = Ax(2.0 * x1 - 0.5 * x2) - (2.0 * ax1 - 0.5 * Ax(x2))
        assert np.abs(lin).max() <= 1e-12 * np.abs(ax1).max()
        lhs, rhs = float(ax1 @ y1), float(x1 @ aty1)
        assert abs(lhs - rhs) <= 1e-10 * max(abs(lhs), abs(rhs), 1.0)
    finally:
        lib.scs_free_lin_sys_work(w)


@pytest.mark.parametrize("m,n,col_nnz,z,seed", CASES[:4])
@pytest.mark.parametrize("warm", [False, True])
def test_solve_lin_sys_matches_reference(lib, reflib, m, n, col_nnz, z, seed, warm):
    rng = np.random.default_rng(100 + seed)
    A = problems.random_sparse_csc(m, n, col_nnz, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, z)
    rhs = rng.standard_normal(n + m)
    tol = 1e-12
    s = None
    if warm:
        # warm start = exact-ish solution of a nearby rhs, as in the ADMM loop
        s = 0.01 * rng.standard_normal(n)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    wr = reflib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert wr
    try:
        mine = rhs.copy()
        ref = rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), capi.dptr(s) if warm else None, tol) == 0
        assert reflib.scs_solve_lin_sys(wr, capi.dptr(ref), capi.dptr(s) if warm else None, tol) == 0
        its = lib.scs_b200_linsys_last_cg_its(w)
        assert its > 0
        r1, r2 = kkt_reduced_residual(A, dr, rhs, mine)
        # the reference's own stop test, recomputed on the host in fp64
        assert r1 < 10 * tol * max(1.0, np.abs(rhs).max() * 10), (r1, its)
        assert r2 < 1e-9 * max(1.0, np.abs(mine[n:]).max())
        err = rel(mine, ref, 0.0)
        print(f"\n[m={m} n={n} warm={warm}] cg_its={its} rel diff vs reference {err:.3e} reduced-res {r1:.2e}")
        assert err <= 1e-10, err
        # update diag_r (scale change) and solve again
        dr2 = diag_r_for(n, m, z, scale=0.37)
        assert lib.scs_update_lin_sys_diag_r(w, capi.dptr(dr2)) == 0
        assert reflib.scs_update_lin_sys_diag_r(wr, capi.dptr(dr2)) == 0
        mine = rhs.copy()
        ref = rhs.copy()
        assert lib.scs_solve_lin_sys(w, capi.dptr(mine), None, tol) == 0
        assert reflib.scs_solve_lin_sys(wr, capi.dptr(ref), None, tol) == 0
        err = rel(mine, ref, 0.0)
        assert err <= 1e-10, err
    finally:
        lib.scs_free_lin_sys_work(w)
        reflib.scs_free_lin_sys_work(wr)


def test_zero_rhs_short_circuit(lib):
    """||b||_inf <= 1e-12 -> b := 0 (reference private.c:296-299)."""
    rng = np.random.default_rng(7)
    m, n = 300, 100
    A = problems.random_sparse_csc(m, n, 5, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, 0)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    try:
        b = np.full(n + m, 1e-13)
        assert lib.scs_solve_lin_sys(w, capi.dptr(b), None, 1e-9) == 0
        assert np.all(b == 0.0)
        assert lib.scs_b200_linsys_last_cg_its(w) == 0
    finally:
        lib.scs_free_lin_sys_work(w)

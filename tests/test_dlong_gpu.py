"""GPU: the DLONG libraries (64-bit scs_int) against the int libraries. Once the 64-bit counts and indices are
checked and narrowed, both widths run the same kernels on the same int32 arrays, so every comparison here is bit
identity, not a tolerance: the solves of the reference's fixtures, of a QP, of a problem over every cone and of the
spectral fixtures; the linear-system plugin with both forms of diag_r; the operator entry points. Also the plugin
path's refusal of a row index that truncation would make valid, and the reference's own suite linked against the
DLONG plugin library where oracle/long.mk built it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import REF_DIR, ROOT
from scs_b200 import capi, problems
from test_dlong_cpu import ensure_built

pytestmark = pytest.mark.gpu
PP = C.POINTER
PROB_DIR = os.path.join(ROOT, "tests", "golden", "problems")
SPECTRAL = ["test_ell1_cone", "test_ell1_and_nuc", "robust_pca", "several_nuc_cone", "several_sum_largest",
            "graph_partitioning"]
INFO_FIELDS = ("iter", "status_val", "pobj", "dobj", "res_pri", "res_dual", "gap", "res_infeas", "res_unbdd_a",
               "res_unbdd_p")

ensure_built()


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def assert_identical(a, b, what=""):
    assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), what


def assert_same_solve(r_int, r_long, what):
    (st_i, info_i, *v_i), (st_l, info_l, *v_l) = r_int, r_long
    assert st_i == st_l, what
    for name, a, b in zip("xys", v_i, v_l):
        assert_identical(a, b, (what, name))
    for f in INFO_FIELDS:
        a, b = getattr(info_i, f), getattr(info_l, f)
        assert (a == b) or (a != a and b != b), (what, f, a, b)  # NaN residuals are NaN in both
    assert info_i.status == info_l.status


def run_scs(lib, long, d, k, s):
    T = capi.abi(long)
    n, m = d.contents.n, d.contents.m
    x, y, sv = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = T.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(sv))
    info = T.ScsInfo()
    status = lib.scs(d, k, s, C.byref(sol), C.byref(info))
    return status, info, x, y, sv


def solve_file(name, spectral=False, **over):
    """the problem file read and solved by the int library and by the DLONG library of the same cone layout"""
    out = []
    for long in (False, True):
        T = capi.abi(long)
        lib = capi.load(spectral=spectral, long=long)
        cone = T.ScsConeSpectral if spectral else T.ScsCone
        lib.scs_b200_read_data.restype = T.int_t
        lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(T.ScsData)), PP(PP(cone)), PP(PP(T.ScsSettings))]
        lib.scs_b200_free_data.argtypes = [PP(T.ScsData), PP(cone), PP(T.ScsSettings)]
        d, k, s = PP(T.ScsData)(), PP(cone)(), PP(T.ScsSettings)()
        assert lib.scs_b200_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
        s.contents.verbose = 0
        for f, v in over.items():
            setattr(s.contents, f, v)
        out.append(run_scs(lib, long, d, k, s))
        lib.scs_b200_free_data(d, k, s)
    return out


def solve_prob(prob, **over):
    out = []
    for long in (False, True):
        lib = capi.load(long=long)
        hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], prob.get("P"), long=long)
        st = capi.default_settings(lib, long=long, verbose=0, **over)
        out.append(run_scs(lib, long, C.pointer(hp.data), C.pointer(hp.cone), C.pointer(st)))
    return out


@pytest.mark.parametrize("name", ["random_prob", "mpc_bug1", "mpc_bug2", "mpc_bug3"])
def test_reference_fixtures_solve_bit_identically(name):
    r_int, r_long = solve_file(name, eps_abs=1e-6, eps_rel=1e-6)
    assert r_int[0] == 1, r_int[1].status
    assert_same_solve(r_int, r_long, name)


@pytest.mark.parametrize("name", SPECTRAL)
def test_spectral_fixtures_solve_bit_identically(name):
    r_int, r_long = solve_file(os.path.join("spectral", name), spectral=True, max_iters=2000)
    assert r_int[1].iter > 0
    assert_same_solve(r_int, r_long, name)


def qp_problem(seed=21):
    import scipy.sparse as sp
    prob = dict(problems.make_problem(400, 100, 8, {"z": 40, "l": 120, "q": [3, 7, 30, 200]}, seed))
    n = prob["n"]
    B = sp.random(30, n, density=0.08, random_state=np.random.RandomState(seed), format="csr")
    P = sp.triu(B.T @ B + 0.1 * sp.identity(n), format="csc")
    P.sort_indices()
    prob["P"] = (P.data.copy(), P.indices, P.indptr, (n, n))
    return prob


def every_cone_problem(seed=5):
    """a problems.make_problem SOCP with box and PSD rows, extended by exponential and power rows whose slack is an
    interior point of their cones (with y = 0 there, the generator's optimum stays optimal)"""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    base = {"z": 10, "l": 40, "bl": -rng.uniform(0.5, 1.5, 9), "bu": rng.uniform(0.5, 1.5, 9), "q": [4, 30, 3],
            "s": [3, 6]}
    prob = problems.make_problem(capi.cone_rows(base), 120, 8, base, seed)
    ep, ed, pw = 4, 3, [0.3, -0.5, 0.8]
    Ax, Ai, Ap, shape = prob["A"]
    A1 = sp.random(3 * (ep + ed + len(pw)), shape[1], density=0.1, random_state=np.random.RandomState(seed),
                   format="csr")
    A = sp.vstack([sp.csc_matrix((Ax, Ai, Ap), shape=shape), A1], format="csc")
    A.sort_indices()
    s1 = np.concatenate([np.tile([0.0, 1.0, 2.0], ep),       # t > s exp(r / s)
                         np.tile([-1.0, 0.0, 1.0], ed),      # e w > -u exp(v / u)
                         np.tile([1.0, 1.0, 0.5], len(pw))])  # x^a y^(1-a) > |r|, and the same for the dual cones
    cone = dict(base, ep=ep, ed=ed, p=pw)
    assert capi.cone_rows(cone) == A.shape[0]
    return {"A": (A.data, A.indices, A.indptr, A.shape), "b": np.concatenate([prob["b"], A1 @ prob["x_opt"] + s1]),
            "c": prob["c"], "cone": cone}


@pytest.mark.parametrize("kind", ["qp", "every_cone"])
def test_generated_problems_solve_bit_identically(kind):
    prob = qp_problem() if kind == "qp" else every_cone_problem()
    for over in (dict(max_iters=1), dict(eps_abs=1e-7, eps_rel=1e-7, max_iters=3000)):
        r_int, r_long = solve_prob(prob, **over)
        assert_same_solve(r_int, r_long, (kind, over))


# ---------------------------------------------------------------------------------------------------- plugin ABI
def diag_r_scs(n, m, z, scale=0.1, rho_x=1e-6):
    d = np.empty(n + m + 1)
    d[:n] = rho_x
    d[n:n + z] = 1.0 / (1000.0 * scale)
    d[n + z:n + m] = 1.0 / scale
    d[n + m] = 10.0
    return d


@pytest.mark.parametrize("with_p", [False, True])
def test_plugin_abi_bit_identical(with_p):
    rng = np.random.default_rng(3)
    m, n, z = 3000, 1000, 300
    A = problems.random_sparse_csc(m, n, 12, rng)
    P = None
    if with_p:
        P = qp_problem()["P"]
        n0 = P[3][0]
        A = problems.random_sparse_csc(m, n0, 12, rng)
        n = n0
    diag_two = diag_r_scs(n, m, z)
    diag_plain = rng.uniform(0.5, 2.0, n + m + 1)          # not SCS's two-value form: R_y as a vector
    b0 = rng.standard_normal(n + m)
    s0 = rng.standard_normal(n)
    x, yv = rng.standard_normal(n), rng.standard_normal(m)
    results = []
    for long in (False, True):
        lib = capi.load(long=long)
        hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m}, P, long=long)
        w = lib.scs_init_lin_sys_work(C.byref(hp.A), C.byref(hp.P) if P is not None else None, capi.dptr(diag_two))
        assert w
        try:
            got = []
            for dr in (diag_two, diag_plain, diag_two):
                assert lib.scs_update_lin_sys_diag_r(w, capi.dptr(dr)) == 0
                for warm in (None, s0):
                    b = b0.copy()
                    assert lib.scs_solve_lin_sys(w, capi.dptr(b), capi.dptr(warm), 1e-9) == 0
                    got.append(b)
                    got.append(np.array([lib.scs_b200_linsys_last_cg_its(w)], dtype=np.float64))
            for acc in (0, 1):
                y = np.ones(m)
                assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(y), acc) == 0
                xt = np.ones(n)
                assert lib.scs_b200_accum_by_atrans(w, capi.dptr(yv), capi.dptr(xt), acc) == 0
                got += [y, xt]
            results.append(got)
        finally:
            lib.scs_free_lin_sys_work(w)
    for i, (a, b) in enumerate(zip(*results)):
        assert_identical(a, b, i)


def test_plugin_refuses_a_row_index_that_truncation_would_make_valid(capfd):
    llib = capi.load(long=True)
    rng = np.random.default_rng(4)
    m, n = 500, 100
    A = problems.random_sparse_csc(m, n, 5, rng)
    good = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m}, long=True)
    w0 = llib.scs_init_lin_sys_work(C.byref(good.A), None, capi.dptr(diag_r_scs(n, m, 0)))
    assert w0  # the matrix without the bad index builds
    llib.scs_free_lin_sys_work(w0)
    bad_rows = np.array(A[1], dtype=np.int64)  # a copy: HostProblem borrows int64 arrays as they are
    bad_rows[7] = 2 ** 32 + 3                  # the valid row 3 once truncated
    hp = capi.HostProblem((A[0], bad_rows, A[2], A[3]), np.zeros(m), np.zeros(n), {"l": m}, long=True)
    launches = llib.scs_b200_launch_count()
    w = llib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(diag_r_scs(n, m, 0)))
    assert not w
    # the narrowing kernel is the only kernel launched: no builder kernel ever read the refused index
    assert llib.scs_b200_launch_count() - launches == 1
    assert "row indices must lie in [0, m)" in capfd.readouterr().err


# ---------------------------------------------------------------------------------------------------- operators
def test_cone_and_aa_operators_bit_identical():
    prob = every_cone_problem()
    cone = prob["cone"]
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(12)
    x0, ry, D = rng.standard_normal(m), rng.uniform(0.5, 2.0, m), rng.uniform(0.5, 2.0, m)
    dim, mem = 2000, 7
    fs = [rng.standard_normal(dim) for _ in range(12)]
    results = []
    for long in (False, True):
        lib = capi.load(long=long)
        k, keep = capi.make_cone(cone, long=long)
        got = []
        for scale in (None, D):
            cw = lib.scs_b200_init_cone(C.byref(k), m, capi.dptr(scale))
            assert cw
            for r in (None, ry):
                out = x0.copy()
                assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(r)) == 0
                got.append(out)
            lib.scs_b200_finish_cone(cw)
        aa = lib.scs_b200_aa_init(dim, mem, mem, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
        assert aa
        try:
            xk = np.zeros(dim)
            for f in fs:
                fk = f.copy()
                nrm = lib.scs_b200_aa_apply(aa, capi.dptr(fk), capi.dptr(xk))
                got += [fk, np.array([nrm])]
                fn, xn = fk + 0.1, xk - 0.1
                rc = lib.scs_b200_aa_safeguard(aa, capi.dptr(fn), capi.dptr(xn))
                got += [fn, xn, np.array([float(rc)])]
                xk = fk
            st = lib.scs_b200_aa_get_stats(aa)
            got.append(np.array([float(getattr(st, f)) for f, _ in st._fields_]))
            lib.scs_b200_aa_reset(aa)
        finally:
            lib.scs_b200_aa_finish(aa)
        results.append(got)
    for i, (a, b) in enumerate(zip(*results)):
        assert_identical(a, b, i)


# ---------------------------------------------------------------------------------------------------- reference suite
def test_reference_suite_with_the_dlong_plugin():
    exe = os.path.join(REF_DIR, "run_tests_b200_long")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/run_tests_b200_long not built (oracle/long.mk needs the reference sources)")
    ob = os.environ.get("SCS_REF_OPENBLAS_DIR",
                        "/opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs")
    env = dict(os.environ, LD_LIBRARY_PATH=ob + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
    r = subprocess.run([exe], cwd=REF_DIR, capture_output=True, text=True, env=env, timeout=1200)
    tail = (r.stdout + r.stderr)[-3000:]
    print(tail)
    assert r.returncode == 0 and "ALL TESTS PASSED" in r.stdout, tail

"""The reference's own binary fixtures (test/problems/{random_prob, mpc_bug1..3}, copied to tests/golden/problems/;
known optima in random_prob.h:6, mpc_bug.h:7-9) read with scs_b200_read_data and solved by the device-resident
driver, checked the way the reference checks them (test/problems/test_prob_from_data_file.h:31-60:
eps 1e-6, status solved, primal and dual objective within 1e-4 of the known optimum).

random_prob exercises every supported cone at once (zero, LP, SOC incl. sizes 0 and 1, PSD incl. orders 0 and
1, primal/dual exponential, primal/dual power); mpc_bug1..3 are QPs. (The file reader itself is verified on the CPU
against the reference's reader in tests/test_rw_cpu.py.)"""
import ctypes as C
import os

import numpy as np
import pytest

from scs_b200 import capi
from reference_replay import rel

pytestmark = pytest.mark.gpu
PP = C.POINTER

FIXTURES = {
    "random_prob": 5.751458006385587,
    "mpc_bug1": -0.473957794500,
    "mpc_bug2": -0.029336830816,
    "mpc_bug3": -0.002215217478,
}


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_reference_fixture_known_optimum(lib, name):
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "problems", name)
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsCone)), PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsCone), PP(capi.ScsSettings)]
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsCone)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    try:
        s.contents.eps_abs = 1e-6
        s.contents.eps_rel = 1e-6
        s.contents.verbose = 0
        n, m = d.contents.n, d.contents.m
        x, y, sv = np.zeros(n), np.zeros(m), np.zeros(m)
        sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(sv))
        info = capi.ScsInfo()
        status = lib.scs(d, k, s, C.byref(sol), C.byref(info))
        opt = FIXTURES[name]
        c = np.ctypeslib.as_array(d.contents.c, (n,))
        b = np.ctypeslib.as_array(d.contents.b, (m,))
        xpx = 0.0
        if d.contents.P:
            P = d.contents.P.contents
            nnz = P.p[P.n]
            import scipy.sparse as sp
            U = sp.csc_matrix((np.ctypeslib.as_array(P.x, (nnz,)), np.ctypeslib.as_array(P.i, (nnz,)),
                               np.ctypeslib.as_array(P.p, (P.n + 1,))), shape=(n, n))
            full = U + sp.triu(U, 1).T
            xpx = float(x @ (full @ x))
        perr = 0.5 * xpx + float(c @ x) - opt
        derr = -0.5 * xpx - float(b @ y) - opt
        print(f"\n[{name}] status={info.status.decode()} iters={info.iter} primal obj error {perr:.3e} dual obj error {derr:.3e}")
        assert status == 1, info.status
        assert abs(perr) < 1e-4 and abs(derr) < 1e-4
    finally:
        lib.scs_b200_free_data(d, k, s)


def test_exp_power_operator_matches_committed_goldens(lib):
    """device exp / power cone kernels under the Moreau wrapper against tests/golden/cone_triples.npz
    (reference outputs); tolerances as in tests/test_cones_gpu.py (1e-8 max with power cones)."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "cone_triples.npz"))
    cone = {"l": 3, "ep": int(g["mixed_ep"]), "ed": int(g["mixed_ed"]), "p": list(g["mixed_p"])}
    m = capi.cone_rows(cone)
    k, keep = capi.make_cone(cone)
    cw = lib.scs_b200_init_cone(C.byref(k), m, None)
    assert cw
    try:
        for tag, ry in (("id", None), ("ry", g["mixed_ry"].copy())):
            out = g["mixed_x"].copy()
            assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(ry)) == 0
            ref = g[f"mixed_out_{tag}"]
            err = np.abs(out - ref) / max(np.abs(ref).max(), 1.0)
            assert err.max() <= 1e-8 and np.median(err) <= 1e-14, (tag, err.max())
    finally:
        lib.scs_b200_finish_cone(cw)


def test_complex_psd_operator_matches_reference(lib, reflib, monkeypatch):
    """complex-PSD kernels (kernels/cones_complex.cu) against the reference's zheevr projection"""
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [PP(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    rng = np.random.default_rng(5)
    for cone in ({"cs": [1, 2, 3, 5, 12, 12, 40]}, {"z": 2, "l": 3, "q": [4], "s": [3], "cs": [4, 7], "ep": 2, "p": [0.4]}):
        m = capi.cone_rows(cone)
        x = rng.standard_normal(m) * 2
        for ry in (None, np.full(m, 10.0)):
            k, keep = capi.make_cone(cone)
            cw = reflib._scs_init_cone(C.byref(k), m)
            ref = x.copy()
            assert reflib._scs_proj_dual_cone(capi.dptr(ref), cw, None, capi.dptr(None if ry is None else ry.copy())) == 0
            reflib._scs_finish_cone(cw)
            k2, keep2 = capi.make_cone(cone)
            mw = lib.scs_b200_init_cone(C.byref(k2), m, None)
            assert mw
            out = x.copy()
            assert lib.scs_b200_proj_dual_cone(mw, capi.dptr(out), capi.dptr(None if ry is None else ry.copy())) == 0
            lib.scs_b200_finish_cone(mw)
            err = rel(out, ref)
            assert err <= (1e-8 if cone.get("p") else 5e-13), (cone, err)


@pytest.mark.parametrize("cfg,steps", [("C3", 25), ("C4", 40), ("C5", 25)])
def test_full_size_configs_are_self_consistent(lib, cfg, steps):
    """BASELINE configs 2-4 at FULL size (C3: LP n=5e6, nnz=5e7; C4: 200 PSD(100) blocks; C5: mixed, n=2e6, nnz=3e7):
    a fixed number of ADMM iterations, then the size-independent checks the reference applies to every solve
    (test/problem_utils.h:209-243): the reported residuals equal the ones recomputed on the host from (x, y, s) in
    fp64, s is in the cone and y in the dual cone, the duality gap is what the objectives say."""
    from scs_b200 import problems
    prob = problems.config(cfg)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(lib, verbose=0, max_iters=steps, eps_abs=1e-12, eps_rel=1e-12)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    status = lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    assert status == 2 and info.iter == steps, (status, info.status)          # solved (inaccurate - reached max_iters)
    A = prob["A"]
    res_pri = np.abs(problems.csc_matvec(A, x) + s - prob["b"]).max()
    res_dual = np.abs(problems.csc_rmatvec(A, y) + prob["c"]).max()
    scale = max(1.0, np.abs(prob["b"]).max(), np.abs(prob["c"]).max())
    assert abs(res_pri - info.res_pri) <= 1e-9 * scale, (res_pri, info.res_pri)
    assert abs(res_dual - info.res_dual) <= 1e-9 * scale, (res_dual, info.res_dual)
    pobj, dobj = float(prob["c"] @ x), -float(prob["b"] @ y)
    assert abs(pobj - info.pobj) <= 1e-9 * max(1.0, abs(pobj)) and abs(dobj - info.dobj) <= 1e-9 * max(1.0, abs(dobj))
    assert abs(abs(pobj - dobj) - info.gap) <= 1e-9 * max(1.0, abs(pobj), abs(dobj))
    # cone membership of the returned s and y (projection is idempotent on them)
    smax = max(1.0, np.abs(s).max())
    assert np.abs(problems.proj_cone(s, prob["cone"]) - s).max() <= 1e-9 * smax
    ymax = max(1.0, np.abs(y).max())
    assert np.abs(problems.proj_dual_cone(y, prob["cone"]) - y).max() <= 1e-9 * ymax


def test_long_row_mode_matches_reference(lib, reflib):
    """v3 long-row mode (virtual rows + combine pass, the default since round 2): both operators and a KKT
    solve on matrices with 700-entry columns and 40-entry rows / very long rows."""
    from scs_b200 import problems
    reflib._scs_accum_by_a.argtypes = [PP(capi.ScsMatrix), capi.c_double_p, capi.c_double_p]
    reflib._scs_accum_by_atrans.argtypes = [PP(capi.ScsMatrix), capi.c_double_p, capi.c_double_p]
    for m, n, col_nnz, seed in ((3000, 50, 700, 4), (64, 5000, 40, 5), (20000, 400, 300, 6)):
        rng = np.random.default_rng(seed)
        A = problems.random_sparse_csc(m, n, col_nnz, rng)
        hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
        dr = np.empty(n + m + 1)
        dr[:n], dr[n:] = 1e-6, 10.0
        w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
        assert w
        try:
            x, yv = rng.standard_normal(n), rng.standard_normal(m)
            mine, ref = np.zeros(m), np.zeros(m)
            assert lib.scs_b200_accum_by_a(w, capi.dptr(x), capi.dptr(mine), 0) == 0
            reflib._scs_accum_by_a(C.byref(hp.A), capi.dptr(x), capi.dptr(ref))
            assert rel(mine, ref, 0.0) <= 1e-13
            mine, ref = np.ones(n), np.ones(n)
            assert lib.scs_b200_accum_by_atrans(w, capi.dptr(yv), capi.dptr(mine), 1) == 0
            reflib._scs_accum_by_atrans(C.byref(hp.A), capi.dptr(yv), capi.dptr(ref))
            assert rel(mine, ref, 0.0) <= 1e-13
            rhs = rng.standard_normal(n + m)
            wr = reflib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
            a, b = rhs.copy(), rhs.copy()
            assert lib.scs_solve_lin_sys(w, capi.dptr(a), None, 1e-12) == 0
            assert reflib.scs_solve_lin_sys(wr, capi.dptr(b), None, 1e-12) == 0
            reflib.scs_free_lin_sys_work(wr)
            assert rel(a, b, 0.0) <= 1e-10
        finally:
            lib.scs_free_lin_sys_work(w)

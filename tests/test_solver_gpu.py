"""Whole-solver parity on the GPU: the device-resident scs_init/scs_solve/
scs_finish against the reference CPU-indirect solver (its answers recorded under
tests/golden/reference/) on the same problems, plus the known optimum the generator builds in."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi, problems
from reference_replay import rel

pytestmark = pytest.mark.gpu


def solve_with(lib, prob, **over):
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], prob.get("P"))
    st = capi.default_settings(lib, verbose=0, **over)
    n, m = hp.n, hp.m
    x, y, s = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    status = lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    return status, info, x, y, s


def small_problem(kind, seed=0):
    if kind == "lp":
        return problems.make_problem(300, 100, 6, {"z": 30, "l": 270}, seed)
    if kind == "socp":
        return problems.make_problem(400, 100, 8, {"z": 40, "l": 120, "q": [3, 7, 30, 200]}, seed)
    if kind == "box":
        rng = np.random.default_rng(seed)
        bl = -rng.uniform(0.5, 1.5, 99)
        bu = rng.uniform(0.5, 1.5, 99)
        return problems.make_problem(300, 80, 6, {"z": 20, "l": 180, "bl": bl, "bu": bu}, seed)
    if kind == "sdp":
        return problems.make_problem(60 + 21 + 36 + 10, 40, 8, {"l": 60, "s": [6, 8, 4]}, seed)
    if kind == "mixed":
        rng = np.random.default_rng(seed)
        bl = -rng.uniform(0.5, 1.5, 19)
        bu = rng.uniform(0.5, 1.5, 19)
        cone = {"z": 10, "l": 50, "bl": bl, "bu": bu, "q": [5, 9000, 12], "s": [5, 1, 9]}
        m = capi.cone_rows(cone)
        return problems.make_problem(m, 300, 12, cone, seed)
    raise KeyError(kind)


@pytest.mark.parametrize("kind", ["lp", "socp", "box", "sdp", "mixed"])
def test_solver_matches_reference(lib, reflib, kind):
    prob = small_problem(kind, seed=11)
    eps = {"lp": 1e-9, "sdp": 1e-9, "socp": 1e-6, "box": 1e-4, "mixed": 1e-5}[kind]
    st_m, info_m, x, y, s = solve_with(lib, prob, eps_abs=eps, eps_rel=eps, max_iters=30000)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, eps_abs=eps, eps_rel=eps, max_iters=30000)
    assert info_r.lin_sys_solver.decode() == "sparse-indirect-scs"   # really the reference
    print(f"\n[{kind}] mine: {info_m.status.decode()} it={info_m.iter} pobj={info_m.pobj:.12e} "
          f"res_pri={info_m.res_pri:.2e} | ref: {info_r.status.decode()} it={info_r.iter} pobj={info_r.pobj:.12e} | "
          f"delta_iter={info_m.iter - info_r.iter:+d}")
    assert st_m == st_r == 1
    assert info_m.lin_sys_solver.decode().startswith("sparse-indirect-b200")
    # converged quantities agree (trajectories are not reproducible even between two CPU
    # builds of the reference -- SURVEY.md section 7 -- so iteration counts may differ)
    assert abs(info_m.pobj - info_r.pobj) <= 100 * eps * max(1.0, abs(info_r.pobj))
    assert abs(info_m.pobj - prob["opt"]) <= 1000 * eps * max(1.0, abs(prob["opt"]))
    # iteration counts / minimisers are not reproducible WITH Anderson acceleration at eps 1e-9 (AA amplifies
    # rounding; degenerate LPs; the reference's own two builds differ by >10x here, DESIGN.md section 4): delta_iter
    # is REPORTED above and bounded loosely; the |delta| <= 25 gate of SURVEY 8(d) is applied where the trajectory is
    # reproducible -- AA off, default eps -- in tests/test_parity_configs_gpu.py
    assert info_m.iter <= 4 * info_r.iter + 100
    # the reference's own universal checker, recomputed here (test/problem_utils.h:107-249)
    A = prob["A"]
    res_pri = np.abs(problems.csc_matvec(A, x) + s - prob["b"]).max()
    res_dual = np.abs(problems.csc_rmatvec(A, y) + prob["c"]).max()
    assert abs(res_pri - info_m.res_pri) < 1e-10
    assert abs(res_dual - info_m.res_dual) < 1e-10
    # cone membership of s (primal) and y (dual)
    assert np.abs(problems.proj_cone(s, prob["cone"]) - s).max() < 1e-5
    assert np.abs(problems.proj_dual_cone(y, prob["cone"]) - y).max() < 1e-5


@pytest.mark.parametrize("kind", ["lp", "socp", "box", "sdp", "mixed"])
def test_one_iteration_matches_reference(lib, reflib, kind):
    """max_iters=1: equilibration + KKT solve at tol 1e-12 + cone projection + un-normalisation,
    end to end through scs(); agreement to 1e-10 relative on x, y, s and the ScsInfo residuals (north star)."""
    prob = small_problem(kind, seed=11)
    st_m, info_m, x, y, s = solve_with(lib, prob, max_iters=1)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, max_iters=1)
    assert info_r.lin_sys_solver.decode() == "sparse-indirect-scs"
    assert st_m == st_r and info_m.iter == info_r.iter == 1
    errs = {}
    for a, b, nm in ((x, xr, "x"), (y, yr, "y"), (s, sr, "s")):
        errs[nm] = rel(a, b)
    for fld in ("pobj", "dobj", "res_pri", "res_dual", "gap"):
        a, b = getattr(info_m, fld), getattr(info_r, fld)
        errs[fld] = abs(a - b) / max(1.0, abs(b))
    print(f"\n[{kind}] one-iteration parity: " + " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v <= 1e-10, (kind, k, v)


def qp_problem(seed):
    """min 1/2 x'Px + c'x s.t. Ax + s = b, s in K: P = B'B + 0.1 I, upper triangle in CSC as
    include/scs.h:60-77 requires (reference QP path: accum_by_p, linsys/scs_matrix.c:206-225)."""
    import scipy.sparse as sp
    prob = problems.make_problem(400, 100, 8, {"z": 40, "l": 120, "q": [3, 7, 30, 200]}, seed)
    rng = np.random.default_rng(seed + 1000)
    n = prob["n"]
    B = sp.random(30, n, density=0.08, random_state=np.random.RandomState(seed), format="csr")
    P = sp.triu(B.T @ B + 0.1 * sp.identity(n), format="csc")
    P.sort_indices()
    prob = dict(prob)
    prob["P"] = (P.data.copy(), P.indices.astype(np.int32), P.indptr.astype(np.int32), (n, n))
    prob["opt"] = None
    del rng
    return prob


def test_qp_matches_reference(lib, reflib):
    """Quadratic objective through the device-resident driver: P in the CG operator and the
    preconditioner, P x in the residuals, x'Px in the objective; one iteration sharp, converged loose."""
    prob = qp_problem(21)
    st_m, info_m, x, y, s = solve_with(lib, prob, max_iters=1)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, max_iters=1)
    assert st_m == st_r and info_m.iter == info_r.iter == 1
    for a, b, nm in ((x, xr, "x"), (y, yr, "y"), (s, sr, "s")):
        err = rel(a, b)
        assert err <= 1e-10, (nm, err)
    for fld in ("pobj", "dobj", "res_pri", "res_dual", "gap"):
        a, b = getattr(info_m, fld), getattr(info_r, fld)
        assert abs(a - b) <= 1e-10 * max(1.0, abs(b)), (fld, a, b)
    eps = 1e-7
    st_m, info_m, x, y, s = solve_with(lib, prob, eps_abs=eps, eps_rel=eps, max_iters=30000)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, eps_abs=eps, eps_rel=eps, max_iters=30000)
    print(f"\n[qp] mine it={info_m.iter} pobj={info_m.pobj:.10e} | ref it={info_r.iter} pobj={info_r.pobj:.10e}")
    assert st_m == st_r == 1
    assert abs(info_m.pobj - info_r.pobj) <= 100 * eps * max(1.0, abs(info_r.pobj))
    assert rel(x, xr) <= 1e-4   # strictly convex in x: unique minimiser


def exp_pow_problem(seed, n=60):
    """Strictly feasible primal-dual pair over z x l x SOC x exp(primal, dual) x power(primal, dual):
    s* in int K, y* in int K*, b = A x* + s*, c = -A'y*  (optimum exists; its value is not known in
    closed form, the reference is the judge). Cone order: include/scs.h:121-172."""
    rng = np.random.default_rng(seed)
    ep, ed = 7, 5
    pw = [0.3, 0.5, 0.8, -0.25, -0.6]
    cone = {"z": 6, "l": 20, "q": [4, 9], "ep": ep, "ed": ed, "p": pw}
    m = capi.cone_rows(cone)
    A = problems.random_sparse_csc(m, n, 9, rng)
    s = np.zeros(m)
    y = rng.uniform(-1, 1, m)                    # zero cone: s = 0, y free
    o = cone["z"]
    s[o:o + 20] = rng.uniform(0.5, 1.5, 20); y[o:o + 20] = rng.uniform(0.5, 1.5, 20); o += 20
    for q in cone["q"]:
        for v in (s, y):
            t = rng.standard_normal(q - 1)
            v[o] = np.linalg.norm(t) + rng.uniform(0.2, 1.0)
            v[o + 1:o + q] = t
        o += q

    def exp_primal(v):   # (r, s, t): s > 0, t > s exp(r/s)
        r, sv = rng.standard_normal(), rng.uniform(0.5, 1.5)
        v[:] = (r, sv, sv * np.exp(r / sv) + rng.uniform(0.1, 1.0))

    def exp_dual(v):     # (u, v, w): u < 0, e w > -u exp(v/u)
        u, vv = -rng.uniform(0.5, 1.5), rng.standard_normal()
        v[:] = (u, vv, -u * np.exp(vv / u) / np.e + rng.uniform(0.1, 1.0))

    for i in range(ep + ed):
        (exp_primal if i < ep else exp_dual)(s[o:o + 3])
        (exp_dual if i < ep else exp_primal)(y[o:o + 3])
        o += 3

    def pow_primal(v, a):   # x^a y^(1-a) > |r|
        xx, yy = rng.uniform(0.5, 1.5, 2)
        v[:] = (xx, yy, rng.uniform(-0.5, 0.5) * xx ** a * yy ** (1 - a))

    def pow_dual(v, a):     # (u/a)^a (v/(1-a))^(1-a) > |w|
        uu, vv = rng.uniform(0.5, 1.5, 2)
        v[:] = (uu, vv, rng.uniform(-0.5, 0.5) * (uu / a) ** a * (vv / (1 - a)) ** (1 - a))

    for a in pw:
        if a >= 0:
            pow_primal(s[o:o + 3], a); pow_dual(y[o:o + 3], a)
        else:
            pow_dual(s[o:o + 3], -a); pow_primal(y[o:o + 3], -a)
        o += 3
    assert o == m
    x = rng.uniform(-1, 1, n)
    b = problems.csc_matvec(A, x) + s
    c = -problems.csc_rmatvec(A, y)
    return {"A": A, "b": b, "c": c, "cone": cone, "n": n, "m": m, "opt": None}


def test_exp_and_power_cones_match_reference(lib, reflib):
    """SURVEY 8(f)-3: exponential and power cones on the device loop (kernels/cone_triples.cu)."""
    prob = exp_pow_problem(31)
    st_m, info_m, x, y, s = solve_with(lib, prob, max_iters=1)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, max_iters=1)
    assert st_m == st_r and info_m.iter == info_r.iter == 1
    for a, b, nm in ((x, xr, "x"), (y, yr, "y"), (s, sr, "s")):
        err = rel(a, b)
        assert err <= 1e-9, (nm, err)
    eps = 1e-6
    st_m, info_m, x, y, s = solve_with(lib, prob, eps_abs=eps, eps_rel=eps, max_iters=50000)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, eps_abs=eps, eps_rel=eps, max_iters=50000)
    print(f"\n[exp/pow] mine it={info_m.iter} pobj={info_m.pobj:.10e} | ref it={info_r.iter} pobj={info_r.pobj:.10e}")
    assert st_m == st_r == 1
    assert abs(info_m.pobj - info_r.pobj) <= 100 * eps * max(1.0, abs(info_r.pobj))
    assert abs(info_m.pobj - info_m.dobj) <= 100 * eps * max(1.0, abs(info_m.pobj))
    A = prob["A"]
    assert abs(np.abs(problems.csc_matvec(A, x) + s - prob["b"]).max() - info_m.res_pri) < 1e-10


def test_c1_shape_default_settings(lib, reflib):
    """BASELINE configs[0]: n=1000, m=4000, 32 nnz/col SOCP at default eps=1e-4."""
    prob = problems.config("C1")
    st_m, info_m, x, y, s = solve_with(lib, prob)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob)
    print(f"\n[C1] mine it={info_m.iter} pobj={info_m.pobj:.8e} solve={info_m.solve_time:.1f}ms "
          f"(lin {info_m.lin_sys_time:.1f} cone {info_m.cone_time:.1f} aa {info_m.accel_time:.1f}) | "
          f"ref it={info_r.iter} pobj={info_r.pobj:.8e} solve={info_r.solve_time:.1f}ms")
    assert st_m == st_r == 1
    assert abs(info_m.pobj - info_r.pobj) <= 2e-3 * max(1.0, abs(info_r.pobj))
    assert info_m.iter <= 4 * info_r.iter + 100


def test_max_iters_and_warm_start(lib):
    prob = small_problem("socp", seed=5)
    st1, info1, x, y, s = solve_with(lib, prob, max_iters=7)
    assert info1.iter == 7 and st1 == 2          # solved (inaccurate - reached max_iters)
    assert b"max_iters" in info1.status
    # warm start from a converged solution needs (almost) no iterations
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(lib, verbose=0, eps_abs=1e-7, eps_rel=1e-7)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    assert w
    n, m = hp.n, hp.m
    x, y, s = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    assert lib.scs_solve(w, C.byref(sol), C.byref(info), 0) == 1
    cold_iters = info.iter
    assert lib.scs_solve(w, C.byref(sol), C.byref(info), 1) == 1
    assert info.iter <= max(25, cold_iters // 4)
    # scs_update with new b, c then re-solve
    b2 = prob["b"] * 1.01
    assert lib.scs_update(w, capi.dptr(b2), None) == 0
    assert lib.scs_solve(w, C.byref(sol), C.byref(info), 1) == 1
    lib.scs_finish(w)


def test_malformed_cone_fails_loudly(lib):
    prob = small_problem("lp", seed=1)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    hp.cone.l -= 4
    hp.cone.cssize = 1          # claims one complex PSD block but gives no array: scs_init must refuse (no crash)
    st = capi.default_settings(lib, verbose=0)
    assert not lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))


def test_complex_psd_cone_matches_reference(lib, reflib):
    """Complex (Hermitian) PSD blocks in the device loop (kernels/cones_complex.cu; reference cones.c:1072-1156), mixed
    with every other dense cone type. The known optimum is built with the reference's own dual-cone projection:
    y = Pi_K*(z), s = y - z, b = A x + s, c = -A'y (same construction as test/problem_utils.h:22-81)."""
    cone = {"z": 3, "l": 10, "q": [4, 9], "s": [3, 5], "cs": [2, 5, 4, 1]}
    m = capi.cone_rows(cone)
    n = 40
    rng = np.random.default_rng(77)
    A = problems.random_sparse_csc(m, n, 9, rng)
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.restype = C.c_int
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    k, keep = capi.make_cone(cone)
    cw = reflib._scs_init_cone(C.byref(k), m)
    zz = rng.uniform(-1, 1, m)
    y = zz.copy()
    assert reflib._scs_proj_dual_cone(capi.dptr(y), cw, None, None) == 0
    reflib._scs_finish_cone(cw)
    sv = y - zz
    x0 = rng.uniform(-1, 1, n)
    prob = {"A": A, "b": problems.csc_matvec(A, x0) + sv, "c": -problems.csc_rmatvec(A, y), "cone": cone}
    opt = float(prob["c"] @ x0)
    st_m, info_m, x, yy, s = solve_with(lib, prob, max_iters=1)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, max_iters=1)
    assert st_m == st_r and info_m.iter == info_r.iter == 1
    for a, b, nm in ((x, xr, "x"), (yy, yr, "y"), (s, sr, "s")):
        err = rel(a, b)
        assert err <= 1e-10, (nm, err)
    eps = 1e-7
    st_m, info_m, x, yy, s = solve_with(lib, prob, eps_abs=eps, eps_rel=eps, max_iters=50000)
    st_r, info_r, xr, yr, sr = solve_with(reflib, prob, eps_abs=eps, eps_rel=eps, max_iters=50000)
    print(f"\n[complex PSD] mine it={info_m.iter} pobj={info_m.pobj:.10e} | ref it={info_r.iter} pobj={info_r.pobj:.10e} "
          f"| known optimum {opt:.10e}")
    assert st_m == st_r == 1
    assert abs(info_m.pobj - info_r.pobj) <= 100 * eps * max(1.0, abs(info_r.pobj))
    assert abs(info_m.pobj - opt) <= 1000 * eps * max(1.0, abs(opt))


def test_csv_trace_matches_reference(lib, reflib, tmp_path):
    """log_csv_filename (reference src/rw.c:707-861): same columns, same format; the row of iteration 0 -- everything
    up to and including the first cone projection and residual computation -- agrees with the reference's to 1e-9;
    later rows are compared loosely (CG at the adaptive tolerance, tests/test_reference_reproducibility_cpu.py)."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import csv_trace_diff
    prob = small_problem("socp", seed=4)
    mine, ref = str(tmp_path / "mine.csv"), str(tmp_path / "ref.csv")
    over = dict(max_iters=30, acceleration_lookback=0, eps_abs=1e-12, eps_rel=1e-12)
    st_m, info_m, *_ = solve_with(lib, prob, log_csv_filename=mine.encode(), **over)
    st_r, info_r, *_ = solve_with(reflib, prob, log_csv_filename=ref.encode(), **over)
    reflib.written_file(ref)
    assert st_m == st_r
    hm, rm = csv_trace_diff.read(mine)
    hr, rr = csv_trace_diff.read(ref)
    assert hm[:62] == hr[:62]                       # identical column names, identical order
    assert len(rm) == len(rr) == 31                 # one row per iteration + the final row
    first, _ = csv_trace_diff.compare(mine, ref, nrows=1)
    worst = max(v[0] for v in first.values())
    print(f"\n[csv trace] iteration-0 row: worst relative difference {worst:.2e} over {len(first)} columns")
    assert worst <= 1e-9, {k: v for k, v in first.items() if v[0] > 1e-9}
    allrows, n = csv_trace_diff.compare(mine, ref)
    print(f"[csv trace] all {n} rows: worst {max(v[0] for v in allrows.values()):.2e} "
          f"(res_pri {allrows['res_pri'][0]:.1e}, pobj {allrows['pobj'][0]:.1e})")
    assert allrows["iter"][0] == 0.0 and allrows["scale"][0] == 0.0


def test_sigint_stops_a_long_solve(lib):
    """Ctrl-C contract of the reference (src/ctrlc.c, src/scs.c:1400-1403): SIGINT during scs_solve ends it with
    SCS_SIGINT (-5) / status "interrupted", NaN solution, and the previous handler is restored afterwards."""
    import os
    import signal
    import threading
    import time
    prob = small_problem("socp", seed=9)
    hits = []
    # a recording Python-level handler for the duration of the test: a SIGINT that lands outside the library's
    # listener window must not raise KeyboardInterrupt (pytest would abort the whole session)
    before = signal.signal(signal.SIGINT, lambda *a: hits.append(1))
    try:
        # two shots: should the first SIGINT land before scs_solve has installed its listener (a slow scs_init on a
        # loaded box) the second one still stops the solve; max_iters is finite so that a missed signal FAILS the
        # test after a minute or two instead of hanging the suite
        timers = [threading.Timer(d, lambda: os.kill(os.getpid(), signal.SIGINT)) for d in (0.5, 3.0)]
        for t in timers:
            t.start()
        try:
            st, info, x, y, s = solve_with(lib, prob, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0, max_iters=300000)
        finally:
            for t in timers:
                t.cancel()
        assert st == -5, (st, info.status)
        assert info.status.decode() == "interrupted" and info.iter == -1 and np.isnan(x).all()
        # the previous handler is back in place: a SIGINT sent now reaches the Python-level handler again
        n0 = len(hits)
        os.kill(os.getpid(), signal.SIGINT)
        for _ in range(100):
            if len(hits) > n0:
                break
            time.sleep(0.01)
        assert len(hits) == n0 + 1
    finally:
        signal.signal(signal.SIGINT, before)
    # and the library still works
    st, info, *_ = solve_with(lib, prob)
    assert st == 1


def test_infeasible_and_unbounded(lib, reflib):
    """status codes on certificates (reference test/problems/infeasible_socp.h, unbounded_socp.h)"""
    rng = np.random.default_rng(2)
    m, n = 60, 20
    A = problems.random_sparse_csc(m, n, 5, rng)
    # infeasible: A x + s = b, s >= 0 with b very negative on rows where A row is zero-ish -> use x>=0, sum x <= -1
    data = np.concatenate([np.ones(n), -np.ones(n)])
    indices = np.concatenate([np.zeros(n), 1 + np.arange(n)]).astype(np.int32)
    order = np.argsort(np.repeat(np.arange(n), 1).tolist() * 2, kind="stable")
    # build CSC: column j has rows 0 (val 1) and 1+j (val -1)
    dat = np.empty(2 * n); idx = np.empty(2 * n, dtype=np.int32)
    dat[0::2] = 1.0; dat[1::2] = -1.0
    idx[0::2] = 0; idx[1::2] = 1 + np.arange(n)
    ptr = (2 * np.arange(n + 1)).astype(np.int32)
    Ainf = (dat, idx, ptr, (n + 1, n))
    b = np.zeros(n + 1); b[0] = -1.0
    c = np.ones(n)
    prob = {"A": Ainf, "b": b, "c": c, "cone": {"l": n + 1}}
    st_m, info_m, *_ = solve_with(lib, prob)
    st_r, info_r, *_ = solve_with(reflib, prob)
    assert st_m == st_r == -2, (st_m, st_r)
    # unbounded: min -sum x s.t. x >= 0 (no upper bound)
    dat = -np.ones(n); idx = np.arange(n, dtype=np.int32); ptr = np.arange(n + 1, dtype=np.int32)
    prob = {"A": (dat, idx, ptr, (n, n)), "b": np.zeros(n), "c": -np.ones(n), "cone": {"l": n}}
    st_m, info_m, *_ = solve_with(lib, prob)
    st_r, info_r, *_ = solve_with(reflib, prob)
    assert st_m == st_r == -1, (st_m, st_r)

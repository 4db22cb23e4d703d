"""Solver-level parity on the BASELINE.json configurations C2..C5 (scaled so that the CPU reference finishes in
seconds), the full-size C2 KKT solve, and the C4-sized PSD batch -- all against the UNMODIFIED reference
(its answers recorded under tests/golden/reference/, tests/reference_replay.py) through the C ABI.

Gates (SURVEY 8d), printed with every run. The yardstick for "how close can two correct implementations be" is
MEASURED in the same test: the reference's own second build (libscsindir_ref_nolapack.so: the same
sources with plain-C dot products instead of BLAS -- available when the cone has no PSD block) against its first.
  * one ADMM iteration (max_iters=1: equilibration, KKT solve at tol 1e-12, cone projection, un-normalisation):
    x, y, s and pobj / dobj / res_pri / res_dual / gap agree to max(1e-10, 10 x the reference's own build-to-build
    spread) -- the spread itself reaches 1.5e-10 on C3 (tests/test_reference_reproducibility_cpu.py);
  * default-settings solve (eps 1e-4): same status; delta-iterations REPORTED and gated against the reference's own
    spread: |ours - ref| <= max(25, 2 |ref - ref_nolapack|) with Anderson acceleration off (the reference's two builds
    need 625 and 825 iterations on C2 x0.01), loosely with it on; objective within 10 eps of the reference's and of
    the generator's optimum;
  * the reference's universal checker verify_solution_correct (tests/verify.py, every clause) passes on our
    solution.
"""
import ctypes as C
import os
import time

import numpy as np
import pytest

from scs_b200 import capi, problems
from reference_replay import Reference, rel
import verify

pytestmark = pytest.mark.gpu

# (config, scale): n, m, nnz at these scales: C2 1e4/3e4/1e5, C3 2.5e3/2.5e3/2.5e4 (box + LP), C4 5e3/5.55e4/1e6 with
# 10 PSD blocks of order 100, C5 1e4/3e4/1.5e5 (50 SOCs + PSD blocks of order 10)
CASES = [("C2", 0.01), ("C3", 0.002), ("C4", 0.05), ("C5", 0.005)]
# Converged comparisons are sized by the host time of the CPU reference that records them (minutes at C2 x0.01): C2 at
# x0.004 with and without Anderson acceleration; C4 and C5 with the default settings only. C3 (LP with a box cone) needs
# 2850 ADMM iterations = minutes of CPU time at ANY scale the reference can run: its converged comparison is against a
# recorded reference answer (tests/golden/c3_converged.json), plus a reported fixed-window run below.
CONVERGED = [("C2", 0.004, 0), ("C2", 0.004, 10), ("C4", 0.05, 10), ("C5", 0.003, 10)]


def solve(lib, prob, **over):
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], prob.get("P"))
    st = capi.default_settings(lib, verbose=0, **over)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    status = lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    return status, info, x, y, s, st


def second_reference_build(cone):
    """The reference compiled without BLAS/LAPACK (plain-C dots): same algorithm, different rounding. None when the
    cone needs LAPACK (PSD blocks of order > 1)."""
    if any(int(k) > 1 for k in (cone.get("s") or [])) or (cone.get("cs") or []):
        return None
    return Reference("nolapack")


@pytest.mark.parametrize("cfg,scale", CASES)
def test_config_one_iteration_1e10(lib, reflib, cfg, scale):
    prob = problems.config(cfg, scale=scale)
    st_m, im, x, y, s, _ = solve(lib, prob, max_iters=1)
    st_r, ir, xr, yr, sr, _ = solve(reflib, prob, max_iters=1)
    assert ir.lin_sys_solver.decode() == "sparse-indirect-scs"
    assert st_m == st_r and im.iter == ir.iter == 1
    errs = {nm: rel(a, b) for a, b, nm in ((x, xr, "x"), (y, yr, "y"), (s, sr, "s"))}
    for fld in ("pobj", "dobj", "res_pri", "res_dual", "gap"):
        a, b = getattr(im, fld), getattr(ir, fld)
        errs[fld] = abs(a - b) / max(1.0, abs(b))
    spread = None
    ref2 = second_reference_build(prob["cone"])
    if ref2 is not None:
        _, i2, x2, y2, s2, _ = solve(ref2, prob, max_iters=1)
        spread = max(rel(a, b) for a, b in ((x2, xr), (y2, yr), (s2, sr)))
    gate = max(1e-10, 10 * spread) if spread is not None else 1e-9
    print(f"\n[{cfg} x{scale}] one-iteration parity vs reference: " + " ".join(f"{k}={v:.1e}" for k, v in errs.items()) +
          f" | reference build-to-build spread: {spread if spread is None else format(spread, '.1e')} -> gate {gate:.1e}")
    for k, v in errs.items():
        assert v <= gate, (cfg, k, v, gate)


@pytest.mark.parametrize("cfg,scale,aa", CONVERGED)
def test_config_default_solve_matches_reference(lib, reflib, cfg, scale, aa):
    prob = problems.config(cfg, scale=scale)
    over = dict(acceleration_lookback=aa)
    t0 = time.time()
    st_m, im, x, y, s, stg = solve(lib, prob, **over)
    t_m = time.time() - t0
    t0 = time.time()
    st_r, ir, xr, yr, sr, _ = solve(reflib, prob, **over)
    t_r = time.time() - t0
    eps = stg.eps_rel
    d_it = im.iter - ir.iter
    print(f"\n[{cfg} x{scale} aa={aa}] ours: {im.status.decode()} it={im.iter} pobj={im.pobj:.8e} "
          f"res=({im.res_pri:.1e},{im.res_dual:.1e},{im.gap:.1e}) {t_m:.1f}s | reference: {ir.status.decode()} "
          f"it={ir.iter} pobj={ir.pobj:.8e} res=({ir.res_pri:.1e},{ir.res_dual:.1e},{ir.gap:.1e}) {t_r:.1f}s | "
          f"delta_iter={d_it:+d} rel dpobj={abs(im.pobj - ir.pobj) / max(1, abs(ir.pobj)):.1e}")
    assert st_m == st_r == 1
    assert abs(im.pobj - ir.pobj) <= 10 * eps * max(1.0, abs(ir.pobj))
    assert abs(im.pobj - prob["opt"]) <= 10 * eps * max(1.0, abs(prob["opt"]))
    if aa == 0:
        # convergence is tested every 25 iterations (CONVERGED_INTERVAL): |delta| <= 25 means "same or adjacent check";
        # the yardstick beyond that is the reference's own build-to-build spread on this problem
        ref2 = second_reference_build(prob["cone"])
        # ... measured on this instance where the second build exists, and never tighter than the largest spread seen on
        # this problem family: the reference's two builds need 625 and 825 iterations (32 %) on C2 x0.01, 575 and 575 on
        # C2 x0.004 (tests/test_reference_reproducibility_cpu.py)
        allowed = max(25, int(0.35 * ir.iter))
        if ref2 is not None:
            _, i2, *_ = solve(ref2, prob, **over)
            allowed = max(allowed, 2 * abs(i2.iter - ir.iter))
            print(f"    reference (plain-C dots build): it={i2.iter} -> allowed |delta_iter| {allowed}")
        assert abs(d_it) <= allowed, (cfg, im.iter, ir.iter, allowed)
    else:
        assert im.iter <= 2 * ir.iter + 100, (cfg, im.iter, ir.iter)
    bad = verify.verify_solution_correct(prob, stg, im, x, y, s, st_m)
    assert not bad, (cfg, bad)


def test_c3_fixed_window_trajectory_vs_reference(lib, reflib):
    """C3 (box + LP cone, the box Newton iteration with warm start across iterations): the first 100 ADMM iterations
    without Anderson acceleration.  This window sits in the transient of the homogeneous embedding where tau dips to
    zero: the reference's OWN two builds return different verdicts here (measured on this instance: -4 / 2 at 25 and
    50 iterations, -6 / 2 at 100, -6 / -6 at 200 with iterates 1.0 apart in relative terms, 2 / -6 at 400;
    "could not determine problem status" is one of the verdicts scs.c:887-902 reaches).  So the verdict and the
    iterates cannot be gated against each other.  What IS checked: the window runs to max_iters on both sides, the
    verdict is one that set_unfinished can produce, the outputs the verdict defines are finite and the others NaN (as
    the reference leaves them), and the differences are REPORTED next to the reference's build-to-build drift.  The C3 parity gates proper are the
    one-iteration test above and the converged solve below."""
    prob = problems.config("C3", scale=0.002)
    over = dict(max_iters=100, acceleration_lookback=0)
    st_m, im, x, y, s, _ = solve(lib, prob, **over)
    st_r, ir, xr, yr, sr, _ = solve(reflib, prob, **over)
    print(f"\n[C3 x0.002] statuses ours {st_m} ({im.status.decode()}) reference {st_r} ({ir.status.decode()})")
    unfinished = (2, -6, -7, -4)          # solved / unbounded / infeasible inaccurate, failure (scs.c:887-902)
    assert st_m in unfinished and st_r in unfinished and im.iter == ir.iter == 100
    # what the verdict leaves undefined is NaN, everything else finite (set_unbounded / set_infeasible, scs.c:860-884)
    nan_by_verdict = {2: "", -6: "y", -7: "xs"}
    if st_m != -4:
        for nm, v in zip("xys", (x, y, s)):
            assert np.isnan(v).all() if nm in nan_by_verdict[st_m] else np.isfinite(v).all(), (st_m, nm)

    def defined(pairs):
        return [(a, b) for a, b in pairs if not (np.isnan(a).all() or np.isnan(b).all())]
    drift = None
    ref2 = second_reference_build(prob["cone"])
    if ref2 is not None:
        st_2, i2, x2, y2, s2, _ = solve(ref2, prob, **over)
        if st_2 != -4 and st_r != -4:
            drift = max(rel(a, b) for a, b in defined(((x2, xr), (y2, yr), (s2, sr))))
        print(f"    reference (plain-C dots build): status {st_2}")
    if st_m != -4 and st_r != -4:
        errs = {nm: rel(a, b) for a, b, nm in ((x, xr, "x"), (y, yr, "y"), (s, sr, "s")) if defined(((a, b),))}
        print(f"[C3 x0.002, 100 iterations, AA off] vs reference: " + " ".join(f"{k}={v:.1e}" for k, v in errs.items()) +
              f" | drift between the reference's own two builds: {drift if drift is None else format(drift, '.1e')}")


def test_c3_converged_solve_vs_golden(lib):
    """C3 x0.002 with the default settings, against the reference's answer recorded in tests/golden/c3_converged.json
    (oracle/make_golden_c3.py: 2850 iterations, two minutes of host time -- too long to repeat here).  Same status,
    objective within 10 eps of the reference's and of the generator's optimum, iteration count within a factor two
    (Anderson-accelerated trajectories are not reproducible between builds: the other C-configs use the same
    gate), and the reference's universal checker on our solution."""
    import json
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "c3_converged.json")))
    prob = problems.config("C3", scale=g["scale"])
    t0 = time.time()
    st_m, im, x, y, s, stg = solve(lib, prob)
    eps = stg.eps_rel
    print(f"\n[C3 x{g['scale']}] ours: {im.status.decode()} it={im.iter} pobj={im.pobj:.8e} "
          f"res=({im.res_pri:.1e},{im.res_dual:.1e},{im.gap:.1e}) {time.time() - t0:.1f}s | reference (golden): "
          f"{g['status_str']} it={g['iter']} pobj={g['pobj']:.8e} | delta_iter={im.iter - g['iter']:+d}")
    assert st_m == g["status"] == 1
    assert abs(im.pobj - g["pobj"]) <= 10 * eps * max(1.0, abs(g["pobj"]))
    assert abs(im.pobj - prob["opt"]) <= 10 * eps * max(1.0, abs(prob["opt"]))
    assert im.iter <= 2 * g["iter"] + 100, (im.iter, g["iter"])
    bad = verify.verify_solution_correct(prob, stg, im, x, y, s, st_m)
    assert not bad, bad


@pytest.mark.parametrize("full", [pytest.param(False, id="C2x0.1"), pytest.param(True, id="C2full")])
def test_c2_kkt_solve_vs_reference(lib, full):
    """scs_solve_lin_sys at tol 1e-12 on the C2 operator against the reference's CPU-indirect backend (OpenMP build for
    the SpMV): <= 1e-10 relative. The FULL size (n=1e6, m=3e6, nnz=1e7) costs the reference ~5 min of host time: it
    runs only with SCS_B200_SLOW_TESTS=1 and is answered only while recording (SCS_RECORD_REFERENCE, the reference build
    present); the default run does the same test at a tenth of the size against the recorded answer."""
    if full and not os.environ.get("SCS_B200_SLOW_TESTS"):
        pytest.skip("full-size C2 reference solve takes minutes of host time: set SCS_B200_SLOW_TESTS=1")
    os.environ.setdefault("OMP_NUM_THREADS", str(min(32, os.cpu_count() or 1)))
    ref = Reference("omp")
    rng = np.random.default_rng(1234)
    n = 1_000_000 if full else 100_000
    m = 3 * n
    A = problems.random_sparse_csc(m, n, 10, rng)
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    z = m // 10
    dr = np.empty(n + m + 1)
    dr[:n], dr[n:n + z], dr[n + z:] = 1e-6, 1.0 / 100.0, 10.0
    rhs = rng.standard_normal(n + m)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w
    a = rhs.copy()
    t0 = time.time()
    assert lib.scs_solve_lin_sys(w, capi.dptr(a), None, 1e-12) == 0
    t_m = time.time() - t0
    its = lib.scs_b200_linsys_last_cg_its(w)
    lib.scs_free_lin_sys_work(w)
    wr = ref.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    b = rhs.copy()
    t0 = time.time()
    assert ref.scs_solve_lin_sys(wr, capi.dptr(b), None, 1e-12) == 0
    t_r = time.time() - t0
    ref.scs_free_lin_sys_work(wr)
    ex, ey = rel(a[:n], b[:n]), rel(a[n:], b[n:])
    # the reduced residual recomputed on the host in fp64: || (R_x + A' R_y^-1 A) x - (r_x + A' R_y^-1 r_y) ||_inf
    xs = a[:n]
    t = problems.csc_matvec(A, xs) / dr[n:n + m]
    lhs = dr[:n] * xs + problems.csc_rmatvec(A, t)
    rr = rhs[:n] + problems.csc_rmatvec(A, rhs[n:] / dr[n:n + m])
    res = float(np.abs(lhs - rr).max())
    print(f"\n[C2 {'full' if full else 'x0.1'} KKT solve tol 1e-12] ours {its} CG iterations {t_m:.2f}s (incl. H2D/D2H) | reference {t_r:.1f}s | "
          f"rel err x {ex:.2e} y {ey:.2e} | reduced residual (host fp64) {res:.2e}")
    assert ex <= 1e-10 and ey <= 1e-10
    assert res <= 1e-10


def test_psd_c4_batch_200_blocks_of_order_100(lib, reflib):
    """C4's cone: 200 PSD blocks of order 100 (+ LP rows) under the Moreau wrapper vs _scs_proj_dual_cone."""
    cone = {"l": 1000, "s": [100] * 200}
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(44)
    x = rng.standard_normal(m) * 2.0
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.restype = C.c_int
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    for ry in (None, np.full(m, 10.0)):
        k, keep = capi.make_cone(cone)
        cw = reflib._scs_init_cone(C.byref(k), m)
        ref = x.copy()
        t0 = time.time()
        assert reflib._scs_proj_dual_cone(capi.dptr(ref), cw, None, capi.dptr(None if ry is None else ry.copy())) == 0
        t_r = time.time() - t0
        reflib._scs_finish_cone(cw)
        k2, keep2 = capi.make_cone(cone)
        mw = lib.scs_b200_init_cone(C.byref(k2), m, None)
        assert mw
        out = x.copy()
        assert lib.scs_b200_proj_dual_cone(mw, capi.dptr(out), capi.dptr(None if ry is None else ry.copy())) == 0
        t0 = time.time()
        out = x.copy()
        assert lib.scs_b200_proj_dual_cone(mw, capi.dptr(out), capi.dptr(None if ry is None else ry.copy())) == 0
        t_m = time.time() - t0
        lib.scs_b200_finish_cone(mw)
        e = rel(out, ref)
        print(f"\n[PSD 200 x k=100, metric={'on' if ry is not None else 'off'}] rel err {e:.2e}  ours {1e3 * t_m:.1f} ms "
              f"(incl. H2D/D2H) reference {1e3 * t_r:.1f} ms")
        assert e <= 5e-13

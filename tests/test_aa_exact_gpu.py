"""Anderson acceleration (kernels/aa.cu) against exact arithmetic, at every history length 1..31 the library accepts.

Every x_k and f_k handed to scs_b200_aa_apply is an integer vector with entries in [-2^10, 2^10]. The library keeps
its own copy of each input before it overwrites f, so its history S, D, Y and g stays integer (entries below 2^12 in
magnitude), exact in fp64, and every Gram entry is an exact int64 (dim 2^24 << 2^53; so are the squared column norms
the device sums in fp64). The reference solves, per apply and per len,

    type-I   (S'Y + r I) gamma = S'g        type-II   (Y'Y + r I) gamma = Y'g

exactly: in integers (fraction-free elimination, then Fractions) for r = 0 and r = 2^-20, in 400-bit mpmath for
r = reg ||A||_F ||Y||_F. From gamma it forms aa_norm = ||gamma||_2 and f_out = beta (f - D gamma) + (1 - beta)(x - S gamma)
in 64-bit-mantissa long double, 2^-60 or better, far below any gate here.

The device result must agree to c kappa_2(M) len 2^-52, where M is the small system above; f_out's bound is scaled
by |beta| (|f|_inf + ||D|| |gamma|) + |1 - beta| (|x|_inf + ||S|| |gamma|), ||D|| the largest row 2-norm of D. Every
kappa_2(M) is asserted <= 1e6, so no gate is loose enough to pass an O(1) error.

One sequence of mem + 6 applies with min_len = 1 solves every len from 1 to mem and wraps the circular column index.
aa_safeguard is not called (a reset would restart the history); test_aa_gpu.py covers it against the reference.
"""
import ctypes as C
import os
from fractions import Fraction

import mpmath
import numpy as np
import pytest

from scs_b200 import capi, problems

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2.0 ** -52
GATE_C = 64          # the c of the gate above
KAPPA_MAX = 1e6
PINNED_REG = -2.0 ** -20
REG_SCALED = 1e-8
MAX_MEM = 31         # AA_MAX_MEM of kernels/aa.cu


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles_past_grid(k):
    """a dim of k 128-row tiles for every CTA of the TSQR grid (2 CTAs per SM), plus one ragged tile"""
    return k * 2 * num_sms() * 128 + 77


def bareiss_solve(K, b):
    """exact solution of the integer system K x = b (lists of Python ints) as Fractions"""
    n = len(K)
    a = [list(map(int, K[i])) + [int(b[i])] for i in range(n)]
    prev = 1
    for k in range(n - 1):
        p = next(i for i in range(k, n) if a[i][k] != 0)
        if p != k:
            a[k], a[p] = a[p], a[k]
        for i in range(k + 1, n):
            for j in range(k + 1, n + 1):
                a[i][j] = (a[i][j] * a[k][k] - a[i][k] * a[k][j]) // prev
            a[i][k] = 0
        prev = a[k][k]
    assert a[n - 1][n - 1] != 0, "singular reference system"
    x = [Fraction(0)] * n
    for i in range(n - 1, -1, -1):
        s = Fraction(a[i][n]) - sum(a[i][j] * x[j] for j in range(i + 1, n))
        x[i] = s / a[i][i]
    return x


def exact_gamma(M, rhs, reg, nrm2_a, nrm2_y):
    """gamma of (M + r I) gamma = rhs, M and rhs int64; returns (gamma as mpf, r as mpf)"""
    n = M.shape[0]
    if reg <= 0:
        r = Fraction(-reg) if reg < 0 else Fraction(0)
        den = r.denominator       # 2^20 or 1: scale to an integer system
        K = [[int(M[i, j]) * den + (r.numerator if i == j else 0) for j in range(n)] for i in range(n)]
        g = bareiss_solve(K, [int(v) * den for v in rhs])
        return [mpmath.mpf(x.numerator) / x.denominator for x in g], mpmath.mpf(r.numerator) / r.denominator
    r = mpmath.mpf(reg) * mpmath.sqrt(int(nrm2_a)) * mpmath.sqrt(int(nrm2_y))
    K = mpmath.matrix([[mpmath.mpf(int(M[i, j])) + (r if i == j else 0) for j in range(n)] for i in range(n)])
    g = mpmath.lu_solve(K, mpmath.matrix([mpmath.mpf(int(v)) for v in rhs]))
    return [g[i] for i in range(n)], r


def split2(v):
    """mpf values -> (hi, lo) float64 arrays with hi + lo = v to ~2^-106 relative"""
    hi = np.array([float(x) for x in v])
    lo = np.array([float(x - mpmath.mpf(h)) for x, h in zip(v, hi)])
    return hi, lo


def ld_combine(base, cols, hi, lo):
    """base - cols' (hi + lo) in long double; cols (len, dim) integer"""
    L = np.longdouble
    c = cols.astype(L)
    return base.astype(L) - (hi.astype(L) @ c) - (lo.astype(L) @ c)


def run_sequence(lib, dim, mem, type1, reg=PINNED_REG, relax=1.0, seed=0):
    """Drives one mem + 6 apply sequence; returns the list of (len, ratio) and the failures found.
    ratio = observed error / gate, the larger of aa_norm's and f_out's."""
    with mpmath.workdps(121):
        return _run_sequence(lib, dim, mem, type1, reg, relax, seed)


def _run_sequence(lib, dim, mem, type1, reg, relax, seed):
    rng = np.random.default_rng([dim, mem, type1, seed, int(relax * 10), 0 if reg == 0 else (1 if reg > 0 else 2)])
    mem_c = min(mem, dim)
    h = lib.scs_b200_aa_init(dim, mem, 1, type1, reg, relax, 1.0, 1e10, 5, 0)
    assert h
    S = np.zeros((mem_c, dim), np.int64)
    D = np.zeros((mem_c, dim), np.int64)
    Y = np.zeros((mem_c, dim), np.int64)
    AY = np.zeros((mem_c, mem_c), np.int64)   # Gram of the filled slots: A' Y, A = S (type-I) or Y (type-II)
    beta = Fraction(relax)
    results, fails = [], []
    x_prev = f_prev = g_prev = None
    try:
        for k in range(mem_c + 6):
            x = rng.integers(-2 ** 10, 2 ** 10 + 1, size=dim)
            f = rng.integers(-2 ** 10, 2 ** 10 + 1, size=dim)
            fo = f.astype(np.float64)
            ret = lib.scs_b200_aa_apply(h, capi.dptr(fo), capi.dptr(x.astype(np.float64)))
            g = x - f
            if k == 0:
                assert ret == 0 and np.array_equal(fo, f)
                x_prev, f_prev, g_prev = x, f, g
                continue
            idx = (k - 1) % mem_c
            S[idx], D[idx], Y[idx] = x - x_prev, f - f_prev, g - g_prev
            x_prev, f_prev, g_prev = x, f, g
            n = min(k, mem_c)
            A = S if type1 else Y
            AY[idx, :n] = Y[:n] @ A[idx]
            AY[:n, idx] = A[:n] @ Y[idx]
            M = AY[:n, :n]
            rhs = A[:n] @ g
            gam, r = exact_gamma(M, rhs, reg, (A * A).sum(), (Y * Y).sum())
            kappa = float(np.linalg.cond(M.astype(np.float64) + float(r) * np.eye(n)))
            assert kappa <= KAPPA_MAX, (n, kappa)
            tol = GATE_C * kappa * n * EPS
            st = lib.scs_b200_aa_get_stats(h)
            norm = mpmath.sqrt(mpmath.fsum(v * v for v in gam))
            hi, lo = split2(gam)
            out = ld_combine(f, D[:n], hi, lo)
            gn = float(norm)
            dnorm = float(np.sqrt((D[:n].astype(np.float64) ** 2).sum(0)).max())
            scale = abs(float(beta)) * (np.abs(f).max() + dnorm * gn)
            if beta != 1:
                xs = ld_combine(x, S[:n], hi, lo)
                out = out * np.longdouble(beta.numerator) / beta.denominator \
                    + xs * np.longdouble((1 - beta).numerator) / (1 - beta).denominator
                snorm = float(np.sqrt((S[:n].astype(np.float64) ** 2).sum(0)).max())
                scale += abs(float(1 - beta)) * (np.abs(x).max() + snorm * gn)
            e_norm = abs(ret - gn) / (tol * gn)
            e_f = float(np.abs(fo.astype(np.longdouble) - out).max()) / (tol * scale)
            e_r = abs(st.last_regularization - float(r)) / (float(r) * 1e-13) if r > 0 else \
                (0.0 if st.last_regularization == 0 else np.inf)
            ratio = max(e_norm, e_f)
            results.append((n, ratio))
            ok = ret > 0 and st.n_accept == k and st.last_rank == n and ratio <= 1.0 and e_r <= 1.0
            if not ok:
                fails.append(dict(len=n, apply=k, aa_norm=ret, exact=gn, ratio_norm=e_norm, ratio_f=e_f,
                                  accepted=st.n_accept, rank=st.last_rank, kappa=kappa, reg=st.last_regularization))
    finally:
        lib.scs_b200_aa_finish(h)
    return results, fails


def check(lib, dim, mem, type1, **kw):
    results, fails = run_sequence(lib, dim, mem, type1, **kw)
    worst = max(results, key=lambda t: t[1])
    print(f"\n[aa exact dim={dim} mem={mem} type{'I' if type1 else 'II'} {kw}] {len(results)} applies, "
          f"worst observed/gate {worst[1]:.3e} at len {worst[0]}")
    assert not fails, f"{len(fails)} applies off the exact answer; lens {sorted({d['len'] for d in fails})}; " \
                      f"first {fails[0]}"


@pytest.mark.parametrize("type1", [1, 0])
@pytest.mark.parametrize("tiles", [0, 3])
def test_every_len_mem31(lib, type1, tiles):
    """every len 1..31; dim 129 (one full tile and one row), and >= 3 tiles per CTA (CTAs eliminate onto a non-zero
    triangle, the combine stacks 128 / len triangles per pass over 2 num_sms of them)"""
    check(lib, tiles_past_grid(tiles) if tiles else 129, MAX_MEM, type1)


@pytest.mark.parametrize("mem,type1", [(13, 1), (14, 1), (27, 0), (28, 0)])
def test_trailing_block_thresholds(lib, mem, type1):
    """the memories at which the trailing block of the first reflector block passes 24 columns"""
    check(lib, 4099, mem, type1)


@pytest.mark.parametrize("mem", [10, MAX_MEM])
@pytest.mark.parametrize("where", ["1", "3", "127", "128", "129", "grid-1", "grid+1"])
def test_tile_and_grid_edges(lib, mem, where):
    """dim < mem (the memory is clamped to dim), one partial / exactly one / one plus one tile, one tile per CTA -+ 1"""
    dim = {"grid-1": 2 * num_sms() * 128 - 1, "grid+1": 2 * num_sms() * 128 + 1}.get(where) or int(where)
    check(lib, dim, mem, 1)


@pytest.mark.parametrize("relax", [1.0, 0.7, 1.5])
@pytest.mark.parametrize("reg", [PINNED_REG, 0.0, REG_SCALED])
@pytest.mark.parametrize("type1", [1, 0])
def test_regularization_and_relaxation(lib, type1, reg, relax):
    check(lib, 2500, 20, type1, reg=reg, relax=relax)


# ---- solver level: long memories inside scs()
SOCP = (400, 100, 8, {"z": 40, "l": 120, "q": [3, 7, 30, 200]})   # test_golden_gpu.py's "socp", seed 11


def _solve(lib, **over):
    prob = problems.make_problem(*SOCP, seed=11)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(lib, verbose=0, **over)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    status = lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    return status, info


@pytest.mark.parametrize("lookback,type1", [(20, 1), (31, 1), (31, 0)])
def test_solver_long_memory(lib, lookback, type1):
    """solved, to the reference's recorded objective (tests/golden/solves.npz, 20000 iterations at eps 1e-9)"""
    eps = 1e-6
    ref = float(np.load(os.path.join(ROOT, "tests", "golden", "solves.npz"))["socp__pobj"])
    status, info = _solve(lib, eps_abs=eps, eps_rel=eps, max_iters=100000, acceleration_lookback=lookback,
                          acceleration_type_1=type1)
    print(f"\n[aa lookback {lookback} type{'I' if type1 else 'II'}] status {status} iters {info.iter} "
          f"pobj {info.pobj:.12e} (reference {ref:.12e}) accepted {info.aa_stats.n_accept} "
          f"rejected {info.rejected_accel_steps}")
    assert status == 1
    assert abs(info.pobj - ref) <= 10 * eps * max(1.0, abs(ref))
    assert info.aa_stats.n_accept > 0


def test_solver_lookback_above_device_limit_runs_unaccelerated(lib):
    """the device holds at most AA_MAX_MEM columns: lookback 32 solves without acceleration (INTEGRATION.md)"""
    eps = 1e-4
    status, info = _solve(lib, eps_abs=eps, eps_rel=eps, max_iters=100000, acceleration_lookback=MAX_MEM + 1)
    assert status == 1
    assert info.accepted_accel_steps == 0 and info.rejected_accel_steps == 0
    assert info.aa_stats.n_accept == 0

"""Seeded inputs of the log-det cone tests (tests/test_logdet_*.py, oracle/make_golden_logdet.py).

Two kinds, for orders 1, 2, 3, 5, 16, 40 and 100:

* operator inputs: one log-det cone's rows (t, v, packed X), projected through the public operator
  (scs_b200_proj_dual_cone / the reference's _scs_proj_dual_cone). X = Q diag(lam) Q' with a seeded orthogonal Q and
  eigenvalues chosen for each branch of the vector step: in the cone, on the v = 0 boundary, in the negative dual
  cone, the analytic v <= 0 <= t case, and plain Newton; plus diagonal X with distinct entries, where both
  eigensolvers are exact and the operator isolates the vector step.
* vector-step inputs (t0, v0, e ascending) for the reference's log_cone_proj_wrapper, called directly: cold Newton,
  Newton warm-started from the previous call on the same state, and inputs the reference sends to the interior-point
  method (variant 0), found by a seeded search near the dual-cone boundary, where Newton's v collapses to 0.

The tests require the reference's Newton record (newton_success, iter) exactly, so every input is screened with
tests/logdet_numpy.py on what the vector step actually receives (robust_record). Newton stops when its decrement
falls to 2e-12: a candidate whose last decrement lies within a factor 2 below that threshold, or whose previous one
within a factor 2 above it, is dropped, since there the last bits of a sum (the reference's OpenBLAS order, numpy's
pairwise order, the device's warp order) could decide the count. The same holds for a candidate whose record changes
under relative perturbations of a few 1e-16.
"""
import numpy as np

import logdet_numpy as ln

ORDERS = [1, 2, 3, 5, 16, 40, 100]
KINDS = ["in_cone", "v0_zero", "neg_dual", "analytic", "newton", "diag"]
TOL = 2e-12


def _rng(*key):
    return np.random.default_rng([20261016, *key])


def _q(rng, n):
    q, r = np.linalg.qr(rng.standard_normal((n, n)))
    return q * np.sign(np.diag(r))


def rows(n):
    return 2 + n * (n + 1) // 2


def _robust(stats):
    dec = stats.get("decrements", [])
    if not dec:
        return True
    last = dec[-1]
    if last <= TOL and last >= TOL / 2:
        return False
    if len(dec) >= 2 and dec[-2] <= 2 * TOL:
        return False
    return True


def robust_record(t0, v0, e):
    """the (newton_success, iter) record of the vector step on (t0, v0, e) by the numpy restatement, or None when
    rounding could decide it: Newton stopped within a factor 2 of its threshold, or relative perturbations of a few
    1e-16 of t0 and e change the record (near the interior-point method's boundaries its count hangs on the last
    bits of its input), or all three methods failed"""
    recs = set()
    for k, f in enumerate((1.0, 1 + 2e-16, 1 - 2e-16, 1 + 1e-15)):
        st = ln.State(e.size)
        status, stats = ln.wrapper(t0 * f, v0, e * f, st)
        if status != 0 or (k == 0 and not _robust(stats)):
            return None
        recs.add((stats["newton_success"], stats["iter"]))
    return recs.pop() if len(recs) == 1 else None


def _step_input(tvX, n):
    """the vector step's input for one cone's rows (t, v, packed X): (sqrt2 t, sqrt2 v, eigenvalues of sqrt2 X)"""
    from spectral_numpy import packed_to_sym
    s2 = np.sqrt(2.0)
    return s2 * tvX[0], s2 * tvX[1], np.linalg.eigvalsh(s2 * packed_to_sym(tvX[2:], n))


# the branch each operator kind must take on the projection's own input, as a test on (record, v0)
BRANCH = {
    "in_cone": lambda rec, v0: rec == (ln.NEWTON_SUCCESS, ln.IN_CONE) and v0 > 0,
    "v0_zero": lambda rec, v0: rec == (ln.NEWTON_SUCCESS, ln.IN_CONE) and v0 == 0,
    "neg_dual": lambda rec, v0: rec == (ln.NEWTON_SUCCESS, ln.IN_NEGATIVE_DUAL_CONE),
    "analytic": lambda rec, v0: rec == (ln.NEWTON_SUCCESS, ln.ANALYTICAL_SOL),
    "newton": lambda rec, v0: rec[0] == ln.NEWTON_SUCCESS and rec[1] > 0,
    "diag": lambda rec, v0: rec[0] == ln.NEWTON_SUCCESS and rec[1] > 0,
}


def operator_input(kind, n, trial=0):
    """x of one log-det cone of order n. scs_b200_proj_dual_cone (as the reference's _scs_proj_dual_cone) returns
    x + Pi_K(-R x) / R, so the projection sees -x (R = I) or -R x: x = -(t, v, packed X) with (t, v, X) chosen for the
    branch `kind`. A candidate is kept when the projection's input without r_y takes that branch and the inputs with
    and without r_y both have a robust record (robust_record)."""
    for attempt in range(100):
        rng = _rng(KINDS.index(kind), n, trial, attempt)
        q = _q(rng, n)
        if kind == "in_cone":
            lam = rng.uniform(0.5, 2.0, n)
            t, v = 10.0 * n + 5.0, 1.0
        elif kind == "v0_zero":
            lam = rng.uniform(0.5, 2.0, n)
            t, v = 1.0, 0.0
        elif kind == "neg_dual":
            lam = -rng.uniform(0.5, 2.0, n)
            t, v = -1.0, -100.0 * n
        elif kind == "analytic":
            lam = rng.standard_normal(n)
            t, v = 1.0 + rng.uniform(), -rng.uniform(0.1, 1.0)
        elif kind == "newton":
            lam = rng.standard_normal(n) * 2
            t, v = -abs(rng.standard_normal()) * n, abs(rng.standard_normal()) + 0.1
        else:  # diag: distinct diagonal entries, Newton
            lam = np.sort(rng.uniform(-1.0, 3.0, n)) + np.arange(n) * 1e-3
            q = np.eye(n)
            t, v = -rng.uniform(1.0, 3.0) * n, rng.uniform(0.2, 2.0)
        M = (q * lam) @ q.T if kind != "diag" else np.diag(rng.permutation(lam))
        M = 0.5 * (M + M.T)
        tvX = np.concatenate(([t, v], _packed(M, n)))
        t0, v0, e = _step_input(tvX, n)
        rec = robust_record(t0, v0, e)
        if rec is None or not BRANCH[kind](rec, v0):
            continue
        if robust_record(*_step_input(r_y(n) * tvX, n)) is None:
            continue
        return -tvX
    raise RuntimeError(f"no robust {kind} input of order {n}")


def _packed(M, n):
    """packed lower triangle, column-major, off-diagonals x sqrt2 (SCS's PSD layout)"""
    out = []
    for j in range(n):
        out.append(M[j, j])
        out.extend(np.sqrt(2.0) * M[j + 1:, j])
    return np.array(out)


def operator_cases():
    """[(name, order, x)]"""
    return [(f"{kind}_{n}", n, operator_input(kind, n)) for n in ORDERS for kind in KINDS]


def r_y(n):
    return np.linspace(0.5, 2.0, rows(n))


def _cold(n, trial):
    for attempt in range(50):
        rng = _rng(100, n, trial, attempt)
        e = np.sort(rng.standard_normal(n) * 2)
        t0, v0 = rng.standard_normal(), abs(rng.standard_normal()) + 0.1
        rec = robust_record(t0, v0, e)
        if rec is not None and rec[0] == ln.NEWTON_SUCCESS and rec[1] > 0:
            return t0, v0, e
    raise RuntimeError(f"no robust cold Newton input of order {n}")


def _ipm(n):
    """a point just above the negative dual cone's boundary v0 = t0 (-n - sum log(x0 / t0)): the projection is near 0,
    Newton's v collapses and the reference falls back to IPM variant 0. Near that boundary the IPM's iteration count
    can hang on the last bits of its input; a point is kept only when relative perturbations of a few 1e-16 leave the
    count unchanged and below the IPM's limit of 100."""
    for attempt in range(200):
        rng = _rng(200, n, attempt)
        e = np.sort(-rng.uniform(0.5, 2.0, n))
        t0 = -rng.uniform(0.5, 2.0)
        bound = (-n - np.sum(np.log(e / t0))) * t0
        v0 = bound + abs(bound) * 10.0 ** rng.uniform(-8, -2)
        rec = robust_record(t0, v0, e)
        if rec is not None and rec[0] == ln.IPM0_SUCCESS and rec[1] < 100:
            return t0, v0, e
    return None


def vector_cases():
    """[(name, [(t0, v0, e), ...])]: each entry is a sequence of calls on one persistent state"""
    out = []
    for n in ORDERS:
        t0, v0, e = _cold(n, 0)
        out.append((f"cold_{n}", [(t0, v0, e)]))
        rng = _rng(300, n)
        for attempt in range(50):
            t1 = t0 + 1e-3 * rng.standard_normal()
            v1 = v0 + 1e-3 * rng.standard_normal()
            e1 = np.sort(e + 1e-3 * rng.standard_normal(n))
            st = ln.State(n)
            ln.wrapper(t0, v0, e.copy(), st)
            _, stats = ln.wrapper(t1, v1, e1.copy(), st)
            if _robust(stats) and stats["newton_success"] == ln.NEWTON_SUCCESS:
                out.append((f"warm_{n}", [(t0, v0, e), (t1, v1, e1)]))
                break
        ip = _ipm(n)
        if ip is not None:
            out.append((f"ipm_{n}", [ip]))
    return out


def replay(cases):
    """the numpy restatement on vector_cases(): {name: [(status, proj, stats), ...]}"""
    res = {}
    for name, calls in cases:
        st = ln.State(calls[0][2].size)
        seq = []
        for t0, v0, e in calls:
            status, stats = ln.wrapper(t0, v0, e.copy(), st)
            seq.append((status, st.proj.copy(), stats))
        res[name] = seq
    return res

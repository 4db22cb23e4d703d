"""numpy restatement of the reference's universal solution checker `verify_solution_correct`
(the reference's test/problem_utils.h:107-249) -- every clause, same tolerances.  Test infrastructure.

All norms are infinity norms (NORM = SCS(norm_inf), problem_utils.h:16).  The cone distances are
||s - Pi_K(s)||_inf = ||Pi_K*(-s)||_inf and ||y - Pi_K*(y)||_inf (problem_utils.h:83-105); they are computed with
the numpy projections of scs_b200/problems.py (zero / LP / box / SOC / PSD) or, when `ref_proj_dual` is given
(a callable x -> Pi_K*(x) backed by the compiled reference), with the reference's own operator."""
import numpy as np

from scs_b200 import problems

SCS_SOLVED, SCS_INFEASIBLE, SCS_UNBOUNDED = 1, -2, -1


def ninf(v):
    return float(np.abs(v).max()) if v.size else 0.0


def sym_from_upper_csc(P, n):
    import scipy.sparse as sp
    U = sp.csc_matrix((P[0], P[1], P[2]), shape=(n, n))
    return U + sp.triu(U, 1).T


def verify_solution_correct(prob, stgs, info, x, y, s, status, ref_proj_dual=None):
    """Returns a list of (clause, value, bound) that FAILED (empty list = the reference's checker passes)."""
    A, b, c, cone = prob["A"], prob["b"], prob["c"], prob["cone"]
    n = c.size
    ax = problems.csc_matvec(A, x)
    primal = ax + s
    res_unbdd_a = ninf(primal)
    res_pri = ninf(primal - b)
    if prob.get("P") is not None:
        px = sym_from_upper_csc(prob["P"], n) @ x
        xt_p_x = float(px @ x)
        res_unbdd_p = ninf(px)
    else:
        px = np.zeros(n)
        xt_p_x, res_unbdd_p = 0.0, 0.0
    aty = problems.csc_rmatvec(A, y)
    res_infeas = ninf(aty)
    res_dual = ninf(aty + px + c)

    def pdual(v):
        return ref_proj_dual(v) if ref_proj_dual is not None else problems.proj_dual_cone(v, cone)

    sdist = ydist = float("nan")
    if status in (SCS_SOLVED, SCS_UNBOUNDED):
        sdist = ninf(pdual(-s))                      # ||s - Pi_K(s)|| = ||Pi_K*(-s)||
    if status in (SCS_SOLVED, SCS_INFEASIBLE):
        ydist = ninf(y - pdual(y))
    sty = float(y @ s)
    bty = float(y @ b)
    ctx = float(x @ c)
    gap = abs(xt_p_x + ctx + bty)
    pobj = xt_p_x / 2.0 + ctx
    dobj = -xt_p_x / 2.0 - bty
    grl = max(abs(xt_p_x), abs(ctx), abs(bty))
    prl = max(ninf(b), ninf(s), ninf(ax))
    drl = max(ninf(c), ninf(px), ninf(aty))
    checks = []

    def less(name, val, bound):
        if not (val < bound):
            checks.append((name, val, bound))

    if status == SCS_SOLVED:
        less("Primal residual ERROR", abs(res_pri - info.res_pri), 1e-10)
        less("Dual residual ERROR", abs(res_dual - info.res_dual), 1e-10)
        less("Gap ERROR", abs(gap - info.gap), 1e-7 * (1 + abs(gap)))
        less("Primal obj ERROR", abs(pobj - info.pobj), 1e-9 * (1 + abs(pobj)))
        less("Dual obj ERROR", abs(dobj - info.dobj), 1e-9 * (1 + abs(dobj)))
        less("Complementary slackness ERROR", abs(sty), 5e-8 * max(ninf(s), ninf(y)))
        less("s cone dist ERROR", abs(sdist), 1e-5)
        less("y cone dist ERROR", abs(ydist), 1e-5)
        less("Primal feas ERROR", res_pri, stgs.eps_abs + stgs.eps_rel * prl)
        less("Dual feas ERROR", res_dual, stgs.eps_abs + stgs.eps_rel * drl)
        less("Gap feas ERROR", gap, stgs.eps_abs + stgs.eps_rel * grl)
    elif status == SCS_INFEASIBLE:
        less("Infeas ERROR", abs(res_infeas - info.res_infeas), 1e-8)
        less("bty ERROR", abs(bty + 1), 1e-12)
        less("y cone dist ERROR", abs(ydist), 1e-5)
        less("Infeas invalid ERROR", res_infeas, stgs.eps_infeas)
    elif status == SCS_UNBOUNDED:
        less("Unbdd_a ERROR", abs(res_unbdd_a - info.res_unbdd_a), 1e-8)
        less("Unbdd_p ERROR", abs(res_unbdd_p - info.res_unbdd_p), 1e-8)
        less("ctx ERROR", abs(ctx + 1), 1e-12)
        less("s cone dist ERROR", abs(sdist), 1e-5)
        less("Unbounded P invalid ERROR", res_unbdd_p, stgs.eps_infeas)
        less("Unbounded A invalid ERROR", res_unbdd_a, stgs.eps_infeas)
    else:
        checks.append(("INVALID STATUS", status, None))
    return checks

"""CPU: tests/verify.py (numpy restatement of the reference's verify_solution_correct,
test/problem_utils.h:107-249) accepts what the UNMODIFIED reference produces (recorded under tests/golden/reference/) -- solved,
infeasible and unbounded outcomes -- and rejects a corrupted solution. Pins the checker the GPU tests use."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi, problems
import reference_replay
import verify


@pytest.fixture(scope="module")
def reflib():
    """the reference's answers stored whole: the checker reads every entry of the solution"""
    return reference_replay.Reference("ref", whole=True)


def ref_solve(reflib, prob, **over):
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], prob.get("P"))
    st = capi.default_settings(reflib, verbose=0, **over)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    status = reflib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    return status, info, x, y, s, st


def test_checker_accepts_reference_solutions(reflib):
    for cone, m, n in (({"z": 30, "l": 270}, 300, 100), ({"z": 40, "l": 120, "q": [3, 7, 30, 200]}, 400, 100),
                       ({"l": 60, "s": [6, 8, 4]}, 127, 40)):
        prob = problems.make_problem(m, n, 8, cone, seed=3)
        status, info, x, y, s, st = ref_solve(reflib, prob)
        assert status == 1
        assert verify.verify_solution_correct(prob, st, info, x, y, s, status) == []
        # a corrupted primal variable must be caught (residual / objective clauses)
        x2 = x.copy()
        x2[0] += 1e-3
        assert verify.verify_solution_correct(prob, st, info, x2, y, s, status)


def test_checker_on_certificates(reflib):
    n = 20
    dat = np.empty(2 * n); idx = np.empty(2 * n, dtype=np.int32)
    dat[0::2], dat[1::2] = 1.0, -1.0
    idx[0::2], idx[1::2] = 0, 1 + np.arange(n)
    ptr = (2 * np.arange(n + 1)).astype(np.int32)
    b = np.zeros(n + 1); b[0] = -1.0
    prob = {"A": (dat, idx, ptr, (n + 1, n)), "b": b, "c": np.ones(n), "cone": {"l": n + 1}}
    status, info, x, y, s, st = ref_solve(reflib, prob)
    assert status == -2
    assert verify.verify_solution_correct(prob, st, info, x, y, s, status) == []
    prob = {"A": (-np.ones(n), np.arange(n, dtype=np.int32), np.arange(n + 1, dtype=np.int32), (n, n)),
            "b": np.zeros(n), "c": -np.ones(n), "cone": {"l": n}}
    status, info, x, y, s, st = ref_solve(reflib, prob)
    assert status == -1
    assert verify.verify_solution_correct(prob, st, info, x, y, s, status) == []

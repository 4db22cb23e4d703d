"""CPU: input validation of the outer ABI (scs_b200/csrc/host/scs_driver.c validate(), mirroring reference
src/scs.c:1005-1084 + src/cones.c:430-700 and the reference's own test/problems/test_validation.h): every
bad input must make scs() return SCS_FAILED (and scs_init NULL) BEFORE any GPU work -- so this runs anywhere --
and the same inputs must be refused by the reference (oracle/_ref) too."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import REF_LIB
from scs_b200 import capi, problems

SCS_FAILED = -4


def base_problem():
    prob = problems.make_problem(30, 10, 3, {"z": 3, "l": 8, "q": [4, 6], "s": [2, 3], "ep": 0}, seed=4)
    return prob


def run(library, prob, cone=None, mutate=None, **over):
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], cone if cone is not None else prob["cone"], prob.get("P"))
    st = capi.default_settings(library, verbose=0, **over)
    if mutate:
        mutate(hp, st)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    return library.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))


def bad_settings():
    nan, inf = float("nan"), float("inf")
    return [dict(eps_abs=-1.0), dict(eps_abs=nan), dict(eps_rel=-1e-3), dict(eps_rel=inf), dict(eps_infeas=-1.0),
            dict(alpha=0.0), dict(alpha=2.0), dict(alpha=nan), dict(rho_x=0.0), dict(rho_x=-1.0), dict(scale=0.0),
            dict(scale=inf), dict(max_iters=0), dict(max_iters=-5), dict(time_limit_secs=-1.0),
            dict(acceleration_interval=0), dict(acceleration_lookback=-1), dict(acceleration_regularization=-1.0),
            dict(acceleration_relaxation=2.5)]


def bad_data():
    def neg_m(hp, st): hp.data.m = -1
    def zero_n(hp, st): hp.data.n = 0
    def dim_mismatch(hp, st): hp.A.m = hp.m + 1
    def p0(hp, st): hp.Ap[0] = 1
    def decreasing(hp, st): hp.Ap[3] = hp.Ap[2] - 1
    def row_oob(hp, st): hp.Ai[0] = hp.m
    def row_neg(hp, st): hp.Ai[1] = -1
    def nonfinite(hp, st): hp.Ax[2] = np.inf
    def no_b(hp, st): hp.data.b = capi.c_double_p()
    return [neg_m, zero_n, dim_mismatch, p0, decreasing, row_oob, row_neg, nonfinite, no_b]


def bad_cones(base):
    out = []
    for upd in (dict(z=-1), dict(l=base["l"] + 1), dict(q=[4, 7]), dict(q=[-1, 11]), dict(s=[2, 4]), dict(s=[-2, 3]),
                dict(ep=-1), dict(ed=2), dict(p=[0.5]), dict(l=base["l"] - 3, p=[1.5]), dict(l=base["l"] - 3, p=[float("nan")])):
        c = dict(base)
        c.update(upd)
        out.append(c)
    bx = dict(base)
    bx["l"] = base["l"] - 3
    bx["bl"], bx["bu"] = [1.0, 0.0], [0.0, 1.0]          # lower > upper
    out.append(bx)
    return out


def struct_cones(base):
    """(cone, mutate) pairs whose fault lies in the struct and not in the dict: a NULL array behind a positive size"""
    def no_q(k): k.q = type(k.q)()
    def no_bl(k): k.bl = capi.c_double_p()
    bx = dict(base, l=base["l"] - 3, bl=[0.0, 0.0], bu=[1.0, 1.0])
    return [(dict(base), no_q), (bx, no_bl)]


def libs(lib):
    pairs = [("scs_b200", lib)]
    if os.path.exists(REF_LIB):
        pairs.append(("reference", capi.load_reference(REF_LIB)))
    return pairs


@pytest.mark.parametrize("over", bad_settings(), ids=lambda d: next(iter(d)) + "=" + str(next(iter(d.values()))))
def test_bad_settings_are_refused(lib, over):
    for name, library in libs(lib):
        assert run(library, base_problem(), **over) == SCS_FAILED, name


@pytest.mark.parametrize("mutate", bad_data(), ids=lambda f: f.__name__)
def test_bad_data_is_refused(lib, mutate):
    for name, library in libs(lib):
        if name == "reference" and mutate.__name__ == "no_b":
            continue   # the reference does not check b / c for NULL (it dereferences them): ours only
        assert run(library, base_problem(), mutate=mutate) == SCS_FAILED, name


@pytest.mark.parametrize("i", range(12))
def test_bad_cones_are_refused(lib, i):
    prob = base_problem()
    cone = bad_cones(prob["cone"])[i]
    for name, library in libs(lib):
        assert run(library, prob, cone=cone) == SCS_FAILED, (name, cone)


def test_bad_P_is_refused(lib):
    import scipy.sparse as sp
    prob = base_problem()
    n = prob["n"]
    L = sp.tril(sp.random(n, n, density=0.5, random_state=np.random.RandomState(0)) + sp.identity(n), format="csc")
    L.sort_indices()
    prob["P"] = (L.data.copy(), L.indices.astype(np.int32), L.indptr.astype(np.int32), (n, n))   # LOWER triangle
    for name, library in libs(lib):
        assert run(library, prob) == SCS_FAILED, name


@pytest.mark.parametrize("i", range(14))
def test_init_cone_refuses_what_scs_init_refuses_with_its_message(lib, capfd, i):
    """scs_b200_init_cone validates like scs_init: the same cones refused, before any device work, with the line
    scs_init prints for them, also where a positive size has no array behind it"""
    prob = base_problem()
    cases = [(c, None) for c in bad_cones(prob["cone"])] + struct_cones(prob["cone"])
    cone, mutate = cases[i]
    capfd.readouterr()
    assert run(lib, prob, cone=cone, mutate=(lambda hp, st: mutate(hp.cone)) if mutate else None) == SCS_FAILED
    init_out = capfd.readouterr().out
    k, keep = capi.make_cone(cone)
    if mutate:
        mutate(k)
    assert not lib.scs_b200_init_cone(C.byref(k), prob["m"], None)
    cone_out = capfd.readouterr().out
    assert cone_out.count("\n") == 1 and init_out.startswith(cone_out), (cone_out, init_out)

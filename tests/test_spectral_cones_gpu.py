"""GPU: the nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones of libscs_b200_spectral.so.

* operator parity: scs_b200_proj_dual_cone against the reference spectral build's _scs_proj_dual_cone recorded in
  tests/golden/spectral_cones.npz (oracle/make_golden_spectral.py) on the seeded inputs of tests/spectral_cases.py,
  with and without r_y: 1e-13 relative for the l1 cone, 5e-13 where an eigen-decomposition is involved (cuSOLVER
  syevd vs LAPACK syev / gesvd), as for PSD;
* solver level on the reference's spectral test problems (tests/golden/problems/spectral/): status solved, objective
  within 10 eps of the known optimum, the reference's checker (tests/verify.py) with the numpy spectral cone distance
  of tests/spectral_numpy.py, one iteration within 1e-10 of the reference's x, y, s, and the iteration count within
  the spread the reference shows between its own builds (DESIGN.md section 4)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import spectral_cases
import spectral_numpy
import verify
from conftest import ROOT
from scs_b200 import capi

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
PROB_DIR = os.path.join(GOLD, "problems", "spectral")
OPS = np.load(os.path.join(GOLD, "spectral_cones.npz"))
SOLVES = np.load(os.path.join(GOLD, "spectral_solves.npz"))
OPTIMA = json.load(open(os.path.join(PROB_DIR, "optima.json")))
PP = C.POINTER


@pytest.fixture(scope="module")
def slib():
    lib = capi.load(spectral=True)
    assert lib.scs_b200_device_ok()
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                       PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    return lib


def project(lib, cone, x, r_y):
    k, keep = capi.make_cone(cone, spectral=True)
    cw = lib.scs_b200_init_cone(C.byref(k), len(x), None)
    assert cw, "scs_b200_init_cone failed"
    out = x.copy()
    assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(r_y)) == 0
    lib.scs_b200_finish_cone(cw)
    return out


@pytest.mark.parametrize("name", [str(n) for n in OPS["names"]])
@pytest.mark.parametrize("metric", [False, True])
def test_proj_dual_cone_matches_reference(slib, name, metric):
    cone, xs = spectral_cases.inputs(name)
    r_y = spectral_cases.r_y(cone) if metric else None
    tol = 1e-13 if name.startswith("ell1") else 5e-13
    assert len(xs) == int(OPS[f"{name}/n"][0])
    for i, x in enumerate(xs):
        spectral_cases.check_regenerated(OPS, name, i, x)
        idx, ref = spectral_cases.recorded(OPS, name, i, metric)
        mine = project(slib, cone, x, r_y)[idx]
        err = np.abs(mine - ref).max() / max(np.abs(ref).max(), np.abs(x).max(), 1e-300)
        assert err <= tol, (name, metric, i, err)


def read_problem(lib, name):
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    return d, k, s


def as_dict(d, k):
    """the problem as numpy arrays + cone dict (for tests/verify.py)"""
    D, K = d.contents, k.contents
    A = D.A.contents
    nnz = A.p[A.n]
    arr = lambda p, n, t: np.ctypeslib.as_array(p, (n,)).astype(t) if n > 0 else np.zeros(0, t)  # noqa: E731
    cone = {"z": K.z, "l": K.l, "q": list(arr(K.q, K.qsize, int)), "s": list(arr(K.s, K.ssize, int)),
            "nuc_m": list(arr(K.nuc_m, K.nucsize, int)), "nuc_n": list(arr(K.nuc_n, K.nucsize, int)),
            "ell1": list(arr(K.ell1, K.ell1_size, int)), "sl_n": list(arr(K.sl_n, K.sl_size, int)),
            "sl_k": list(arr(K.sl_k, K.sl_size, int))}
    assert K.bsize == 0 and K.cssize == 0 and K.ep == 0 and K.ed == 0 and K.psize == 0 and not D.P
    Acsc = (arr(A.x, nnz, np.float64), arr(A.i, nnz, np.int32), arr(A.p, A.n + 1, np.int32), (D.m, D.n))
    return {"A": Acsc, "b": arr(D.b, D.m, np.float64), "c": arr(D.c, D.n, np.float64), "cone": cone, "P": None}


def solve(lib, d, k, s, **over):
    st = capi.ScsSettings.from_buffer_copy(s.contents)
    st.verbose = 0
    for key, v in over.items():
        setattr(st, key, v)
    m, n = d.contents.m, d.contents.n
    x, y, z = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(z))
    info = capi.ScsInfo()
    flag = lib.scs(d, k, C.byref(st), C.byref(sol), C.byref(info))
    return flag, info, st, x, y, z


@pytest.mark.parametrize("name", sorted(OPTIMA))
def test_reference_spectral_problem(slib, name):
    d, k, s = read_problem(slib, name)
    try:
        prob = as_dict(d, k)
        # one iteration: the reference's own answer
        _, _, _, x1, y1, s1 = solve(slib, d, k, s, max_iters=1)
        for mine, key in ((x1, "x1"), (y1, "y1"), (s1, "s1")):
            ref = SOLVES[f"{name}/{key}"]
            err = np.abs(mine - ref).max() / max(1.0, np.abs(ref).max())
            assert err <= 1e-10, (name, key, err)
        # converged solve
        flag, info, st, x, y, z = solve(slib, d, k, s)
        ref_flag, ref_iter = SOLVES[f"{name}/info"][:2]
        assert flag == 1 and int(ref_flag) == 1, (name, flag, info.status)
        opt = OPTIMA[name]
        assert abs(info.pobj - opt) <= 10 * st.eps_abs * max(1.0, abs(opt)), (name, info.pobj, opt)
        fails = verify.verify_solution_correct(prob, st, info, x, y, z, flag,
                                               ref_proj_dual=lambda v: spectral_numpy.proj_dual_cone(v, prob["cone"]))
        assert not fails, (name, fails)
        # the reference's two builds differ by a factor 1.32 in iterations (DESIGN.md section 4); allow 1.5 and one
        # convergence-check interval
        assert ref_iter / 1.5 - 25 <= info.iter <= 1.5 * ref_iter + 25, (name, info.iter, ref_iter)
        print(f"{name}: iters {info.iter} (reference {int(ref_iter)}) pobj {info.pobj:.12g} opt {opt:.12g}")
    finally:
        slib.scs_b200_free_data(d, k, s)

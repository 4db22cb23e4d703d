"""GPU parity of the cone operator (zero / LP / box / SOC / PSD / exponential / power under the Moreau
wrapper) against the reference's own _scs_proj_dual_cone (src/cones.c:1552-1596)
recorded under tests/golden/reference/, on identical inputs. Tolerance: 1e-13 relative (SURVEY 8d)."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi
from reference_replay import amax, rel

pytestmark = pytest.mark.gpu


def ref_proj(reflib, cone, m, x, r_y):
    k, keep = capi.make_cone(cone)
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.restype = C.c_int
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    cw = reflib._scs_init_cone(C.byref(k), m)
    assert cw
    out = x.copy()
    ry = None if r_y is None else r_y.copy()
    assert reflib._scs_proj_dual_cone(capi.dptr(out), cw, None, capi.dptr(ry)) == 0
    reflib._scs_finish_cone(cw)
    return out


def mine_proj(lib, cone, m, x, r_y, reps=1):
    k, keep = capi.make_cone(cone)
    cw = lib.scs_b200_init_cone(C.byref(k), m, None)
    assert cw, "scs_b200_init_cone failed"
    out = x.copy()
    for _ in range(reps):
        out = x.copy()
        assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(r_y)) == 0
    lib.scs_b200_finish_cone(cw)
    return out


def r_y_for(cone, m, scale=0.1):
    r = np.full(m, 1.0 / scale)
    r[: cone.get("z", 0)] = 1.0 / (1000 * scale)
    return r


CONES = [
    {"z": 5, "l": 9},
    {"z": 3, "l": 4, "q": [1, 2, 3, 5, 17, 64, 1000]},
    {"l": 2, "q": [20000, 3, 9000, 8193]},                    # big (chunked) SOCs + small ones
    {"z": 2, "l": 3, "bl": [-1.0, -0.5, 0.0, -2.0] * 50, "bu": [1.0, 0.5, 3.0, 0.0] * 50},
    {"l": 1, "s": [1, 2, 3, 5, 12]},
    {"z": 1, "s": [40, 40, 40, 7]},
    {"z": 4, "l": 6, "bl": [-1.0] * 9, "bu": [2.0] * 9, "q": [4, 30], "s": [6, 3]},
]


@pytest.mark.parametrize("ci", range(len(CONES)))
@pytest.mark.parametrize("metric", [False, True])
def test_proj_dual_cone_matches_reference(lib, reflib, ci, metric):
    cone = CONES[ci]
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(ci)
    for trial in range(3):
        x = rng.standard_normal(m) * (10.0 ** rng.integers(-2, 3))
        r_y = r_y_for(cone, m) if metric else None
        ref = ref_proj(reflib, cone, m, x, r_y)
        mine = mine_proj(lib, cone, m, x, r_y)
        scale = max(amax(ref), np.abs(x).max(), 1e-300)
        err = np.nanmax(np.abs(mine - ref)) / scale
        has_psd = bool(cone.get("s"))
        tol = 5e-13 if has_psd else 1e-13   # eigen-decompositions differ (cuSOLVER vs LAPACK syevr)
        assert err <= tol, (ci, metric, trial, err)


TRIPLE_CONES = [
    {"ep": 400},
    {"ed": 400},
    {"z": 2, "l": 3, "q": [5], "ep": 150, "ed": 150},
    {"p": list(np.linspace(0.05, 0.95, 200))},
    {"p": list(-np.linspace(0.05, 0.95, 200))},
    {"l": 4, "s": [3], "ep": 50, "ed": 40, "p": [0.5, -0.5, 0.1, -0.9, 1.0 / 3]},
]


@pytest.mark.parametrize("ci", range(len(TRIPLE_CONES)))
@pytest.mark.parametrize("metric", [False, True])
def test_exp_power_cones_match_reference(lib, reflib, ci, metric):
    """Exponential / power cones (reference src/exp_cone.c, src/cones.c:1282-1332) vs the reference itself.
    The restatement itself is bit-identical to the reference when compiled for the host with the same flags
    (tests/test_cone_triples_cpu.py); on the device exp/log/pow come from the CUDA math library and FMA
    contraction differs, and both feed Newton stop tests: on the CPU alone, gcc with vs without contraction
    already differs by up to 1.3e-10 on 0.07 % of ill-conditioned triples. Asserted: max 1e-9 (exp) /
    1e-8 (power: its Newton stops at |f| < 1e-9, reference POW_CONE_TOL), and the MEDIAN error <= 1e-14."""
    cone = TRIPLE_CONES[ci]
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(50 + ci)
    for trial in range(4):
        x = rng.standard_normal(m) * (10.0 ** rng.integers(-2, 3))
        if trial == 3:
            x[rng.random(m) < 0.3] = 0.0          # boundary / degenerate triples
        r_y = r_y_for(cone, m) if metric else None
        ref = ref_proj(reflib, cone, m, x, r_y)
        mine = mine_proj(lib, cone, m, x, r_y)
        scale = max(amax(ref), np.abs(x).max(), 1e-300)
        err = np.abs(mine - ref) / scale
        tol = 1e-8 if cone.get("p") else 1e-9
        assert np.nanmax(err) <= tol, (ci, metric, trial, np.nanmax(err))
        assert np.nanmedian(err) <= 1e-14


def test_soc_edge_cases(lib, reflib):
    """inside the cone, inside the polar cone, boundary, zero vector"""
    cone = {"q": [4, 4, 4, 4, 1, 1, 2]}
    m = capi.cone_rows(cone)
    x = np.array([5, 1, 1, 1,   -5, 1, 1, 1,   1, 1, 0, 0,   0, 0, 0, 0,   -2.0,   3.0,   0.5, -0.5])
    for r_y in (None, np.full(m, 10.0)):
        ref = ref_proj(reflib, cone, m, x, r_y)
        mine = mine_proj(lib, cone, m, x, r_y)
        assert np.nanmax(np.abs(mine - ref)) <= 1e-14


def test_box_warm_start_repeat(lib, reflib):
    """the Newton warm start t carries across calls (cones.c:1376-1378)"""
    cone = {"bl": list(-np.linspace(0.1, 2, 300)), "bu": list(np.linspace(0.2, 3, 300))}
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(3)
    k, keep = capi.make_cone(cone)
    cw = lib.scs_b200_init_cone(C.byref(k), m, None)
    assert cw
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    k2, keep2 = capi.make_cone(cone)
    rw = reflib._scs_init_cone(C.byref(k2), m)
    for it in range(5):
        x = rng.standard_normal(m) * 3
        a, b = x.copy(), x.copy()
        assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(a), None) == 0
        assert reflib._scs_proj_dual_cone(capi.dptr(b), rw, None, None) == 0
        assert rel(a, b) <= 1e-12
    lib.scs_b200_finish_cone(cw)
    reflib._scs_finish_cone(rw)

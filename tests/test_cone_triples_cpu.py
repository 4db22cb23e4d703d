"""CPU check of the exp / power cone restatement in scs_b200/csrc/kernels/cone_triples.cu: the SAME
source, compiled for the host by oracle/Makefile (libtriples_host.so, test-only), against the
UNMODIFIED reference (oracle/_ref: src/exp_cone.c proj_pd_exp_cone, src/cones.c proj_power_cone via
_scs_proj_dual_cone) on random and degenerate triples. On the host both sides use glibc's exp/log/pow,
so the branch decisions are identical and the results agree to rounding."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, REF_LIB
from scs_b200 import capi

HOST_LIB = os.path.join(ROOT, "oracle", "libtriples_host.so")
pytestmark = pytest.mark.skipif(not os.path.exists(HOST_LIB), reason="oracle/libtriples_host.so not built")
needs_reference = pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle/_ref not built")


def triples(rng, n):
    x = rng.standard_normal((n, 3)) * (10.0 ** rng.integers(-3, 4, size=(n, 1)))
    x[rng.random((n, 3)) < 0.08] = 0.0                      # degenerate coordinates
    k = n // 10
    s = rng.uniform(0.1, 3, k)                               # points near / on the cone boundary
    r = rng.standard_normal(k)
    x[:k] = np.stack([r, s, s * np.exp(r / s) * (1 + 1e-9 * rng.standard_normal(k))], axis=1)
    return x


@needs_reference
def test_exp_cone_host_restatement_matches_reference():
    host = C.CDLL(HOST_LIB)
    host.b200_triples_host_exp.argtypes = [capi.c_double_p, C.c_int]
    ref = capi.load_reference(REF_LIB)
    ref._scs_proj_pd_exp_cone.restype = C.c_double
    ref._scs_proj_pd_exp_cone.argtypes = [capi.c_double_p, C.c_int]
    rng = np.random.default_rng(1)
    worst = 0.0
    for v in triples(rng, 20000):
        for primal in (1, 0):
            a, b = v.copy(), v.copy()
            host.b200_triples_host_exp(capi.dptr(a), primal)
            ref._scs_proj_pd_exp_cone(capi.dptr(b), primal)
            worst = max(worst, np.abs(a - b).max() / max(1.0, np.abs(b).max(), np.abs(v).max()))
    assert worst <= 1e-13, worst


@needs_reference
def test_power_cone_host_restatement_matches_reference():
    host = C.CDLL(HOST_LIB)
    host.b200_triples_host_pow.argtypes = [capi.c_double_p, C.c_double]
    ref = capi.load_reference(REF_LIB)
    ref._scs_init_cone.restype = C.c_void_p
    ref._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    ref._scs_proj_dual_cone.restype = C.c_int
    ref._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    ref._scs_finish_cone.argtypes = [C.c_void_p]
    rng = np.random.default_rng(2)
    n = 4000
    pw = np.concatenate([rng.uniform(0.02, 0.98, n // 2), -rng.uniform(0.02, 0.98, n // 2)])
    x = triples(rng, n)
    # reference: proj_dual_cone(x) = x + Pi_K(-x)  ->  Pi_K(v) = proj_dual_cone(-v) + v
    k, keep = capi.make_cone({"p": list(pw)})
    cw = ref._scs_init_cone(C.byref(k), 3 * n)
    out = (-x).reshape(-1).copy()
    assert ref._scs_proj_dual_cone(capi.dptr(out), cw, None, None) == 0
    ref._scs_finish_cone(cw)
    ref_proj = out.reshape(n, 3) + x
    worst = 0.0
    for i in range(n):
        a = x[i].copy()
        host.b200_triples_host_pow(capi.dptr(a), float(pw[i]))
        worst = max(worst, np.abs(a - ref_proj[i]).max() / max(1.0, np.abs(x[i]).max()))
    assert worst <= 1e-12, worst


def test_host_restatement_matches_committed_goldens():
    """same check against tests/golden/cone_triples.npz (generated from the reference by
    oracle/make_golden_triples.py), so it also runs where oracle/_ref is absent"""
    host = C.CDLL(HOST_LIB)
    host.b200_triples_host_exp.argtypes = [capi.c_double_p, C.c_int]
    host.b200_triples_host_pow.argtypes = [capi.c_double_p, C.c_double]
    g = np.load(os.path.join(ROOT, "tests", "golden", "cone_triples.npz"))
    x = g["x"]
    for primal, key in ((1, "exp_primal"), (0, "exp_dual")):
        for i in range(len(x)):
            a = x[i].copy()
            host.b200_triples_host_exp(capi.dptr(a), primal)
            assert np.abs(a - g[key][i]).max() <= 1e-13 * max(1.0, np.abs(x[i]).max()), (key, i)
    for i in range(len(x)):
        a = x[i].copy()
        host.b200_triples_host_pow(capi.dptr(a), float(g["pow_params"][i]))
        assert np.abs(a - g["pow_proj"][i]).max() <= 1e-12 * max(1.0, np.abs(x[i]).max()), i

"""GPU parity of Anderson acceleration (device TSQR + host pivoted QR) against
the reference's aa_apply / aa_safeguard (src/aa.c:822-901), recorded under tests/golden/reference/, on
an identical fixed-point sequence."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi
from reference_replay import rel

pytestmark = pytest.mark.gpu


def decl_ref(reflib):
    reflib.aa_init.restype = C.c_void_p
    reflib.aa_init.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                               C.c_double, C.c_int, C.c_int]
    reflib.aa_apply.restype = C.c_double
    reflib.aa_apply.argtypes = [capi.c_double_p, capi.c_double_p, C.c_void_p]
    reflib.aa_safeguard.restype = C.c_int
    reflib.aa_safeguard.argtypes = [capi.c_double_p, capi.c_double_p, C.c_void_p]
    reflib.aa_finish.argtypes = [C.c_void_p]
    reflib.aa_reset.argtypes = [C.c_void_p]


def known_or(xr, xm):
    """the reference's iterate where it is stored, ours elsewhere: long vectors are recorded as a sample, and the next
    map application needs every entry (the two agree to 1e-9, so the sampled entries stay a sharp check)"""
    return np.where(np.isnan(xr), xm, xr)


def contraction(dim, seed):
    """x -> M x + b with spectral radius < 1 (a linear fixed-point map)."""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.2, 0.97, size=dim)
    b = rng.standard_normal(dim)
    shift = rng.integers(1, dim)

    def F(x):
        return d * x + 0.02 * np.roll(x, shift) + b
    return F


def steps(mem):
    """40 map applications, and more for long memories: the first solve comes at the mem-th apply (min_len = mem)"""
    return max(40, mem + 30)


@pytest.mark.parametrize("dim,mem,type1,relax", [
    (50, 5, 1, 1.0), (5000, 10, 1, 1.0), (5000, 10, 0, 1.0), (3001, 7, 1, 0.8), (200000, 10, 1, 1.0),
    (4099, 14, 1, 1.0), (4099, 31, 1, 1.0), (4099, 31, 0, 1.0), (50000, 20, 1, 1.5),
])
def test_aa_sequence_matches_reference(lib, reflib, dim, mem, type1, relax):
    decl_ref(reflib)
    F = contraction(dim, dim + mem)
    reg = 1e-8 if type1 else 1e-12
    mine = lib.scs_b200_aa_init(dim, mem, mem, type1, reg, relax, 1.0, 1e10, 5, 0)
    ref = reflib.aa_init(dim, mem, mem, type1, reg, relax, 1.0, 1e10, 5, 0)
    assert mine and ref
    xm = np.zeros(dim)
    xr = np.zeros(dim)
    worst = 0.0
    n_acc = 0
    for i in range(steps(mem)):
        # same driver as the reference's documented usage pattern (include/aa.h:66-84)
        if i > 0:
            nm = lib.scs_b200_aa_apply(mine, capi.dptr(xm), capi.dptr(xm_prev))
            nr = reflib.aa_apply(capi.dptr(xr), capi.dptr(xr_prev), ref)
            xr = known_or(xr, xm)
            assert (nm > 0) == (nr > 0), (i, nm, nr)
            if nr > 0:
                n_acc += 1
                assert abs(nm - nr) <= 1e-6 * abs(nr), (i, nm, nr)
        xm_prev, xr_prev = xm.copy(), xr.copy()
        xm, xr = F(xm), F(xr)
        sm = lib.scs_b200_aa_safeguard(mine, capi.dptr(xm), capi.dptr(xm_prev))
        sr = reflib.aa_safeguard(capi.dptr(xr), capi.dptr(xr_prev), ref)
        assert sm == sr, (i, sm, sr)
        worst = max(worst, rel(xm, xr, 1e-300))
        xr = known_or(xr, xm)
    print(f"\n[dim={dim} mem={mem} type1={type1}] accepted={n_acc} worst rel diff {worst:.3e}")
    assert n_acc > 10
    assert worst <= 1e-9
    st = lib.scs_b200_aa_get_stats(mine)
    assert st.n_accept == n_acc
    lib.scs_b200_aa_finish(mine)
    reflib.aa_finish(ref)


def test_aa_rank_deficient_history_matches_reference(lib, reflib):
    """One apply handed the inputs of the apply before it: its S, D and Y columns are exactly zero. Without
    regularization the pivoted QR then truncates the rank (last_rank < len) until a reset or until that column is
    overwritten mem applies later; the truncated solve is not the exact one, so only the reference can check it."""
    decl_ref(reflib)
    dim, mem, repeat = 3001, 8, 12
    F = contraction(dim, 77)
    mine = lib.scs_b200_aa_init(dim, mem, mem, 1, 0.0, 1.0, 1.0, 1e10, 5, 0)
    ref = reflib.aa_init(dim, mem, mem, 1, 0.0, 1.0, 1.0, 1e10, 5, 0)
    assert mine and ref
    xm = np.zeros(dim)
    xr = np.zeros(dim)
    worst = 0.0
    n_acc = 0
    truncated = []
    for i in range(40):
        if i > 0:
            if i == repeat:
                fm, fr = xm.copy(), xr.copy()   # the same inputs once more right after: a zero history column
                nm = lib.scs_b200_aa_apply(mine, capi.dptr(fm), capi.dptr(xm_prev))
                nr = reflib.aa_apply(capi.dptr(fr), capi.dptr(xr_prev), ref)
                assert (nm > 0) == (nr > 0), (i, nm, nr)
                n_acc += nr > 0
            nm = lib.scs_b200_aa_apply(mine, capi.dptr(xm), capi.dptr(xm_prev))
            nr = reflib.aa_apply(capi.dptr(xr), capi.dptr(xr_prev), ref)
            xr = known_or(xr, xm)
            assert (nm > 0) == (nr > 0), (i, nm, nr)
            if nr > 0:
                n_acc += 1
                assert abs(nm - nr) <= 1e-6 * abs(nr), (i, nm, nr)
            st = lib.scs_b200_aa_get_stats(mine)
            if nm > 0 and st.last_rank < min(st.iter - 1, mem):
                truncated.append((i, st.last_rank))
        xm_prev, xr_prev = xm.copy(), xr.copy()
        xm, xr = F(xm), F(xr)
        sm = lib.scs_b200_aa_safeguard(mine, capi.dptr(xm), capi.dptr(xm_prev))
        sr = reflib.aa_safeguard(capi.dptr(xr), capi.dptr(xr_prev), ref)
        assert sm == sr, (i, sm, sr)
        worst = max(worst, rel(xm, xr, 1e-300))
        xr = known_or(xr, xm)
    print(f"\n[rank-deficient history] accepted={n_acc} truncated (step, rank) {truncated} worst rel diff {worst:.3e}")
    assert truncated and truncated[0] == (repeat, mem - 1)
    assert n_acc > 10
    assert worst <= 1e-9
    assert lib.scs_b200_aa_get_stats(mine).n_accept == n_acc
    lib.scs_b200_aa_finish(mine)
    reflib.aa_finish(ref)

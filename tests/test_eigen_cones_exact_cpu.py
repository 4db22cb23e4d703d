"""CPU: the exact references of tests/test_eigen_cones_exact_gpu.py (tests/eigen_exact.py) are exact, are the
projections they claim to be, and their gate rejects the defects a tiled, chunked eigen-reconstruction can have.

* the orthogonal and unitary factors satisfy Q* Q = I exactly and mix every coordinate;
* every input matrix is representable in fp64 (the builders assert it) and the only input rounding is the sqrt2 of
  the packed off-diagonals (and the division by r = 10), which delta_in measures;
* each reference meets the optimality conditions of its projection exactly: for PSD, Q' Pi Q >= 0 and
  Q' (X - Pi) Q <= 0 are diagonal and <Pi, X - Pi> = 0; for the nuclear-norm and sum-of-largest cones the vector-level
  conditions (primal and polar feasibility, complementarity) and <Pi, X - Pi> + t' (t - t') = 0;
* the exact vector projections agree with the float restatements of tests/spectral_numpy.py;
* three planted defects, applied to the exact PSD reference, exceed the gate by at least 100x: the last positive
  32-column eigen-chunk dropped, a chunk straddling zero left unclamped, and the first row of the second 32 x 32
  output tile left unwritten."""
from fractions import Fraction

import numpy as np
import pytest

import eigen_exact as ee
import spectral_numpy


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 16, 17, 33, 64, 65, 129])
@pytest.mark.parametrize("phases", [False, True])
def test_factors_are_exactly_orthogonal_and_mix_every_coordinate(k, phases):
    Q = ee.orthogonal(k, np.random.default_rng(k), phases=phases)
    assert ee.check_orthogonal(Q)
    Z = Q.Z[0] if phases else Q.Z
    nnz = np.count_nonzero(Z, axis=0) + (np.count_nonzero(Q.Z[1], axis=0) if phases else 0)
    if k >= 4:  # below order 4 there is no reflector: a signed (or phased) permutation
        assert nnz.min() >= 4, nnz.min()
        assert not phases or np.count_nonzero(Q.Z[1]) > 0


def _sorted_positions(lam):
    """original indices of lam in ascending order (the eigensolver's column order)"""
    return sorted(range(len(lam)), key=lambda i: lam[i])


def _psd_blocks(k):
    return ee.psd_order_blocks(k)


@pytest.mark.parametrize("k", [2, 3, 31, 32, 33, 64, 65])
def test_psd_references_are_the_projections(k):
    for name, b in _psd_blocks(k):
        Q, lam, X, P = b.parts["Q"], b.parts["lam"], b.parts["X"], b.parts["P"]
        assert ee.check_orthogonal(Q)
        d = ee.congruence_diagonal(Q, P)
        assert d is not None and sorted(d) == sorted(max(v, 0) for v in lam), name
        r = ee.congruence_diagonal(Q, X - P)
        assert r is not None and all(v <= 0 for v in r), name
        assert ee.inner(P, X - P) == 0, name


@pytest.mark.parametrize("kc", [1, 2, 16, 17, 33])
def test_complex_psd_references_are_the_projections(kc):
    for name, b in ee.cpsd_order_blocks(kc):
        Q, lam, (Xr, Xi), (Pr, Pi) = b.parts["Q"], b.parts["lam"], b.parts["X"], b.parts["P"]
        assert ee.check_orthogonal(Q)
        d = ee.congruence_diagonal(Q, (Pr, Pi))
        assert d is not None and sorted(d) == sorted(max(v, 0) for v in lam), name
        r = ee.congruence_diagonal(Q, (Xr - Pr, Xi - Pi))
        assert r is not None and all(v <= 0 for v in r), name
        assert ee.inner((Pr, Pi), (Xr - Pr, Xi - Pi)) == 0, name


@pytest.mark.parametrize("mn", ee.NUC_SHAPES, ids=lambda mn: f"{mn[0]}x{mn[1]}")
def test_nuclear_references_are_the_projections(mn):
    m, n = mn
    wheres = set()
    for name, b in ee.nuc_shape_blocks(m, n):
        p = b.parts
        assert ee.check_orthogonal(p["U"]) and ee.check_orthogonal(p["V"])
        t, tn, sig, sn = p["t"], p["tn"], p["sig"], p["sn"]
        assert sum(sn) <= tn and all(v >= 0 for v in sn), name                  # in the cone
        mu = tn - t
        assert mu >= 0 and all(abs(a - b) <= mu for a, b in zip(sig, sn)), name  # residual in the polar cone
        assert tn * (t - tn) + sum(a * (s - a) for a, s in zip(sn, sig)) == 0, name
        # the matrix level: <Pi, X - Pi> + t' (t - t') = 0 on the vector the device sees
        v = [a for a, _ in b.v]
        out = [a for a, _ in b.out]
        pi = [a + o for a, o in zip(v, out)]
        assert sum(a * o for a, o in zip(pi, out)) == 0, name
        wheres.add("inside" if mu == 0 else ("polar" if tn == 0 else "between"))
        ref_t, ref_s = spectral_numpy.proj_ell1(float(t), np.array([float(s) for s in sig]))
        assert abs(ref_t - float(tn)) <= 1e-13 * max(1.0, abs(float(tn))), name
        assert np.abs(ref_s - np.array([float(s) for s in sn])).max() <= 1e-13 * max(1.0, float(max(sig))), name
    assert wheres == {"inside", "polar", "between"}


@pytest.mark.parametrize("n", ee.SL_ORDERS)
def test_sum_largest_references_are_the_projections(n):
    for name, b in ee.sl_order_blocks(n):
        p = b.parts
        assert ee.check_orthogonal(p["Q"])
        t, tn, lam, xn, k = p["t"], p["tn"], p["lam"], p["xn"], p["k"]
        assert ee.sum_largest(xn, k) <= tn, name                                  # in the cone
        eta = tn - t
        assert eta >= 0, name
        if eta == 0:
            assert xn == lam, name
        else:                                                                     # residual (-eta, eta w) in the polar
            w = [(a - b) / eta for a, b in zip(lam, xn)]
            assert all(0 <= v <= 1 for v in w) and sum(w) == k, name
        assert tn * (t - tn) + sum(a * (l - a) for a, l in zip(xn, lam)) == 0, name
        # <Pi, Pi - v> on the packed rows, whose off-diagonals carry sqrt2
        assert sum((a + o) * o * (2 if s else 1) for (a, s), (o, _) in zip(b.v, b.out)) == 0, name
        if "between" in name:
            ref_t, ref_x = spectral_numpy.proj_sum_largest_vec(float(t), np.array([float(v) for v in lam]), k)
            assert abs(ref_t - float(tn)) <= 1e-12 * max(1.0, abs(float(tn))), name
            assert np.abs(ref_x - np.array([float(v) for v in xn])).max() <= 1e-12 * max(1.0, abs(float(tn))), name


def _psd_output(X, P, r):
    """the float vector closest to (Pi - X) / r, packed: what a device without any rounding would return"""
    return np.array([float(ee.mp_value(a, s) / r) for a, s in ee.packed_sym(P - X)])


def _defects(b):
    """{defect name: Pi'} for the defects that change this block's projection"""
    Q, lam, X = b.parts["Q"], b.parts["lam"], b.parts["X"]
    k = len(lam)
    asc = _sorted_positions(lam)
    chunk = {i: pos // 32 for pos, i in enumerate(asc)}
    out = {}
    last = chunk[asc[-1]]
    if lam[asc[-1]] > 0:
        w = [0 if chunk[i] == last else max(v, 0) for i, v in enumerate(lam)]
        out["last positive chunk dropped"] = ee.qdq(Q, w)
    for c in set(chunk.values()):
        vals = [lam[i] for i in asc if chunk[i] == c]
        if min(vals) < 0 < max(vals):
            w = [v if chunk[i] == c else max(v, 0) for i, v in enumerate(lam)]
            out["straddling chunk not clamped"] = ee.qdq(Q, w)
            break
    if k > 32:
        P = b.parts["P"].copy()
        P[32, :] = P[:, 32] = Fraction(0)  # the first row of the second output tile never written
        out["tile edge row 32 unwritten"] = P
    return out


@pytest.mark.parametrize("k,name", [(33, "p32"), (33, "p31"), (64, "p33"), (65, "p31"), (65, "zeros31_32"),
                                    (129, "p33")])
@pytest.mark.parametrize("r", [1, 10])
def test_gate_rejects_planted_defects(k, name, r):
    b = dict(_psd_blocks(k))[name]
    x = b.x(r)
    X, P = b.parts["X"], b.parts["P"]
    assert b.ratio(_psd_output(X, P, r), x, r) <= 1e-3  # the rounded exact answer passes with room
    defects = _defects(b)
    assert "tile edge row 32 unwritten" in defects and len(defects) >= 2, sorted(defects)
    for what, Pd in defects.items():
        ratio = b.ratio(_psd_output(X, Pd, r), x, r)
        assert ratio >= 100, (k, name, what, ratio)


def test_every_defect_is_planted_somewhere():
    seen = set()
    for k, name in [(33, "p32"), (33, "p31"), (64, "p33"), (65, "p31"), (65, "zeros31_32"), (129, "p33")]:
        seen |= set(_defects(dict(_psd_blocks(k))[name]))
    assert seen == {"last positive chunk dropped", "straddling chunk not clamped", "tile edge row 32 unwritten"}

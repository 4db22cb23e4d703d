"""CPU: the index arithmetic of the complex-PSD kernels (scs_b200/csrc/kernels/cones_complex.cu:
k_cpsd_unpack / k_cpsd_reconstruct -- packed Hermitian block <-> real embedding [[A, -B], [B, A]] of order 2k),
restated in numpy line by line and checked against the reference's zheevr-based projection
(src/cones.c:1072-1156 through _scs_proj_dual_cone; its answer recorded under tests/golden/reference/)."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi
import reference_replay

SQRT2 = 1.4142135623730951


def embed(kc, p):
    """k_cpsd_unpack"""
    K = 2 * kc
    M = np.zeros((K, K))

    def entry(i, j):  # i >= j
        base = j * (2 * kc - j)
        if i == j:
            return p[base] * SQRT2, 0.0
        return p[base + 1 + 2 * (i - j - 1)], p[base + 2 + 2 * (i - j - 1)]

    for e in range(K * K):
        I, J = e % K, e // K
        i, j, bi, bj = I % kc, J % kc, I // kc, J // kc
        if i >= j:
            re, im = entry(i, j)
        else:
            re, im = entry(j, i)
            im = -im
        M[I, J] = re if bi == bj else (im if bi == 1 else -im)
    return M


def repack(kc, X):
    """writer of k_cpsd_reconstruct: top-left block -> real parts, bottom-left block -> imaginary parts"""
    K = 2 * kc
    out = np.zeros(kc * kc)
    for I in range(K):
        for J in range(min(I, kc - 1) + 1):
            col = J * (2 * kc - J)
            if I < kc:
                if I == J:
                    out[col] = X[I, J] * 0.7071067811865476
                else:
                    out[col + 1 + 2 * (I - J - 1)] = X[I, J]
            else:
                i = I - kc
                if i > J:
                    out[col + 2 + 2 * (i - J - 1)] = X[I, J]
    return out


def reference_projection(reflib, orders, x):
    reflib._scs_init_cone.restype = C.c_void_p
    reflib._scs_init_cone.argtypes = [C.POINTER(capi.ScsCone), C.c_int]
    reflib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    reflib._scs_finish_cone.argtypes = [C.c_void_p]
    k, keep = capi.make_cone({"cs": list(orders)})
    cw = reflib._scs_init_cone(C.byref(k), x.size)
    v = (-x).copy()
    assert reflib._scs_proj_dual_cone(capi.dptr(v), cw, None, None) == 0
    reflib._scs_finish_cone(cw)
    return v + x        # Pi_K(x) = Pi_K*(-x) + x  (the cone is self-dual)


@pytest.fixture(scope="module")
def reflib():
    """the reference's answers stored whole: every block of the projection is compared"""
    return reference_replay.Reference("ref", whole=True)


def test_embedding_reproduces_the_reference(reflib):
    rng = np.random.default_rng(0)
    orders = [1, 2, 3, 5, 8, 13]
    x = rng.standard_normal(sum(k * k for k in orders)) * 3
    ref = reference_projection(reflib, orders, x)
    pos = 0
    for kc in orders:
        p = x[pos:pos + kc * kc]
        M = embed(kc, p)
        assert np.allclose(M, M.T)
        lam, V = np.linalg.eigh(M)
        X = (V * np.maximum(lam, 0.0)) @ V.T
        got = repack(kc, X)
        assert np.abs(got - ref[pos:pos + kc * kc]).max() <= 1e-13 * max(1.0, np.abs(p).max()), kc
        pos += kc * kc

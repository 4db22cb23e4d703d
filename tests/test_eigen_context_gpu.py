"""GPU: every eigen-decomposition family of one cone workspace shares one eigensolver context (one cuSOLVER handle, one
device and one host workspace of the largest queried size, one status-word array for the largest group). Each
family's projection must not depend on the other families it shares them with: one spectral-library cone with real
PSD, complex PSD, log-det, nuclear-norm, sum-of-largest and l1 cones is projected in one call, and each family's rows
must be bit for bit what a workspace of that family alone returns.

The groups are added to the context in the order real PSD (by order), log-det, nuclear norm, sum of largest, complex
PSD. The real PSD family has 4097 order-2 blocks (one full sub-batch and one block): the largest batch, which sizes the
status-word array, followed by groups of orders 33 and 100 of one and three blocks. The complex PSD family, added
last, has 4096 blocks of order 2, decomposed through embeddings of order 4: on an H100 with cuSOLVER 11.7.5 their
workspace query is the largest, so the shared workspace grows after the groups of the other families have been sized,
and the largest workspace and the largest batch come from different groups."""
import ctypes as C

import numpy as np
import pytest

import logdet_cases
from scs_b200 import capi

pytestmark = pytest.mark.gpu

# (family, cone), in the row order of the spectral ScsCone
FAMILIES = [
    ("psd", {"s": [1] + [2] * 4097 + [33, 100, 100, 100]}),
    ("complex psd", {"cs": [3, 17] + [2] * 4096}),
    ("log-det", {"d": [1, 5]}),
    ("nuclear", {"nuc_m": [7], "nuc_n": [4]}),
    ("l1", {"ell1": [9]}),
    ("sum-of-largest", {"sl_n": [6], "sl_k": [2]}),
]


@pytest.fixture(scope="module")
def slib():
    lib = capi.load(spectral=True)
    assert lib.scs_b200_device_ok()
    return lib


def project(lib, cone, x, r_y):
    k, keep = capi.make_cone(cone, spectral=True)
    cw = lib.scs_b200_init_cone(C.byref(k), len(x), None)
    assert cw, "scs_b200_init_cone failed"
    out = x.copy()
    try:
        rc = lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(r_y))
    finally:
        lib.scs_b200_finish_cone(cw)
    assert rc == 0, "scs_b200_proj_dual_cone failed"
    return out


def family_inputs():
    """x of each family: Gaussian entries, and log-det cones that take Newton's branch"""
    rng = np.random.default_rng(20261017)
    xs = []
    for name, cone in FAMILIES:
        if name == "log-det":
            xs.append(np.concatenate([logdet_cases.operator_input("newton", d) for d in cone["d"]]))
        else:
            xs.append(rng.standard_normal(capi.cone_rows(cone)))
    return xs


@pytest.mark.parametrize("r", [None, 4.0, 10.0])
def test_families_sharing_one_context_match_each_family_alone(slib, r):
    xs = family_inputs()
    cone = {}
    for _, c in FAMILIES:
        cone.update(c)
    x = np.concatenate(xs)
    assert capi.cone_rows(cone) == x.size
    together = project(slib, cone, x, None if r is None else np.full(x.size, r))
    pos = 0
    for (name, c), xf in zip(FAMILIES, xs):
        alone = project(slib, c, xf, None if r is None else np.full(xf.size, r))
        assert not np.array_equal(alone, xf), name  # the projection moved every family
        assert np.array_equal(together[pos:pos + xf.size], alone), (name, r)
        pos += xf.size

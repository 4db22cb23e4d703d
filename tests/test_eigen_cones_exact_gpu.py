"""GPU: the eigen-decomposition cones (real PSD, complex PSD, nuclear norm, sum of largest eigenvalues, log-det) at
their tile, chunk and batch edges.

* More than 65535 blocks of one order: the unpack, embed and reconstruct kernels put the block index in gridDim.y or
  gridDim.z, which stop at 65535, and the batched eigensolver needs about 0.5 MB of workspace per matrix, so the host
  launchers split every group into sub-batches of at most 4096 blocks (one batched eigensolver call each). Checked at
  65535, 65536, 65537 and 131071 order-2 PSD blocks behind an order-3 block, at 65537 blocks of every other family,
  and with one scs() solve over 65537 2 x 2 blocks. The
  references are batched numpy eigendecompositions at the suite's 5e-13 parity gate; the log-det cones reuse the
  recorded reference answers of tests/golden/logdet_cones.npz at tests/test_logdet_gpu.py's gate.
* Exact references (tests/eigen_exact.py): inputs with exactly known eigen- or singular-value decompositions at the
  32 x 32 tile edges of the reconstruction and the 32-column chunk edges of its positive-eigenvalue skip (real PSD
  k = 2 ... 200 with 0, 1, 31, 32, 33, k - 1 or k positive eigenvalues, exact zeros, multiple eigenvalues, a 2^+-30
  spread, several blocks per call and interleaved orders; complex PSD kc = 1 ... 33; nuclear norm up to 100 x 7 and
  65 x 65, full rank, rank deficient and repeated; sum of largest eigenvalues with ties at the k-th), without r_y and
  with r_y = 4 and 10. Each block must lie within delta_in + 64 N 2^-53 ||x||_2 of its exact projection. Gaussian
  inputs against 40-digit mpmath decompositions check that the structure of those inputs hides nothing."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse

import eigen_exact as ee
import logdet_cases
import logdet_numpy
from conftest import ROOT
from scs_b200 import capi

pytestmark = pytest.mark.gpu
SQRT2 = np.sqrt(2.0)
GRID_YZ = 65535  # largest gridDim.y / gridDim.z
SUB_BATCH = 4096  # B200_EIG_BATCH (scs_b200/csrc/eigen.cuh)


@pytest.fixture(scope="module")
def slib():
    lib = capi.load(spectral=True)
    assert lib.scs_b200_device_ok()
    return lib


def project(lib, cone, x, r_y=None, spectral=None):
    """scs_b200_proj_dual_cone: x + Pi_K(-R x) / R; spectral=True: the ScsCone layout of the spectral library"""
    k, keep = capi.make_cone(cone, spectral=spectral)
    cw = lib.scs_b200_init_cone(C.byref(k), len(x), None)
    assert cw, "scs_b200_init_cone failed"
    out = x.copy()
    try:
        rc = lib.scs_b200_proj_dual_cone(cw, capi.dptr(out), capi.dptr(r_y))
    finally:
        lib.scs_b200_finish_cone(cw)
    assert rc == 0, "scs_b200_proj_dual_cone failed"
    return out


def rel(mine, ref, x):
    return np.abs(mine - ref).max() / max(np.abs(ref).max(), np.abs(x).max())


# ---------------------------------------------------------------------------------------------- batched references
def psd2_dual(x):
    """x + Pi_PSD(-x) for rows of packed 2 x 2 blocks (a, sqrt2 b, d), shape (N, 3)"""
    M = np.empty((len(x), 2, 2))
    M[:, 0, 0], M[:, 1, 1] = -x[:, 0], -x[:, 2]
    M[:, 0, 1] = M[:, 1, 0] = -x[:, 1] / SQRT2
    lam, V = np.linalg.eigh(M)
    P = np.einsum("bik,bk,bjk->bij", V, np.maximum(lam, 0.0), V)
    return x + np.stack([P[:, 0, 0], SQRT2 * P[:, 1, 0], P[:, 1, 1]], axis=1)


def psd_dual(x, k):
    """x + Pi_PSD(-x) for one packed block of order k"""
    import spectral_numpy as sn
    lam, V = np.linalg.eigh(sn.packed_to_sym(-x, k))
    return x + sn.sym_to_packed((V * np.maximum(lam, 0.0)) @ V.T)


def hermitian(p, kc):
    """the Hermitian matrix of a packed complex PSD block (column j at j (2 kc - j): diagonal, then (re, im) * sqrt2)"""
    H = np.zeros((kc, kc), complex)
    for j in range(kc):
        base = j * (2 * kc - j)
        H[j, j] = p[base]
        for i in range(j + 1, kc):
            H[i, j] = (p[base + 1 + 2 * (i - j - 1)] + 1j * p[base + 2 + 2 * (i - j - 1)]) / SQRT2
            H[j, i] = np.conj(H[i, j])
    return H


def hermitian_packed(H):
    kc = H.shape[0]
    out = np.zeros(kc * kc)
    for j in range(kc):
        base = j * (2 * kc - j)
        out[base] = H[j, j].real
        for i in range(j + 1, kc):
            out[base + 1 + 2 * (i - j - 1)] = SQRT2 * H[i, j].real
            out[base + 2 + 2 * (i - j - 1)] = SQRT2 * H[i, j].imag
    return out


def cpsd_dual(x, kc):
    lam, V = np.linalg.eigh(hermitian(-x, kc))
    return x + hermitian_packed((V * np.maximum(lam, 0.0)) @ V.conj().T)


def cycled(blocks, count):
    """count blocks, block i a copy of blocks[i % len(blocks)]: a sub-batch that read or wrote its neighbour's rows
    (an offset off by a sub-batch or by 65535 or 65536, none a multiple of len(blocks)) gets another block's answer"""
    assert SUB_BATCH % len(blocks) and GRID_YZ % len(blocks) and (GRID_YZ + 1) % len(blocks)
    return np.tile(np.stack(blocks), ((count + len(blocks) - 1) // len(blocks), 1))[:count]


# ---------------------------------------------------------------------------------------------- batch limit
@pytest.mark.parametrize("count", [GRID_YZ, GRID_YZ + 1, GRID_YZ + 2, 2 * GRID_YZ + 1])
def test_psd_blocks_beyond_the_grid_limit(lib, count):
    """one order-3 block, then `count` order-2 blocks, every one distinct; with and without r_y"""
    cone = {"l": 1, "s": [3] + [2] * count}
    m = capi.cone_rows(cone)
    rng = np.random.default_rng(count)
    x = rng.standard_normal(m)
    ref = np.empty(m)
    ref[0] = max(x[0], 0.0)
    ref[1:7] = psd_dual(x[1:7], 3)
    ref[7:] = psd2_dual(x[7:].reshape(count, 3)).ravel()
    err = rel(project(lib, cone, x), ref, x)
    assert err <= 5e-13, (count, err)
    if count == GRID_YZ + 2:
        r = 10.0
        err = rel(project(lib, cone, x, np.full(m, r)), ref, x)  # the cone is homogeneous: the same answer
        assert err <= 5e-13, (count, r, err)


def test_complex_psd_blocks_beyond_the_grid_limit(lib):
    count = GRID_YZ + 2
    cone = {"cs": [2] + [1] * count}
    rng = np.random.default_rng(1)
    x = rng.standard_normal(capi.cone_rows(cone))
    ref = np.concatenate([cpsd_dual(x[:4], 2), x[4:] + np.maximum(-x[4:], 0.0)])
    err = rel(project(lib, cone, x), ref, x)
    assert err <= 5e-13, err


def test_nuclear_cones_beyond_the_grid_limit(slib):
    """(2, 1): X is a 2-vector, the cone a second-order cone of dimension 3"""
    import spectral_numpy as sn
    count = GRID_YZ + 2
    rng = np.random.default_rng(2)
    blocks = [rng.standard_normal(3) * s for s in (1.0, 0.5, 2.0, 3.0, 0.1, 1.5, 0.7)]
    blocks[1][0] = 5.0    # -(t, X) in the polar cone: Pi(-x) = 0
    blocks[2][0] = -9.0   # -(t, X) inside the cone: Pi(-x) = -x
    x = cycled(blocks, count).ravel()
    ref = np.empty_like(x)
    for i, b in enumerate(blocks):
        tn, Xn = sn.proj_nuclear(-b[0], -b[1:].reshape(2, 1))
        ref.reshape(count, 3)[i::len(blocks)] = b + np.concatenate(([tn], Xn.ravel()))
    err = rel(project(slib, {"nuc_m": [2] * count, "nuc_n": [1] * count}, x), ref, x)
    assert err <= 5e-13, err


def test_sum_largest_cones_beyond_the_grid_limit(slib):
    import spectral_numpy as sn
    count = GRID_YZ + 2
    rng = np.random.default_rng(3)
    blocks = [rng.standard_normal(4) for _ in range(7)]
    blocks[3][0] = -50.0  # -(t, X) inside the cone
    x = cycled(blocks, count).ravel()
    ref = np.empty_like(x)
    for i, b in enumerate(blocks):
        tn, pn = sn.proj_sum_largest(-b[0], -b[1:], 2, 1)
        ref.reshape(count, 4)[i::len(blocks)] = b + np.concatenate(([tn], pn))
    err = rel(project(slib, {"sl_n": [2] * count, "sl_k": [1] * count}, x), ref, x)
    assert err <= 5e-13, err


def test_logdet_cones_beyond_the_grid_limit(slib):
    """the six recorded order-2 operator inputs, cycled; each at tests/test_logdet_gpu.py's gate: 10 x the numpy
    restatement's distance to the reference's recorded answer, at least 5e-13"""
    ops = np.load(os.path.join(ROOT, "tests", "golden", "logdet_cones.npz"))
    count = GRID_YZ + 2
    cases = [(f"{kind}_2", logdet_cases.operator_input(kind, 2)) for kind in logdet_cases.KINDS]
    x = cycled([c[1] for c in cases], count).ravel()
    mine = project(slib, {"d": [2] * count}, x).reshape(count, 5)
    for i, (name, xi) in enumerate(cases):
        ref = ops[f"{name}/out"]
        _, p, _ = logdet_numpy.proj_logdet(-xi, 2, logdet_numpy.State(2))
        gate = max(5e-13, 10 * rel(xi + p, ref, xi))
        err = np.abs(mine[i::len(cases)] - ref).max() / max(np.abs(ref).max(), np.abs(xi).max())
        assert err <= gate, (name, err, gate)


def test_scs_solves_an_sdp_with_65537_blocks(lib):
    """minimise sum_i tr X_i subject to X_i[0, 1] = 1, X_i PSD (2 x 2): the optimum is X_i = [[1, 1], [1, 1]], 2 N"""
    N = GRID_YZ + 2
    # x = (a_i, b_i, d_i) per block; rows: N zero rows b_i = 1, then s_i = (a_i, sqrt2 b_i, d_i) = -A x in the PSD cone
    i = np.arange(N)
    rows = np.concatenate((i, N + 3 * i, N + 3 * i + 1, N + 3 * i + 2))
    cols = np.concatenate((3 * i + 1, 3 * i, 3 * i + 1, 3 * i + 2))
    vals = np.concatenate((np.ones(N), np.full(N, -1.0), np.full(N, -SQRT2), np.full(N, -1.0)))
    A = scipy.sparse.csc_matrix((vals, (rows, cols)), shape=(4 * N, 3 * N))
    b = np.concatenate((np.ones(N), np.zeros(3 * N)))
    c = np.tile([1.0, 0.0, 1.0], N)
    cone = {"z": N, "s": [2] * N}
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone)
    st = capi.default_settings(lib, verbose=0)
    x, y, s = np.zeros(3 * N), np.zeros(4 * N), np.zeros(4 * N)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    flag = lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    assert flag == 1, (flag, info.status)
    assert abs(info.pobj - 2 * N) <= 10 * st.eps_abs * 2 * N, info.pobj
    X = x.reshape(N, 3)
    assert np.abs(X[:, 1] - 1.0).max() <= 10 * st.eps_abs
    print(f"scs: {N} blocks, {info.iter} iterations, pobj {info.pobj:.9g}, solve {info.solve_time:.0f} ms")


# ---------------------------------------------------------------------------------------------- exact references
# Each block within ||dev - ref||_2 <= delta_in + 64 N 2^-53 ||x||_2 of its exact projection (tests/eigen_exact.py);
# the largest ratio per family is printed.
WORST = {}


def _check_blocks(lib, cone, blocks, r, family, spectral=None):
    """one call on all blocks; r = 1 without r_y, else a constant r_y = r"""
    xs = [b.x(r) for _, b in blocks]
    x = np.concatenate(xs)
    dev = project(lib, cone, x, None if r == 1 else np.full(x.size, float(r)), spectral)
    pos, worst = 0, 0.0
    for (name, b), xb in zip(blocks, xs):
        ratio = b.ratio(dev[pos:pos + xb.size], xb, r)
        worst = max(worst, ratio)
        assert ratio <= 1.0, (family, name, r, ratio)
        pos += xb.size
    assert pos == x.size
    WORST[family] = max(WORST.get(family, 0.0), worst)
    print(f"{family}: worst err / gate so far {WORST[family]:.3g}")


@pytest.mark.parametrize("r", [1, 4, 10])
@pytest.mark.parametrize("k", ee.PSD_ORDERS)
def test_psd_exact(lib, k, r):
    """several blocks of order k in one call, the positive / non-positive boundary at columns 0, 1, 31, 32, 33,
    k - 1 and k, exact zeros at columns 31 and 32, multiple eigenvalues and a 2^+-30 spread; the main and the
    spectral library"""
    blocks = ee.psd_order_blocks(k)
    cone = {"s": [k] * len(blocks)}
    _check_blocks(lib, cone, blocks, r, "psd")
    if r == 1:
        _check_blocks(capi.load(spectral=True), cone, blocks, r, "psd", spectral=True)


@pytest.mark.parametrize("r", [1, 4, 10])
def test_psd_mixed_orders_exact(lib, r):
    blocks = list(enumerate(ee.mixed_blocks()))
    _check_blocks(lib, {"s": ee.MIXED_ORDERS}, blocks, r, "psd")


@pytest.mark.parametrize("r", [1, 4, 10])
@pytest.mark.parametrize("kc", ee.CPSD_ORDERS)
def test_complex_psd_exact(lib, kc, r):
    blocks = ee.cpsd_order_blocks(kc)
    _check_blocks(lib, {"cs": [kc] * len(blocks)}, blocks, r, "complex psd")


@pytest.mark.parametrize("r", [1, 4, 10])
@pytest.mark.parametrize("mn", ee.NUC_SHAPES, ids=lambda mn: f"{mn[0]}x{mn[1]}")
def test_nuclear_exact(slib, mn, r):
    blocks = ee.nuc_shape_blocks(*mn)
    cone = {"nuc_m": [mn[0]] * len(blocks), "nuc_n": [mn[1]] * len(blocks)}
    _check_blocks(slib, cone, blocks, r, "nuclear")


@pytest.mark.parametrize("r", [1, 4, 10])
@pytest.mark.parametrize("n", ee.SL_ORDERS)
def test_sum_largest_exact(slib, n, r):
    blocks = ee.sl_order_blocks(n)
    cone = {"sl_n": [n] * len(blocks), "sl_k": [b.parts["k"] for _, b in blocks]}
    _check_blocks(slib, cone, blocks, r, "sum-largest")


# ---------------------------------------------------------------------------------------------- Gaussian inputs
def _mp_rows(v):
    """rows of 40-digit values as [(Fraction, False)] (exact binary values of the mpf numbers)"""
    return [(ee.mpf_fraction(a), False) for a in v]


@pytest.mark.parametrize("k", [5, 33, 40])
def test_psd_gaussian_against_mpmath(lib, k):
    """no structure a Householder construction could share with the eigensolver: Gaussian X, the projection from a
    40-digit mpmath eigendecomposition of the packed input itself (delta_in = 0)"""
    rng = np.random.default_rng(k)
    x = rng.standard_normal(k * (k + 1) // 2)
    ref = x + ee.mp_psd_packed(-x, k)
    b = ee.Block([(ee.mpf_fraction(-a), False) for a in x], _mp_rows(ref), k)
    _check_blocks(lib, {"s": [k]}, [("gaussian", b)], 1, "psd gaussian")


def test_complex_psd_gaussian_against_mpmath(lib):
    kc = 12
    x = np.random.default_rng(12).standard_normal(kc * kc)
    ref = x + ee.mp_cpsd_packed(-x, kc)
    b = ee.Block([(ee.mpf_fraction(-a), False) for a in x], _mp_rows(ref), 2 * kc)
    _check_blocks(lib, {"cs": [kc]}, [("gaussian", b)], 1, "complex psd gaussian")


def test_nuclear_gaussian_against_mpmath(slib):
    m, n = 20, 7
    rng = np.random.default_rng(20)
    x = np.concatenate(([-2.0], rng.standard_normal(m * n)))
    ref = x + ee.mp_nuclear(-x, m, n)
    b = ee.Block([(ee.mpf_fraction(-a), False) for a in x], _mp_rows(ref), m + n)
    _check_blocks(slib, {"nuc_m": [m], "nuc_n": [n]}, [("gaussian", b)], 1, "nuclear gaussian")

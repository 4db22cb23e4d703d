"""Seeded operator inputs of the spectral cones, shared by oracle/make_golden_spectral.py (which records the
reference's projections of them in tests/golden/spectral_cones.npz) and the tests that compare against that record.

Only the answers are stored: the inputs are regenerated here from fixed seeds. A projection is nonexpansive, so an
input that differed in its last bits (another BLAS in np.linalg) could move the answer by no more than that.
Answers of up to FULL_ROWS rows are stored whole; longer ones as SAMPLE seeded entries plus the largest one."""
import numpy as np

from scs_b200 import capi

FULL_ROWS = 1000
SAMPLE = 64
X_CHECK = 16  # entries of every input stored as well, to confirm that the regeneration matches


def sym_packed(M):
    """packed lower triangle, column-major, off-diagonals * sqrt2 (the PSD cone's vectorisation)"""
    n = M.shape[0]
    return np.concatenate([np.concatenate([[M[j, j]], np.sqrt(2.0) * M[j + 1:, j]]) for j in range(n)])


def _ell1_points(rng, n):
    v = rng.standard_normal(n)
    pts = [np.concatenate([[rng.standard_normal() * np.abs(v).sum() / 3], v])]
    pts.append(np.concatenate([[1.5 * np.abs(v).sum()], v]))      # inside the cone
    pts.append(np.concatenate([[-1.5 * np.abs(v).max()], v]))     # inside the polar cone
    w = np.round(v * 2) / 2                                       # repeated magnitudes
    pts.append(np.concatenate([[0.3 * np.abs(w).sum()], w]))
    return pts


def _nuc_points(rng, m, n):
    X = rng.standard_normal((m, n))
    U, s, Vt = np.linalg.svd(X, full_matrices=False)
    sr = np.repeat(np.abs(rng.standard_normal((n + 2) // 3)) + 0.5, 3)[:n]   # repeated singular values
    Xr = (U * sr) @ Vt
    pts = [np.concatenate([[rng.standard_normal() * s.sum() / 3], X.ravel(order="F")])]
    pts.append(np.concatenate([[1.5 * s.sum()], X.ravel(order="F")]))      # inside the cone
    pts.append(np.concatenate([[-1.5 * s.max()], X.ravel(order="F")]))     # inside the polar cone
    pts.append(np.concatenate([[0.4 * sr.sum()], Xr.ravel(order="F")]))
    pts.append(np.concatenate([[0.7], np.zeros(m * n)]))                   # zero matrix
    return pts


def _sl_points(rng, n, k):
    A = rng.standard_normal((n, n))
    A = (A + A.T) / 2
    lam, V = np.linalg.eigh(A)
    lr = np.repeat(rng.standard_normal((n + 2) // 3), 3)[:n]                 # repeated eigenvalues
    Ar = (V * lr) @ V.T
    top = np.sort(lam)[::-1][:k].sum()
    w = rng.random(n)
    w = np.minimum(w * k / w.sum(), 1.0)
    W = (V * w) @ V.T                                                       # 0 <= W <= I, tr W <= k
    pts = [np.concatenate([[top + rng.standard_normal()], sym_packed(A)])]
    pts.append(np.concatenate([[top + 1.0], sym_packed(A)]))               # inside the cone
    pts.append(np.concatenate([[-2.0], sym_packed(2.0 * W)]))              # inside the polar cone
    pts.append(np.concatenate([[np.sort(lr)[::-1][:k].sum() - 0.5], sym_packed(Ar)]))
    pts.append(np.concatenate([[-0.3], np.zeros(n * (n + 1) // 2)]))       # zero matrix
    return pts


def _join(rng, make, shapes):
    return [np.concatenate(parts) for parts in zip(*[make(rng, *sh) for sh in shapes])]


# name -> (seed, cone); the l1 cone of 9000 entries takes the chunked path (above 8192), sl_100_1 is the C4 shape
CASES = {
    "ell1_5": (11, {"ell1": [1, 2, 5]}),
    "ell1_200": (12, {"ell1": [64, 200]}),
    "ell1_9000": (13, {"ell1": [9000]}),
    "nuc_5x2": (21, {"nuc_m": [1, 3, 5], "nuc_n": [1, 3, 2]}),
    "nuc_20x5": (22, {"nuc_m": [12, 20], "nuc_n": [12, 5]}),
    "nuc_100x60": (23, {"nuc_m": [100, 120], "nuc_n": [60, 4]}),
    "sl_5_4": (31, {"sl_n": [2, 3, 3, 5], "sl_k": [1, 1, 2, 4]}),
    "sl_16_15": (32, {"sl_n": [10, 10, 16, 16], "sl_k": [1, 9, 7, 15]}),
    "sl_40_39": (33, {"sl_n": [40, 40], "sl_k": [7, 39]}),
    "sl_100_1": (34, {"sl_n": [100], "sl_k": [1]}),
    "mixed": (41, {"z": 2, "l": 3, "q": [4, 10], "s": [3, 5], "nuc_m": [4, 6], "nuc_n": [3, 6], "ell1": [5, 120],
                   "sl_n": [4, 12], "sl_k": [1, 11]}),
}
BIG_POINTS = (0, 2, 3)  # cases over FULL_ROWS rows keep the random, polar and repeated-value points only


def inputs(name):
    """the cone dict and the list of input vectors of case `name`"""
    seed, cone = CASES[name]
    rng = np.random.default_rng(seed)
    if name == "mixed":
        m = capi.cone_rows(cone)
        return cone, [rng.standard_normal(m) * 10.0 ** e for e in (-1, 0, 2)]
    if "ell1" in cone:
        xs = _join(rng, _ell1_points, [(n,) for n in cone["ell1"]])
    elif "nuc_m" in cone:
        xs = _join(rng, _nuc_points, list(zip(cone["nuc_m"], cone["nuc_n"])))
    else:
        xs = _join(rng, _sl_points, list(zip(cone["sl_n"], cone["sl_k"])))
    return cone, (xs if len(xs[0]) <= FULL_ROWS else [xs[i] for i in BIG_POINTS])


def r_y(cone):
    ry = np.full(capi.cone_rows(cone), 10.0)
    ry[: cone.get("z", 0)] = 1e-2
    return ry


def stored_index(m, out):
    """which entries of an answer of length m are stored: all (recorded as an empty index), or SAMPLE seeded ones
    plus the largest"""
    if m <= FULL_ROWS:
        return np.zeros(0, dtype=np.int32)
    idx = np.random.default_rng(m).choice(m, SAMPLE, replace=False)
    return np.unique(np.append(idx, int(np.argmax(np.abs(out)))))


def check_index(m):
    return np.random.default_rng(m + 1).choice(m, min(m, X_CHECK), replace=False)


def recorded(gold, name, i, metric):
    """(entry indices, reference values) of answer i of case `name` (metric: with r_y)"""
    tag = "ry" if metric else ""
    idx, out = gold[f"{name}/idx{tag}{i}"], gold[f"{name}/out{tag}{i}"]
    return (idx if idx.size else np.arange(out.size)), out


def check_regenerated(gold, name, i, x):
    ci = check_index(x.size)
    assert np.allclose(x[ci], gold[f"{name}/xcheck{i}"], rtol=1e-14, atol=1e-14), \
        f"{name}: regenerated input {i} does not match the recorded one"

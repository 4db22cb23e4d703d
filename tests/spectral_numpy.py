"""numpy restatement of the nuclear-norm, l1-norm and sum-of-largest-eigenvalues cone projections, written from the
math (not from any C source). Used by tests/test_spectral_cones_cpu.py against the recorded reference answers and as
the cone-distance clause of the spectral solves in tests/test_spectral_cones_gpu.py.

Vectorisations (SCS): l1 cone (t, x), 1 + n rows; nuclear-norm cone (t, X) with X m x n column-major, m >= n;
sum-of-largest cone (t, X) with X symmetric n x n as its packed lower triangle, column-major, off-diagonals * sqrt2.
"""
import numpy as np

from scs_b200 import problems

SQRT2 = np.sqrt(2.0)
SL_TOL = 1e-9  # SCS stops the sum-of-largest vector step once S_k <= t + 1e-9 (in the sqrt2-scaled units)


def proj_ell1(t, v):
    """Pi onto {(t, v): ||v||_1 <= t}: (t + mu, sign(v) max(|v| - mu, 0)), mu >= 0 solving
    sum max(|v_i| - mu, 0) = t + mu."""
    a = np.abs(v)
    if a.size == 0 or -t >= a.max():
        return 0.0, np.zeros_like(v)
    if a.sum() <= t:
        return t, v.copy()
    s = np.sort(a)[::-1]
    cs = np.cumsum(s)
    k = np.arange(1, s.size + 1)
    mus = (cs - t) / (k + 1)
    nxt = np.append(s[1:], 0.0)
    ok = np.nonzero((s > mus) & (nxt <= mus))[0]
    mu = mus[ok[0]] if ok.size else mus[-1]
    mu = max(mu, 0.0)
    return t + mu, np.sign(v) * np.maximum(a - mu, 0.0)


def proj_nuclear(t, X):
    """Pi onto {(t, X): ||X||_* <= t}: the l1 projection of (t, sigma), then U diag(sigma') V'."""
    U, s, Vt = np.linalg.svd(X, full_matrices=False)
    tn, sn = proj_ell1(t, s)
    return tn, (U * sn) @ Vt


def _theta(lam, eta, k):
    """theta with sum_i clip((lam_i - theta) / eta, 0, 1) = k (piecewise linear, decreasing in theta)"""
    pts = np.sort(np.concatenate([lam, lam - eta]))

    def h(th):
        return np.clip((lam - th) / eta, 0.0, 1.0).sum() - k

    hv = np.array([h(p) for p in pts])
    i = np.nonzero(hv <= 0)[0][0]  # h decreasing; h(min pt) = n - k > 0 ... first breakpoint with h <= 0
    lo, hi = pts[i - 1], pts[i]
    return lo + (hi - lo) * hv[i - 1] / (hv[i - 1] - hv[i])


def proj_sum_largest_vec(t, lam, k):
    """Pi onto {(t, x): sum of the k largest x_i <= t}. KKT: x = lam - eta w, t' = t + eta, with w in
    {0 <= w <= 1, sum w = k} maximising w'x; i.e. x_i = min(lam_i, max(lam_i - eta, theta)) and eta >= 0 the root of
    S_k(x(eta)) = t + eta (decreasing in eta), found by bisection to the last bit."""
    def x_of(eta):
        th = _theta(lam, eta, k)
        return np.minimum(lam, np.maximum(lam - eta, th))

    def g(eta):
        return np.sort(x_of(eta))[::-1][:k].sum() - t - eta

    lo, hi = 0.0, max(np.sort(lam)[::-1][:k].sum() - t, 1e-300)
    for _ in range(2000):
        mid = 0.5 * (lo + hi)
        if mid <= lo or mid >= hi:
            break
        if g(mid) > 0:
            lo = mid
        else:
            hi = mid
    eta = hi
    return t + eta, x_of(eta)


def packed_to_sym(p, n):
    M = np.zeros((n, n))
    pos = 0
    for j in range(n):
        M[j:, j] = p[pos:pos + n - j]
        pos += n - j
    M = M + np.tril(M, -1).T
    return M / SQRT2 + np.diag(np.diag(M)) * (1 - 1 / SQRT2)


def sym_to_packed(M):
    n = M.shape[0]
    return np.concatenate([np.concatenate([[M[j, j]], SQRT2 * M[j + 1:, j]]) for j in range(n)])


def proj_sum_largest(t, p, n, k):
    """Pi onto {(t, X): sum of the k largest eigenvalues of X <= t}, X packed"""
    M = packed_to_sym(p, n)
    lam, V = np.linalg.eigh(M)
    if np.sort(SQRT2 * lam)[::-1][:k].sum() <= SQRT2 * t + SL_TOL:
        return t, p.copy()
    tn, ln = proj_sum_largest_vec(t, lam, k)
    return tn, sym_to_packed((V * ln) @ V.T)


def proj_spectral(v, cone):
    """Pi_K on the spectral rows v (nuclear, then l1, then sum-of-largest cones)"""
    out = np.empty_like(v)
    pos = 0
    for m, n in zip(cone.get("nuc_m", []) or [], cone.get("nuc_n", []) or []):
        tn, Xn = proj_nuclear(v[pos], v[pos + 1:pos + 1 + m * n].reshape((m, n), order="F"))
        out[pos], out[pos + 1:pos + 1 + m * n] = tn, Xn.ravel(order="F")
        pos += 1 + m * n
    for n in cone.get("ell1", []) or []:
        out[pos], out[pos + 1:pos + 1 + n] = proj_ell1(v[pos], v[pos + 1:pos + 1 + n])
        pos += 1 + n
    for n, k in zip(cone.get("sl_n", []) or [], cone.get("sl_k", []) or []):
        r = n * (n + 1) // 2
        out[pos], out[pos + 1:pos + 1 + r] = proj_sum_largest(v[pos], v[pos + 1:pos + 1 + r], n, k)
        pos += 1 + r
    assert pos == v.size
    return out


def base_cone(cone):
    return {key: val for key, val in cone.items() if key not in ("d", "nuc_m", "nuc_n", "ell1", "sl_n", "sl_k")}


def proj_dual_cone(v, cone, r_y=None):
    """SCS's Moreau wrapper x + R^-1 Pi_K^R(-R x) ... restated for R = I on the spectral rows: Pi_K*(v) = v + Pi_K(-v);
    the other rows by scs_b200.problems.proj_dual_cone. r_y must be None."""
    assert r_y is None
    from scs_b200 import capi
    m0 = capi.cone_rows(base_cone(cone))
    out = np.empty_like(v)
    out[:m0] = problems.proj_dual_cone(v[:m0], base_cone(cone)) if m0 else v[:0]
    out[m0:] = v[m0:] + proj_spectral(-v[m0:], cone)
    return out

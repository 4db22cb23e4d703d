"""Inputs with exactly known eigen- and singular-value decompositions for the eigen-decomposition cones, and their
projections in exact arithmetic (tests/test_eigen_cones_exact_cpu.py checks the references themselves,
tests/test_eigen_cones_exact_gpu.py the device against them).

Orthogonal factors: products of layers of Householder reflectors H = I - 2 v v' / (v'v), v in {0, +-1}^k with
nnz(v) = 4^j (4, 16 or 64), so 2 / (v'v) is a power of two and every entry dyadic. A layer is a set of disjoint
reflectors that covers every coordinate (the last one overlapping its neighbour when the order is not a multiple of
its size); layers of different sizes are joined by random permutations and signs, so their supports overlap. With
the layers' factors 2^-1, 2^-3, 2^-5, Q = Z / 2^D for an integer matrix Z. Unitary factors of the complex cone put a
diagonal of phases in {+-1, +-i} between the layers (a phase next to a real diagonal Lambda would cancel).

All matrix arithmetic is on integers (numpy int64 where a bound shows the products cannot overflow, Python ints
otherwise) and Fractions. The packed vectors carry sqrt(2) on their off-diagonals, so the distance of a device answer
to an exact reference, and the input rounding delta_in = ||x~ - x_exact||_2, are evaluated with mpmath at 40
significant digits from the exact values; that evaluation error (~1e-40 relative) is far below anything gated.

The gate: every map here is a Euclidean projection onto a closed convex cone in the sqrt2-scaled vector space (the
Moreau wrapper x + Pi_K(-r x) / r = Pi_K*(x) for a constant r > 0 included), hence 1-Lipschitz, so a backward-stable
eigensolver keeps the device within
    ||dev - ref||_2 <= delta_in + C N 2^-53 ||x||_2,   N the order the eigensolver sees (k, 2 kc or m + n), C = 64,
whatever the eigenvalue gaps are."""
import functools
import math
import zlib
from fractions import Fraction

import mpmath
import numpy as np

C_GATE = 64
U = 2.0 ** -53
mpmath.mp.dps = 40
SQ2 = mpmath.sqrt(2)
INT64_SAFE = 2 ** 62


# ---------------------------------------------------------------------------------------------- exact integer algebra
def imatmul(A, B):
    """exact product of integer matrices: int64 when max|A| max|B| inner < 2^62, Python ints otherwise"""
    A, B = np.asarray(A), np.asarray(B)
    amax = max((abs(int(v)) for v in A.flat), default=0)
    bmax = max((abs(int(v)) for v in B.flat), default=0)
    if amax * bmax * max(A.shape[-1], 1) < INT64_SAFE:
        return A.astype(np.int64) @ B.astype(np.int64)
    return A.astype(object) @ B.astype(object)


def cmatmul(A, B):
    """exact product of Gaussian-integer matrices given as (re, im) pairs"""
    (a, b), (c, d) = A, B
    return imatmul(a, c) - imatmul(b, d), imatmul(a, d) + imatmul(b, c)


def ctrans(A):
    return A[0].T.copy(), -A[1].T


class Factor:
    """Q = Z / 2^D (real: Z an integer matrix; complex: Z = (re, im))"""

    def __init__(self, Z, D):
        self.Z, self.D = Z, D

    def is_complex(self):
        return isinstance(self.Z, tuple)


def orthogonal(k, rng, sizes=None, phases=False):
    """Q = P_L S_L H_L ... P_1 S_1 H_1 (P permutations, S signs or phases, H layers), as a Factor. sizes: the layers'
    reflector sizes (default: every one of 4, 16, 64 not above k; none below order 4, leaving a signed permutation)"""
    if sizes is None:
        sizes = [s for s in (4, 16, 64) if s <= k]
    Z = np.eye(k, dtype=np.int64)
    Zc = (Z, np.zeros((k, k), np.int64))
    D = 0
    for s in list(sizes) + [None]:
        if s is not None:
            # disjoint reflectors commute: the layer is I - (2/s) sum_a v_a v_a', scaled by s/2 to stay integral;
            # when s does not divide k, one more reflector on the last s coordinates follows
            starts = list(range(0, k - s + 1, s))
            groups = [starts] + ([[k - s]] if starts[-1] + s < k else [])
            for group in groups:
                H = np.eye(k, dtype=np.int64) * (s // 2)
                for a in group:
                    v = np.zeros(k, np.int64)
                    v[a:a + s] = rng.choice([-1, 1], s)
                    H -= np.outer(v, v)
                Zc = (imatmul(H, Zc[0]), imatmul(H, Zc[1]))
                D += {4: 1, 16: 3, 64: 5}[s]
        perm = rng.permutation(k)
        if phases:
            ph = rng.integers(0, 4, k)  # i^ph
            re = np.where(ph == 0, 1, np.where(ph == 2, -1, 0))
            im = np.where(ph == 1, 1, np.where(ph == 3, -1, 0))
            a, b = Zc[0][perm], Zc[1][perm]
            Zc = (re[:, None] * a - im[:, None] * b, re[:, None] * b + im[:, None] * a)
        else:
            sg = rng.choice([-1, 1], k)
            Zc = (sg[:, None] * Zc[0][perm], sg[:, None] * Zc[1][perm])
    return Factor(Zc if phases else Zc[0], D)


def check_orthogonal(Q):
    """Q* Q = I exactly, i.e. Z* Z = 4^D I"""
    k = (Q.Z[0] if Q.is_complex() else Q.Z).shape[0]
    I4 = np.eye(k, dtype=object) * (4 ** Q.D)
    if Q.is_complex():
        re, im = cmatmul(ctrans(Q.Z), Q.Z)
        return bool(np.all(re.astype(object) == I4) and np.all(im == 0))
    return bool(np.all(imatmul(Q.Z.T, Q.Z).astype(object) == I4))


# ---------------------------------------------------------------------------------------------- exact spectra
def _common(w):
    """[Fraction] -> (integer numerators as objects, common denominator)"""
    fr = [Fraction(v) for v in w]
    L = math.lcm(*(f.denominator for f in fr))
    return np.array([int(f * L) for f in fr], dtype=object), L


def fractions(M, den):
    """integer matrix / den -> Fraction matrix (object array)"""
    return np.vectorize(lambda v: Fraction(int(v), den), otypes=[object])(M)


def qdq(Q, w):
    """Q diag(w) Q* exactly: a Fraction matrix, or a (re, im) pair of them for a unitary Q"""
    num, L = _common(w)
    den = 4 ** Q.D * L
    if Q.is_complex():
        Zl = (Q.Z[0].astype(object) * num[None, :], Q.Z[1].astype(object) * num[None, :])
        return tuple(fractions(m, den) for m in cmatmul(Zl, ctrans(Q.Z)))
    return fractions(imatmul(Q.Z.astype(object) * num[None, :], Q.Z.T), den)


def udv(Uf, Vf, w):
    """U[:, :n] diag(w) V' exactly (U of order m >= n = order of V)"""
    num, L = _common(w)
    n = len(w)
    return fractions(imatmul(Uf.Z[:, :n].astype(object) * num[None, :], Vf.Z.T), 2 ** (Uf.D + Vf.D) * L)


def exact_float(F):
    """float64 matrix of a Fraction matrix; asserts each entry is exactly representable"""
    out = np.array([float(v) for v in F.flat]).reshape(F.shape)
    bad = [v for v, f in zip(F.flat, out.flat) if Fraction(f) != v]
    assert not bad, f"{len(bad)} entries are not representable in fp64, e.g. {bad[0]}"
    return out


# ---------------------------------------------------------------------------------------------- packing (sqrt2 scaled)
def packed_sym(F):
    """Fraction matrix -> [(value, scaled)] of the packed lower triangle, column-major; scaled: carries sqrt2"""
    k = F.shape[0]
    return [(F[i, j], i != j) for j in range(k) for i in range(j, k)]


def packed_herm(Fre, Fim):
    """Hermitian (Fraction re, im) -> [(value, scaled)] in the complex PSD layout"""
    k = Fre.shape[0]
    out = []
    for j in range(k):
        out.append((Fre[j, j], False))
        for i in range(j + 1, k):
            out += [(Fre[i, j], True), (Fim[i, j], True)]
    return out


def mp_value(v, scaled):
    a = mpmath.mpf(int(v.numerator)) / int(v.denominator)
    return SQ2 * a if scaled else a


def float_input(entries, r=1):
    """x~: the float64 vector the device is given for the exact vector entries / r (rounded once per entry)"""
    return np.array([float(mp_value(v, s) / r) for v, s in entries])


def mp_dist(a, entries, r=1):
    """||a - entries / r||_2 with a float64, at 40 digits"""
    return mpmath.sqrt(mpmath.fsum((mpmath.mpf(float(x)) - mp_value(v, s) / r) ** 2 for x, (v, s) in zip(a, entries)))


def gate(delta_in, N, x):
    return float(delta_in) + C_GATE * N * U * float(np.linalg.norm(x))


# ---------------------------------------------------------------------------------------------- projections, exactly
def ell1_threshold(t, a):
    """exact mu >= 0 of Pi onto {(t, a): ||a||_1 <= t} for a >= 0 (Fractions): (t + mu, max(a - mu, 0)); mu = None when
    -t >= max a (Pi = 0). a may also be a numpy integer array with an integer t (the path for long vectors)."""
    if isinstance(a, np.ndarray):
        return _ell1_threshold_int(t, a)
    if not a or -t >= max(a):
        return None
    if sum(a) <= t:
        return Fraction(0)
    s = sorted(a, reverse=True)
    cs = Fraction(0)
    for j, v in enumerate(s):
        cs += v
        mu = (cs - t) / (j + 2)
        nxt = s[j + 1] if j + 1 < len(s) else Fraction(0)
        if v > mu >= nxt:
            return mu
    raise AssertionError("no threshold")


def _ell1_threshold_int(t, a):
    """ell1_threshold for integer magnitudes (numpy, sum below 2^62) and an integer t: the same sorted scan on int64
    prefix sums, the threshold (cs_j - t) / (j + 2) compared by cross-multiplication"""
    T = int(t)
    assert T == t and a.dtype.kind in "iu"
    a = a.astype(np.int64)
    if a.size == 0 or -T >= int(a.max()):
        return None
    if int(a.sum()) <= T:
        return Fraction(0)
    s = np.sort(a)[::-1]
    cs = np.cumsum(s)
    j2 = np.arange(2, s.size + 2, dtype=np.int64)
    nxt = np.append(s[1:], 0)
    ok = np.nonzero((s * j2 > cs - T) & (cs - T >= nxt * j2))[0]
    assert ok.size, "no threshold"
    return Fraction(int(cs[ok[0]]) - T, int(j2[ok[0]]))


def proj_ell1_exact(t, a):
    mu = ell1_threshold(t, a)
    if mu is None:
        return Fraction(0), [Fraction(0)] * len(a)
    return t + mu, [max(v - mu, Fraction(0)) for v in a]


def proj_sum_largest_exact(t, lam, k):
    """exact Pi onto {(t, x): sum of the k largest x_i <= t} (Fractions): x = lam - eta w with w in the capped simplex
    {0 <= w <= 1, sum w = k}, t' = t + eta. With lam sorted descending: the first u entries drop by eta, the next s
    are cut to a level theta (lam_i - eta <= theta <= lam_i), the rest stay (lam_i <= theta); every (u, s) is tried and
    the one whose solution meets these conditions is returned (the projection is unique)."""
    order = sorted(range(len(lam)), key=lambda i: -lam[i])
    L = [lam[i] for i in order]
    n = len(L)
    if sum(L[:k]) <= t:
        return t, list(lam)
    for u in range(0, k + 1):
        for s in range(0, n - u + 1):
            if s == 0:
                if u != k:
                    continue
                eta = (sum(L[:k]) - t) / (k + 1)
                theta = L[k - 1] - eta
                ok = eta >= 0 and all(L[i] <= theta for i in range(k, n))
            else:
                if not u < k < u + s + 1 or k - u > s:
                    continue
                # sum_{i<u} (L_i - eta) + (k - u) theta = t + eta ; sum_tie L_i - s theta = (k - u) eta
                A, T = sum(L[:u]), sum(L[u:u + s])
                # from the second: theta = (T - (k - u) eta) / s; substitute into the first
                # A - u eta + (k - u) (T - (k - u) eta) / s = t + eta
                den = (u + 1) + Fraction((k - u) ** 2, s)
                eta = (A + Fraction(k - u, s) * T - t) / den
                theta = (T - (k - u) * eta) / s
                ok = (eta >= 0 and all(L[i] - eta >= theta for i in range(u))
                      and all(L[i] - eta <= theta <= L[i] for i in range(u, u + s))
                      and all(L[i] <= theta for i in range(u + s, n)))
            if ok:
                x = [None] * n
                for pos, i in enumerate(order):
                    x[i] = L[pos] - eta if pos < u else (theta if pos < u + s else L[pos])
                return t + eta, x
    raise AssertionError("no active set")


def sum_largest(x, k):
    return sum(sorted(x, reverse=True)[:k])


# ---------------------------------------------------------------------------------------------- blocks
class Block:
    """one cone block: v, the rows the projection sees, and Pi(v) - v, both as [(Fraction, carries sqrt2)]; N the
    order the eigensolver sees. The device is given x = -v / r and returns x + Pi_K(-r x) / r = (Pi(v) - v) / r."""

    def __init__(self, v, out, N, **parts):
        self.v, self.out, self.N = v, out, N
        self.parts = parts

    def x(self, r=1):
        """x~ = fl(-v / r), rounded once per entry"""
        return np.array([float(-mp_value(a, s) / r) for a, s in self.v])

    def delta_in(self, x, r=1):
        """||x~ - x_exact||_2"""
        return mp_dist(x, [(-a, s) for a, s in self.v], r)

    def ratio(self, dev, x, r=1):
        """||dev - ref||_2 / (delta_in + C N 2^-53 ||x~||_2)"""
        return float(mp_dist(dev, self.out, r)) / gate(self.delta_in(x, r), self.N, x)


def _sub(A, B):
    return np.vectorize(lambda a, b: a - b, otypes=[object])(A, B)


def psd_block(k, lam, rng, sizes=None):
    Q = orthogonal(k, rng, sizes)
    lam = [Fraction(v) for v in lam]
    X, P = qdq(Q, lam), qdq(Q, [max(v, 0) for v in lam])
    exact_float(X)
    return Block(packed_sym(X), packed_sym(_sub(P, X)), k, Q=Q, lam=lam, X=X, P=P)


def cpsd_block(kc, lam, rng):
    Q = orthogonal(kc, rng, phases=True)
    lam = [Fraction(v) for v in lam]
    (Xr, Xi), (Pr, Pi) = qdq(Q, lam), qdq(Q, [max(v, 0) for v in lam])
    exact_float(Xr), exact_float(Xi)
    return Block(packed_herm(Xr, Xi), packed_herm(_sub(Pr, Xr), _sub(Pi, Xi)), 2 * kc, Q=Q, lam=lam, X=(Xr, Xi),
                 P=(Pr, Pi))


def nuc_block(m, n, sig, t, rng):
    """(t, X) with X = U[:, :n] diag(sig) V', m x n column-major"""
    Uf, Vf = orthogonal(m, rng), orthogonal(n, rng)
    sig, t = [Fraction(v) for v in sig], Fraction(t)
    tn, sn = proj_ell1_exact(t, sig)
    X, P = udv(Uf, Vf, sig), udv(Uf, Vf, sn)
    exact_float(X)
    flat = lambda M: [(v, False) for v in M.flatten(order="F")]  # noqa: E731
    return Block([(t, False)] + flat(X), [(tn - t, False)] + flat(_sub(P, X)), m + n, U=Uf, V=Vf, sig=sig, t=t,
                 tn=tn, sn=sn)


def sl_block(n, k, lam, t, rng):
    """(t, X) with X = Q diag(lam) Q', packed"""
    Q = orthogonal(n, rng)
    lam, t = [Fraction(v) for v in lam], Fraction(t)
    tn, xn = proj_sum_largest_exact(t, lam, k)
    X, P = qdq(Q, lam), qdq(Q, xn)
    exact_float(X)
    return Block([(t, False)] + packed_sym(X), [(tn - t, False)] + packed_sym(_sub(P, X)), n, Q=Q, lam=lam, t=t,
                 tn=tn, xn=xn, k=k)


# ---------------------------------------------------------------------------------------------- the cases
def _rng(*key):
    return np.random.default_rng([20261017, *[zlib.crc32(v.encode()) if isinstance(v, str) else v for v in key]])


def psd_spectrum(k, p, rng, zeros=()):
    """k eigenvalues, p of them positive (small integers and halves), the rest <= 0; exact zeros at the ascending
    positions `zeros`"""
    neg = sorted(Fraction(-int(v), 2) for v in rng.integers(1, 9, k - p))
    pos = sorted(Fraction(int(v), 2) for v in rng.integers(1, 9, p))
    lam = neg + pos
    for i in zeros:
        lam[i] = Fraction(0)
    return [lam[i] for i in rng.permutation(k)]


PSD_ORDERS = [2, 3, 31, 32, 33, 63, 64, 65, 97, 128, 129, 200]


@functools.lru_cache(maxsize=None)
def psd_order_blocks(k):
    """the blocks of order k: p in {0, 1, 31, 32, 33, k-1, k} positive eigenvalues, exact zeros at ascending positions
    31 and 32, c I, c I plus rank one of either sign, and eigenvalues 2^-30 ... 2^30 (with a signed permutation for
    Q: no nontrivial Q keeps such a matrix representable) and 2^-16 ... 2^16 (one layer of 4-reflectors)"""
    rng = _rng("psd", k)
    out = []
    for p in sorted({p for p in (0, 1, 31, 32, 33, k - 1, k) if 0 <= p <= k}):
        out.append((f"p{p}", psd_block(k, psd_spectrum(k, p, rng), rng)))
    if k >= 34:
        out.append(("zeros31_32", psd_block(k, psd_spectrum(k, k - 33, rng, zeros=(31, 32)), rng)))
    out.append(("cI", psd_block(k, [Fraction(3, 2)] * k, rng)))
    out.append(("-cI", psd_block(k, [Fraction(-3, 2)] * k, rng)))
    out.append(("-cI+rank1", psd_block(k, [Fraction(-1)] * (k - 1) + [Fraction(5, 2)], rng)))
    out.append(("cI-rank1", psd_block(k, [Fraction(2)] * (k - 1) + [Fraction(-3)], rng)))
    e30 = [Fraction(2) ** int(e) * int(sg) for e, sg in zip(rng.integers(-30, 31, k), rng.choice([-1, 1], k))]
    out.append(("spread30", psd_block(k, e30, rng, sizes=())))
    if k >= 4:
        e16 = [Fraction(2) ** int(e) * int(sg) for e, sg in zip(rng.integers(-16, 17, k), rng.choice([-1, 1], k))]
        out.append(("spread16", psd_block(k, e16, rng, sizes=(4,))))
    return out


MIXED_ORDERS = [1, 2, 33, 2, 1, 65, 33]


@functools.lru_cache(maxsize=None)
def mixed_blocks():
    """interleaved orders in one cone, each block with its own number of positive eigenvalues"""
    rng = _rng("mixed")
    ps = [1, 0, 32, 2, 0, 33, 1]
    return [psd_block(k, psd_spectrum(k, p, rng), rng) for k, p in zip(MIXED_ORDERS, ps)]


CPSD_ORDERS = [1, 2, 15, 16, 17, 31, 32, 33]


@functools.lru_cache(maxsize=None)
def cpsd_order_blocks(kc):
    rng = _rng("cpsd", kc)
    return [(f"p{p}", cpsd_block(kc, psd_spectrum(kc, p, rng), rng))
            for p in sorted({0, 1, kc // 2, kc - 1, kc})]


NUC_SHAPES = [(1, 1), (2, 1), (32, 32), (33, 32), (33, 1), (64, 33), (65, 65), (100, 7)]


@functools.lru_cache(maxsize=None)
def nuc_shape_blocks(m, n):
    """full rank, rank deficient (half the singular values 0) and repeated singular values, each with t inside the
    cone, in the polar cone and in between"""
    rng = _rng("nuc", m, n)
    out = []
    full = [Fraction(int(v), 2) for v in rng.integers(1, 9, n)]
    deficient = [v if i % 2 else Fraction(0) for i, v in enumerate(full)] if n > 1 else [Fraction(0)]
    repeated = [Fraction(3, 2)] * n
    for name, sig in (("full", full), ("deficient", deficient), ("repeated", repeated)):
        s1, smax = sum(sig), max(sig)
        for where, t in (("inside", s1 + 1), ("polar", -smax - 1), ("between", (s1 - smax) / 2 if s1 > 0 else -1)):
            if name == "deficient" and n == 1 and where == "between":
                t = Fraction(-1, 2)
            out.append((f"{name}_{where}", nuc_block(m, n, sig, t, rng)))
    return out


SL_ORDERS = [2, 31, 32, 33, 65]


@functools.lru_cache(maxsize=None)
def sl_order_blocks(n):
    """k in {1, n // 2, n - 1}; ties at the k-th largest eigenvalue; t between the cone and its polar (S_k - t >= 1)
    and inside"""
    rng = _rng("sl", n)
    out = []
    for k in sorted({1, n // 2, n - 1}):
        lam = sorted((Fraction(int(v), 2) for v in rng.integers(-8, 9, n)), reverse=True)
        tied = list(lam)
        lo = max(k - 2, 0)
        for i in range(lo, min(k + 2, n)):
            tied[i] = lam[k - 1]  # the k-th largest and its neighbours equal
        for name, l in (("plain", lam), ("ties", tied)):
            sk = sum(sorted(l, reverse=True)[:k])
            for where, t in (("between", sk - 3), ("far", sk - 40), ("inside", sk + 1)):
                out.append((f"k{k}_{name}_{where}", sl_block(n, k, [l[i] for i in rng.permutation(n)], t, rng)))
    return out


# ---------------------------------------------------------------------------------------------- 40-digit references
def mpf_fraction(a):
    """the exact binary value of a float or an mpf"""
    if isinstance(a, float) or isinstance(a, np.floating):
        return Fraction(float(a))
    sign, man, exp, _ = a._mpf_
    f = Fraction(int(man) * 2 ** exp) if exp >= 0 else Fraction(int(man), 2 ** -exp)
    return -f if sign else f


def _mp_sym(v, k):
    M = mpmath.matrix(k, k)
    pos = 0
    for j in range(k):
        for i in range(j, k):
            M[i, j] = M[j, i] = mpmath.mpf(float(v[pos])) / (1 if i == j else SQ2)
            pos += 1
    return M


def mp_psd_packed(v, k):
    """Pi_PSD of the packed (sqrt2-scaled) float vector v, from mpmath.eigsy at 40 digits, packed"""
    E, Q = mpmath.eigsy(_mp_sym(v, k))
    P = Q * mpmath.diag([max(e, 0) for e in E]) * Q.T
    return np.array([P[i, j] * (SQ2 if i != j else 1) for j in range(k) for i in range(j, k)], dtype=object)


def mp_cpsd_packed(v, kc):
    H = mpmath.matrix(kc, kc)
    for j in range(kc):
        base = j * (2 * kc - j)
        H[j, j] = mpmath.mpf(float(v[base]))
        for i in range(j + 1, kc):
            z = mpmath.mpc(float(v[base + 1 + 2 * (i - j - 1)]), float(v[base + 2 + 2 * (i - j - 1)])) / SQ2
            H[i, j], H[j, i] = z, mpmath.conj(z)
    E, Q = mpmath.eighe(H)
    P = Q * mpmath.diag([max(e, 0) for e in E]) * Q.transpose_conj()
    out = []
    for j in range(kc):
        out.append(mpmath.re(P[j, j]))
        for i in range(j + 1, kc):
            out += [SQ2 * mpmath.re(P[i, j]), SQ2 * mpmath.im(P[i, j])]
    return np.array(out, dtype=object)


def mp_nuclear(v, m, n):
    """Pi onto the nuclear-norm cone of (t, X) (X m x n column-major) from mpmath.svd_r at 40 digits"""
    X = mpmath.matrix(m, n)
    for j in range(n):
        for i in range(m):
            X[i, j] = mpmath.mpf(float(v[1 + i + j * m]))
    Um, S, Vm = mpmath.svd_r(X)
    tn, sn = proj_ell1_exact(Fraction(float(v[0])), [mpf_fraction(s) for s in S])
    P = Um * mpmath.diag([mpmath.mpf(s.numerator) / s.denominator for s in sn]) * Vm
    return np.array([mpmath.mpf(tn.numerator) / tn.denominator] + [P[i, j] for j in range(n) for i in range(m)],
                    dtype=object)


# ---------------------------------------------------------------------------------------------- checks of the references
def congruence_diagonal(Q, F):
    """Q* F Q for a Fraction matrix F (a (re, im) pair for a unitary Q), exactly: its diagonal when it is diagonal,
    else None. With Q orthogonal (check_orthogonal), a nonnegative diagonal proves F PSD, a nonpositive one F NSD."""
    parts = F if Q.is_complex() else (F,)
    num, L = _common([v for part in parts for v in part.flat])
    k = parts[0].shape[0]
    ints = [num[i * k * k:(i + 1) * k * k].reshape(k, k) for i in range(len(parts))]
    if Q.is_complex():
        W, Wi = cmatmul(cmatmul(ctrans(Q.Z), tuple(ints)), Q.Z)
        if np.any(Wi != 0):
            return None
    else:
        W = imatmul(imatmul(Q.Z.T, ints[0]), Q.Z)
    W = W.astype(object)
    if np.any(W - np.diag(np.diag(W)) != 0):
        return None
    return [Fraction(int(v), 4 ** Q.D * L) for v in np.diag(W)]


def inner(A, B):
    """<A, B> of Fraction matrices (or (re, im) pairs: the real part of tr(A* B))"""
    if isinstance(A, tuple):
        return sum(inner(a, b) for a, b in zip(A, B))
    return sum(a * b for a, b in zip(A.flat, B.flat))

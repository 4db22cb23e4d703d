"""Inputs with exactly known projections for the second-order, box and l1-norm cones, and those projections in
integer and Fraction arithmetic (tests/test_vector_cones_exact_cpu.py checks the references themselves,
tests/test_vector_cones_exact_gpu.py the device against them).

Every block is v * 2^e with v an integer vector (entries below 2^53) and e a per-block exponent, so the device input
x = -v 2^e / r is exact for every power-of-two r and the input rounding delta_in is 0. Each block holds the exact
Pi(v) - v, and `out` its entries rounded once to fp64 (Python's int / int division rounds correctly); the device
answer for (e, r) is out 2^e / r, an exact rescaling.

* SOC: Pythagorean vectors. For a in Z^k and an integer p, (2 p a, p^2 - ||a||^2) has norm p^2 + ||a||^2 exactly, so
  s = ||v_{1:}|| is an integer and every branch of the projection (s <= v_1, s <= -v_1, in between) is decided
  exactly; the in-between answer ((s + v_1) / 2, (s + v_1) / (2 s) v_{1:}) is rational.
* box: dyadic x, bounds in {0, +-2^j, +-inf} and power-of-two weights rho_j = 1 / r_j, so every breakpoint v_j / b_j
  of the optimality condition g(t) = rho_0 (t - v_0) + sum_j rho_j (t b_j - v_j) b_j [b_j the bound row j is clipped
  to] is an exact fp64 number. g is linear between breakpoints and increasing, so g(t) = 0 certifies t = t*; up to
  ROOT_ROWS rows t* is also found by bisection over the sorted breakpoints. `newton` restates the reference's Newton
  on t (src/cones.c proj_box_cone, its stop rules included) in exact arithmetic.
* l1: integer v and t; the threshold mu is eigen_exact.ell1_threshold (its integer path for long vectors), and
  `michelot` replays the device's active-set iteration exactly, pass by pass.

The gate (as eigen_exact.gate): every map is a projection, hence 1-Lipschitz, and so is the Moreau wrapper at a
constant r, so a device that rounds each operation once stays within
    ||dev - ref||_2 <= delta_in + C N 2^-53 ||x||_2,   N the cone's dimension, C = 64,
and the box adds the reference's own stop slack 1e-11 max(t*, 1) (1 + ||clipped bounds||_2), in output units (/ r).
The distance to the exact answer is bounded from above by ||dev - fl(ref)|| (1 + 1e-9) + 2^-52 ||fl(ref)||."""
import functools
import math
import zlib
from fractions import Fraction

import numpy as np

import eigen_exact as ee

C_GATE = ee.C_GATE
U = ee.U
SOC_BIG, SOC_CHUNK, SOC_BATCH_ROWS, SOC_ITEM_CONES = 8192, 4096, 4096, 4096  # kernels/cones.cu
ELL1_INLINE, ELL1_CHUNK = 8192, 4096                                          # kernels/cones_spectral.cu
BOX_BLOCK_ROWS = 2048   # grid_for(bsize - 1, B200_RED_THREADS * 4): rows per block of the Newton grid
BOX_MAX_ITERS = 25
NEWTON_STEPS_ALLOWED = 20
ROOT_ROWS = 20000
INT53 = 2 ** 53


def _rng(*key):
    return np.random.default_rng([20261018, *[zlib.crc32(v.encode()) if isinstance(v, str) else v for v in key]])


def to_float(num, den):
    """correctly rounded fp64 of num / den (integers, or object / int64 arrays of them)"""
    if isinstance(num, np.ndarray):
        return np.array([int(a) / int(den) for a in num.tolist()], dtype=np.float64) if num.size else np.zeros(0)
    return int(num) / int(den)


def err_bound(dev, ref):
    """an upper bound of ||dev - exact|| from ref = fl(exact) (each entry within 2^-53 of its exact value)"""
    return float(np.linalg.norm(dev - ref)) * (1 + 1e-9) + 2.0 ** -52 * float(np.linalg.norm(ref))


# ---------------------------------------------------------------------------------------------- blocks
class Block:
    """one cone: v (integer numpy array, the rows the projection sees, unscaled), e (v is scaled by 2^e), out (fp64 of
    Pi(v) - v, unscaled) and N (the cone's dimension). The device is given x = -v 2^e / r and must return
    x + Pi_K(-r x) / r = (Pi(v) - v) 2^e / r."""

    def __init__(self, kind, v, out, e=0, **parts):
        self.kind, self.v, self.out, self.e = kind, np.asarray(v, dtype=np.int64), np.asarray(out, np.float64), e
        self.N = self.v.size
        self.parts = parts
        assert self.v.size == 0 or int(np.abs(self.v).max()) < INT53

    def scaled(self, e):
        return Block(self.kind, self.v, self.out, e, **self.parts)

    def x(self, r=1.0):
        return np.ldexp(-self.v.astype(np.float64), self.e) / r

    def ref(self, r=1.0):
        return np.ldexp(self.out, self.e) / r

    def slack(self, r=1.0):
        return 0.0

    def ratio(self, dev, r=1.0):
        x = self.x(r)
        gate = C_GATE * max(self.N, 1) * U * float(np.linalg.norm(x)) + self.slack(r)
        err = err_bound(dev, self.ref(r))
        if gate == 0:
            return 0.0 if err == 0 else math.inf
        return err / gate


# ---------------------------------------------------------------------------------------------- second-order cone
SOC_KINDS = ["inside", "polar", "above", "below_polar", "edge_in", "edge_polar", "mid", "zero_tail_pos",
             "zero_tail_neg", "zero"]


def soc_tail(q, rng):
    """(tail, s): an integer tail of length q - 1 with integer norm s"""
    if q <= 1:
        return np.zeros(0, np.int64), 0
    if q == 2:
        w = int(rng.integers(1, 50)) * int(rng.choice([-1, 1]))
        return np.array([w], np.int64), abs(w)
    a = rng.integers(-3, 4, q - 2).astype(np.int64)
    if not a.any():
        a[0] = 1
    na = int(a @ a)
    p = int(rng.integers(1, 2 * math.isqrt(na) + 3))
    tail = np.concatenate((2 * p * a, [p * p - na])).astype(np.int64)
    s = p * p + na
    assert int(tail @ tail) == s * s
    return tail, s


def soc_head(kind, s, rng):
    return {"inside": s, "polar": -s, "above": s + 1, "below_polar": -s - 1, "edge_in": s - 1, "edge_polar": 1 - s,
            "mid": int(rng.integers(-s + 1, s)) if s > 1 else 0, "zero_tail_pos": 3, "zero_tail_neg": -3,
            "zero": 0}[kind]


def soc_out(v1, tail, s):
    """fp64 of Pi(v) - v for v = (v1, tail), ||tail|| = s"""
    q = 1 + tail.size
    if s <= v1:
        return np.zeros(q)
    if s <= -v1:
        return -np.concatenate(([v1], tail)).astype(np.float64)
    # Pi = ((s + v1) / 2, (s + v1) / (2 s) tail): Pi - v = ((s - v1) / 2, (v1 - s) / (2 s) tail)
    return np.concatenate(([to_float(s - v1, 2)], to_float(tail.astype(object) * (v1 - s), 2 * s)))


def soc_block(q, kind, rng, e=0):
    if q == 0:
        return Block("soc", [], [], e, s=0, q=0)
    tail, s = soc_tail(q, rng) if not kind.startswith("zero") else (np.zeros(q - 1, np.int64), 0)
    v1 = soc_head(kind, s, rng)
    if q == 1:  # the ray: Pi = max(v1, 0)
        return Block("soc", [v1], [float(max(-v1, 0))], e, s=0, q=1)
    return Block("soc", np.concatenate(([v1], tail)), soc_out(v1, tail, s), e, s=s, q=q)


SOC_SIZES = [0, 1, 2, 3, 31, 32, 33, 4095, 4096, 4097, 8191, 8192, 8193, 12288, 12289, 131072, 131073, 131074, 200001]


@functools.lru_cache(maxsize=None)
def soc_size_blocks(q):
    """cones of dimension q, one per decision branch; the big ones (q > SOC_BIG) at the three branches that move
    every row, and the in-between ones scaled by 2^+-200 next to unscaled ones"""
    rng = _rng("soc", q)
    kinds = SOC_KINDS if q <= SOC_BIG else ["mid", "edge_in", "edge_polar", "inside", "polar"]
    out = []
    for i, kind in enumerate(kinds):
        b = soc_block(q, kind, rng)
        out.append((kind, b))
        if kind == "mid" and q > 1:
            out.append(("mid_2^200", soc_block(q, kind, rng, 200)))
            out.append(("mid_2^-200", soc_block(q, kind, rng, -200)))
    return out


def soc_cone(blocks):
    return [b.N for _, b in blocks]


# ---------------------------------------------------------------------------------------------- l1-norm cone
def michelot(T, a):
    """the device's active-set iteration (kernels/cones_spectral.cu ell1_threshold) in exact arithmetic on the
    integer magnitudes a >= 0 and integer t = T: the list of thresholds of every pass; [] when mu = 0 at once, None
    for the polar exit"""
    a = np.asarray(a, dtype=np.int64)
    if a.size == 0 or -T >= int(a.max()):
        return None
    cnt, S = a.size, int(a.sum())
    mu = Fraction(S - T, cnt + 1)
    if not mu > 0:
        return []
    mus = [mu]
    while True:
        act = a * mu.denominator > mu.numerator
        c, s = int(act.sum()), int(a[act].sum())
        if c >= cnt:
            return mus
        cnt = c
        mu = Fraction(s - T, c + 1)
        mus.append(mu)


def ell1_out(T, v, mu):
    """fp64 of Pi(v) - v for (T, v) with threshold mu (None: polar, Pi = 0)"""
    if mu is None:
        return -np.concatenate(([T], v)).astype(np.float64)
    if mu == 0:
        return np.zeros(1 + v.size)
    fmu = to_float(mu.numerator, mu.denominator)
    # Pi - v = (mu, -sign(v) min(|v|, mu)); min(|v_i|, fl(mu)) = fl(min(|v_i|, mu)) as v_i is an fp64 number
    return np.concatenate(([fmu], -np.sign(v) * np.minimum(np.abs(v).astype(np.float64), fmu)))


def ell1_block(T, v, e=0):
    v = np.asarray(v, dtype=np.int64)
    mu = ee.ell1_threshold(Fraction(T), np.abs(v))
    return Block("ell1", np.concatenate(([T], v)), ell1_out(T, v, mu), e, T=T, mu=mu, mus=michelot(T, np.abs(v)))


def ell1_magnitudes(n, rng):
    """magnitudes spread over several scales, so that Michelot's iteration takes several passes"""
    scale = 2 ** rng.integers(0, 12, n)
    return (rng.integers(1, 8, n) * scale).astype(np.int64)


ELL1_SIZES = [1, 255, 256, 257, 8191, 8192, 8193, 12289, 131073]


@functools.lru_cache(maxsize=None)
def ell1_size_blocks(n):
    """polar exit (-t = max|v| exactly and beyond), in the cone (and on its boundary), v = 0, and thresholds at many
    passes, with ties |v_i| = mu"""
    rng = _rng("ell1", n)
    sg = rng.choice([-1, 1], n).astype(np.int64)
    a = ell1_magnitudes(n, rng)
    v = sg * a
    out = [("polar_edge", ell1_block(-int(a.max()), v)), ("polar", ell1_block(-int(a.max()) - 1, v)),
           ("inside", ell1_block(int(a.sum()) + 5, v)), ("boundary", ell1_block(int(a.sum()), v)),
           ("zero", ell1_block(3, np.zeros(n, np.int64))), ("zero_neg_t", ell1_block(-3, np.zeros(n, np.int64)))]
    for name, T in (("between", int(a.sum()) // 3), ("deep", -int(a.max()) + 1), ("t0", 0)):
        out.append((name, ell1_block(T, v)))
    out.append(("between_2^200", ell1_block(int(a.sum()) // 5, v, 200)))
    out.append(("between_2^-200", ell1_block(int(a.sum()) // 5, v, -200)))
    if n >= 3:
        out.append(("tie", ell1_tie_block(n, rng)))
    return out


def ell1_tie_block(n, rng):
    """|v_i| = mu exactly for some i: k entries of 4 M + a_i, ties at 2 M, the rest below; t chosen so mu = 2 M"""
    k = max(1, n // 3)
    ties = max(1, n // 4)
    M = 1 << 20
    big = (4 * M + rng.integers(0, 1000, k)).astype(np.int64)
    small = rng.integers(0, M, n - k - ties).astype(np.int64)
    mag = np.concatenate((big, np.full(ties, 2 * M, np.int64), small))
    mu = 2 * M
    T = int((big - mu).sum()) - mu   # sum_i max(|v_i| - mu, 0) = t + mu
    perm = rng.permutation(n)
    v = (mag * rng.choice([-1, 1], n))[perm]
    b = ell1_block(T, v)
    assert b.parts["mu"] == mu
    return b


# ---------------------------------------------------------------------------------------------- box cone
INF = math.inf


class BoxBlock(Block):
    """(t, s) rows; bl, bu the bounds the projection sees (Fractions of the form 0, +-2^j, or +-inf), rho the metric
    weights (powers of two; rho_j = 1 / r_j), t0 the warm start of the call. `raw` / D: the bounds and the row
    scaling given to the library (bounds at +-1e15 become +-inf under a D)."""

    def slack(self, r=1.0):
        t = self.parts["t"]
        tf = float(t)
        clipped = self.parts["clipped"]
        rmin = float(np.min(r)) if np.ndim(r) else float(r)
        return 1e-11 * max(tf, 1.0) * (1.0 + clipped) * 2.0 ** self.e / rmin

    def x(self, r=1.0):
        return np.ldexp(-self.v.astype(np.float64), self.e) / r

    def ref(self, r=1.0):
        return np.ldexp(self.out, self.e) / r


def _fr(a):
    return Fraction(a) if a not in (INF, -INF) else a


def _ints(vals):
    """Fractions (finite) -> (int64 or object numerators, common power-of-two denominator)"""
    den = 1
    for f in vals:
        den = max(den, f.denominator)
    assert den & (den - 1) == 0
    nums = [int(f * den) for f in vals]
    big = max((abs(a) for a in nums), default=0) >= 2 ** 62
    return np.array(nums, dtype=object if big else np.int64), den


class BoxProblem:
    """the exact piecewise-linear optimality condition of one box projection, vectorised over its rows"""

    def __init__(self, v0, v, bl, bu, rho0=Fraction(1), rho=None):
        n = len(v)
        self.n = n
        self.v0, self.rho0 = Fraction(v0), Fraction(rho0)
        self.v = np.asarray(v, dtype=np.int64)                 # integer x rows
        if isinstance(bl, np.ndarray):  # integer bounds, all finite (long cones)
            self.bl, self.bu = None, None
            self.lfin = self.ufin = np.ones(n, bool)
            self.bden, self.L, self.U = 1, bl.astype(np.int64), bu.astype(np.int64)
        else:
            self.bl, self.bu = list(bl), list(bu)
            self.lfin = np.array([b != -INF for b in bl], bool)
            self.ufin = np.array([b != INF for b in bu], bool)
            L, Ld = _ints([b if f else Fraction(0) for b, f in zip(bl, self.lfin)])
            Uu, Ud = _ints([b if f else Fraction(0) for b, f in zip(bu, self.ufin)])
            self.bden = max(Ld, Ud)
            self.L, self.U = L * (self.bden // Ld), Uu * (self.bden // Ud)   # bounds * bden, integers
        rho = [Fraction(1)] * n if rho is None else [Fraction(r) for r in rho]
        self.R, self.rden = _ints(rho + [self.rho0])
        self.R0, self.R = int(self.R[-1]), self.R[:-1]

    def active(self, t):
        """(hi, lo) masks at t: v_j > t u_j, v_j < t l_j (an infinite side never active, also at t = 0)"""
        P, Q = t.numerator, t.denominator
        lhs = self.v.astype(object) * (Q * self.bden) if abs(int(np.abs(self.v).max(initial=0))) * Q * self.bden >= 2 ** 62 \
            else self.v * (Q * self.bden)
        big = P * max(int(np.abs(self.U).max(initial=0)), int(np.abs(self.L).max(initial=0))) >= 2 ** 62
        Ut = self.U.astype(object) * P if big else self.U * P
        Lt = self.L.astype(object) * P if big else self.L * P
        return (lhs > Ut) & self.ufin, (lhs < Lt) & self.lfin

    def newton_point(self, hi, lo):
        """(Num, Den) with N_A / D_A: rho_0 v_0 + sum_A rho_j v_j b_j over rho_0 + sum_A rho_j b_j^2 (the Newton
        iterate of every t with this active set, and g(t) = t D_A - N_A)"""
        B = np.where(hi, self.U, np.where(lo, self.L, 0))
        act = hi | lo
        R, V, B = self.R[act], self.v[act], B[act]
        mx = [int(np.abs(a).max(initial=0)) for a in (R, V, B)]
        if max(mx[0] * mx[1] * mx[2], mx[0] * mx[2] * mx[2]) * max(int(act.sum()), 1) >= 2 ** 62:
            R, V, B = R.astype(object), V.astype(object), B.astype(object)
        num = Fraction(int((R * V * B).sum()) if act.any() else 0, self.rden * self.bden) + self.rho0 * self.v0
        den = Fraction(int((R * B * B).sum()) if act.any() else 0, self.rden * self.bden ** 2) + self.rho0
        return num, den

    def g(self, t):
        num, den = self.newton_point(*self.active(t))
        return t * den - num, den

    def root(self):
        """t* >= 0: bisection of the increasing g over the sorted breakpoints, then the linear piece's zero"""
        if self.g(Fraction(0))[0] >= 0:
            return Fraction(0)
        bps = set()
        for B, fin in ((self.U, self.ufin), (self.L, self.lfin)):
            nz = fin & (B != 0)
            for vj, bj in zip(self.v[nz].tolist(), B[nz].tolist()):
                f = Fraction(vj * self.bden, bj)
                if f > 0:
                    bps.add(f)
        pts = sorted(bps)
        lo, hi = 0, len(pts)   # g(0) < 0; find the first breakpoint with g >= 0
        while lo < hi:
            mid = (lo + hi) // 2
            if self.g(pts[mid])[0] >= 0:
                hi = mid
            else:
                lo = mid + 1
        left = pts[lo - 1] if lo > 0 else Fraction(0)
        right = pts[lo] if lo < len(pts) else None   # None: beyond the last breakpoint
        num, den = self.newton_point(*self.active((left + right) / 2 if right is not None else left + 1))
        t = num / den
        assert left <= t and (right is None or t <= right) and self.g(t)[0] == 0, (left, t, right)
        return t

    def newton(self, t0):
        """the reference's Newton (src/cones.c proj_box_cone) in exact arithmetic from t0: its iterates"""
        t, its = Fraction(t0), []
        for _ in range(BOX_MAX_ITERS):
            g, h = self.g(t)
            tn = max(t - g / max(h, Fraction(1e-8)), Fraction(0))
            its.append(tn)
            stop = abs(g / max(h, Fraction(1e-6))) < Fraction(1e-12) * max(tn, 1) or \
                abs(tn - t) < Fraction(1e-11) * max(tn, 1)
            t = tn
            if stop:
                break
        return its

    def out(self, t):
        """fp64 of Pi(v) - v at t (row 0 then the s rows)"""
        hi, lo = self.active(t)
        P, Q = t.numerator, t.denominator
        B = np.where(hi, self.U, np.where(lo, self.L, 0))
        # clipped row: t b_j - v_j = (P B_j - Q bden v_j) / (Q bden)
        numer = B.astype(object) * P - self.v.astype(object) * (Q * self.bden)
        res = np.zeros(self.n)
        act = hi | lo
        if act.any():
            res[act] = to_float(numer[act], Q * self.bden)
        head = t - self.v0
        return np.concatenate(([to_float(head.numerator, head.denominator)], res))

    def clipped_norm(self, t):
        hi, lo = self.active(t)
        B = np.where(hi, self.U, np.where(lo, self.L, 0)).astype(np.float64) / self.bden
        return float(np.linalg.norm(B))


def box_block(v0, v, bl, bu, t0=Fraction(1), rho0=Fraction(1), rho=None, raw=None, D=None, e=0):
    """one box cone; the exact Newton from the call's warm start t0 must reach t* within NEWTON_STEPS_ALLOWED steps"""
    bp = BoxProblem(v0, v, bl, bu, rho0, rho)
    its = bp.newton(t0)
    t = its[-1]
    # g is increasing with slope >= rho_0 > 0, so g(t) = 0 (or t = 0 with g(0) >= 0) certifies t = t*; below
    # ROOT_ROWS rows the sorted-breakpoint root is computed as well
    g0 = bp.g(t)[0]
    assert g0 == 0 or (t == 0 and g0 >= 0), (float(t), float(g0))
    if bp.n <= ROOT_ROWS:
        assert bp.root() == t
    reach = next((i + 1 for i, ti in enumerate(its) if ti == t), None)
    assert reach is not None and reach <= NEWTON_STEPS_ALLOWED, (float(t), [float(a) for a in its[-3:]], len(its))
    assert int(v0) == v0
    return BoxBlock("box", np.concatenate(([int(v0)], bp.v)), bp.out(t), e, t=t, its=its, bp=bp,
                    clipped=bp.clipped_norm(t), raw=raw, D=D, rho0=rho0, rho=rho, t0=Fraction(t0))


def box_long(n, name="long"):
    """a box cone of n rows with integer bounds l in {0, -1, -2, -4}, u in {0, 1, 2, 4} (some l = u = 0)"""
    rng = _rng("box", name, n)
    bl = -(2 ** rng.integers(0, 3, n)) * (rng.random(n) < 0.8)
    bu = (2 ** rng.integers(0, 3, n)) * (rng.random(n) < 0.8)
    bu[bl == 0] = np.maximum(bu[bl == 0], 0)
    v = rng.integers(-2 ** 12, 2 ** 12, n).astype(np.int64)
    return box_block(int(rng.integers(1, 64)), v, bl.astype(np.int64), bu.astype(np.int64))


def box_warm_sequence(n=3000):
    """three calls on one workspace, t* = T, 2^40 T, T: each call starts Newton from the previous call's t*"""
    rng = _rng("box", "warm", n)
    bl, bu = box_bounds(n, rng)
    v = rng.integers(-2 ** 12, 2 ** 12, n).astype(np.int64)
    v0 = int(rng.integers(1, 64))
    out, t0 = [], Fraction(1)
    for sc in (1, 2 ** 40, 1):
        b = box_block(v0 * sc, v * sc, bl, bu, t0)
        out.append(b)
        t0 = b.parts["t"]
    return out


def pow2(rng, lo, hi, n):
    return [Fraction(2) ** int(k) for k in rng.integers(lo, hi + 1, n)]


def box_bounds(n, rng, inf_frac=0.0, equal_frac=0.1):
    """bounds in {0, +-2^j} with l <= u, some l = u, and a share of infinite sides"""
    bl, bu = [], []
    for _ in range(n):
        kind = rng.random()
        a, b = pow2(rng, -1, 3, 2)
        if kind < equal_frac:
            c = a * int(rng.choice([-1, 1])) if rng.random() < 0.8 else Fraction(0)
            lo, hi = c, c
        elif kind < 0.5:
            lo, hi = -a, b
        elif kind < 0.75:
            lo, hi = Fraction(0), b
        else:
            lo, hi = a, max(a, b)
        if rng.random() < inf_frac:
            lo = -INF
        if rng.random() < inf_frac:
            hi = INF
        bl.append(lo)
        bu.append(hi)
    return bl, bu


@functools.lru_cache(maxsize=None)
def box_case(name, n, weighted=False):
    """named box cones of n = bsize - 1 rows (all with the default warm start t0 = 1, one call)"""
    rng = _rng("box", name, n, int(weighted))
    rho = pow2(rng, -3, 3, n) if weighted else None
    rho0 = pow2(rng, -2, 2, 1)[0] if weighted else Fraction(1)
    inf_frac = 0.2 if name in ("inf", "inf_D") else 0.0
    bl, bu = box_bounds(n, rng, inf_frac)
    v = rng.integers(-2 ** 12, 2 ** 12, n).astype(np.int64)
    v0 = {"plain": int(rng.integers(1, 64)), "inf": int(rng.integers(1, 64)), "inf_D": int(rng.integers(1, 64)),
          "zero": -2 ** 40, "far": 2 ** 30}[name]
    raw, D = None, None
    if name == "inf_D":
        # the library is given +-1e15 and a row scaling by powers of two; it turns those bounds into +-inf and
        # multiplies the others by D[j + 1] / D[0]
        D = np.array([2.0 ** int(k) for k in rng.integers(-2, 3, n + 1)])
        f = [Fraction(D[j + 1]) / Fraction(D[0]) for j in range(n)]
        raw = ([-1e15 if b == -INF else float(b / fj) for b, fj in zip(bl, f)],
               [1e15 if b == INF else float(b / fj) for b, fj in zip(bu, f)])
    return box_block(v0, v, bl, bu, Fraction(1), rho0, rho, raw=raw, D=D)


def box_library_bounds(b):
    """(bl, bu, D) as given to the library for a box block"""
    if b.parts["raw"] is not None:
        return b.parts["raw"][0], b.parts["raw"][1], b.parts["D"]
    bp = b.parts["bp"]
    return [float(a) if a != -INF else -INF for a in bp.bl], [float(a) if a != INF else INF for a in bp.bu], None


# ---------------------------------------------------------------------------------------------- Moreau checks
def moreau_soc(b):
    """exact: Pi in K, Pi - v in K (self-dual, -(polar)), <Pi, Pi - v> = 0; via the integer norm"""
    v = b.v
    if v.size <= 1:
        p = max(int(v[0]), 0) if v.size else 0
        return v.size == 0 or (p >= 0 and p - int(v[0]) >= 0 and p * (p - int(v[0])) == 0)
    s, v1 = b.parts["s"], int(v[0])
    if int(v[1:].astype(object) @ v[1:].astype(object)) != s * s:
        return False
    if s <= v1:
        a, sc = Fraction(v1), Fraction(1)
    elif s <= -v1:
        a, sc = Fraction(0), Fraction(0)
    else:
        a, sc = Fraction(s + v1, 2), Fraction(s + v1, 2 * s)
    # Pi = (a, sc tail): ||Pi tail|| = sc s; Pi - v = (a - v1, (sc - 1) tail): norm |sc - 1| s
    in_k = sc * s <= a
    res_in_k = abs(sc - 1) * s <= a - v1
    inner = a * (a - v1) + sc * (sc - 1) * s * s
    return in_k and res_in_k and inner == 0


def moreau_ell1(b):
    """exact: Pi in K (||x||_1 <= t), Pi - v in K* (||.||_inf <= t'), <Pi, Pi - v> = 0"""
    T, mu = b.parts["T"], b.parts["mu"]
    v = [Fraction(int(a)) for a in b.v[1:]]
    if mu is None:
        pi_t, pi = Fraction(0), [Fraction(0)] * len(v)
    else:
        pi_t = T + mu
        pi = [(1 if a > 0 else -1) * max(abs(a) - mu, 0) for a in v]
    d_t, d = pi_t - T, [p - a for p, a in zip(pi, v)]
    return (sum(abs(p) for p in pi) <= pi_t and max((abs(a) for a in d), default=0) <= d_t
            and pi_t * d_t + sum(p * a for p, a in zip(pi, d)) == 0)


def moreau_box(b):
    """exact, in the metric W = diag(rho): Pi in K, W (Pi - v) in K* = {(tau, y): tau + sum_j min(y_j l_j, y_j u_j)
    >= 0} (y_j of the sign that keeps an infinite bound's term finite), <Pi, W (Pi - v)> = 0"""
    bp, t = b.parts["bp"], b.parts["t"]
    rho = [Fraction(r) for r in (b.parts["rho"] or [1] * bp.n)]
    hi, lo = bp.active(t)
    pi = []
    for j in range(bp.n):
        vj = Fraction(int(bp.v[j]))
        pi.append(t * bp.bu[j] if hi[j] else (t * bp.bl[j] if lo[j] else vj))
    y = [r * (p - int(a)) for r, p, a in zip(rho, pi, bp.v)]
    tau = bp.rho0 * (t - bp.v0)
    ok = t >= 0
    for j in range(bp.n):
        l, u = bp.bl[j], bp.bu[j]
        lo_ok = l == -INF or t * l <= pi[j]
        hi_ok = u == INF or pi[j] <= t * u
        ok = ok and lo_ok and hi_ok
    supp = Fraction(0)
    for j in range(bp.n):
        l, u, yj = bp.bl[j], bp.bu[j], y[j]
        if yj > 0:
            if l == -INF:
                return False
            supp += yj * l
        elif yj < 0:
            if u == INF:
                return False
            supp += yj * u
    ok = ok and tau + supp >= 0
    return ok and t * tau + sum(p * yj for p, yj in zip(pi, y)) == 0

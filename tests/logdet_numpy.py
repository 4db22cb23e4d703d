"""A numpy restatement of the reference's log-cone projection (src/spectral_cones/logdeterminant/
log_cone_{wrapper,Newton,IPM}.c) and of the log-det cone projection built on it (logdet_cone.c).

It follows the reference step by step, with its constants, branches and in-place updates; sums are numpy's (pairwise)
rather than the reference's OpenBLAS order or the device's warp order, so its answers differ from both in the last
bits. tests/test_logdet_cpu.py measures that spread against the recorded reference, and the device is held to a
multiple of it. It is also the exact cone distance tests/verify.py needs for log-det problems.

The IPM's third column of G \\ C is taken as -e_r (its mathematical value). The reference reads the rest of that
column from workspace it never writes, which is zero for every workspace that has only served cones of one order.
"""
import numpy as np

NEWTON_SUCCESS, IPM0_SUCCESS, IPM1_SUCCESS = 1, 2, 3
IN_CONE, IN_NEGATIVE_DUAL_CONE, ANALYTICAL_SOL = -1, -2, -3
TERMINATE_DUE_TO_ZEROS, MAX_GRAD_STEPS_REACHED = -5, -6


class State:
    """one cone's persistent state: the warm-start flag and the previous projection (t, v, x)"""

    def __init__(self, n):
        self.warm = False
        self.proj = np.zeros(n + 2)


def _obj(v, x, t0, v0, x0):
    n = x.size
    sx = -(v * np.sum(np.log(x)) - n * v * np.log(v))
    return 0.5 * (sx - t0) ** 2 + 0.5 * (v - v0) ** 2 + np.sum(0.5 * (x - x0) ** 2)


def newton(t0, v0, x0, st, stats):
    """log_cone_Newton; returns 0 or -1, writes st.proj and stats['iter']; also every Newton decrement
    (stats['decrements'])"""
    n = x0.size
    u = st.proj
    nonneg, pos = bool(np.all(x0 >= 0)), bool(np.all(x0 > 0))
    if (v0 > 0 and pos and -v0 * (np.sum(np.log(x0)) - n * np.log(v0)) <= t0) or (v0 == 0 and nonneg and t0 >= 0):
        u[0], u[1], u[2:] = t0, v0, x0
        stats["iter"] = IN_CONE
        st.warm = True
        return 0
    if t0 < 0 and np.all(x0 < 0):
        s = (-n - np.sum(np.log(x0 / t0))) * t0
        if v0 <= s:
            u[:] = 0.0
            stats["iter"] = IN_NEGATIVE_DUAL_CONE
            st.warm = False
            return 0
    if v0 <= 0 and t0 >= 0:
        u[0], u[1], u[2:] = t0, 0.0, np.maximum(x0, 0.0)
        stats["iter"] = ANALYTICAL_SOL
        st.warm = True
        return 0
    if not st.warm:
        u[1] = v0 if v0 > 1 else 1.0
        u[2:] = np.where(x0 > 1, x0, 1.0)
    obj_old = _obj(u[1], u[2:], t0, v0, x0)
    grad_steps = 0
    it = 1
    while it <= 100:
        v = u[1]
        if v < 1e-14:
            stats["iter"] = TERMINATE_DUE_TO_ZEROS
            return -1
        u[2:] = np.maximum(u[2:], 1e-17)
        x = u[2:]
        temp0 = -np.sum(np.log(x)) + n * np.log(v)
        a = v * temp0 - t0
        c = temp0 + n
        v_inv = 1 / v
        xi = 1 / x
        grad = np.concatenate(([a * c + v - v0], -(a * v) * xi + x - x0))
        d = np.concatenate(([1 + a * (-a * (v_inv * v_inv) + n * v_inv - 2 * c * v_inv)], 1 + (a * v) * (xi * xi)))
        w = np.concatenate(([-(a + v * c) * v_inv], v * xi))
        du = -grad / d
        temp1 = w / d
        den = 1 + np.sum(w * temp1)
        if abs(den) < 1e-14:
            stats["iter"] = TERMINATE_DUE_TO_ZEROS
            return -1
        du = du + (-np.sum(w * du) / den) * temp1
        dirder = np.sum(grad * du)
        if dirder > 0:
            if grad_steps >= 5:
                stats["iter"] = MAX_GRAD_STEPS_REACHED
                return -1
            grad_steps += 1
            du = -grad
            dirder = -np.sum(grad * grad)
        stats.setdefault("decrements", []).append(-dirder)
        if -dirder <= 2e-12:
            break
        step = 1.0
        neg = du < 0
        if np.any(neg):
            step = min(step, float(np.min(-0.99 * u[1:][neg] / du[neg])))
        while True:
            un = u[1:] + step * du
            new_obj = _obj(un[0], un[1:], t0, v0, x0)
            if not ((1 - 1e-14) * new_obj > obj_old + 0.01 * step * dirder):
                break
            step *= 0.8
        obj_old = new_obj
        u[1:] = un
        it += 1
    u[0] = -u[1] * (np.sum(np.log(u[2:])) - n * np.log(u[1]))
    st.warm = True
    stats["iter"] = it
    return 0


def check_opt(tvx, t0, v0, x0):
    n = x0.size
    t, v, x = tvx[0], tvx[1], tvx[2:]
    dt = t - t0
    if abs(dt) < 1e-8:
        dt = 1e-8
    dv = v - v0
    dx = x - x0
    dx = np.where(np.abs(dx) < 1e-8, 1e-8, dx)
    comp = t * dt + v * dv + np.sum(dx * x)
    if v > 0 and np.all(x > 0):
        pri = -v * (np.sum(np.log(x)) - n * np.log(v)) - t
    else:
        pri = v * v + (t * t if t < 0 else 0.0) + np.sum(np.where(x < 0, x * x, 0.0))
    if dt > 0 and np.all(dx > 0):
        dual = dt * (n * np.log(dt) - n - np.sum(np.log(dx))) - dv
    else:
        dual = dt * dt + (dv * dv if dv < 0 else 0.0) + np.sum(np.where(dx < 0, dx * dx, 0.0))
    dn = np.sqrt(dt * dt + dv * dv + np.sum(dx * dx))
    pn = np.sqrt(np.sum(tvx * tvx))
    return np.array([dual / max(dn, 1.0), pri / max(pn, 1.0), comp / max(max(pn, 1.0), dn)])


def _oracle(u1, r, t0, v0, x0):
    n = x0.size
    v, x = u1[1], u1[2:]
    xi = 1 / x
    g0 = np.concatenate(([u1[0] - t0, v - v0], x - x0, [-1.0]))
    slxv = np.sum(np.log(x)) - n * np.log(v)
    nrm = np.sqrt(np.sum(g0[2:n + 2] ** 2))
    f = np.array([0.5 * (g0[0] ** 2 + g0[1] ** 2 + nrm * nrm) - r, -v * slxv - u1[0], -v])
    g1 = np.concatenate(([-1.0, n - slxv], xi * -v, [0.0]))
    return xi, f, g0, g1


def _residuals(g0, g1, z, f, s):
    n3 = g0.size
    rx = g0 * z[0] + z[1] * g1
    rx[1] -= z[2]
    rx[n3 - 1] += 1
    return rx, f + s


def ipm(t0, v0, x0, u1, variant):
    """log_cone_IPM; x0 (a float array) is scaled in place and unscaled at the end, as in the reference. Returns the
    iteration count."""
    n = x0.size
    ud = n + 3
    sc = max(float(np.max(np.abs(x0))) if n else 0.0, 0.0)
    sc = t0 if t0 > sc else sc
    sc = v0 if v0 > sc else sc
    sc = 1 / sc
    t0, v0 = t0 * sc, v0 * sc
    x0 *= sc
    u1[:] = 1.0
    r, dr = 0.0, 0.0
    z, s = np.ones(3), np.ones(3)
    dz, ds = np.zeros(3), np.zeros(3)
    relaxed = 0
    keep = None
    it = 0
    while it < 100:
        gap = float(np.sum(z * s))
        mu = gap / 3
        xi, f, g0, g1 = _oracle(u1, r, t0, v0, x0)
        rx, rznl = _residuals(g0, g1, z, f, s)
        dres = float(np.sqrt(np.sum(rx * rx)))
        pres = float(np.sqrt(np.sum(rznl * rznl)))
        norm_rx, norm_rznl = dres, pres
        if it == 0:
            pres0, dres0 = max(pres, 1.0), max(dres, 1.0)
            th1, th2, th3 = 1.0 / gap, 1.0 / dres0, 1.0 / pres0
        pres, dres = pres / pres0, dres / dres0
        relgap = gap / max(r, 1.0)
        if dres < 1e-7 and pres < 1e-7 and (gap < 1e-7 or relgap <= 1e-6):
            break
        w, lm = np.sqrt(s / z), np.sqrt(s * z)
        g0 = g0 * (1 / w[0])
        g1 = g1 * (1 / w[1])
        v = u1[1]
        # KKT_precompute
        a = z[0] + 1 / (w[2] * w[2]) + z[1] * n / v
        temp1 = z[0] + (z[1] * v) * (xi * xi)
        temp2 = xi / temp1
        coeff = a - z[1] * z[1] * np.sum((xi * xi) / temp1)

        def ginv(res):
            out = np.empty(ud)
            out[0] = res[0] / z[0]
            out[1] = (res[1] + z[1] * np.sum(res[2:n + 2] * temp2)) / coeff
            out[2:n + 2] = (res[2:n + 2] + (z[1] * out[1]) * xi) / temp1
            out[n + 2] = -res[n + 2]
            return out

        C0, C1 = ginv(g0), ginv(g1)
        C2 = np.zeros(ud)
        C2[n + 2] = -1.0
        R = np.zeros(9)
        R[0] = 1 + np.sum(g0 * C0)
        R[3] = np.sum(g0 * C1)
        R[6] = np.sum(g0 * C2)
        R[1] = np.sum(g1 * C0)
        R[4] = 1 + np.sum(g1 * C1)
        R[2] = C0[n + 2]

        def kkt_solve(rhs1, rhs2):
            rr = rhs1.copy()
            rr[ud:] -= w * (rhs2 / lm)
            bnew = rr[:ud].copy()
            bnew += (rr[n + 3] / w[0]) * g0
            bnew += (rr[n + 4] / w[1]) * g1
            bnew[1] -= rr[n + 5] / (w[2] * w[2])
            res = bnew.copy()
            du1 = np.zeros(n + 2)
            dr_ = 0.0
            for k in range(3):
                G = ginv(res)
                ctg = np.array([np.sum(g0 * G), np.sum(g1 * G), G[n + 2]])
                ri = np.zeros(3)
                ri[0] = ctg[2] / R[2]
                ri[1] = (ctg[1] - R[1] * ri[0]) / R[4]
                ri[2] = (ctg[0] - R[0] * ri[0] - R[3] * ri[1]) / R[6]
                G = G - (C0 * ri[0] + C1 * ri[1] + C2 * ri[2])
                du1 += G[:n + 2]
                dr_ += G[n + 2]
                if k != 2:
                    Gdu = np.empty(ud)
                    Gdu[0] = z[0] * du1[0]
                    Gdu[1] = (z[0] + 1 / (w[2] * w[2])) * du1[1] + z[1] * (n / v * du1[1] - np.sum(xi * du1[2:]))
                    Gdu[2:n + 2] = z[0] * du1[2:] + z[1] * (-du1[1] * xi + v * du1[2:] * xi * xi)
                    Gdu[n + 2] = -dr_
                    c0 = np.sum(g0[:n + 2] * du1) + g0[n + 2] * dr_
                    c1 = np.sum(g1[:n + 2] * du1) + g1[n + 2] * dr_
                    cct = g0 * c0 + c1 * g1
                    cct[n + 2] += dr_
                    res = bnew - (Gdu + cct)
            dz_ = rr[ud:].copy()
            dz_[0] -= w[0] * (np.sum(g0[:n + 2] * du1) + g0[n + 2] * dr_)
            dz_[1] -= w[1] * (np.sum(g1[:n + 2] * du1) + g1[n + 2] * dr_)
            dz_[2] += du1[1]
            dz_ = -dz_ / (w * w)
            ds_ = w * (rhs2 / lm - w * dz_)
            return du1, dr_, dz_, ds_

        rhs2 = -lm * lm
        rhs1 = -np.concatenate((rx, rznl))
        sigma = 0.0
        phi = th1 * gap + th2 * norm_rx + th3 * norm_rznl
        dphi = -th1 * (1 - sigma) * gap - th2 * norm_rx - th3 * norm_rznl
        for j in range(2):
            if j == 1 and variant == 0:
                rhs1 = rhs1 * (1 - sigma)
                rhs2 = rhs2 + (sigma * mu - ds * dz)
            du1, dr, dz, ds = kkt_solve(rhs1, rhs2)
            smax = 10.0
            for k in range(3):
                if dz[k] < 0:
                    smax = min(smax, -z[k] / dz[k])
                if ds[k] < 0:
                    smax = min(smax, -s[k] / ds[k])
            dom = 10.0
            neg = du1[1:] < 0
            if np.any(neg):
                dom = min(dom, float(np.min(-u1[1:][neg] / du1[1:][neg])))
            step = min(1.0, 0.99 * smax)
            while step > dom:
                step *= 0.5
            while True:
                u1n = u1 + step * du1
                rn = r + step * dr
                zn, sn = z + step * dz, s + step * ds
                _, fn, g0n, g1n = _oracle(u1n, rn, t0, v0, x0)
                rxn, rzn = _residuals(g0n, g1n, zn, fn, sn)
                gapn = float(np.sum(zn * sn))
                phin = th1 * gapn + th2 * np.sqrt(np.sum(rxn * rxn)) + th3 * np.sqrt(np.sum(rzn * rzn))
                if j == 0:
                    if phin <= (1 - 0.01 * step) * phi:
                        sigma = gapn / gap
                        if sigma < 1:
                            sigma *= sigma * sigma
                        break
                    step *= 0.5
                elif relaxed == -1:
                    if phin <= phi + 0.01 * step * dphi:
                        break
                    step *= 0.5
                elif relaxed == 0:
                    if not (phin <= phi + 0.01 * step * dphi):
                        relaxed = 1
                        keep = (u1.copy(), r, z.copy(), s.copy(), du1.copy(), dr, dz.copy(), ds.copy(), phi, dphi,
                                step)
                    break
                elif relaxed == 8:
                    if phin <= keep[8] + 0.01 * keep[10] * keep[9]:
                        break
                    relaxed = -1
                    u1[:], r, z, s, du1, dr, dz, ds, phi, dphi, step = (keep[0], keep[1], keep[2].copy(),
                                                                         keep[3].copy(), keep[4].copy(), keep[5],
                                                                         keep[6].copy(), keep[7].copy(), keep[8],
                                                                         keep[9], keep[10])
                else:
                    if phin <= keep[8] + 0.01 * keep[10] * keep[9]:
                        relaxed = 0
                    else:
                        relaxed += 1
                    break
        u1[:] = u1n
        r, z, s = rn, zn, sn
        it += 1
    sc = 1 / sc
    x0 *= sc
    u1 *= sc
    return it


def _accept(res):
    return res[0] < 1e-2 and res[1] < 1e-2 and abs(res[2]) < 1e-2


def wrapper(t0, v0, x0, st):
    """log_cone_proj_wrapper on (t0, v0, x0) with the cone state st. x0 may be modified in its last bits (the IPM's
    scaling round trip), as in the reference. Returns (status, stats) with stats = {iter, newton_success, res,
    decrements}."""
    stats = {"iter": 0, "newton_success": 0, "res": np.zeros(3)}
    status = newton(t0, v0, x0, st, stats)
    if st.proj[0] >= t0 - 0.1 * abs(t0):
        stats["res"] = check_opt(st.proj, t0, v0, x0)
    else:
        status = -1
    if status == 0 and _accept(stats["res"]):
        stats["newton_success"] = NEWTON_SUCCESS
        return 0, stats
    for variant in (0, 1):
        stats["iter"] = ipm(t0, v0, x0, st.proj, variant)
        stats["res"] = check_opt(st.proj, t0, v0, x0)
        if variant == 0:
            st.warm = True
        if _accept(stats["res"]):
            stats["newton_success"] = IPM0_SUCCESS + variant
            return 0, stats
    return -1, stats


def proj_logdet(tvX, n, st):
    """proj_logdet_cone (logdet_cone.c) on one cone's rows (t, v, packed X); returns (status, projection, stats)"""
    from spectral_numpy import packed_to_sym, sym_to_packed
    sqrt2 = np.sqrt(2.0)
    e, V = np.linalg.eigh(sqrt2 * packed_to_sym(tvX[2:], n))  # the reference's unpack: sqrt2 X
    status, stats = wrapper(sqrt2 * tvX[0], sqrt2 * tvX[1], e, st)
    lam = st.proj[2:]
    out = np.empty_like(tvX)
    out[0], out[1] = st.proj[0] / sqrt2, st.proj[1] / sqrt2
    out[2:] = sym_to_packed(((V * lam) @ V.T) / sqrt2)
    return status, out, stats


def proj_dual_cone(v, cone):
    """SCS's Moreau wrapper Pi_K*(v) = v + Pi_K(-v) (R = I) for cones whose spectral part is log-det cones only: the
    rows before them by scs_b200.problems.proj_dual_cone, each log-det block from a fresh (cold) state"""
    from scs_b200 import problems
    ds = [int(d) for d in cone.get("d", [])]
    base = {k: val for k, val in cone.items() if k != "d"}
    out = np.array(v, dtype=float)
    row = out.size - sum(d * (d + 1) // 2 + 2 for d in ds)
    if row:
        out[:row] = problems.proj_dual_cone(out[:row], base)
    for d in ds:
        k = d * (d + 1) // 2 + 2
        _, p, _ = proj_logdet(-out[row:row + k].copy(), d, State(d))
        out[row:row + k] = out[row:row + k] + p
        row += k
    return out

"""The operator-level device twins on the GPU (include/scs_b200.h group (3)): each computes the same bits as its host
twin, orders itself with the caller's stream, moves no vector across PCIe, refuses bad pointers before writing
anything, and works one workspace per thread. Also the PyTorch classes of scs_b200/torch_ops.py built on them."""
import ctypes as C
import functools
import threading

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from scs_b200 import capi, problems, torch_ops
import logdet_cases
import spectral_cases
from test_aa_gpu import contraction
from test_cones_gpu import CONES, TRIPLE_CONES, r_y_for

pytestmark = pytest.mark.gpu
_libc = C.CDLL(None)


def dp(t):
    return C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p) if t is not None else None


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def same_bits(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def printed(capfd):
    _libc.fflush(None)
    return capfd.readouterr().out


# ------------------------------------------------------------------ 1. cone projection, device door = host door
def _logdet_stats(lib, w):
    it, ok, res = C.c_int(), C.c_int(), (C.c_double * 3)()
    rc = lib.scs_b200_cone_logdet_stats(w, C.byref(it), C.byref(ok), res)
    return rc, it.value, ok.value, tuple(res)


def check_cone_sequence(cone, xs, metric, D=None, ry=None):
    """five successive projections on two workspaces, one per door: the same bits and log-det stats after each, and
    r_y left as it was"""
    spectral = capi.is_spectral(cone)
    lib = capi.load(spectral=spectral)
    m = capi.cone_rows(cone)
    k, _keep = capi.make_cone(cone, spectral=spectral)
    hw = lib.scs_b200_init_cone(C.byref(k), m, capi.dptr(D))
    dw = lib.scs_b200_init_cone(C.byref(k), m, capi.dptr(D))
    assert hw and dw
    if metric and ry is None:
        ry = r_y_for(cone, m)
    ry = ry if metric else None
    d_ry = cuda(ry) if metric else None
    try:
        for i, x in enumerate(xs):
            h = x.copy()
            d = cuda(x)
            rh = lib.scs_b200_proj_dual_cone(hw, capi.dptr(h), capi.dptr(ry))
            rd = lib.scs_b200_proj_dual_cone_device(dw, dp(d), dp(d_ry), stream())
            assert rh == rd and (rh == 0 or cone.get("d")), (cone, metric, i, rh, rd)
            assert same_bits(h, d), (cone, metric, i, np.nanmax(np.abs(h - d.cpu().numpy())))
            assert _logdet_stats(lib, hw) == _logdet_stats(lib, dw), (cone, i)
        if metric:
            assert same_bits(d_ry, ry)
    finally:
        lib.scs_b200_finish_cone(hw)
        lib.scs_b200_finish_cone(dw)


def random_inputs(m, seed, count=5):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal(m) * 10.0 ** rng.integers(-2, 3) for _ in range(count)]


BOX = {"z": 2, "l": 3, "bl": [-1.0, -0.5, 0.0, -2.0, -1e15] * 40, "bu": [1.0, 0.5, 3.0, 0.0, 1e15] * 40}
SOC_EDGE = {"q": [4, 4, 4, 4, 1, 1, 2]}
PLAIN = CONES + [SOC_EDGE, {"s": [100] * 200}] + TRIPLE_CONES + [{"z": 1, "l": 2, "cs": [1, 2, 3, 17]}]
LOGDET = [{"d": [1, 2, 3, 5, 16, 40]}, {"l": 4, "q": [5], "s": [4], "d": [3, 100]}, {"d": [100] * 12}]


@pytest.mark.parametrize("metric", [False, True])
@pytest.mark.parametrize("ci", range(len(PLAIN)))
def test_projection_doors_agree(ci, metric):
    cone = PLAIN[ci]
    m = capi.cone_rows(cone)
    xs = random_inputs(m, 100 + ci)
    if cone is SOC_EDGE:
        xs[0] = np.array([5, 1, 1, 1, -5, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, -2.0, 3.0, 0.5, -0.5])
    check_cone_sequence(cone, xs, metric)


@pytest.mark.parametrize("metric", [False, True])
def test_box_projection_doors_agree_with_D(metric):
    m = capi.cone_rows(BOX)
    D = np.random.default_rng(5).uniform(0.5, 2.0, m)
    check_cone_sequence(BOX, random_inputs(m, 6), metric, D=D)


@pytest.mark.parametrize("metric", [False, True])
@pytest.mark.parametrize("name", sorted(spectral_cases.CASES))
def test_spectral_projection_doors_agree(name, metric):
    cone, xs = spectral_cases.inputs(name)
    xs = (list(xs) + random_inputs(capi.cone_rows(cone), 7))[:5]
    check_cone_sequence(cone, xs, metric)


@functools.lru_cache(maxsize=None)
def _logdet_block(kind, n):
    return logdet_cases.operator_input(kind, n)


def logdet_inputs(cone, seed):
    """five inputs: the log-det rows from logdet_cases (a different branch per cone and call), the other rows random;
    the fourth is the third moved by 1e-3, so that the warm starts carry over between close inputs"""
    rng = np.random.default_rng(seed)
    head = capi.cone_rows({key: v for key, v in cone.items() if key != "d"})
    xs = []
    for call in range(5):
        parts = [rng.standard_normal(head)]
        for j, n in enumerate(cone["d"]):
            kinds = logdet_cases.KINDS
            parts.append(_logdet_block(kinds[(call + j) % len(kinds)], n))
        xs.append(np.concatenate(parts))
    xs[3] = xs[2] * (1 + 1e-3 * rng.standard_normal(xs[2].size))
    return xs


@pytest.mark.parametrize("metric", [False, True])
@pytest.mark.parametrize("ci", range(len(LOGDET)))
def test_logdet_projection_doors_agree(ci, metric):
    cone = LOGDET[ci]
    head = r_y_for({key: v for key, v in cone.items() if key != "d"}, capi.cone_rows(cone) - sum(
        logdet_cases.rows(n) for n in cone["d"]))
    ry = np.concatenate([head] + [logdet_cases.r_y(n) for n in cone["d"]])  # the metric logdet_cases chose inputs for
    check_cone_sequence(cone, logdet_inputs(cone, 200 + ci), metric, ry=ry)


# ------------------------------------------------------------------ 2. the primal projection of ConeProjector
@pytest.mark.parametrize("cone", [{"z": 7}, {"l": 50}, {"z": 3, "l": 4, "q": [1, 2, 3, 17, 300]},
                                  {"l": 2, "s": [1, 2, 3, 5, 12, 40]}])
def test_primal_projection_matches_numpy(cone):
    m = capi.cone_rows(cone)
    proj = torch_ops.ConeProjector(cone)
    for x in random_inputs(m, 11, 3):
        got = proj.project(cuda(x)).cpu().numpy()
        want = problems.proj_cone(x, cone)
        assert np.abs(got - want).max() <= 1e-13 * max(1.0, np.abs(x).max())
        y = proj.project_dual(cuda(x)).cpu().numpy()
        assert np.abs(y - problems.proj_dual_cone(x, cone)).max() <= 1e-13 * max(1.0, np.abs(x).max())
    proj.close()


# ------------------------------------------------------------------ 3. SpMV, 4. KKT solve
def random_csc(m, n, density, seed, empty_rows=(), empty_cols=(), dense_cols=()):
    A = sp.random(m, n, density=density, random_state=seed, format="csc")
    if dense_cols:  # columns of m entries: rows of A' far longer than one warp's tile
        rows, cols = np.tile(np.arange(m), len(dense_cols)), np.repeat(dense_cols, m)
        vals = np.random.default_rng(seed).uniform(-1, 1, rows.size)
        A = (A + sp.csc_matrix((vals, (rows, cols)), shape=(m, n))).tocsc()
    keep = np.ones(m)
    keep[list(empty_rows)] = 0
    A = sp.diags(keep) @ A
    colkeep = np.ones(n)
    colkeep[list(empty_cols)] = 0
    A = (A @ sp.diags(colkeep)).tocsc()
    A.eliminate_zeros()
    A.sort_indices()
    return A


def upper_P(n, seed):
    M = sp.random(n, n, density=4.0 / n, random_state=seed, format="csc")
    return sp.triu(M @ M.T + sp.eye(n), format="csc")


class Pair:
    """a host-made and a device-made plugin workspace of the same A, P and diag_r, in one library flavour"""

    def __init__(self, A, P, diag_r, long=False):
        self.lib = capi.load(long=long)
        self.T = capi.abi(long)
        self.m, self.n = A.shape
        idx = np.int64 if long else np.int32
        self.keep = []

        def host(M):
            x, i, p = (np.ascontiguousarray(M.data, np.float64), np.ascontiguousarray(M.indices, idx),
                       np.ascontiguousarray(M.indptr, idx))
            self.keep += [x, i, p]
            ip = capi.lptr if long else capi.iptr
            return self.T.ScsMatrix(capi.dptr(x), ip(i), ip(p), M.shape[0], M.shape[1])

        def dev(M):
            x, i, p = cuda(M.data), torch.from_numpy(M.indices.astype(idx)).cuda(), torch.from_numpy(
                M.indptr.astype(idx)).cuda()
            self.keep += [x, i, p]
            cast = lambda t: C.cast(C.c_void_p(t.data_ptr()), self.T.int_p)  # noqa: E731
            return self.T.ScsMatrix(dp(x), cast(i), cast(p), M.shape[0], M.shape[1])

        hA, hP = host(A), host(P) if P is not None else None
        self.h = self.lib.scs_init_lin_sys_work(C.byref(hA), C.byref(hP) if hP else None, capi.dptr(diag_r))
        self.dA, self.dP = dev(A), dev(P) if P is not None else None
        self.d = self.lib.scs_b200_init_lin_sys_work_device(C.byref(self.dA), C.byref(self.dP) if self.dP else None,
                                                            dp(cuda(diag_r)), stream())
        assert self.h and self.d

    def solve_host(self, w, b, s, tol):
        out = b.copy()
        assert self.lib.scs_solve_lin_sys(w, capi.dptr(out), capi.dptr(s), tol) == 0
        return out, self.lib.scs_b200_linsys_last_cg_its(w)

    def solve_dev(self, w, b, s, tol):
        out = cuda(b)
        d_s = cuda(s) if s is not None else None
        assert self.lib.scs_b200_solve_lin_sys_device(w, dp(out), dp(d_s), tol, stream()) == 0
        if s is not None:
            assert same_bits(d_s, s)
        return out.cpu().numpy(), self.lib.scs_b200_linsys_last_cg_its(w)

    def close(self):
        self.lib.scs_free_lin_sys_work(self.h)
        self.lib.scs_free_lin_sys_work(self.d)


SPMV_MATS = {
    "empty rows and columns": lambda: random_csc(3000, 1200, 0.004, 1, empty_rows=range(0, 3000, 7),
                                                 empty_cols=range(5, 1200, 11)),
    "long columns": lambda: random_csc(60000, 300, 0.0005, 2, dense_cols=(0, 17, 299)),
}


@pytest.mark.parametrize("name", sorted(SPMV_MATS))
def test_spmv_doors_agree(name):
    A = SPMV_MATS[name]()
    m, n = A.shape
    pair = Pair(A, None, np.ones(n + m))
    rng = np.random.default_rng(3)
    for w in (pair.h, pair.d):
        for accumulate in (0, 1):
            for f_host, f_dev, nin, nout in ((pair.lib.scs_b200_accum_by_a, pair.lib.scs_b200_accum_by_a_device, n, m),
                                             (pair.lib.scs_b200_accum_by_atrans,
                                              pair.lib.scs_b200_accum_by_atrans_device, m, n)):
                x, y0 = rng.standard_normal(nin), rng.standard_normal(nout)
                h = y0.copy()
                assert f_host(w, capi.dptr(x), capi.dptr(h), accumulate) == 0
                d_x, d_y = cuda(x), cuda(y0)
                assert f_dev(w, dp(d_x), dp(d_y), accumulate, stream()) == 0
                assert same_bits(h, d_y) and same_bits(d_x, x)
                want = (A @ x if nout == m else A.T @ x) + (y0 if accumulate else 0)
                assert np.abs(h - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    pair.close()


def kkt_problem(with_P, seed=4):
    A = random_csc(2000, 700, 0.01, seed, empty_rows=(5, 77))
    m, n = A.shape
    diag_r = np.concatenate((np.full(n, 1e-3), np.full(m, 0.5)))
    diag_r[n:n + 10] = 5e-4  # two values of R_y, as SCS sets them for zero-cone rows
    return A, (upper_P(n, seed) if with_P else None), diag_r


@pytest.mark.parametrize("with_P", [False, True])
@pytest.mark.parametrize("long", [False, True])
def test_kkt_solve_doors_agree(long, with_P):
    A, P, diag_r = kkt_problem(with_P)
    m, n = A.shape
    pair = Pair(A, P, diag_r, long=long)
    rng = np.random.default_rng(9)

    def compare(b, s, tol):
        ref = pair.solve_host(pair.h, b, s, tol)
        for got in (pair.solve_dev(pair.d, b, s, tol), pair.solve_dev(pair.h, b, s, tol),
                    pair.solve_host(pair.d, b, s, tol)):  # the two doors and the two mixed uses
            assert same_bits(got[0], ref[0]) and got[1] == ref[1], (long, with_P, tol, got[1], ref[1])
        return ref

    for step in range(2):
        b = rng.standard_normal(n + m)
        x, its = compare(b, None, 1e-12)
        assert its > 0
        s = x[:n] + 1e-3 * rng.standard_normal(n)
        compare(b + 1e-3 * rng.standard_normal(n + m), s, 1e-4)
        new_r = diag_r * rng.uniform(0.5, 2.0, n + m)
        assert pair.lib.scs_update_lin_sys_diag_r(pair.h, capi.dptr(new_r)) == 0
        assert pair.lib.scs_b200_update_lin_sys_diag_r_device(pair.d, dp(cuda(new_r)), stream()) == 0
    pair.close()


def test_row_index_out_of_range_is_refused_with_init_message(capfd):
    lib = capi.load()
    A, _, diag_r = kkt_problem(False)
    m, n = A.shape
    i = torch.from_numpy(A.indices.astype(np.int32)).cuda()
    i[17] = m
    x, p = cuda(A.data), torch.from_numpy(A.indptr.astype(np.int32)).cuda()
    cast = lambda t: C.cast(C.c_void_p(t.data_ptr()), capi.c_int_p)  # noqa: E731
    M = capi.ScsMatrix(dp(x), cast(i), cast(p), m, n)
    printed(capfd)
    assert not lib.scs_b200_init_lin_sys_work_device(C.byref(M), None, dp(cuda(diag_r)), stream())
    assert f"A row index {m} outside valid range [0, {m - 1}]" in printed(capfd)


# ------------------------------------------------------------------ 5. Anderson acceleration
@pytest.mark.parametrize("dim,mem,type1,relax,guard", [
    (5000, 10, 1, 1.0, 1.0), (5000, 10, 0, 1.0, 1.0), (3001, 7, 1, 1.5, 1.0), (4099, 14, 0, 1.5, 1.0),
    (2000, 5, 1, 1.0, 0.05),
])
def test_aa_doors_agree(dim, mem, type1, relax, guard):
    lib = capi.load()
    F = contraction(dim, dim + mem)
    reg = 1e-8 if type1 else 1e-12
    hw = lib.scs_b200_aa_init(dim, mem, mem, type1, reg, relax, guard, 1e10, 5, 0)
    dw = lib.scs_b200_aa_init(dim, mem, mem, type1, reg, relax, guard, 1e10, 5, 0)
    assert hw and dw
    x = np.zeros(dim)
    for i in range(max(40, mem + 30)):
        if i > 0:
            h, d = x.copy(), cuda(x)
            d_prev = cuda(x_prev)
            nh = lib.scs_b200_aa_apply(hw, capi.dptr(h), capi.dptr(x_prev))
            nd = lib.scs_b200_aa_apply_device(dw, dp(d), dp(d_prev), stream())
            assert same_bits(np.array([nh]), np.array([nd])) and same_bits(h, d) and same_bits(d_prev, x_prev), i
            x = h
        x_prev = x.copy()
        x = F(x)
        h, hp = x.copy(), x_prev.copy()
        d, d_p = cuda(x), cuda(x_prev)
        sh = lib.scs_b200_aa_safeguard(hw, capi.dptr(h), capi.dptr(hp))
        sd = lib.scs_b200_aa_safeguard_device(dw, dp(d), dp(d_p), stream())
        assert sh == sd and same_bits(h, d) and same_bits(hp, d_p), i
        x, x_prev = h, hp
    sh, sd = lib.scs_b200_aa_get_stats(hw), lib.scs_b200_aa_get_stats(dw)
    for f, _ in capi.AaStats._fields_:
        assert same_bits(np.array([getattr(sh, f)]), np.array([getattr(sd, f)])), f
    assert sh.n_accept > 5
    if guard < 1.0:
        assert sh.n_safeguard_reject > 0
    lib.scs_b200_aa_finish(hw)
    lib.scs_b200_aa_finish(dw)


def test_anderson_class_matches_the_host_door():
    lib = capi.load()
    dim, mem = 3000, 6
    F = contraction(dim, 12)
    hw = lib.scs_b200_aa_init(dim, mem, mem, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
    aa = torch_ops.Anderson(dim, mem=mem)
    x, xt = np.zeros(dim), torch.zeros(dim, dtype=torch.float64, device="cuda")
    for i in range(30):
        if i > 0:
            nh = lib.scs_b200_aa_apply(hw, capi.dptr(x), capi.dptr(x_prev))
            assert aa.apply(xt, xt_prev) == nh
        x_prev, xt_prev = x.copy(), xt.clone()
        x, xt = F(x), cuda(F(xt.cpu().numpy()))
        assert lib.scs_b200_aa_safeguard(hw, capi.dptr(x), capi.dptr(x_prev)) == aa.safeguard(xt, xt_prev)
        assert same_bits(x, xt)
    assert aa.stats()["n_accept"] == lib.scs_b200_aa_get_stats(hw).n_accept > 5
    aa.reset()
    assert aa.stats()["iter"] == 0
    lib.scs_b200_aa_finish(hw)
    aa.close()


# ------------------------------------------------------------------ 6. stream ordering
def test_work_is_ordered_with_a_side_stream():
    cone = {"z": 10, "l": 3000, "q": [40] * 50, "s": [30] * 10}
    m = capi.cone_rows(cone)
    A, _, diag_r = kkt_problem(False)
    mA, n = A.shape
    kkt = torch_ops.LinSys(torch.sparse_csc_tensor(torch.from_numpy(A.indptr), torch.from_numpy(A.indices),
                                                   torch.from_numpy(A.data), size=A.shape).cuda(), cuda(diag_r))
    proj = torch_ops.ConeProjector(cone)
    rng = np.random.default_rng(1)
    xc, xa, b = cuda(rng.standard_normal(m)), cuda(rng.standard_normal(n)), cuda(rng.standard_normal(n + mA))
    sync = (proj.project_dual(xc).cpu(), kkt.A_mul(xa).cpu(), kkt.solve(b, tol=1e-10).cpu())
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs = []
        for f, x in ((lambda v: proj.project_dual_(v), xc), (kkt.A_mul, xa), (lambda v: kkt.solve(v, tol=1e-10), b)):
            torch.cuda._sleep(100_000_000)  # the input is produced well after the call is made on the host
            v = x * 1.0
            outs.append(f(v).clone())  # consumed on the side stream, no host synchronisation in between
    side.synchronize()
    for got, want in zip(outs, sync):
        assert same_bits(got, want)
    kkt.close()
    proj.close()


# ------------------------------------------------------------------ 7. no vector crosses PCIe
def transfers(lib, f):
    stats = (C.c_longlong * 4)()
    torch.cuda.synchronize()
    lib.scs_b200_transfer_stats_reset()
    f()
    torch.cuda.synchronize()
    lib.scs_b200_transfer_stats(stats)
    return list(stats)


def test_no_vector_crosses_pcie():
    lib = capi.load()
    totals = []
    for m in (10_000, 1_000_000):
        cone = {"z": 100, "l": m // 2 - 100, "q": [50] * (m // 100)}
        k, _keep = capi.make_cone(cone)
        cw = lib.scs_b200_init_cone(C.byref(k), m, None)
        n = m // 10
        data, indices, indptr, shape = problems.random_sparse_csc(m, n, 80, np.random.default_rng(5))
        A = sp.csc_matrix((data, indices, indptr), shape=shape)
        pair = Pair(A, None, np.concatenate((np.full(n, 1e-3), np.full(m, 0.5))))
        aw = lib.scs_b200_aa_init(m, 5, 5, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
        rng = np.random.default_rng(0)
        x, ry, xn, ym, bb = (cuda(rng.standard_normal(size)) for size in (m, m, n, m, n + m))
        f_prev, x_prev = cuda(rng.standard_normal(m)), cuda(rng.standard_normal(m))
        diag = cuda(np.concatenate((np.full(n, 2e-3), np.full(m, 0.25))))

        def calls():
            assert lib.scs_b200_proj_dual_cone_device(cw, dp(x), dp(ry), stream()) == 0
            assert lib.scs_b200_accum_by_a_device(pair.d, dp(xn), dp(ym), 1, stream()) == 0
            assert lib.scs_b200_accum_by_atrans_device(pair.d, dp(ym), dp(xn), 0, stream()) == 0
            assert lib.scs_b200_update_lin_sys_diag_r_device(pair.d, dp(diag), stream()) == 0
            assert lib.scs_b200_solve_lin_sys_device(pair.d, dp(bb), dp(xn), 1e-4, stream()) == 0
            for i in range(8):  # from the 6th apply on, each runs the TSQR and the small solve
                f = f_prev * 0.9 + 0.01 * i
                nrm = lib.scs_b200_aa_apply_device(aw, dp(f), dp(x_prev), stream())
                assert nrm == nrm
                lib.scs_b200_aa_safeguard_device(aw, dp(f), dp(x_prev), stream())
        st = transfers(lib, calls)
        assert st[1] < 4096 and st[3] < 4096, (m, st)
        # scalars only (CG control blocks, AA's small factor): far below one vector even at m = 10^4 (80 kB)
        assert st[0] < 32768 and st[2] < 32768, (m, st)
        totals.append((st[0], st[2]))
        lib.scs_b200_finish_cone(cw)
        lib.scs_b200_aa_finish(aw)
        pair.close()
    print(f"\nbytes host to device, device to host at m = 1e4 and 1e6: {totals}")


# ------------------------------------------------------------------ 8. refusals
def test_refusals_write_nothing(capfd):
    lib = capi.load()
    cone = {"l": 100}
    k, _keep = capi.make_cone(cone)
    cw = lib.scs_b200_init_cone(C.byref(k), 100, None)
    A, _, diag_r = kkt_problem(False)
    m, n = A.shape
    pair = Pair(A, None, diag_r)
    aw = lib.scs_b200_aa_init(100, 5, 5, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
    big = cuda(np.arange(2 * (n + m), dtype=np.float64))
    host = np.arange(n + m, dtype=np.float64)
    snapshot = (big.clone(), host.copy())
    printed(capfd)
    S = stream()
    cases = [
        ("host x", lambda: lib.scs_b200_proj_dual_cone_device(cw, capi.dptr(host), None, S), -1, "device memory"),
        ("x / r_y overlap", lambda: lib.scs_b200_proj_dual_cone_device(cw, dp(big), dp(big[50:]), S), -1, "overlap"),
        ("NULL cone", lambda: lib.scs_b200_proj_dual_cone_device(None, dp(big), None, S), -1, "missing"),
        ("host y", lambda: lib.scs_b200_accum_by_a_device(pair.d, dp(big), capi.dptr(host), 0, S), -1, "device memory"),
        ("x / y overlap", lambda: lib.scs_b200_accum_by_atrans_device(pair.d, dp(big), dp(big[m - 1:]), 1, S), -1,
         "overlap"),
        ("NULL linsys", lambda: lib.scs_b200_accum_by_a_device(None, dp(big), dp(big[n:]), 0, S), -1, "missing"),
        ("host b", lambda: lib.scs_b200_solve_lin_sys_device(pair.d, capi.dptr(host), None, 1e-4, S), -1,
         "device memory"),
        ("b / s overlap", lambda: lib.scs_b200_solve_lin_sys_device(pair.d, dp(big), dp(big[n + m - 4:]), 1e-4, S), -1,
         "overlap"),
        ("NULL solve", lambda: lib.scs_b200_solve_lin_sys_device(None, dp(big), None, 1e-4, S), -1, "missing"),
        ("host diag_r", lambda: lib.scs_b200_update_lin_sys_diag_r_device(pair.d, capi.dptr(host), S), -1,
         "device memory"),
        ("host f", lambda: lib.scs_b200_aa_apply_device(aw, capi.dptr(host), dp(big), S), None, "device memory"),
        ("f / x overlap", lambda: lib.scs_b200_aa_apply_device(aw, dp(big), dp(big[99:]), S), None, "overlap"),
        ("NULL aa", lambda: lib.scs_b200_aa_apply_device(None, dp(big), dp(big[100:]), S), None, "missing"),
        ("f_new / x_new overlap", lambda: lib.scs_b200_aa_safeguard_device(aw, dp(big), dp(big[10:]), S), -1,
         "overlap"),
        ("host diag_r at init", lambda: lib.scs_b200_init_lin_sys_work_device(C.byref(pair.dA), None,
                                                                             capi.dptr(host), S), 0, "device memory"),
    ]
    for name, call, want, message in cases:
        rc = call()
        if want is None:
            assert rc != rc, name  # NaN
        elif want == 0:
            assert not rc, name
        else:
            assert rc == want, name
        assert message in printed(capfd), name
        torch.cuda.synchronize()
        assert same_bits(big, snapshot[0]) and same_bits(host, snapshot[1]), name
    assert lib.scs_b200_aa_get_stats(aw).iter == 0
    lib.scs_b200_finish_cone(cw)
    lib.scs_b200_aa_finish(aw)
    pair.close()


# ------------------------------------------------------------------ 9. one workspace per thread
def test_threads_with_their_own_workspaces_match_the_serial_run():
    cone = {"z": 5, "l": 2000, "q": [30] * 40, "s": [20] * 8}
    m = capi.cone_rows(cone)
    A, _, diag_r = kkt_problem(False)
    mA, n = A.shape
    A_t = torch.sparse_csc_tensor(torch.from_numpy(A.indptr), torch.from_numpy(A.indices), torch.from_numpy(A.data),
                                  size=A.shape).cuda()
    d_r = cuda(diag_r)
    inputs = [[(cuda(np.random.default_rng(100 * t + i).standard_normal(m)),
                cuda(np.random.default_rng(100 * t + i).standard_normal(n + mA))) for i in range(20)] for t in range(4)]
    torch.cuda.synchronize()

    def run(t, out):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            proj, kkt = torch_ops.ConeProjector(cone), torch_ops.LinSys(A_t, d_r)
            res = []
            for x, b in inputs[t]:
                res.append((proj.project_dual(x), kkt.solve(b, tol=1e-8), kkt.At_mul(b[n:])))
            s.synchronize()
            out[t] = [tuple(r.cpu() for r in rr) for rr in res]
            kkt.close()
            proj.close()

    serial = {}
    for t in range(4):
        run(t, serial)
    threaded = {}
    threads = [threading.Thread(target=run, args=(t, threaded)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for t in range(4):
        for a, b in zip(serial[t], threaded[t]):
            assert all(same_bits(x, y) for x, y in zip(a, b)), t

"""GPU: the second-order, box and l1-norm cones against exactly known projections (tests/vector_exact.py) at their
warp, chunk and batch edges.

* SOC: q = 0 ... 200001 around one warp per cone (q <= 8192), 4096-row chunks and more than 32 chunks per cone (each
  lane of pass 2 adds several partials); 4096 and 4097 rays and 9000 cones of 0 or 1 rows (the 4096-cone item cap),
  small cones whose rows cross 4096 inside an item, big cones first, last, back to back and between small ones.
* box: bsize 1, 2, 3; 2047 ... 2049 rows (the Newton grid's second block) and more rows than 2048 x 8 x SMs (the
  capped grid, blocks loop); infinite bounds given directly and from +-1e15 under a D; t* = 0; t* far from the warm
  start; three calls on one workspace whose t* differ by 2^40 (Newton starts from the previous call's t) and a fresh
  workspace (t = 1 again); per-row power-of-two r_y.
* l1: n = 1 ... 131073 around the 256- and 1024-thread CTAs and the 8192-entry inline limit; 70 000 cones of n = 1;
  small and big cones in one vector; ties at mu, the polar edge -t = max|v|, v = 0.
* one vector with every family behind z and l rows; three scs() solves with known optima through the fused path.

Every projection runs without r_y and with r_y = 4 and 1/8, through the host door and the device door, which must
agree bit for bit. Each cone must lie within 64 N 2^-53 ||x||_2 of its exact projection (delta_in = 0: every input is
exact), the box within that plus the reference's stop slack; the largest ratio per family is printed."""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.sparse
import torch

import spectral_numpy
import vector_exact as ve
import verify
from scs_b200 import capi

pytestmark = pytest.mark.gpu
RS = [1.0, 4.0, 0.125]
WORST = {}


@pytest.fixture(scope="module")
def slib():
    lib = capi.load(spectral=True)
    assert lib.scs_b200_device_ok()
    return lib


def _dp(t):
    return C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p) if t is not None else None


def project(lib, cone, x, r_y=None, D=None, spectral=None, cw=None):
    """the host door and the device door on workspaces of their own (or both on cw, one after the other when
    cw = (host workspace, device workspace)); they must give the same bits. Returns the answer."""
    k, keep = capi.make_cone(cone, spectral=spectral)
    m = x.size
    own = cw is None
    if own:
        cw = tuple(lib.scs_b200_init_cone(C.byref(k), m, capi.dptr(D)) for _ in range(2))
        assert cw[0] and cw[1], "scs_b200_init_cone failed"
    try:
        h = x.copy()
        assert lib.scs_b200_proj_dual_cone(cw[0], capi.dptr(h), capi.dptr(r_y)) == 0
        d = torch.from_numpy(x.copy()).cuda()
        d_ry = torch.from_numpy(r_y.copy()).cuda() if r_y is not None else None
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.scs_b200_proj_dual_cone_device(cw[1], _dp(d), _dp(d_ry), st) == 0
        dev = d.cpu().numpy()
        assert np.array_equal(h.view(np.uint64), dev.view(np.uint64)), "device door differs from the host door"
    finally:
        if own:
            for w in cw:
                lib.scs_b200_finish_cone(w)
    return h


def check(lib, cone, blocks, r, family, head=(), spectral=None, D=None, r_y=None):
    """one call on all blocks (after `head`: z / l rows given as (x, expected)); r a constant r_y (1: none) unless
    r_y (per row) is given"""
    hx = np.concatenate([h[0] for h in head]) if head else np.zeros(0)
    pos0 = hx.size
    parts, rr = [hx], []
    pos = pos0
    for b in blocks:
        rb = r if r_y is None else r_y[pos:pos + b.N]
        parts.append(b.x(rb))
        rr.append(rb)
        pos += b.N
    x = np.concatenate(parts)
    ry = r_y if r_y is not None else (None if r == 1 else np.full(x.size, float(r)))
    dev = project(lib, cone, x, ry, D=D, spectral=spectral)
    if head:
        exp = np.concatenate([h[1] for h in head])
        assert np.array_equal(dev[:pos0], exp)
    pos, worst = pos0, 0.0
    for b, rb in zip(blocks, rr):
        ratio = b.ratio(dev[pos:pos + b.N], rb)
        worst = max(worst, ratio)
        assert ratio <= 1.0, (family, b.kind, b.N, r, ratio)
        pos += b.N
    assert pos == x.size
    WORST[family] = max(WORST.get(family, 0.0), worst)
    print(f"{family}: worst err / gate so far {WORST[family]:.3g}")
    return dev


# ---------------------------------------------------------------------------------------------- SOC
@pytest.mark.parametrize("r", RS)
@pytest.mark.parametrize("q", ve.SOC_SIZES)
def test_soc_sizes(lib, q, r):
    """q = 0: the empty cones behind one LP row (a workspace needs at least one row)"""
    blocks = [b for _, b in ve.soc_size_blocks(q)]
    head = [(np.array([-3.0 / r]), np.array([0.0]))] if q == 0 else ()
    check(lib, {"l": len(head), "q": [b.N for b in blocks]}, blocks, r, "soc", head=head)


def _rays(count, rng):
    return [ve.soc_block(1, ["above", "below_polar", "zero"][i % 3], rng) for i in range(count)]


@pytest.mark.parametrize("r", RS)
def test_soc_item_edges(lib, r):
    """4096 and 4097 rays (one item full, then one spilling into the next); 9000 cones of 0 or 1 rows, whose 4096-cone
    cap ends items before their rows do; small cones whose rows cross 4096 inside an item"""
    rng = np.random.default_rng(11)
    for count in (ve.SOC_ITEM_CONES, ve.SOC_ITEM_CONES + 1):
        blocks = _rays(count, rng)
        check(lib, {"q": [1] * count}, blocks, r, "soc")
    blocks = [ve.soc_block(int(q), "mid" if q > 1 else "below_polar", rng) for q in rng.integers(0, 2, 9000)]
    check(lib, {"q": [b.N for b in blocks]}, blocks, r, "soc")
    qs = [1000, 1500, 1700, 33, 4000, 97, 8192, 1, 4095, 2, 3]
    blocks = [ve.soc_block(q, ve.SOC_KINDS[i % len(ve.SOC_KINDS)], rng) for i, q in enumerate(qs)]
    check(lib, {"q": qs}, blocks, r, "soc")


@pytest.mark.parametrize("r", RS)
def test_soc_big_cone_placement(lib, r):
    """big cones first, last, back to back and between small ones, some scaled by 2^+-200"""
    rng = np.random.default_rng(12)
    layout = [(12289, "mid", 0), (3, "mid", 0), (8193, "edge_in", 200), (131073, "mid", -200), (5, "edge_polar", 0),
              (1, "below_polar", 0), (16385, "polar", 0), (33, "mid", 200), (8193, "mid", 0)]
    blocks = [ve.soc_block(q, kind, rng, e) for q, kind, e in layout]
    check(lib, {"q": [q for q, _, _ in layout]}, blocks, r, "soc")


# ---------------------------------------------------------------------------------------------- l1
@pytest.mark.parametrize("r", RS)
@pytest.mark.parametrize("n", ve.ELL1_SIZES)
def test_ell1_sizes(slib, n, r):
    blocks = [b for _, b in ve.ell1_size_blocks(n)]
    check(slib, {"ell1": [n] * len(blocks)}, blocks, r, "l1")


@pytest.mark.parametrize("r", RS)
def test_ell1_many_and_mixed(slib, r):
    rng = np.random.default_rng(13)
    T = rng.integers(-5, 6, 70000)
    v = rng.integers(-5, 6, 70000)
    blocks = [ve.ell1_block(int(t), [int(a)]) for t, a in zip(T, v)]
    check(slib, {"ell1": [1] * len(blocks)}, blocks, r, "l1")
    sizes = [8193, 3, 12289, 256, 1, 8192, 4097, 257]
    blocks = [dict(ve.ell1_size_blocks(n))["between"] if n in ve.ELL1_SIZES else
              ve.ell1_block(int(n), ve.ell1_magnitudes(n, rng) * rng.choice([-1, 1], n)) for n in sizes]
    check(slib, {"ell1": sizes}, blocks, r, "l1")


# ---------------------------------------------------------------------------------------------- box
def _box_cone(b):
    bl, bu, D = ve.box_library_bounds(b)
    return {"bl": bl, "bu": bu}, D


@pytest.mark.parametrize("name", ["plain", "inf", "inf_D", "zero", "far"])
@pytest.mark.parametrize("n", [0, 1, 2, 2047, 2048, 2049])
def test_box(lib, name, n):
    """constant r_y and per-row power-of-two r_y (the weighted metric of the Newton step)"""
    if n == 0:
        b = ve.box_block(int(np.random.default_rng(1).integers(-9, 9)), np.zeros(0, np.int64), [], [])
        cone, D = {"bsize": 1}, None
    else:
        b = ve.box_case(name, n)
        cone, D = _box_cone(b)
    for r in RS:
        check(lib, cone, [b], r, "box", D=D)
    if n:
        bw = ve.box_case(name, n, True)
        cone, D = _box_cone(bw)
        r_y = np.array([1.0 / float(bw.parts["rho0"])] + [1.0 / float(a) for a in bw.parts["rho"]])
        check(lib, cone, [bw], 1, "box", D=D, r_y=r_y)


def test_box_capped_grid(lib):
    """more rows than 2048 x 8 x SMs: the Newton grid is capped and its blocks loop"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = ve.BOX_BLOCK_ROWS * 8 * sms + 3 * ve.BOX_BLOCK_ROWS + 5
    b = ve.box_long(n)
    bp = b.parts["bp"]
    cone = {"bl": bp.L.astype(np.float64), "bu": bp.U.astype(np.float64)}
    for r in RS:
        check(lib, cone, [b], r, "box")


def test_box_warm_start_across_calls(lib):
    """three calls on one workspace pair, t* = T, 2^40 T, T; then a fresh workspace for the last input starts from
    t = 1 again (its exact Newton from 1 must also reach t*)"""
    seq = ve.box_warm_sequence()
    cone, _ = _box_cone(seq[0])
    k, keep = capi.make_cone(cone)
    m = seq[0].N
    cw = tuple(lib.scs_b200_init_cone(C.byref(k), m, None) for _ in range(2))
    try:
        for i, b in enumerate(seq):
            dev = project(lib, cone, b.x(), cw=cw)
            ratio = b.ratio(dev)
            assert ratio <= 1.0, (i, ratio)
            WORST["box"] = max(WORST.get("box", 0.0), ratio)
    finally:
        for w in cw:
            lib.scs_b200_finish_cone(w)
    last = seq[-1]
    bp = last.parts["bp"]
    fresh = ve.box_block(int(last.v[0]), bp.v, bp.bl, bp.bu, 1)
    assert fresh.parts["t"] == last.parts["t"]
    check(lib, cone, [fresh], 1, "box")


# ---------------------------------------------------------------------------------------------- everything at once
@pytest.mark.parametrize("r", RS)
def test_mixed_vector(slib, r):
    """z and l rows, then a box, SOCs and l1 cones in one call of the spectral library"""
    rng = np.random.default_rng(14)
    z, l = 7, 9
    zx = rng.integers(-50, 50, z).astype(np.float64)
    lv = rng.integers(-50, 50, l)
    box = ve.box_case("inf", 300)
    socs = [ve.soc_block(q, kind, rng) for q, kind in ((33, "mid"), (8193, "edge_in"), (1, "below_polar"),
                                                       (3, "polar"))]
    l1s = [dict(ve.ell1_size_blocks(n))[name] for n, name in ((257, "tie"), (8193, "between"), (1, "polar_edge"))]
    bl, bu, _ = ve.box_library_bounds(box)
    cone = {"z": z, "l": l, "bl": bl, "bu": bu, "q": [b.N for b in socs], "ell1": [b.N - 1 for b in l1s]}
    # zero cone rows: x + Pi_{0}(-r x) / r = x; LP rows: x + max(-r x, 0) / r, exact for power-of-two r
    head = [(zx / r, zx / r), (-lv / r, np.maximum(lv, 0) / r - lv / r)]
    check(slib, cone, [box] + socs + l1s, r, "mixed", head=head, spectral=True)


# ---------------------------------------------------------------------------------------------- solves
def _solve(library, A, b, c, cone, **over):
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone)
    st = capi.default_settings(library, verbose=0, **over)
    x, y, s = np.zeros(A.shape[1]), np.zeros(A.shape[0]), np.zeros(A.shape[0])
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    flag = library.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    prob = {"A": (A.data, A.indices, A.indptr, A.shape), "b": b, "c": c, "cone": cone}
    return flag, info, st, x, y, s, prob


def _norm_ball(n):
    """rows (t, x) = b - A x with t = 1: A = [0; -I], b = e_0"""
    A = scipy.sparse.vstack([scipy.sparse.csc_matrix((1, n)), -scipy.sparse.identity(n, format="csc")]).tocsc()
    b = np.zeros(n + 1)
    b[0] = 1.0
    return A, b


def test_scs_soc_solve(lib):
    """minimise -a'x s.t. ||x||_2 <= 1, a Pythagorean of length 131072 (one cone of 33 chunks): optimum -||a||"""
    tail, s = ve.soc_tail(131073, np.random.default_rng(21))
    a = tail.astype(np.float64)
    A, b = _norm_ball(a.size)
    cone = {"q": [a.size + 1]}
    t0 = time.time()
    flag, info, st, x, y, z, prob = _solve(lib, A, b, -a, cone)
    assert flag == 1, info.status
    fails = verify.verify_solution_correct(prob, st, info, x, y, z, flag)
    assert not fails, fails
    assert abs(info.pobj + s) <= 1e-4 * max(1.0, s), (info.pobj, -s)
    print(f"soc solve: {info.iter} iterations, pobj {info.pobj:.12g}, opt {-s}, {time.time() - t0:.1f} s")


def test_scs_ell1_solve(slib):
    """minimise -a'x s.t. ||x||_1 <= 1, n = 8193: optimum -||a||_inf"""
    rng = np.random.default_rng(22)
    n = 8193
    a = (rng.integers(-1000, 1000, n) / 8.0)
    a[4097] = 200.0
    A, b = _norm_ball(n)
    cone = {"ell1": [n]}
    flag, info, st, x, y, z, prob = _solve(slib, A, b, -a, cone)
    assert flag == 1, info.status
    fails = verify.verify_solution_correct(prob, st, info, x, y, z, flag,
                                           ref_proj_dual=lambda v: spectral_numpy.proj_dual_cone(v, cone))
    assert not fails, fails
    opt = -float(np.abs(a).max())
    assert abs(info.pobj - opt) <= 1e-4 * max(1.0, abs(opt)), (info.pobj, opt)
    print(f"l1 solve: {info.iter} iterations, pobj {info.pobj:.12g}, opt {opt}")


def test_scs_box_solve(lib):
    """minimise c'x s.t. l <= x <= u as a box cone with t fixed to 1, some bounds at +-1e15 (c signed so the problem
    stays bounded): optimum sum_j min(c_j l_j, c_j u_j) over the finite bounds"""
    rng = np.random.default_rng(23)
    n = 5000
    bl = -rng.integers(1, 8, n) / 4.0
    bu = rng.integers(1, 8, n) / 4.0
    c = rng.integers(-20, 21, n) / 8.0
    c[c == 0] = 0.5
    up_inf = rng.random(n) < 0.1
    lo_inf = (rng.random(n) < 0.1) & ~up_inf
    bu[up_inf] = 1e15
    c[up_inf] = np.abs(c[up_inf])         # pushed towards the finite lower bound
    bl[lo_inf] = -1e15
    c[lo_inf] = -np.abs(c[lo_inf])        # pushed towards the finite upper bound
    opt = float(np.where(c > 0, c * bl, c * bu).sum())
    A, b = _norm_ball(n)
    cone = {"bl": bl, "bu": bu}
    flag, info, st, x, y, z, prob = _solve(lib, A, b, c, cone)
    assert flag == 1, info.status
    fails = verify.verify_solution_correct(prob, st, info, x, y, z, flag)
    assert not fails, fails
    assert abs(info.pobj - opt) <= 1e-4 * max(1.0, abs(opt)), (info.pobj, opt)
    print(f"box solve: {info.iter} iterations, pobj {info.pobj:.12g}, opt {opt}")


def test_zz_report():
    print("largest err / gate per family:", {k: f"{v:.3g}" for k, v in sorted(WORST.items())})

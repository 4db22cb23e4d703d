"""scs_b200_update_matrix_device and SCS.update(A=, P=): new values of A and P on the pattern a workspace was built
with leave it acting exactly like a fresh init on the new data. Every comparison is by bits: x, y, s and the
iteration record of the next solve, cold or warm from the same given x, y, s."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from scs_b200 import capi, problems, torch_solver
from test_device_data_gpu import CASES, INFO_EQUAL, PROBLEMS, assert_same, c2_like, read_fixture, to_torch

pytestmark = pytest.mark.gpu
INFO = INFO_EQUAL + ("scale", "res_infeas", "res_unbdd_a", "res_unbdd_p", "comp_slack")
ST = dict(eps_abs=1e-6, eps_rel=1e-6)


def perturbed(A, P, seed=11):
    """A with every value times (1 + 0.1 N(0, 1)), one value exactly 0.0 and one sign flipped; P times 1.3. The
    pattern, explicit zeros included, is A's and P's."""
    rng = np.random.default_rng(seed)
    A2 = sp.csc_matrix((A.data * (1 + 0.1 * rng.standard_normal(A.nnz)), A.indices.copy(), A.indptr.copy()),
                       shape=A.shape)
    A2.data[A.nnz // 3] = 0.0
    A2.data[A.nnz // 2] *= -1.0
    P2 = None if P is None else sp.csc_matrix((P.data * 1.3, P.indices.copy(), P.indptr.copy()), shape=P.shape)
    return A2, P2


def record(r):
    return (r["x"].cpu().numpy(), r["y"].cpu().numpy(), r["s"].cpu().numpy(), {k: r["info"][k] for k in INFO})


def warm_from(first):
    """the given warm start: the first problem's solution as CUDA tensors"""
    return {k: torch.tensor(v, device=torch_solver._library_device()) for k, v in zip("xys", first[:3])}


def fresh(A2, P2, b, c, cone, warm=None, idx=torch.int32, **st):
    solver = torch_solver.SCS(to_torch(A2, P2, b, c, idx), cone, verbose=0, **st)
    try:
        return record(solver.solve(warm_start=False) if warm is None else solver.solve(warm_start=True, **warm))
    finally:
        solver.close()


def updated(A, P, A2, P2, b, c, cone, warm=None, idx=torch.int32, first=None, **st):
    """init(A, P) -> solve -> update(A2, P2) -> solve (cold, or warm from `warm`); (first solve, solve after)"""
    solver = torch_solver.SCS(to_torch(A, P, b, c, idx), cone, verbose=0, **st)
    try:
        r0 = record(solver.solve(warm_start=False))
        if first is not None:
            first.append(r0)
        d2 = to_torch(A2, P2, b, c, idx)
        solver.update(A=d2["A"], P=d2.get("P"))
        r = solver.solve(warm_start=False) if warm is None else solver.solve(warm_start=True, **warm)
        return r0, record(r)
    finally:
        solver.close()


def check_both_starts(A, P, b, c, cone, idx=torch.int32, **st):
    A2, P2 = perturbed(A, P)
    r0, cold = updated(A, P, A2, P2, b, c, cone, idx=idx, **st)
    assert_same([fresh(A2, P2, b, c, cone, idx=idx, **st)], [cold])
    warm = warm_from(r0)
    _, hot = updated(A, P, A2, P2, b, c, cone, warm=warm, idx=idx, **st)
    assert_same([fresh(A2, P2, b, c, cone, warm=warm, idx=idx, **st)], [hot])
    return r0


@pytest.mark.parametrize("max_iters", [1, 100000])
@pytest.mark.parametrize("name,normalize", CASES)
def test_update_equals_a_fresh_init(name, normalize, max_iters):
    A, P, b, c, cone = PROBLEMS[name]()
    check_both_starts(A, P, b, c, cone, normalize=normalize, max_iters=max_iters, **ST)


def test_scale_goes_back_to_the_setting():
    """a first solve that has moved the scale: the update restores stgs->scale and diag_r"""
    A, P, b, c, cone = c2_like(scale=0.02)
    r0 = check_both_starts(A, P, b, c, cone, scale=1e4, max_iters=2000, **ST)
    assert r0[3]["scale_updates"] > 0, r0[3]


@pytest.mark.parametrize("max_iters", [1, 100000])
def test_c2_shaped_socp_with_the_packed_cg_pair(max_iters):
    check_both_starts(*c2_like(scale=0.1), max_iters=max_iters)


def special_shapes(seed=4):
    """an empty row and an empty column, a row and a column of more than 124 entries (virtual rows in A and in A'),
    and a box cone whose bounds the equilibration rescales; primal-dual feasible by construction"""
    rng = np.random.default_rng(seed)
    bs = 31
    cone = {"z": 20, "l": 150, "bl": -rng.uniform(0.5, 1.5, bs - 1), "bu": rng.uniform(0.5, 1.5, bs - 1), "q": [199]}
    m, n = 20 + 150 + bs + 199, 150
    Ad = np.where(rng.random((m, n)) < 0.03, rng.uniform(-1, 1, (m, n)), 0.0)
    Ad[5, :] = rng.uniform(-1, 1, n)
    Ad[:, 7] = rng.uniform(-1, 1, m)
    Ad[300, :] = 0.0
    Ad[:, 100] = 0.0
    A = sp.csc_matrix(Ad)
    assert A.getnnz(axis=1)[5] > 124 and A.getnnz(axis=0)[7] > 124
    assert A.getnnz(axis=1)[300] == 0 and A.getnnz(axis=0)[100] == 0
    zz = rng.uniform(-1, 1, m)
    y = problems.proj_dual_cone(zz, cone)
    x = rng.uniform(-1, 1, n)
    return A, None, A @ x + (y - zz), -(A.T @ y), cone


@pytest.mark.parametrize("max_iters", [1, 100000])
def test_empty_and_long_rows_and_columns_with_a_box_cone(max_iters):
    check_both_starts(*special_shapes(), max_iters=max_iters)


def _device_matrix(M, T, keep):
    """a ScsMatrix of device pointers into `keep`'s torch copies of M (int32 or int64 as T)"""
    dev = torch_solver._library_device()
    it = torch.int64 if T is capi.Long else torch.int32
    p, i = torch.tensor(M.indptr, dtype=it, device=dev), torch.tensor(M.indices, dtype=it, device=dev)
    x = torch.tensor(M.data, dtype=torch.float64, device=dev)
    keep += [p, i, x]
    ptr = lambda t, ty: C.cast(C.c_void_p(t.data_ptr()), ty)
    return T.ScsMatrix(ptr(x, capi.c_double_p), ptr(i, T.int_p), ptr(p, T.int_p), M.shape[0], M.shape[1])


def host_door(A, P, b, c, cone, A2=None, P2=None, **st):
    """scs_init(A, P) -> scs_solve -> scs_b200_update_matrix_device(A2, P2) -> scs_solve, or with A2 = None a fresh
    scs_init(A, P) -> scs_solve: the last solve's record"""
    lib = capi.load()
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone,
                          None if P is None else (P.data, P.indices, P.indptr, P.shape))
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0, **st)))
    assert w
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    keep = []
    try:
        steps = [0] if A2 is None else [0, 1]
        for step in steps:
            if step:
                Am = _device_matrix(A2, capi.Int, keep)
                Pm = None if P2 is None else C.byref(_device_matrix(P2, capi.Int, keep))
                assert lib.scs_b200_update_matrix_device(w, C.byref(Am), Pm, None) == 0
            sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
            lib.scs_solve(w, C.byref(sol), C.byref(info), 0)
        return x.copy(), y.copy(), s.copy(), {k: getattr(info, k) for k in INFO}
    finally:
        lib.scs_finish(w)


@pytest.mark.parametrize("name,normalize", [("random_prob", 1), ("mpc_bug1", 1), ("mpc_bug1", 0)])
def test_host_door_workspaces(name, normalize):
    """scs_init -> update equals a fresh scs_init on A2: P = 0 equilibrated on the pair of A, P != 0 with the P-aware
    equilibration, and P != 0 without equilibration"""
    A, P, b, c, cone = read_fixture(name)
    A2, P2 = perturbed(A, P)
    st = dict(ST, normalize=normalize)
    assert_same([host_door(A2, P2, b, c, cone, **st)], [host_door(A, P, b, c, cone, A2, P2, **st)])


@pytest.mark.parametrize("name", ["random_prob", "mpc_bug1"])
def test_int64_indices_with_the_dlong_library(name):
    A, P, b, c, cone = read_fixture(name)
    check_both_starts(A, P, b, c, cone, idx=torch.int64, **ST)


def test_combined_update_equals_a_fresh_init():
    A, P, b, c, cone = read_fixture("mpc_bug2")
    A2, P2 = perturbed(A, P)
    rng = np.random.default_rng(2)
    b2, c2 = b * (1 + 0.05 * rng.standard_normal(b.size)), c * 1.2
    ref = fresh(A2, P2, b2, c2, cone, **ST)
    for single_call in (False, True):
        solver = torch_solver.SCS(to_torch(A, P, b, c), cone, verbose=0, **ST)
        solver.solve()
        d2 = to_torch(A2, P2, b2, c2)
        if single_call:
            solver.update(A=d2["A"], P=d2["P"], b=d2["b"], c=d2["c"])
        else:
            solver.update(A=d2["A"], P=d2["P"])
            solver.update(d2["b"], d2["c"])
        got = record(solver.solve(warm_start=False))
        solver.close()
        assert_same([ref], [got])


def _moved_row(A):
    """A with one row index moved to a row its column does not hold"""
    A = A.copy()
    A.indices = A.indices.copy()
    for j in range(A.shape[1]):
        rows = set(A.indices[A.indptr[j]:A.indptr[j + 1]])
        if A.indptr[j + 1] > A.indptr[j]:
            free = [r for r in range(A.shape[0]) if r not in rows]
            A.indices[A.indptr[j]] = free[0]
            return A
    raise AssertionError("no column to move")


def _moved_pointer(A):
    A = A.copy()
    A.indptr = A.indptr.copy()
    j = next(j for j in range(A.shape[1] - 1) if A.indptr[j + 1] > A.indptr[j])
    A.indptr[j + 1] -= 1
    return A


REFUSALS = {
    "moved row index": (lambda A, P: (_moved_row(A), P), "the pattern of A differs"),
    "changed p": (lambda A, P: (_moved_pointer(A), P), "the pattern of A differs"),
    "moved P entry": (lambda A, P: (A, _p_moved(P)), "the pattern of P differs"),
    "wrong shape": (lambda A, P: (sp.csc_matrix((A.data, A.indices, A.indptr), shape=(A.shape[0] + 1, A.shape[1])), P),
                    "the workspace was built for"),
    "P missing": (lambda A, P: (A, None), "the workspace was built with P, and no P is given"),
    "nan in A": (lambda A, P: (sp.csc_matrix((np.where(np.arange(A.nnz) == 3, np.nan, A.data), A.indices, A.indptr),
                                             shape=A.shape), P), "A contains a non-finite entry"),
    "P below the diagonal": (lambda A, P: (A, _p_lower(P)), "P is not upper triangular"),
}


def _p_moved(P):
    """P with the row of one strictly upper entry moved to another row above the diagonal that its column lacks"""
    P = P.copy()
    P.indices = P.indices.copy()
    for j in range(P.shape[1]):
        rows = set(P.indices[P.indptr[j]:P.indptr[j + 1]])
        free = [r for r in range(j + 1) if r not in rows]
        if P.indptr[j + 1] > P.indptr[j] and free:
            P.indices[P.indptr[j]] = free[0]
            return P
    raise AssertionError("no entry of P to move")


def _p_lower(P):
    """one entry of P moved below the diagonal, same nnz"""
    P = P.copy()
    P.indices = P.indices.copy()
    j = next(j for j in range(P.shape[1] - 1) if P.indptr[j + 1] > P.indptr[j])
    P.indices[P.indptr[j]] = P.shape[0] - 1
    return P


def _raw_update(solver, A, P, host=False):
    """scs_b200_update_matrix_device on the solver's workspace without the front end's checks"""
    keep = []
    T = solver._T
    if host:
        hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), np.zeros(A.shape[0]), np.zeros(A.shape[1]),
                              {"l": A.shape[0]}, None if P is None else (P.data, P.indices, P.indptr, P.shape))
        return solver._lib.scs_b200_update_matrix_device(solver._work, C.byref(hp.A),
                                                         None if P is None else C.byref(hp.P), None)
    Am = _device_matrix(A, T, keep)
    Pm = None if P is None else C.byref(_device_matrix(P, T, keep))
    rc = solver._lib.scs_b200_update_matrix_device(solver._work, C.byref(Am), Pm, None)
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("case", sorted(REFUSALS) + ["P without a workspace P", "host pointer"])
def test_refusals_leave_the_workspace_untouched(capfd, case):
    name = "random_prob" if case == "P without a workspace P" else "mpc_bug1"
    A, P, b, c, cone = read_fixture(name)
    ref = fresh(A, P, b, c, cone, **ST)
    solver = torch_solver.SCS(to_torch(A, P, b, c), cone, verbose=0, **ST)
    capfd.readouterr()
    if case == "P without a workspace P":
        rc, message = _raw_update(solver, A, sp.csc_matrix(sp.eye(A.shape[1]))), "the workspace was built without P"
    elif case == "host pointer":
        rc, message = _raw_update(solver, A, P, host=True), "must point to device memory"
    else:
        make, message = REFUSALS[case]
        rc = _raw_update(solver, *make(A, P))
    out = capfd.readouterr().out
    assert rc == -1 and message in out, out
    got = record(solver.solve(warm_start=False))
    solver.close()
    assert_same([ref], [got])


def test_front_end_value_errors_before_the_library():
    A, P, b, c, cone = read_fixture("mpc_bug1")
    solver = torch_solver.SCS(to_torch(A, P, b, c), cone, verbose=0)
    d = to_torch(A, P, b, c)
    d64 = to_torch(A, P, b, c, idx=torch.int64)
    lib, solver._lib = solver._lib, None  # any library call below would raise AttributeError
    try:
        bad = [({"P": d["P"]}, "pass A as well"), ({"A": d["A"]}, "pass P together with A"),
               ({"A": d["A"].to_dense(), "P": d["P"]}, "sparse_csc"),
               ({"A": d64["A"], "P": d64["P"]}, "torch.int32 indices"),
               ({"A": d["P"], "P": d["P"]}, "must have shape"),
               ({"A": d["A"].cpu(), "P": d["P"].cpu()}, "must be a CUDA tensor")]
        for kw, message in bad:
            with pytest.raises(ValueError, match=message):
                solver.update(**kw)
    finally:
        solver._lib = lib
        solver.close()
    A0, _, b0, c0, cone0 = read_fixture("random_prob")
    solver = torch_solver.SCS(to_torch(A0, None, b0, c0), cone0, verbose=0)
    d0 = to_torch(A0, sp.csc_matrix(sp.eye(A0.shape[1])), b0, c0)
    with pytest.raises(ValueError, match="built without P"):
        solver.update(A=d0["A"], P=d0["P"])
    solver.close()


def test_update_moves_no_problem_sized_transfer():
    lib = capi.load()
    A, P, b, c, cone = c2_like(scale=0.02)
    dense = sp.random(A.shape[0], A.shape[1], density=min(1.0, 25.0 * sum(A.shape) / (A.shape[0] * A.shape[1])),
                      random_state=1, format="csc")
    A = (A + dense).tocsc()
    assert A.nnz >= 20 * sum(A.shape)
    A2, _ = perturbed(A, None)
    solver = torch_solver.SCS(to_torch(A, None, b, c), cone, verbose=0, max_iters=50)
    solver.solve()
    d2 = to_torch(A2, None, b, c)
    torch.cuda.synchronize()
    stats = (C.c_longlong * 4)()
    lib.scs_b200_transfer_stats_reset()
    solver.update(A=d2["A"])
    torch.cuda.synchronize()
    lib.scs_b200_transfer_stats(stats)
    solver.close()
    bound = 16 * sum(A.shape) + 4096
    assert stats[0] <= bound and stats[2] <= bound, (list(stats), bound, A.nnz)


def test_side_stream_and_caller_memory():
    A, P, b, c, cone = read_fixture("mpc_bug3")
    A2, P2 = perturbed(A, P)
    ref = fresh(A2, P2, b, c, cone)
    solver = torch_solver.SCS(to_torch(A, P, b, c), cone, verbose=0)
    solver.solve()
    d2 = to_torch(A2, P2, b, c)
    before = {k: (v.values().clone(), v.row_indices().clone(), v.ccol_indices().clone()) for k, v in d2.items()
              if v.layout != torch.strided}
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        vals = d2["A"].values()
        torch.cuda._sleep(50_000_000)  # the update below must wait for this stream's work
        A2t = torch.sparse_csc_tensor(d2["A"].ccol_indices(), d2["A"].row_indices(), vals * 1.0, size=A.shape)
        solver.update(A=A2t, P=d2["P"])
        got = record(solver.solve(warm_start=False))
    solver.close()
    assert_same([ref], [got])
    for k, (v, i, p) in before.items():
        assert torch.equal(v, d2[k].values()) and torch.equal(i, d2[k].row_indices())
        assert torch.equal(p, d2[k].ccol_indices())

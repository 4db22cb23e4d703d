"""The device-data entry points (scs_b200_init_device / _update_device / _solve_device) and their PyTorch front end
against the host API on the same data: solutions equal by bits, the same iteration record, the same refusals, and no
problem-sized copy across PCIe."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from scs_b200 import capi, problems, torch_solver

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "problems")
INFO_EQUAL = ("iter", "status_val", "pobj", "dobj", "res_pri", "res_dual", "gap", "scale_updates",
              "accepted_accel_steps", "rejected_accel_steps")
PP = C.POINTER


def read_fixture(name):
    """(A csc, P csc or None, b, c, cone dict) of a reference fixture, read with scs_b200_read_data"""
    lib = capi.load()
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsCone)), PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsCone), PP(capi.ScsSettings)]
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsCone)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(os.path.join(GOLDEN, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    try:
        D, K = d.contents, k.contents
        arr = lambda p, n, t=np.int32: np.ctypeslib.as_array(p, (n,)).astype(t).copy() if n > 0 else np.zeros(0, t)

        def mat(M):
            M = M.contents
            nnz = M.p[M.n]
            return sp.csc_matrix((arr(M.x, nnz, np.float64), arr(M.i, nnz), arr(M.p, M.n + 1)), shape=(M.m, M.n))
        cone = {"z": K.z, "l": K.l, "ep": K.ep, "ed": K.ed, "q": list(arr(K.q, K.qsize)), "s": list(arr(K.s, K.ssize)),
                "p": list(arr(K.p, K.psize, np.float64))}
        if K.bsize > 1:
            cone["bu"], cone["bl"] = list(arr(K.bu, K.bsize - 1, np.float64)), list(arr(K.bl, K.bsize - 1, np.float64))
        else:
            cone["bsize"] = K.bsize
        return (mat(D.A), mat(D.P) if D.P else None, arr(D.b, D.m, np.float64), arr(D.c, D.n, np.float64), cone)
    finally:
        lib.scs_b200_free_data(d, k, s)


def c2_like(scale=0.1, seed=3):
    """an SOCP shaped like C2 (n : m : nnz = 1 : 3 : 10) at `scale` of 1e5 columns"""
    n = int(1e5 * scale)
    m = 3 * n
    q = [3] * ((m - n) // 3)
    cone = {"z": n // 2, "l": m - n // 2 - 3 * len(q), "q": q}
    prob = problems.make_problem(m, n, 10, cone, seed=seed)
    A = sp.csc_matrix((prob["A"][0], prob["A"][1], prob["A"][2]), shape=prob["A"][3])
    return A, None, prob["b"], prob["c"], prob["cone"]


def exp_pow():
    """the exponential and power cone problem of test_solver_gpu.py"""
    from test_solver_gpu import exp_pow_problem
    prob = exp_pow_problem(31)
    return sp.csc_matrix(prob["A"][:3], shape=prob["A"][3]), None, prob["b"], prob["c"], prob["cone"]


def complex_psd():
    """the complex PSD problem of test_solver_gpu.py, its optimum built with this library's own dual-cone projection"""
    lib = capi.load()
    cone = {"z": 3, "l": 10, "q": [4, 9], "s": [3, 5], "cs": [2, 5, 4, 1]}
    m, n = capi.cone_rows(cone), 40
    rng = np.random.default_rng(77)
    A = problems.random_sparse_csc(m, n, 9, rng)
    k, keep = capi.make_cone(cone)
    cw = lib.scs_b200_init_cone(C.byref(k), m, None)
    zz = rng.uniform(-1, 1, m)
    y = zz.copy()
    assert lib.scs_b200_proj_dual_cone(cw, capi.dptr(y), None) == 0
    lib.scs_b200_finish_cone(cw)
    x0 = rng.uniform(-1, 1, n)
    return (sp.csc_matrix(A[:3], shape=A[3]), None, problems.csc_matvec(A, x0) + (y - zz), -problems.csc_rmatvec(A, y),
            cone)


def spectral(name):
    """a reference spectral fixture (nuclear-norm and l1 cones), read with the spectral library"""
    from test_spectral_cones_gpu import as_dict
    lib = capi.load(spectral=True)
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                       PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(os.path.join(GOLDEN, "spectral", name).encode(), C.byref(d), C.byref(k),
                                  C.byref(s)) == 0
    try:
        prob = as_dict(d, k)
    finally:
        lib.scs_b200_free_data(d, k, s)
    assert capi.is_spectral(prob["cone"])
    return sp.csc_matrix(prob["A"][:3], shape=prob["A"][3]), None, prob["b"], prob["c"], prob["cone"]


PROBLEMS = {"random_prob": lambda: read_fixture("random_prob"), "mpc_bug1": lambda: read_fixture("mpc_bug1"),
            "mpc_bug2": lambda: read_fixture("mpc_bug2"), "mpc_bug3": lambda: read_fixture("mpc_bug3"),
            "exp_pow": exp_pow, "complex_psd": complex_psd, "spectral_ell1_nuc": lambda: spectral("test_ell1_and_nuc")}


def host_solve(A, P, b, c, cone, seq=(), long=False, **st):
    """scs_init + scs_solve (+ scs_update / scs_solve for each (b, c) of seq) on the library the device door picks for
    this problem (spectral cones: the spectral flavour; long: the DLONG one): a list of (x, y, s, info)"""
    lib = capi.load(spectral=capi.is_spectral(cone), long=long)
    T = capi.abi(long)
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone,
                          None if P is None else (P.data, P.indices, P.indptr, P.shape), long=long)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone),
                     C.byref(capi.default_settings(lib, long=long, verbose=0, **st)))
    assert w
    out = []
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    try:
        for step in [None] + list(seq):
            if step is not None:
                bb, cc = [None if v is None else np.ascontiguousarray(v, dtype=np.float64) for v in step]
                assert lib.scs_update(w, capi.dptr(bb), capi.dptr(cc)) == 0
            sol = T.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
            info = T.ScsInfo()
            lib.scs_solve(w, C.byref(sol), C.byref(info), 1 if step is not None else 0)
            out.append((x.copy(), y.copy(), s.copy(), {k: getattr(info, k) for k in INFO_EQUAL}))
    finally:
        lib.scs_finish(w)
    return out


def to_torch(A, P, b, c, idx=torch.int32):
    dev = torch.device("cuda", torch_solver._library_device())
    t = lambda M: torch.sparse_csc_tensor(torch.tensor(M.indptr, dtype=idx), torch.tensor(M.indices, dtype=idx),
                                          torch.tensor(M.data, dtype=torch.float64), size=M.shape, device=dev)
    d = {"A": t(A), "b": torch.tensor(b, device=dev), "c": torch.tensor(c, device=dev)}
    if P is not None:
        d["P"] = t(P)
    return d


def device_solve(A, P, b, c, cone, seq=(), idx=torch.int32, **st):
    solver = torch_solver.SCS(to_torch(A, P, b, c, idx), cone, verbose=0, **st)
    out = []
    try:
        for step in [None] + list(seq):
            if step is not None:
                solver.update(*[None if v is None else torch.tensor(v, device=solver.device) for v in step])
            r = solver.solve(warm_start=step is not None)
            out.append((r["x"].cpu().numpy(), r["y"].cpu().numpy(), r["s"].cpu().numpy(),
                        {k: r["info"][k] for k in INFO_EQUAL}))
    finally:
        solver.close()
    return out


def assert_same(h, d):
    assert len(h) == len(d)
    for (xh, yh, sh, ih), (xd, yd, sd, idv) in zip(h, d):
        for u, v in ((xh, xd), (yh, yd), (sh, sd)):
            assert u.tobytes() == v.tobytes(), np.abs(u - v).max()
        assert {k: np.float64(ih[k]).tobytes() for k in ih} == {k: np.float64(idv[k]).tobytes() for k in idv}, (ih, idv)


CASES = [("random_prob", 1), ("mpc_bug1", 1), ("mpc_bug1", 0), ("mpc_bug2", 1), ("mpc_bug2", 0), ("mpc_bug3", 1),
         ("mpc_bug3", 0), ("exp_pow", 1), ("complex_psd", 1), ("spectral_ell1_nuc", 1)]


@pytest.mark.parametrize("max_iters", [1, 100000])
@pytest.mark.parametrize("name,normalize", CASES)
def test_device_api_equals_host_api(name, normalize, max_iters):
    prob = PROBLEMS[name]()
    st = dict(normalize=normalize, max_iters=max_iters, eps_abs=1e-6, eps_rel=1e-6)
    h = host_solve(*prob, **st)
    if max_iters > 1:
        assert h[0][3]["status_val"] == 1, h[0][3]
    assert_same(h, device_solve(*prob, **st))


@pytest.mark.parametrize("max_iters", [1, 100000])
def test_c2_shaped_socp_equals_host_api(max_iters):
    prob = c2_like()
    assert_same(host_solve(*prob, max_iters=max_iters), device_solve(*prob, max_iters=max_iters))


@pytest.mark.parametrize("max_iters", [1, 100000])
@pytest.mark.parametrize("name", ["random_prob", "mpc_bug1"])
def test_int64_indices_equal_the_dlong_host_api(name, max_iters):
    prob = PROBLEMS[name]()
    st = dict(max_iters=max_iters, eps_abs=1e-6, eps_rel=1e-6)
    assert_same(host_solve(*prob, long=True, **st), device_solve(*prob, idx=torch.int64, **st))


@pytest.mark.parametrize("name", ["random_prob", "mpc_bug2"])
def test_update_and_warm_start_sequence_equals_host_api(name):
    A, P, b, c, cone = prob = read_fixture(name)
    rng = np.random.default_rng(5)
    seq = [(b * (1 + 0.1 * rng.standard_normal(b.size)), None), (None, c * 1.3), (b, c)]
    assert_same(host_solve(*prob, seq=seq), device_solve(*prob, seq=seq))


def test_front_end_leaves_update_and_warm_start_inputs_unchanged():
    """update(b) and solve(x=, y=, s=) read the caller's tensors only, and the warm start from them equals the host
    API's warm start from the same vectors"""
    lib = capi.load()
    A, P, b, c, cone = read_fixture("mpc_bug2")
    rng = np.random.default_rng(9)
    b2 = b * 1.05
    x0, y0, s0 = rng.uniform(-1, 1, A.shape[1]), rng.uniform(-1, 1, A.shape[0]), rng.uniform(0, 1, A.shape[0])
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone, (P.data, P.indices, P.indptr, P.shape))
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0)))
    assert w and lib.scs_update(w, capi.dptr(b2), None) == 0
    x, y, s = x0.copy(), y0.copy(), s0.copy()
    sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 1)
    lib.scs_finish(w)
    ref = [(x, y, s, {k: getattr(info, k) for k in INFO_EQUAL})]
    solver = torch_solver.SCS(to_torch(A, P, b, c), cone, verbose=0)
    dev = solver.device
    inputs = {k: torch.tensor(v, device=dev) for k, v in (("b", b2), ("x", x0), ("y", y0), ("s", s0))}
    before = {k: v.clone() for k, v in inputs.items()}
    solver.update(b=inputs["b"])
    r = solver.solve(warm_start=True, x=inputs["x"], y=inputs["y"], s=inputs["s"])
    got = [(r["x"].cpu().numpy(), r["y"].cpu().numpy(), r["s"].cpu().numpy(), {k: r["info"][k] for k in INFO_EQUAL})]
    solver.close()
    for k in inputs:
        assert torch.equal(inputs[k], before[k]), k
    assert_same(ref, got)


def _raw_device(lib, d_tensors, cone):
    """scs_b200_init_device on torch tensors without the front end: (work, keep-alive)"""
    T = capi.Int
    ptr = lambda t, p: C.cast(C.c_void_p(t.data_ptr()), p)
    A = d_tensors["A"]
    mats = [T.ScsMatrix(ptr(A.values(), capi.c_double_p), ptr(A.row_indices(), capi.c_int_p),
                        ptr(A.ccol_indices(), capi.c_int_p), A.shape[0], A.shape[1])]
    if "P" in d_tensors:
        P = d_tensors["P"]
        mats.append(T.ScsMatrix(ptr(P.values(), capi.c_double_p), ptr(P.row_indices(), capi.c_int_p),
                                ptr(P.ccol_indices(), capi.c_int_p), P.shape[0], P.shape[1]))
    data = T.ScsData(A.shape[0], A.shape[1], C.pointer(mats[0]), C.pointer(mats[1]) if len(mats) > 1 else
                     C.POINTER(T.ScsMatrix)(), ptr(d_tensors["b"], capi.c_double_p), ptr(d_tensors["c"], capi.c_double_p))
    k, keep = capi.make_cone(cone)
    w = lib.scs_b200_init_device(C.byref(data), C.byref(k), C.byref(capi.default_settings(lib, verbose=0)), None)
    return w, (mats, data, k, keep)


def test_mixed_sequences_and_user_memory_unchanged():
    lib = capi.load()
    A, P, b, c, cone = prob = read_fixture("mpc_bug1")
    ref = host_solve(*prob, seq=[(b * 1.1, None)])
    d = to_torch(*prob[:4])
    before = {k: (v.values().clone(), v.row_indices().clone(), v.ccol_indices().clone()) if v.layout != torch.strided
              else v.clone() for k, v in d.items()}
    # device init, host update and host solves
    w, keep = _raw_device(lib, d, cone)
    assert w
    x, y, s = np.zeros(A.shape[1]), np.zeros(A.shape[0]), np.zeros(A.shape[0])
    got = []
    for step, bb in ((0, None), (1, b * 1.1)):
        if bb is not None:
            assert lib.scs_update(w, capi.dptr(np.ascontiguousarray(bb)), None) == 0
        sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
        lib.scs_solve(w, C.byref(sol), C.byref(info), step)
        got.append((x.copy(), y.copy(), s.copy(), {k: getattr(info, k) for k in INFO_EQUAL}))
    lib.scs_finish(w)
    assert_same(ref, got)
    # host init, device update and device solves
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone, (P.data, P.indices, P.indptr, P.shape))
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0)))
    dx = torch.zeros(A.shape[1], dtype=torch.float64, device="cuda")
    dy, ds = (torch.zeros(A.shape[0], dtype=torch.float64, device="cuda") for _ in range(2))
    p = lambda t: C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p)
    got = []
    b2 = torch.tensor(b * 1.1, device="cuda")
    for step in (0, 1):
        if step:
            assert lib.scs_b200_update_device(w, p(b2), None, None) == 0
        sol, info = capi.ScsSolution(p(dx), p(dy), p(ds)), capi.ScsInfo()
        lib.scs_b200_solve_device(w, C.byref(sol), C.byref(info), step, None)
        torch.cuda.synchronize()
        got.append((dx.cpu().numpy(), dy.cpu().numpy(), ds.cpu().numpy(), {k: getattr(info, k) for k in INFO_EQUAL}))
    lib.scs_finish(w)
    assert_same(ref, got)
    for k, v in d.items():
        if v.layout != torch.strided:
            for u, t in zip(before[k], (v.values(), v.row_indices(), v.ccol_indices())):
                assert torch.equal(u, t)
        else:
            assert torch.equal(before[k], v)


def _csv_bc_norms(path):
    """(b_nrm_inf, c_nrm_inf) of every row of a CSV trace"""
    import csv
    with open(path) as f:
        return [(float(r["b_nrm_inf"]), float(r["c_nrm_inf"])) for r in csv.DictReader(f)]


def test_nan_in_b_and_c_is_skipped_by_both_doors_and_updates_keep_the_other_original(tmp_path):
    """max |b| and max |c| of the data as given skip a NaN, as the reference's norm_inf does, whichever door the data
    comes through; an update of b alone keeps c, and one of c alone keeps b"""
    prob = problems.make_problem(30, 10, 3, {"z": 3, "l": 17, "q": [4, 6]}, seed=4)
    A, cone = sp.csc_matrix(prob["A"][:3], shape=prob["A"][3]), prob["cone"]
    b, c = prob["b"].copy(), prob["c"].copy()
    j, mid = int(np.argmax(np.abs(b))), b.size // 2
    b[[j, mid]] = b[[mid, j]]
    b[mid + 1] = np.nan  # after the largest |b|: a maximum restarted at the NaN would miss it
    c[-1] = np.nan
    seq = [(2.0 * b, None), (None, 3.0 * c)]
    want, bb, cc = [], b, c
    for step in [(None, None)] + seq:
        bb = bb if step[0] is None else step[0]
        cc = cc if step[1] is None else step[1]
        want.append((np.nanmax(np.abs(bb)), np.nanmax(np.abs(cc))))
    lib = capi.load()
    host_csv = str(tmp_path / "host.csv")
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone),
                     C.byref(capi.default_settings(lib, verbose=0, max_iters=1, log_csv_filename=host_csv.encode())))
    assert w
    host = []
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    try:
        for step in [None] + seq:
            if step is not None:
                assert lib.scs_update(w, *[capi.dptr(np.ascontiguousarray(v)) if v is not None else None
                                           for v in step]) == 0
            sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
            lib.scs_solve(w, C.byref(sol), C.byref(info), 0)
            host.append(_csv_bc_norms(host_csv))
    finally:
        lib.scs_finish(w)
    dev_csv = str(tmp_path / "device.csv")
    solver = torch_solver.SCS(to_torch(A, None, b, c), cone, verbose=0, max_iters=1, log_csv_filename=dev_csv.encode())
    device = []
    try:
        for step in [None] + seq:
            if step is not None:
                solver.update(*[None if v is None else torch.tensor(v, device=solver.device) for v in step])
            solver.solve(warm_start=False)
            device.append(_csv_bc_norms(dev_csv))
    finally:
        solver.close()
    assert host == device
    for rows, nm in zip(host, want):
        assert len(rows) >= 2 and all(r == nm for r in rows), (rows, nm)


def _bad(name):
    A, P, b, c, cone = read_fixture("mpc_bug1")
    A, P = A.copy(), P.copy()
    if name == "p0":
        A.indptr = A.indptr.copy(); A.indptr[0] = 1
        return A, P, b, c, cone, "A->p[0] must equal 0"
    if name == "decreasing":
        A.indptr = A.indptr.copy(); A.indptr[2], A.indptr[3] = A.indptr[3], A.indptr[2]
        return A, P, b, c, cone, "must be nonnegative and nondecreasing"
    if name == "row >= m":
        A.indices = A.indices.copy(); A.indices[5] = A.shape[0]
        return A, P, b, c, cone, f"A row index {A.shape[0]} outside valid range"
    if name == "row < 0":
        A.indices = A.indices.copy(); A.indices[7] = -2
        return A, P, b, c, cone, "A row index -2 outside valid range"
    if name == "nan in A":
        A.data = A.data.copy(); A.data[3] = np.nan
        return A, P, b, c, cone, "A contains a non-finite entry"
    if name == "inf in P":
        P.data = P.data.copy(); P.data[0] = np.inf
        return A, P, b, c, cone, "P contains a non-finite entry"
    if name == "P below the diagonal":
        P = sp.csc_matrix(P.toarray() + np.eye(P.shape[0], k=-1))
        return A, P, b, c, cone, "P is not upper triangular"
    raise KeyError(name)


@pytest.mark.parametrize("name", ["p0", "decreasing", "row >= m", "row < 0", "nan in A", "inf in P",
                                  "P below the diagonal"])
def test_invalid_device_data_is_refused_with_the_host_message(capfd, name):
    lib = capi.load()
    A, P, b, c, cone, message = _bad(name)
    capfd.readouterr()  # the fixture reader's own output
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone, (P.data, P.indices, P.indptr, P.shape))
    assert not lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0)))
    host_out = capfd.readouterr().out
    assert message in host_out
    w, keep = _raw_device(lib, to_torch(A, P, b, c), cone)
    assert not w
    assert capfd.readouterr().out == host_out


def test_host_pointer_is_refused(capfd):
    lib = capi.load()
    A, P, b, c, cone = read_fixture("mpc_bug1")
    hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone, (P.data, P.indices, P.indptr, P.shape))
    assert not lib.scs_b200_init_device(C.byref(hp.data), C.byref(hp.cone),
                                        C.byref(capi.default_settings(lib, verbose=0)), None)
    assert "must point to device memory" in capfd.readouterr().out


def test_mismatched_device_is_refused_before_the_library(monkeypatch):
    A, P, b, c, cone = read_fixture("mpc_bug1")
    data = to_torch(A, P, b, c)
    monkeypatch.setattr(torch_solver, "_library_device", lambda: data["A"].device.index + 1)
    monkeypatch.setattr(capi, "load", lambda *a, **k: pytest.fail("the library was loaded"))
    with pytest.raises(ValueError, match="the library drives cuda:"):
        torch_solver.SCS(data, cone)


def test_no_problem_sized_transfer():
    lib = capi.load()
    A, P, b, c, cone = c2_like(scale=0.02)
    # the C2 shape has nnz = 2.5 (m + n): add entries until nnz >= 20 (m + n)
    dense = sp.random(A.shape[0], A.shape[1], density=min(1.0, 25.0 * sum(A.shape) / (A.shape[0] * A.shape[1])),
                      random_state=1, format="csc")
    A = (A + dense).tocsc()
    nnz = A.nnz
    assert nnz >= 20 * sum(A.shape)
    stats = (C.c_longlong * 4)()
    d = to_torch(A, None, b, c)
    torch.cuda.synchronize()
    lib.scs_b200_transfer_stats_reset()
    solver = torch_solver.SCS(d, cone, verbose=0, max_iters=200)
    lib.scs_b200_transfer_stats(stats)
    init_max = max(stats[1], stats[3])
    lib.scs_b200_transfer_stats_reset()
    solver.solve()
    lib.scs_b200_transfer_stats(stats)
    assert max(stats[1], stats[3]) <= 4096, list(stats)
    solver.close()
    assert init_max < 4 * nnz, (init_max, nnz)
    lib.scs_b200_transfer_stats_reset()
    host_solve(A, None, b, c, cone, max_iters=200)
    lib.scs_b200_transfer_stats(stats)
    assert stats[1] >= 8 * nnz, (list(stats), nnz)


def test_front_end_orders_with_a_non_default_stream():
    A, P, b, c, cone = read_fixture("mpc_bug3")
    ref = host_solve(A, P, b * 2.0, c, cone)
    d = to_torch(A, P, b, c)
    solver = torch_solver.SCS(d, cone, verbose=0)
    side = torch.cuda.Stream()
    bt = torch.tensor(b, device="cuda")
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # the update below must wait for this stream's work
        b2 = bt * 2.0
        solver.update(b=b2)
        r = solver.solve(warm_start=False)
        x, y, s = r["x"].cpu(), r["y"].cpu(), r["s"].cpu()
    solver.close()
    assert_same(ref, [(x.numpy(), y.numpy(), s.numpy(), {k: r["info"][k] for k in INFO_EQUAL})])

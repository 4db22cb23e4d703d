"""Independent solves on several host threads at once (include/scs_b200.h, "Threading"): every workspace solves on an
execution context of its own, and each solve returns the same bits as when it runs alone. Every test first solves its
problems serially in this process; that run is the reference. ctypes releases the GIL, so the threads of
concurrent.futures enter the library concurrently. Bit identity does not need convergence: the larger problems run a
capped number of iterations."""
import ctypes as C
import os
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from scs_b200 import capi, problems, torch_solver
from test_device_data_gpu import c2_like, complex_psd, read_fixture, to_torch

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "problems")
INFO_BITS = ("iter", "status_val", "pobj", "dobj")
PP = C.POINTER


def _csc(prob):
    A = prob["A"]
    return sp.csc_matrix((A[0], A[1], A[2]), shape=A[3])


def generated(name, scale, seed=1234):
    prob = problems.config(name, scale=scale, seed=seed)
    return _csc(prob), None, prob["b"], prob["c"], prob["cone"]


# (problem, settings): the C2-shaped ones and the PSD one capped so that each solve takes at most a few seconds
def distinct_problems():
    return {
        "C1": (generated("C1", 1.0), {}),
        "C2x0.01": (generated("C2", 0.01, seed=11), {"max_iters": 300}),
        "C2x0.1": (generated("C2", 0.1, seed=12), {"max_iters": 60}),
        "C4_psd": (generated("C4", 0.05), {"max_iters": 40}),
        "random_prob": (read_fixture("random_prob"), {}),
        "mpc_bug1": (read_fixture("mpc_bug1"), {}),
        "complex_psd": (complex_psd(), {}),
    }


def host_problem(prob, long=False):
    A, P, b, c, cone = prob
    return capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, cone,
                            None if P is None else (P.data, P.indices, P.indptr, P.shape), long=long)


def run_host(prob, settings, long=False):
    """scs_init -> scs_solve -> scs_b200_get_stats / scs_b200_cg_k34_paths -> scs_finish on host buffers (long: the
    DLONG flavour)"""
    lib = capi.load(spectral=capi.is_spectral(prob[4]), long=long)
    T = capi.abi(long)
    hp = host_problem(prob, long)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone),
                     C.byref(capi.default_settings(lib, long=long, verbose=0, **settings)))
    assert w
    try:
        x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
        sol, info = T.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), T.ScsInfo()
        lib.scs_solve(w, C.byref(sol), C.byref(info), 0)
        stats = T.ScsB200Stats()
        assert lib.scs_b200_get_stats(w, C.byref(stats)) == 0
        paths = (C.c_longlong * 2)()
        assert lib.scs_b200_cg_k34_paths(w, paths) == 0
    finally:
        lib.scs_finish(w)
    return {"x": x.tobytes(), "y": y.tobytes(), "s": s.tobytes(),
            "info": {k: np.float64(getattr(info, k)).tobytes() for k in INFO_BITS},
            "cg_iters": stats.cg_iters, "solves": stats.lin_sys_solves, "paths": (paths[0], paths[1]),
            "times": (info.lin_sys_time, info.cone_time, info.accel_time, info.solve_time)}


def run_scs(prob, settings):
    """scs() on host buffers: x, y, s and the info bits"""
    lib = capi.load(spectral=capi.is_spectral(prob[4]))
    hp = host_problem(prob)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
    lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0, **settings)),
            C.byref(sol), C.byref(info))
    return {"x": x.tobytes(), "y": y.tobytes(), "s": s.tobytes(),
            "info": {k: np.float64(getattr(info, k)).tobytes() for k in INFO_BITS}}


def same(a, b, keys=("x", "y", "s", "info")):
    for k in keys:
        assert a[k] == b[k], k


def threaded(jobs, workers):
    """run the callables of `jobs` on `workers` threads, in the given order of submission"""
    with ThreadPoolExecutor(max_workers=workers) as ex:
        futures = [ex.submit(f) for f in jobs]
        return [f.result() for f in futures]


def test_distinct_problems_on_eight_threads_equal_serial():
    probs = distinct_problems()
    names = sorted(probs)
    serial = {n: run_host(*probs[n]) for n in names}
    rng = random.Random(3)
    for _ in range(3):
        order = names + names[:1]  # 8 solves: the first problem twice at once
        rng.shuffle(order)
        out = threaded([lambda n=n: (n, run_host(*probs[n])) for n in order], 8)
        for n, r in out:
            same(r, serial[n])
            assert r["cg_iters"] == serial[n]["cg_iters"], n
            lin, cone, accel, total = r["times"]
            assert min(lin, cone, accel) >= 0.0, (n, r["times"])
            assert lin + cone + accel <= total, (n, r["times"])


def test_allocator_churn_is_bit_identical():
    # same shapes, different seeds: the blocks one thread's workspace frees are reused by another thread's next one
    seeds = [[100 + 5 * t + k for k in range(5)] for t in range(8)]
    prob = {sd: (generated("C1", 0.5, seed=sd), {"max_iters": 400}) for row in seeds for sd in row}
    serial = {sd: run_scs(*prob[sd]) for sd in prob}

    def worker(row):
        return [(sd, run_scs(*prob[sd])) for sd in row]

    for rows in threaded([lambda row=row: worker(row) for row in seeds], 8):
        for sd, r in rows:
            same(r, serial[sd])


# the fused kernel's grid: 4096 elements of x per block (kernels/cg.cu k34_grid); larger n needs more than one block
K34_PER_BLOCK = 4096


def test_fused_cg_token_totals():
    # C2 x 0.01 .. x 0.3 (n = 10^4 .. 3 10^5: fused grids of 3 to 74 blocks): at most one of them runs the fused kernel
    # at a time, the others take the pair
    probs = {s: (generated("C2", s, seed=20 + i), {"max_iters": 100}) for i, s in enumerate((0.01, 0.03, 0.1, 0.3))}
    assert all(p[0][0].shape[1] > K34_PER_BLOCK for p in probs.values())
    serial = {s: run_host(*probs[s]) for s in probs}
    for s, r in serial.items():  # alone, every KKT solve holds the token
        assert r["paths"] == (r["solves"], 0), (s, r["paths"], r["solves"])
    out = threaded([lambda s=s: (s, run_host(*probs[s])) for s in probs], 4)
    fused = 0
    for s, r in out:
        same(r, serial[s])
        assert r["cg_iters"] == serial[s]["cg_iters"]
        assert r["paths"][0] + r["paths"][1] == r["solves"], (s, r["paths"], r["solves"])
        fused += r["paths"][0]
    assert fused >= 1


def test_every_flavour_shares_the_token():
    # one token per process, in libscs_b200_token.so: held here, the int and the DLONG flavour both run the pair
    prob = (generated("C2", 0.03, seed=5), {"max_iters": 60})
    assert prob[0][0].shape[1] > K34_PER_BLOCK
    free = run_host(*prob)
    assert free["paths"] == (free["solves"], 0)
    token = C.CDLL(os.path.join(os.path.dirname(capi.LIB_PATH), "libscs_b200_token.so"))
    assert token.b200_k34_token_take() == 1
    try:
        held = [run_host(*prob), run_host(*prob, long=True)]
    finally:
        token.b200_k34_token_give_back()
    for r in held:
        assert r["paths"] == (0, free["solves"]), r["paths"]
        same(r, free)
    again = run_host(*prob, long=True)
    assert again["paths"] == (free["solves"], 0)
    same(again, free)


def torch_sequence(prob, settings):
    """solve -> update(b=) -> solve(warm) -> update(A=) -> solve, on the current torch stream; results read there"""
    A, P, b, c, cone = prob
    data = to_torch(A, P, b, c)
    solver = torch_solver.SCS(data, cone, verbose=0, **settings)
    out = []
    try:
        r = solver.solve(warm_start=False)
        out.append(r)
        solver.update(b=data["b"] * 1.05)
        out.append(solver.solve(warm_start=True))
        A2 = A.copy()
        A2.data = A2.data * 0.9
        solver.update(A=to_torch(A2, None, b, c)["A"])
        out.append(solver.solve(warm_start=True))
        res = [(r["x"].cpu().numpy().tobytes(), r["y"].cpu().numpy().tobytes(), r["s"].cpu().numpy().tobytes(),
                {k: np.float64(r["info"][k]).tobytes() for k in INFO_BITS}) for r in out]
    finally:
        solver.close()
    return res


def test_torch_front_end_one_solver_per_thread():
    probs = {"C1": (generated("C1", 0.5), {}), "C2x0.01": (c2_like(0.01, seed=31), {"max_iters": 200}),
             "random_prob": (read_fixture("random_prob"), {}), "complex_psd": (complex_psd(), {})}
    serial = {n: torch_sequence(*probs[n]) for n in probs}
    dev = torch.device("cuda", torch_solver._library_device())

    def worker(n):
        stream = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(stream):
            return n, torch_sequence(*probs[n])

    for n, r in threaded([lambda n=n: worker(n) for n in probs], 4):
        assert r == serial[n], n


def read_spectral(path):
    lib = capi.load(spectral=True)
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                       PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    return lib, d, k, s


def run_spectral(lib, d, k, s):
    st = capi.ScsSettings.from_buffer_copy(s.contents)
    st.verbose, st.max_iters = 0, min(st.max_iters, 2000)
    m, n = d.contents.m, d.contents.n
    x, y, z = np.zeros(n), np.zeros(m), np.zeros(m)
    sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(z)), capi.ScsInfo()
    lib.scs(d, k, C.byref(st), C.byref(sol), C.byref(info))
    return {"x": x.tobytes(), "y": y.tobytes(), "s": z.tobytes(),
            "info": {key: np.float64(getattr(info, key)).tobytes() for key in INFO_BITS}}


def test_spectral_cones_each_workspace_its_own_eigensolver():
    paths = [os.path.join(GOLDEN, "logdet", f) for f in ("dopt_24", "exp_design", "several_logdet_cones")]
    paths += [os.path.join(GOLDEN, "spectral", f) for f in ("several_nuc_cone", "several_sum_largest",
                                                            "test_ell1_and_nuc")]
    read = [read_spectral(p) for p in paths]
    try:
        serial = [run_spectral(*r) for r in read]
        out = threaded([lambda r=r: run_spectral(*r) for r in read], len(read))
        for p, a, b in zip(paths, out, serial):
            assert a == b, p
    finally:
        for lib, d, k, s in read:
            lib.scs_b200_free_data(d, k, s)


def test_plugin_linear_systems_on_four_threads():
    lib = capi.load()
    cases = []
    for t in range(4):
        A, _, b, c, cone = c2_like(0.01 * (t + 1), seed=40 + t)
        hp = host_problem((A, None, b, c, cone))
        rng = np.random.default_rng(t)
        diag_r = np.concatenate([np.full(hp.n, 1e-6), rng.uniform(0.5, 2.0, hp.m), [10.0]])
        rhs = [rng.standard_normal(hp.n + hp.m) for _ in range(4)]
        cases.append((hp, diag_r, rhs))

    def solve_all(case):
        hp, diag_r, rhs = case
        w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(diag_r))
        assert w
        out = []
        try:
            warm = None
            for r in rhs:
                v = r.copy()
                assert lib.scs_solve_lin_sys(w, capi.dptr(v), capi.dptr(warm), 1e-9) == 0
                out.append(v.tobytes())
                warm = np.ascontiguousarray(v[:hp.n])
        finally:
            lib.scs_free_lin_sys_work(w)
        return out

    serial = [solve_all(cs) for cs in cases]
    assert threaded([lambda cs=cs: solve_all(cs) for cs in cases], 4) == serial


def test_refused_init_leaves_a_concurrent_solve_untouched():
    prob = (generated("C1", 1.0, seed=77), {})
    A, _, b, c, cone = prob[0]
    bad = dict(cone)
    bad["l"] = cone["l"] + 1  # cone rows no longer add up to m
    lib = capi.load()
    serial = run_host(*prob)

    def refused():
        hp = capi.HostProblem((A.data, A.indices, A.indptr, A.shape), b, c, bad)
        return lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(capi.default_settings(lib, verbose=0)))

    w, r = threaded([refused, lambda: run_host(*prob)], 2)
    assert not w
    same(r, serial)
    assert r["cg_iters"] == serial["cg_iters"]

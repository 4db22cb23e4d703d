"""GPU: the log-det cone of libscs_b200_spectral.so.

* operator: scs_b200_proj_dual_cone against the reference's _scs_proj_dual_cone recorded in tests/golden/logdet_cones.npz
  (oracle/make_golden_logdet.py) on the inputs of tests/logdet_cases.py, with and without r_y, each input within
  max(5e-13, 10 x the spread between tests/logdet_numpy.py and the reference on that input), and with the reference's
  Newton record (newton_success, iter; scs_b200_cone_logdet_stats); on diagonal inputs, where both eigensolvers are
  exact, the operator reproduces the reference's recorded vector step and its record, warm-started second calls on
  one cone workspace included;
* solver, on tests/golden/problems/logdet/: one iteration within 1e-10 of the reference's x, y, s; status solved,
  objective within 10 eps of the optimum (or 10x the reference's own distance to it); tests/verify.py clean with the
  numpy log-det projection, complementary slackness within what the reference's own recorded solution reaches; the
  iteration count within 1.5x + 25 of the range the reference itself shows when b moves by a few ulps (its
  iteration counts on these problems are that sensitive); the CSV trace's Newton columns as the reference wrote them
  (row 0 exactly, the branch and count of the first 12 rows);
* the same bits through every door: the DLONG library, torch_solver.SCS on CUDA tensors, and update(A=...) against a
  fresh device init (exp_design, whose log-det warm starts change the iterates)."""
import csv
import ctypes as C
import json
import os

import numpy as np
import pytest

import logdet_cases
import logdet_numpy
import verify
from conftest import ROOT
from scs_b200 import capi

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
PROB_DIR = os.path.join(GOLD, "problems", "logdet")
OPS = np.load(os.path.join(GOLD, "logdet_cones.npz"))
SOLVES = np.load(os.path.join(GOLD, "logdet_solves.npz"))
OPTIMA = json.load(open(os.path.join(PROB_DIR, "optima.json")))
NEWTON_COLS = ["spectral_Newton_iter", "plain_Newton_success", "res_dual_spectral", "res_pri_spectral",
               "comp_spectral"]
PP = C.POINTER


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def slib():
    lib = capi.load(spectral=True)
    assert lib.scs_b200_device_ok()
    lib.scs_b200_read_data.restype = C.c_int
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                       PP(PP(capi.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    return lib


class Cone:
    """one scs_b200 cone workspace of a single log-det cone of order n (its warm-start state persists across calls)"""

    def __init__(self, lib, n):
        self.lib = lib
        self.k, self.keep = capi.make_cone({"d": [n]}, spectral=True)
        self.m = logdet_cases.rows(n)
        self.cw = lib.scs_b200_init_cone(C.byref(self.k), self.m, None)
        assert self.cw, "scs_b200_init_cone failed"

    def proj(self, x, r_y=None):
        out = x.copy()
        assert self.lib.scs_b200_proj_dual_cone(self.cw, capi.dptr(out), capi.dptr(r_y)) == 0
        return out

    def record(self):
        """(iter, newton_success) of the last projection"""
        it, ok, res = C.c_int(), C.c_int(), np.zeros(3)
        assert self.lib.scs_b200_cone_logdet_stats(self.cw, C.byref(it), C.byref(ok), capi.dptr(res)) == 0
        return it.value, ok.value

    def close(self):
        self.lib.scs_b200_finish_cone(self.cw)


def _rel(a, ref, x):
    return np.abs(a - ref).max() / max(np.abs(ref).max(), np.abs(x).max())


@pytest.mark.parametrize("metric", [False, True])
def test_proj_dual_cone_matches_reference(slib, metric):
    """each input has its own gate: the numpy restatement's distance to the reference on that input (x + Pi(-R x) / R)
    times 10, at least 5e-13"""
    cases = {name: (n, x) for name, n, x in logdet_cases.operator_cases()}
    assert sorted(cases) == sorted(str(s) for s in OPS["names"])
    tag = "ry" if metric else ""
    worst = 0.0
    for name, (n, x) in cases.items():
        np.testing.assert_array_equal(x, OPS[f"{name}/x"])
        r = logdet_cases.r_y(n) if metric else np.ones(x.size)
        ref, rec = OPS[f"{name}/out{tag}"], OPS[f"{name}/rec{tag}"]
        _, p, _ = logdet_numpy.proj_logdet(-r * x, n, logdet_numpy.State(n))
        gate = max(5e-13, 10 * _rel(x + p / r, ref, x))
        c = Cone(slib, n)
        try:
            mine = c.proj(x, r if metric else None)
            record = c.record()
        finally:
            c.close()
        err = _rel(mine, ref, x)
        worst = max(worst, err / gate)
        assert err <= gate, (name, metric, err, gate)
        assert record == (int(rec[1]), int(rec[2])), (name, metric, record, rec[1:3])
    print(f"operator: worst error / gate {worst:.3f}")


def _diag_input(t0, v0, e):
    """operator rows whose Moreau dual projection runs the vector step on exactly (t0, v0, e): x = -(t, v, X) with
    X = diag(e) / sqrt2 (the unpack scales the diagonal by sqrt2), e ascending along the diagonal"""
    n = e.size
    s2 = np.sqrt(2.0)
    packed = []
    for j in range(n):
        packed.append(e[j] / s2)
        packed.extend([0.0] * (n - 1 - j))
    return -np.concatenate(([t0 / s2, v0 / s2], packed))


def _diag_out(x, out, n):
    """the projection's (t, v, diag X) from the operator's Moreau answer, scaled back to the vector step's units"""
    p = out - x
    s2 = np.sqrt(2.0)
    diag = []
    k = 2
    for j in range(n):
        diag.append(p[k])
        k += n - j
    return np.concatenate(([p[0] * s2, p[1] * s2], np.array(diag) * s2))


def test_vector_step_matches_the_reference_on_diagonal_inputs(slib):
    """the recorded log_cone_proj_wrapper answers and records, including warm-started second calls on one workspace.
    Each call's gate is 10x the numpy restatement's distance to the reference on it, at least 5e-13 (the
    interior-point answers agree with the reference only to the IPM's tolerances)."""
    replay = logdet_cases.replay(logdet_cases.vector_cases())
    for name in OPS["vnames"]:
        name = str(name)
        n = int(name.rsplit("_", 1)[1])
        c = Cone(slib, n)
        try:
            for j, (_, proj, _) in enumerate(replay[name]):
                tve = OPS[f"v/{name}/in{j}"]
                ref, rec = OPS[f"v/{name}/proj{j}"], OPS[f"v/{name}/rec{j}"]
                assert rec[0] == 0
                gate = max(5e-13, 10 * _rel(proj, ref, tve))
                x = _diag_input(tve[0], tve[1], tve[2:])
                mine = _diag_out(x, c.proj(x), n)
                err = _rel(mine, ref, tve)
                assert err <= gate, (name, j, err, gate)
                assert c.record() == (int(rec[1]), int(rec[2])), (name, j, c.record(), rec[1:3])
        finally:
            c.close()


def read_problem(lib, name):
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert lib.scs_b200_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    return d, k, s


def as_dict(d, k):
    D, K = d.contents, k.contents
    A = D.A.contents
    nnz = A.p[A.n]
    arr = lambda p, n, t: np.ctypeslib.as_array(p, (n,)).astype(t) if n > 0 else np.zeros(0, t)  # noqa: E731
    cone = {"z": K.z, "l": K.l, "q": list(arr(K.q, K.qsize, int)), "s": list(arr(K.s, K.ssize, int)),
            "d": list(arr(K.d, K.dsize, int))}
    assert K.bsize == 0 and K.cssize == 0 and K.ep == 0 and K.ed == 0 and K.psize == 0 and not D.P
    assert K.nucsize == 0 and K.ell1_size == 0 and K.sl_size == 0
    Acsc = (arr(A.x, nnz, np.float64), arr(A.i, nnz, np.int32), arr(A.p, A.n + 1, np.int32), (D.m, D.n))
    return {"A": Acsc, "b": arr(D.b, D.m, np.float64), "c": arr(D.c, D.n, np.float64), "cone": cone, "P": None}


def solve(lib, d, k, s, **over):
    st = capi.ScsSettings.from_buffer_copy(s.contents)
    st.verbose = 0
    for key, v in over.items():
        setattr(st, key, v)
    m, n = d.contents.m, d.contents.n
    x, y, z = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(z))
    info = capi.ScsInfo()
    flag = lib.scs(d, k, C.byref(st), C.byref(sol), C.byref(info))
    return flag, info, st, x, y, z


@pytest.mark.parametrize("name", sorted(OPTIMA))
def test_reference_logdet_problem(slib, name, tmp_path):
    d, k, s = read_problem(slib, name)
    try:
        prob = as_dict(d, k)
        _, _, _, x1, y1, s1 = solve(slib, d, k, s, max_iters=1)
        for mine, key in ((x1, "x1"), (y1, "y1"), (s1, "s1")):
            ref = SOLVES[f"{name}/{key}"]
            err = np.abs(mine - ref).max() / max(1.0, np.abs(ref).max())
            assert err <= 1e-10, (name, key, err)
        flag, info, st, x, y, z = solve(slib, d, k, s)
        ref_flag, ref_iter = SOLVES[f"{name}/info"][:2]
        assert flag == 1 and int(ref_flag) == 1, (name, flag, info.status)
        opt = OPTIMA[name]
        # dopt_24's objective is only as accurate as its residuals allow: the reference itself stops 5e-6 from the
        # certified optimum at eps 1e-7, so the gate is 10 eps or 10 times the reference's own distance
        ref_err = abs(SOLVES[f"{name}/info"][2] - opt)
        assert abs(info.pobj - opt) <= max(10 * st.eps_abs * max(1.0, abs(opt)), 10 * ref_err), (name, info.pobj, opt)
        pdual = lambda v: logdet_numpy.proj_dual_cone(v, prob["cone"])  # noqa: E731
        fails = verify.verify_solution_correct(prob, st, info, x, y, z, flag, ref_proj_dual=pdual)
        # verify.py bounds |s'y| by 5e-8 max(|s|, |y|). The reference's own solution (recorded) can miss that bound
        # on these problems; complementary slackness is then held to twice the reference's own |s'y| / bound
        ys, ss = SOLVES[f"{name}/yf"], SOLVES[f"{name}/sf"]
        ref_ratio = abs(float(ys @ ss)) / (5e-8 * max(np.abs(ss).max(), np.abs(ys).max()))
        for what, val, bound in fails:
            assert what == "Complementary slackness ERROR" and val <= 2 * max(1.0, ref_ratio) * bound, \
                (name, fails, ref_ratio)
        # the reference's iteration count moves a lot when b changes by a few ulps: the window is 1.5x + 25 around
        # the range of its recorded perturbed runs
        spread = SOLVES[f"{name}/iters_spread"]
        lo, hi = min(spread.min(), ref_iter), max(spread.max(), ref_iter)
        assert lo / 1.5 - 25 <= info.iter <= 1.5 * hi + 25, (name, info.iter, ref_iter, spread)
        # the CSV trace copies every iterate to the host: its first row comes from a short run
        log = str(tmp_path / "trace.csv")
        ref_rows = SOLVES[f"{name}/csv"]
        solve(slib, d, k, s, max_iters=len(ref_rows), log_csv_filename=log.encode())
        rows = list(csv.DictReader(open(log)))
        mine = [float(rows[0][c]) for c in NEWTON_COLS]
        ref = ref_rows[0]
        assert np.allclose(mine[2:], ref[2:], rtol=0, atol=1e-9), (name, mine, ref)
        for r, ref in zip(rows, ref_rows):  # the same branch and Newton iteration count, row by row
            assert [float(r[c]) for c in NEWTON_COLS[:2]] == list(ref[:2]), (name, r, ref)
        print(f"{name}: iters {info.iter} (reference {int(ref_iter)}, {int(lo)}..{int(hi)} under ulp changes of b) "
              f"pobj {info.pobj:.12g} opt {opt:.12g} "
              f"Newton row 0 {mine[:2]}")
    finally:
        slib.scs_b200_free_data(d, k, s)


def _solve_file_with(long, name, **over):
    T = capi.abi(long)
    lib = capi.load(spectral=True, long=long)
    cone = T.ScsConeSpectral
    lib.scs_b200_read_data.restype = T.int_t
    lib.scs_b200_read_data.argtypes = [C.c_char_p, PP(PP(T.ScsData)), PP(PP(cone)), PP(PP(T.ScsSettings))]
    lib.scs_b200_free_data.argtypes = [PP(T.ScsData), PP(cone), PP(T.ScsSettings)]
    d, k, s = PP(T.ScsData)(), PP(cone)(), PP(T.ScsSettings)()
    assert lib.scs_b200_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    s.contents.verbose = 0
    for f, v in over.items():
        setattr(s.contents, f, v)
    n, m = d.contents.n, d.contents.m
    x, y, sv = np.zeros(n), np.zeros(m), np.zeros(m)
    sol = T.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(sv))
    info = T.ScsInfo()
    flag = lib.scs(d, k, s, C.byref(sol), C.byref(info))
    lib.scs_b200_free_data(d, k, s)
    return flag, info.iter, x, y, sv


@pytest.mark.parametrize("name", ["exp_design", "several_logdet_cones"])
def test_dlong_library_gives_the_same_bits(name):
    r_int = _solve_file_with(False, name, max_iters=2000)
    r_long = _solve_file_with(True, name, max_iters=2000)
    assert r_int[:2] == r_long[:2]
    for a, b in zip(r_int[2:], r_long[2:]):
        assert np.array_equal(bits(a), bits(b))


def _torch_data(prob):
    import torch
    from scs_b200 import torch_solver
    dev = torch.device("cuda", torch_solver._library_device())
    x, i, p, shape = prob["A"]
    A = torch.sparse_csc_tensor(torch.tensor(p), torch.tensor(i), torch.tensor(x), size=shape, device=dev)
    return {"A": A, "b": torch.tensor(prob["b"], device=dev), "c": torch.tensor(prob["c"], device=dev)}


def test_torch_front_end_and_update_give_the_same_bits(slib):
    """exp_design through scs() on host arrays, through torch_solver.SCS on CUDA tensors (which must pick the
    spectral library), and through update(A=A') on a workspace that has solved the original A, against a fresh init
    on A': the update must reset the log-det warm starts, or the first projection of the next solve differs"""
    from scs_b200 import torch_solver
    d, k, s = read_problem(slib, "exp_design")
    try:
        prob = as_dict(d, k)
        st = {"max_iters": 300, "eps_abs": 1e-7, "eps_rel": 1e-7}
        flag, info, _, x, y, z = solve(slib, d, k, s, **st)
    finally:
        slib.scs_b200_free_data(d, k, s)
    cone = {"z": prob["cone"]["z"], "l": prob["cone"]["l"], "d": prob["cone"]["d"]}
    solver = torch_solver.SCS(_torch_data(prob), cone, verbose=0, **st)
    try:
        assert solver._lib is capi.load(spectral=True)
        r = solver.solve(warm_start=False)
        for a, b in ((r["x"], x), (r["y"], y), (r["s"], z)):
            assert np.array_equal(bits(a.cpu().numpy()), bits(b))
        # a new A on the same pattern
        xA, iA, pA, shape = prob["A"]
        rng = np.random.default_rng(7)
        A2 = (xA * (1 + 0.05 * rng.standard_normal(xA.size)), iA, pA, shape)
        prob2 = dict(prob, A=A2)
        d2 = _torch_data(prob2)
        solver.update(A=d2["A"])
        r_up = solver.solve(warm_start=False)
    finally:
        solver.close()
    fresh = torch_solver.SCS(_torch_data(prob2), cone, verbose=0, **st)
    try:
        r_fr = fresh.solve(warm_start=False)
        r_again = fresh.solve(warm_start=False)  # the same workspace keeps its log-det warm starts
    finally:
        fresh.close()
    assert r_up["info"]["iter"] == r_fr["info"]["iter"]
    for key in "xys":
        assert np.array_equal(bits(r_up[key].cpu().numpy()), bits(r_fr[key].cpu().numpy())), key
    # warm starts change the bits, so the equality above needs the update's reset
    assert not all(np.array_equal(bits(r_again[key].cpu().numpy()), bits(r_fr[key].cpu().numpy())) for key in "xys")

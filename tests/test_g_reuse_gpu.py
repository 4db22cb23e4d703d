"""scs_solve reuses g = (R + M)^{-1} [c; -b] from the workspace's previous solve when nothing g depends on has changed
since it was computed (DESIGN.md section 3.2, "Reusing g"). Every sequence runs twice, with the reuse and with
SCS_B200_G_REUSE=0, which re-solves g at every scs_solve: x, y, s and the ScsInfo results must be the same bits, and a
solve that reuses g must do exactly one linear-system solve fewer, and fewer CG iterations, than its re-solving twin.
Where A, P, b, c or the scale changed, both arms must do the same work."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from scs_b200 import capi, problems, torch_solver

pytestmark = pytest.mark.gpu
INFO = ("iter", "status_val", "pobj", "dobj", "res_pri", "res_dual", "gap", "res_infeas", "res_unbdd_a", "res_unbdd_p",
        "scale", "scale_updates", "comp_slack", "accepted_accel_steps", "rejected_accel_steps")
ST = dict(verbose=0, max_iters=300, eps_abs=1e-7, eps_rel=1e-7)


def socp(n=3000, seed=3, box=False):
    """a random SOCP shaped like the benchmark's C2 (m = 3 n, 10 entries per column), optionally with a box cone"""
    m = 3 * n
    q = [3] * (n // 3) + [40] * 5
    cone = {"z": n // 4, "q": q}
    rest = m - cone["z"] - sum(q)
    if box:
        rng = np.random.default_rng(seed)
        cone["bl"], cone["bu"] = list(-rng.uniform(0.5, 1.5, 99)), list(rng.uniform(0.5, 1.5, 99))
        rest -= 100
    cone["l"] = rest
    return problems.make_problem(m, n, 10, cone, seed=seed)


def stats(lib, work, long=False):
    s = capi.abi(long).ScsB200Stats()
    assert lib.scs_b200_get_stats(work, C.byref(s)) == 0
    return s.cg_iters, s.lin_sys_solves


class Host:
    """scs_init on host buffers (the default library, or the DLONG one)"""

    def __init__(self, prob, long=False, **st):
        self.long = long
        self.lib = capi.load(long=long)
        self.hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], long=long)
        s = capi.default_settings(self.lib, long=long, **{**ST, **st})
        self.work = self.lib.scs_init(C.byref(self.hp.data), C.byref(self.hp.cone), C.byref(s))
        assert self.work
        self.sol = [np.zeros(self.hp.n), np.zeros(self.hp.m), np.zeros(self.hp.m)]

    def solve(self, warm=False):
        T = capi.abi(self.long)
        sol = T.ScsSolution(*(capi.dptr(a) for a in self.sol))
        info = T.ScsInfo()
        self.lib.scs_solve(self.work, C.byref(sol), C.byref(info), int(warm))
        return [a.copy() for a in self.sol] + [{k: getattr(info, k) for k in INFO}] + list(stats(self.lib, self.work,
                                                                                                   self.long))

    def update(self, b=None, c=None):
        assert self.lib.scs_update(self.work, capi.dptr(b), capi.dptr(c)) == 0

    def close(self):
        self.lib.scs_finish(self.work)


def dev_tensors(prob, seed=None):
    """the problem as CUDA tensors for the device door; with `seed`, A's values times (1 + 0.1 N(0, 1))"""
    dev = torch.device("cuda", torch_solver._library_device())
    Ax, Ai, Ap, shape = prob["A"]
    if seed is not None:
        Ax = Ax * (1 + 0.1 * np.random.default_rng(seed).standard_normal(len(Ax)))
    A = torch.sparse_csc_tensor(torch.tensor(Ap, dtype=torch.int32), torch.tensor(Ai, dtype=torch.int32),
                                torch.tensor(Ax, dtype=torch.float64), size=shape, device=dev)
    return {"A": A, "b": torch.tensor(prob["b"], device=dev), "c": torch.tensor(prob["c"], device=dev)}


class Device:
    """scs_b200_init_device through the PyTorch front end"""

    def __init__(self, prob, **st):
        self.prob = prob
        self.s = torch_solver.SCS(dev_tensors(prob), prob["cone"], **{**ST, **st})

    def solve(self, warm=False):
        r = self.s.solve(warm_start=warm)
        return ([r[k].cpu().numpy() for k in "xys"] + [{k: r["info"][k] for k in INFO if k in r["info"]}] +
                list(stats(self.s._lib, self.s._work)))

    def update(self, b=None, c=None, A_seed=None):
        d = dev_tensors(self.prob, A_seed)
        self.s.update(b=None if b is None else torch.tensor(b, device=d["b"].device),
                      c=None if c is None else torch.tensor(c, device=d["c"].device),
                      A=None if A_seed is None else d["A"])

    def close(self):
        self.s.close()


def both_arms(run, monkeypatch):
    """run(), which returns the records of its solves, with the reuse and with SCS_B200_G_REUSE=0"""
    out = []
    for reuse in ("1", "0"):
        monkeypatch.setenv("SCS_B200_G_REUSE", reuse)
        out.append(run())
    monkeypatch.delenv("SCS_B200_G_REUSE")
    return out


def check(on, off, reused):
    """solve k of `on` reused g iff reused[k]; the results are the same bits in both arms"""
    assert len(on) == len(off) == len(reused)
    for k, (a, b, r) in enumerate(zip(on, off, reused)):
        for name, u, v in zip("xys", a[:3], b[:3]):
            assert u.tobytes() == v.tobytes(), (k, name, np.abs(u - v).max())
        assert {f: np.float64(a[3][f]).tobytes() for f in a[3]} == {f: np.float64(b[3][f]).tobytes() for f in b[3]}, \
            (k, a[3], b[3])
        (cg_on, solves_on), (cg_off, solves_off) = a[4:], b[4:]
        if r:
            assert solves_on == solves_off - 1, (k, solves_on, solves_off)
            assert cg_on < cg_off, (k, cg_on, cg_off)
        else:
            assert (cg_on, solves_on) == (cg_off, solves_off), (k, cg_on, cg_off, solves_on, solves_off)


def sequence(make, steps):
    """make() a workspace, then each step: "cold", "warm", or a callable that updates the workspace"""
    def run():
        w = make()
        try:
            recs = []
            for step in steps:
                if callable(step):
                    step(w)
                else:
                    recs.append(w.solve(warm=step == "warm"))
            return recs
        finally:
            w.close()
    return run


@pytest.mark.parametrize("second", ["cold", "warm"])
def test_solve_then_solve(second, monkeypatch):
    prob = socp()
    on, off = both_arms(sequence(lambda: Host(prob), ["cold", second, second]), monkeypatch)
    check(on, off, [False, True, True])


def test_after_a_scale_update(monkeypatch):
    """update_scale re-solves g at the new scale inside the solve; the next solve reuses that g"""
    prob = socp()
    on, off = both_arms(sequence(lambda: Host(prob, scale=1e-3, max_iters=400, eps_abs=0.0, eps_rel=0.0),
                                 ["cold", "cold"]), monkeypatch)
    assert on[0][3]["scale_updates"] >= 1 and on[0][3]["scale"] != 1e-3
    check(on, off, [False, True])


@pytest.mark.parametrize("which", ["b", "c", "both", "neither"])
def test_scs_update_invalidates(which, monkeypatch):
    prob = socp()
    rng = np.random.default_rng(5)
    b = prob["b"] * (1 + 1e-3 * rng.standard_normal(len(prob["b"]))) if which in ("b", "both") else None
    c = prob["c"] * (1 + 1e-3 * rng.standard_normal(len(prob["c"]))) if which in ("c", "both") else None
    on, off = both_arms(sequence(lambda: Host(prob), ["cold", lambda w: w.update(b, c), "warm", "cold"]), monkeypatch)
    check(on, off, [False, False, True])


def test_dlong_library(monkeypatch):
    prob = socp(seed=4)
    on, off = both_arms(sequence(lambda: Host(prob, long=True), ["cold", "cold", lambda w: w.update(b=prob["b"] * 2),
                                                                  "cold"]), monkeypatch)
    check(on, off, [False, True, False])


@pytest.mark.parametrize("box", [False, True])
def test_device_door(box, monkeypatch):
    """init_device / solve_device; scs_b200_update_device (new b, new c) and scs_b200_update_matrix_device (new values
    of A, which also renormalise the box bounds) each make the next solve re-solve g"""
    prob = socp(seed=6, box=box)
    steps = ["cold", "warm", lambda w: w.update(b=prob["b"] * 0.5), "cold", "cold",
             lambda w: w.update(c=prob["c"] * 0.5), "warm", lambda w: w.update(A_seed=9), "cold", "warm"]
    on, off = both_arms(sequence(lambda: Device(prob), steps), monkeypatch)
    check(on, off, [False, True, False, True, False, False, True])


def test_box_cone_host(monkeypatch):
    prob = socp(seed=7, box=True)
    on, off = both_arms(sequence(lambda: Host(prob), ["cold", "cold", lambda w: w.update(c=prob["c"] + 0.1), "cold"]),
                        monkeypatch)
    check(on, off, [False, True, False])

"""One call of each operator-level entry point through the host door (host arrays, staged through HBM) and through
its device twin (CUDA tensors, no copy), in the same process, alternating call by call:

- the cone projection of C4 (200 PSD(100) + 1e5 LP rows) and of C2 (z 3e5, l 9e5, 50 SOCs of 36 000 rows);
- 200 log-det cones of order 100 (libscs_b200_spectral.so);
- accum_by_a / accum_by_atrans and a tolerance-1e-4 warm-started KKT solve on C2's A (scs_b200/problems.py);
- one aa_apply at C2's dimension n + m + 1 with memory 10, on a contraction's iterates.

Each call is bracketed by CUDA events on the current stream, and the stream is drained after each, so a figure is the
time from the call to its last result: for the host door that includes the copies in and out. The two doors run on
separate workspaces fed the same inputs, and the outputs of every call are compared bit for bit. Prints the card's
name and power limit, one line per operator (median and range in ms) and one JSON line.

    python scripts/bench_operators_device.py [--calls 50] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi, problems  # noqa: E402
from bench_device_data import card  # noqa: E402


def dp(t):
    return C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p) if t is not None else None


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def timed(call):
    """ms from the call to its last result, on the current stream's clock"""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    call()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def same(h, d):
    return np.asarray(h).tobytes() == d.detach().cpu().numpy().tobytes()


class Bench:
    def __init__(self, calls, warmup):
        self.calls, self.warmup = calls, warmup
        self.rows = {}

    def run(self, name, step):
        """step(i) -> (host_call, device_call, check): check() after both says whether the outputs agree"""
        ms = {"host": [], "device": []}
        identical = True
        for i in range(self.warmup + self.calls):
            host, device, check = step(i)
            th, td = timed(host), timed(device)
            identical &= bool(check())
            if i >= self.warmup:
                ms["host"].append(th)
                ms["device"].append(td)
        row = {door: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v))}
               for door, v in ms.items()}
        row["bit_identical"] = identical
        self.rows[name] = row
        print(f"{name:<34} host {row['host']['median_ms']:9.3f} ms [{row['host']['min_ms']:.3f}, "
              f"{row['host']['max_ms']:.3f}]   device {row['device']['median_ms']:9.3f} ms "
              f"[{row['device']['min_ms']:.3f}, {row['device']['max_ms']:.3f}]   bit-identical {identical}", flush=True)


def bench_cone(b, name, cone):
    spectral = capi.is_spectral(cone)
    lib = capi.load(spectral=spectral)
    m = capi.cone_rows(cone)
    k, _keep = capi.make_cone(cone, spectral=spectral)
    hw, dw = lib.scs_b200_init_cone(C.byref(k), m, None), lib.scs_b200_init_cone(C.byref(k), m, None)
    assert hw and dw
    rng = np.random.default_rng(1)
    x = rng.standard_normal(m)
    d_x0 = torch.from_numpy(x).cuda()
    buf = {}

    def step(i):
        buf["h"], buf["d"] = x.copy(), d_x0.clone()
        return (lambda: lib.scs_b200_proj_dual_cone(hw, capi.dptr(buf["h"]), None),
                lambda: lib.scs_b200_proj_dual_cone_device(dw, dp(buf["d"]), None, stream()),
                lambda: same(buf["h"], buf["d"]))
    b.run(name, step)
    lib.scs_b200_finish_cone(hw)
    lib.scs_b200_finish_cone(dw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_operators_device.py needs the H100; there is no CPU measurement")
    print(f"card: {card()}", flush=True)
    b = Bench(a.calls, a.warmup)
    bench_cone(b, "proj_dual_cone C4 (200 PSD(100))", {"l": 100_000, "s": [100] * 200})
    c2 = problems.config("C2")
    bench_cone(b, "proj_dual_cone C2 (50 SOC)", c2["cone"])
    bench_cone(b, "proj_dual_cone 200 log-det(100)", {"d": [100] * 200})

    lib = capi.load()
    Ax, Ai, Ap, (m, n) = c2["A"]
    Ax, Ai, Ap = (np.ascontiguousarray(v) for v in (Ax, Ai.astype(np.int32), Ap.astype(np.int32)))
    A = capi.ScsMatrix(capi.dptr(Ax), capi.iptr(Ai), capi.iptr(Ap), m, n)
    z = c2["cone"]["z"]
    diag_r = np.concatenate((np.full(n, 1e-6), np.full(m, 10.0)))  # SCS's R at scale 0.1
    diag_r[n:n + z] = 1e-2
    d_A = [torch.from_numpy(v).cuda() for v in (Ax, Ai, Ap)]
    Ad = capi.ScsMatrix(dp(d_A[0]), C.cast(C.c_void_p(d_A[1].data_ptr()), capi.c_int_p),
                        C.cast(C.c_void_p(d_A[2].data_ptr()), capi.c_int_p), m, n)
    hw = lib.scs_init_lin_sys_work(C.byref(A), None, capi.dptr(diag_r))
    dw = lib.scs_b200_init_lin_sys_work_device(C.byref(Ad), None, dp(torch.from_numpy(diag_r).cuda()), stream())
    assert hw and dw
    rng = np.random.default_rng(2)
    buf = {}
    for name, host_f, dev_f, nin, nout in (("accum_by_a C2", lib.scs_b200_accum_by_a, lib.scs_b200_accum_by_a_device,
                                            n, m),
                                           ("accum_by_atrans C2", lib.scs_b200_accum_by_atrans,
                                            lib.scs_b200_accum_by_atrans_device, m, n)):
        x = rng.standard_normal(nin)
        d_x = torch.from_numpy(x).cuda()

        def step(i, x=x, d_x=d_x, nout=nout, host_f=host_f, dev_f=dev_f):
            buf["h"] = np.empty(nout)
            buf["d"] = torch.empty(nout, dtype=torch.float64, device="cuda")
            return (lambda: host_f(hw, capi.dptr(x), capi.dptr(buf["h"]), 0),
                    lambda: dev_f(dw, dp(d_x), dp(buf["d"]), 0, stream()),
                    lambda: same(buf["h"], buf["d"]))
        b.run(name, step)

    rhs = rng.standard_normal(n + m)
    sol = rhs.copy()
    assert lib.scs_solve_lin_sys(hw, capi.dptr(sol), None, 1e-4) == 0
    warm = sol[:n] + 1e-3 * rng.standard_normal(n)
    rhs2 = rhs + 1e-3 * rng.standard_normal(n + m)
    d_rhs2, d_warm = torch.from_numpy(rhs2).cuda(), torch.from_numpy(warm).cuda()
    its = []

    def step_solve(i):
        buf["h"], buf["d"] = rhs2.copy(), d_rhs2.clone()

        def dev():
            lib.scs_b200_solve_lin_sys_device(dw, dp(buf["d"]), dp(d_warm), 1e-4, stream())
            its.append((lib.scs_b200_linsys_last_cg_its(hw), lib.scs_b200_linsys_last_cg_its(dw)))
        return (lambda: lib.scs_solve_lin_sys(hw, capi.dptr(buf["h"]), capi.dptr(warm), 1e-4), dev,
                lambda: same(buf["h"], buf["d"]) and its[-1][0] == its[-1][1])
    b.run("KKT solve C2, warm, tol 1e-4", step_solve)
    b.rows["KKT solve C2, warm, tol 1e-4"]["cg_its"] = its[-1][0]
    lib.scs_free_lin_sys_work(hw)
    lib.scs_free_lin_sys_work(dw)

    dim = n + m + 1
    ha = lib.scs_b200_aa_init(dim, 10, 10, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
    da = lib.scs_b200_aa_init(dim, 10, 10, 1, 1e-8, 1.0, 1.0, 1e10, 5, 0)
    assert ha and da
    g = torch.Generator(device="cuda").manual_seed(3)
    decay = torch.rand(dim, dtype=torch.float64, device="cuda", generator=g) * 0.7 + 0.2
    shift = torch.randn(dim, dtype=torch.float64, device="cuda", generator=g)
    state = {"x": torch.zeros(dim, dtype=torch.float64, device="cuda")}
    norms = []

    def step_aa(i):
        x = state["x"]
        f = decay * x + shift  # one application of the contraction, on the device
        buf["xh"], buf["h"], buf["d"] = x.cpu().numpy(), f.cpu().numpy(), f

        def dev():
            norms.append(lib.scs_b200_aa_apply_device(da, dp(buf["d"]), dp(x), stream()))

        def check():
            ok = same(buf["h"], buf["d"]) and norms[-1] == buf["nh"]
            state["x"] = buf["d"]
            return ok

        def host():
            buf["nh"] = lib.scs_b200_aa_apply(ha, capi.dptr(buf["h"]), capi.dptr(buf["xh"]))
        return host, dev, check
    b.run("aa_apply C2 dimension, memory 10", step_aa)
    accepted = lib.scs_b200_aa_get_stats(da).n_accept
    b.rows["aa_apply C2 dimension, memory 10"]["accepted"] = accepted
    lib.scs_b200_aa_finish(ha)
    lib.scs_b200_aa_finish(da)
    print(json.dumps({"card": card(), "calls": a.calls, "warmup": a.warmup, "operators": b.rows}))


if __name__ == "__main__":
    main()

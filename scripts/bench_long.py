"""The DLONG library (64-bit scs_int) against the int library on the C2 workload (random sparse SOCP n = 1e6,
m = 3e6, nnz = 1e7; scs_b200/problems.py config("C2"), seed 1234), end to end through scs().

Prints the card's name and power limit first. Then --runs alternating runs per width (int, long, int, long, ...),
each a cold scs() of exactly --iters ADMM iterations (eps = 0, SCS defaults otherwise), and for each the setup time
ScsInfo.setup_time (for the DLONG library: the 8-byte index upload and the device narrowing pass included) and the
solve throughput ScsInfo.iter / ScsInfo.solve_time. After the narrowing both widths run the same kernels on the same
int32 arrays: x, y and s of every run must be bit-identical, which the script checks. The last line is one JSON
record of the medians.

usage: python scripts/bench_long.py [--runs 3] [--iters 200] [--scale 1.0]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi, problems  # noqa: E402


def run(long, hp, iters):
    T = capi.abi(long)
    lib = capi.load(long=long)
    st = capi.default_settings(lib, long=long, verbose=0, max_iters=iters, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = T.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = T.ScsInfo()
    lib.scs(C.byref(hp.data), C.byref(hp.cone), C.byref(st), C.byref(sol), C.byref(info))
    if info.iter != iters:
        raise SystemExit(f"{'long' if long else 'int'}: ran {info.iter} iterations, not {iters}: {info.status}")
    return {"setup_ms": info.setup_time, "solve_ms": info.solve_time, "it_per_s": 1e3 * info.iter / info.solve_time,
            "xys": (x, y, s)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--scale", type=float, default=1.0)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    card = card[0] if card else "unknown"
    print(f"card: {card}")
    if not capi.load().scs_b200_device_ok():
        raise SystemExit("no usable sm_90 device")
    prob = problems.config("C2", scale=a.scale, seed=1234)
    hps = {long: capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"], long=long) for long in (False, True)}
    print(f"C2 at scale {a.scale}: n = {hps[False].n}, m = {hps[False].m}, nnz = {len(hps[False].Ax)}; "
          f"{a.iters} iterations per run")
    res = {False: [], True: []}
    first = None
    for r in range(a.runs):
        for long in (False, True):
            out = run(long, hps[long], a.iters)
            xys = out.pop("xys")
            if first is None:
                first = xys
            identical = all(np.array_equal(u.view(np.uint64), v.view(np.uint64)) for u, v in zip(first, xys))
            if not identical:
                raise SystemExit(f"run {r} ({'long' if long else 'int'}): x, y, s differ from the first run")
            res[long].append(out)
            print(f"run {r} {'long' if long else 'int ':4s}: setup {out['setup_ms']:9.1f} ms, solve "
                  f"{out['solve_ms']:9.1f} ms, {out['it_per_s']:7.2f} it/s, x y s bit-identical to the first run")
    med = {("long" if long else "int"): {k: float(np.median([o[k] for o in res[long]])) for k in res[long][0]}
           for long in (False, True)}
    spread = {("long" if long else "int"): [min(o["it_per_s"] for o in res[long]), max(o["it_per_s"] for o in res[long])]
              for long in (False, True)}
    print(json.dumps({"card": card, "workload": "C2", "scale": a.scale, "iters": a.iters, "runs": a.runs,
                      "median": med, "it_per_s_range": spread, "bit_identical": True}))


if __name__ == "__main__":
    main()

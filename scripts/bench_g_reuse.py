"""A warm re-solve of the C2 problem (scs_b200/problems.py config("C2")) with and without the reuse of g.

Each arm runs in a process of its own, which reads the switch from its environment: SCS_B200_G_REUSE=1 (the default,
g is reused when A, P, b, c and the scale are unchanged) or SCS_B200_G_REUSE=0 (every scs_solve re-solves g, as the
reference does). In each process: scs_init, a cold solve of `--iters` iterations with eps = 0, then the timed warm
solve of `--iters` more. The arms alternate over `--runs` runs. Prints one JSON line with every run's solve time, CG
iterations and linear-system solves of the timed solve, the card and its power limit, and whether the two arms
returned the same bits.

    python scripts/bench_g_reuse.py [--scale 1.0] [--iters 200] [--runs 3]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(scale, iters):
    from scs_b200 import capi, problems
    lib = capi.load()
    prob = problems.config("C2", scale)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(lib, verbose=0, max_iters=iters, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    if not w:
        raise SystemExit("scs_init failed")
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 0)
    lib.scs_solve(w, C.byref(sol), C.byref(info), 1)  # timed: solve_time is the library's own clock
    stats = capi.ScsB200Stats()
    lib.scs_b200_get_stats(w, C.byref(stats))
    lib.scs_finish(w)
    digest = hashlib.sha256(b"".join(a.tobytes() for a in (x, y, s)) +
                            np.array([info.pobj, info.dobj, info.res_pri, info.res_dual, info.gap, info.scale])
                            .tobytes()).hexdigest()[:16]
    print("RESULT " + json.dumps({"reuse": lib.scs_b200_g_reuse(), "solve_ms": info.solve_time,
                                  "lin_sys_ms": info.lin_sys_time, "cg_iters": stats.cg_iters,
                                  "lin_sys_solves": stats.lin_sys_solves, "iters": info.iter, "digest": digest}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_g_reuse.py needs the H100; there is no CPU measurement")
    from bench_device_data import card
    runs = {"1": [], "0": []}
    for _ in range(a.runs):
        for arm in ("1", "0"):
            env = dict(os.environ, SCS_B200_G_REUSE=arm, SCS_G_REUSE_CHILD=json.dumps([a.scale, a.iters]))
            p = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True)
            lines = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
            if p.returncode != 0 or not lines:
                raise SystemExit(f"arm SCS_B200_G_REUSE={arm} failed: {p.stderr[-800:]}")
            runs[arm].append(json.loads(lines[0][len("RESULT "):]))
    on, off = runs["1"], runs["0"]
    print(json.dumps({"card": card(), "problem": f"C2 at scale {a.scale}", "window": f"warm solve of {a.iters} "
                      f"iterations after a cold solve of {a.iters}", "reuse": on, "no_reuse": off,
                      "median_solve_ms": {"reuse": float(np.median([r["solve_ms"] for r in on])),
                                          "no_reuse": float(np.median([r["solve_ms"] for r in off]))},
                      "same_bits": len({r["digest"] for r in on + off}) == 1}))


if __name__ == "__main__":
    if os.environ.get("SCS_G_REUSE_CHILD"):
        child(*json.loads(os.environ["SCS_G_REUSE_CHILD"]))
    else:
        main()

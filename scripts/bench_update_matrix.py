"""A fresh device-door init against a matrix update on the C2 problem (scs_b200/problems.py config("C2")).

Arms, alternated over `--runs` runs: (a) torch_solver.SCS built on A2; (b) a solver built on A (outside the timing),
then update(A=A2). Each arm ends in torch.cuda.synchronize(). Then `--iters` cold iterations with eps = 0 on both,
checked to be bit-identical. A2 has A's pattern and values times (1 + 0.1 N(0, 1)). Prints one JSON line with the
medians, the spread, the card and its power limit. SCS_B200_SETUP_TIMING=1 prints where the update's time goes.

    python scripts/bench_update_matrix.py [--scale 1.0] [--iters 200] [--runs 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_device_data import card  # noqa: E402
from scs_b200 import problems, torch_solver  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update_matrix.py needs the H100; there is no CPU measurement")
    prob = problems.config("C2", a.scale)
    dev = torch.device("cuda", torch_solver._library_device())
    Ax, Ai, Ap, shape = prob["A"]
    Ax2 = Ax * (1 + 0.1 * np.random.default_rng(7).standard_normal(len(Ax)))
    p, i = torch.tensor(Ap, dtype=torch.int32, device=dev), torch.tensor(Ai, dtype=torch.int32, device=dev)
    A = torch.sparse_csc_tensor(p, i, torch.tensor(Ax, device=dev), size=shape)
    A2 = torch.sparse_csc_tensor(p, i, torch.tensor(Ax2, device=dev), size=shape)
    b, c = torch.tensor(prob["b"], device=dev), torch.tensor(prob["c"], device=dev)
    st = dict(verbose=0, max_iters=a.iters, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)

    def fresh():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s = torch_solver.SCS({"A": A2, "b": b, "c": c}, prob["cone"], **st)
        torch.cuda.synchronize()
        return s, time.perf_counter() - t0

    def updated():
        s = torch_solver.SCS({"A": A, "b": b, "c": c}, prob["cone"], **st)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.update(A=A2)
        torch.cuda.synchronize()
        return s, time.perf_counter() - t0

    for arm in (fresh, updated):  # warm-up: module load, allocator pool
        arm()[0].close()
    times = {"init_s": [], "update_s": []}
    same = True
    for _ in range(a.runs):
        s1, t1 = fresh()
        r1 = s1.solve(warm_start=False)
        s1.close()
        s2, t2 = updated()
        r2 = s2.solve(warm_start=False)
        s2.close()
        times["init_s"].append(t1)
        times["update_s"].append(t2)
        same &= all(torch.equal(r1[k].view(torch.int64), r2[k].view(torch.int64)) for k in "xys")
    print(json.dumps({"card": card(), "problem": {"m": shape[0], "n": shape[1], "nnz": int(len(Ax))},
                      "iters": a.iters, "runs": times,
                      "median": {k: float(np.median(v)) for k, v in times.items()},
                      "spread": {k: float(np.max(v) - np.min(v)) for k, v in times.items()},
                      "bit_identical": bool(same)}))


if __name__ == "__main__":
    main()

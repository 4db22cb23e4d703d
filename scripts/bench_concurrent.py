"""Throughput of independent solves on several host threads of one process (include/scs_b200.h, "Threading").

Three workloads of distinct problems, each with its own seed: 64 of C1 size, 32 of C2 x 0.01 and 8 of C2 x 0.1
(scs_b200/problems.py). Each workload is solved serially and on 2, 4 and 8 threads (scs_init -> scs_solve ->
scs_finish per problem on host buffers, default settings), the arms alternating, three repeats each. Printed per arm:
solves per second (median and range over the repeats), the share of KKT solves that ran the fused K3 + K4 kernel
(scs_b200_cg_k34_paths), and whether every solution is bit-identical to the serial arm's. The card's name and power
limit are read in the same run.

    python scripts/bench_concurrent.py [--repeats 3] [--threads 2 4 8] [--max-iters N] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scs_b200 import capi, problems  # noqa: E402

WORKLOADS = (("C1", "C1", 1.0, 64), ("C2x0.01", "C2", 0.01, 32), ("C2x0.1", "C2", 0.1, 8))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def solve(lib, hp, settings):
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(settings))
    if not w:
        raise RuntimeError("scs_init failed")
    try:
        x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
        info = capi.ScsInfo()
        lib.scs_solve(w, C.byref(capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))), C.byref(info), 0)
        paths = (C.c_longlong * 2)()
        lib.scs_b200_cg_k34_paths(w, paths)
    finally:
        lib.scs_finish(w)
    return x.tobytes() + y.tobytes() + s.tobytes(), paths[0], paths[1]


def run_arm(lib, hps, settings, threads):
    t0 = time.perf_counter()
    if threads == 1:
        out = [solve(lib, hp, settings) for hp in hps]
    else:
        with ThreadPoolExecutor(max_workers=threads) as ex:
            out = list(ex.map(lambda hp: solve(lib, hp, settings), hps))
    return len(hps) / (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--threads", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--max-iters", type=int, default=None, help="cap on ADMM iterations (default: SCS's)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    lib = capi.load()
    if not lib.scs_b200_device_ok():
        raise SystemExit("no usable sm_90 device")
    over = {"verbose": 0}
    if args.max_iters:
        over["max_iters"] = args.max_iters
    settings = capi.default_settings(lib, **over)
    print(f"card: {card()}", flush=True)
    arms = [1] + list(args.threads)
    report = {"card": card(), "workloads": {}}
    for label, name, scale, count in WORKLOADS:
        hps = []
        for i in range(count):
            prob = problems.config(name, scale=scale, seed=1000 + i)
            hps.append(capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"]))
        run_arm(lib, hps[:2], settings, 1)  # warm-up: module load and the first blocks of the allocator
        rates = {a: [] for a in arms}
        fused = {a: [0, 0] for a in arms}
        identical = {a: True for a in arms}
        reference = None
        for _ in range(args.repeats):
            for a in arms:
                rate, out = run_arm(lib, hps, settings, a)
                print(f"  {label} threads={a}: {rate:.2f} solves/s", flush=True)
                rates[a].append(rate)
                for _, f, p in out:
                    fused[a][0] += f
                    fused[a][1] += p
                bits = [o[0] for o in out]
                if reference is None:
                    reference = bits
                identical[a] = identical[a] and bits == reference
        print(f"\n{label}: {count} problems, {args.repeats} repeats")
        print(f"  {'threads':>7} {'solves/s median':>16} {'range':>21} {'fused share':>12} {'bit-identical':>14}")
        rows = {}
        for a in arms:
            r = sorted(rates[a])
            share = fused[a][0] / max(1, fused[a][0] + fused[a][1])
            print(f"  {a:>7} {np.median(r):>16.2f} {f'[{r[0]:.2f}, {r[-1]:.2f}]':>21} {share:>12.3f} "
                  f"{str(identical[a]):>14}", flush=True)
            rows[a] = {"median": float(np.median(r)), "min": r[0], "max": r[-1], "fused_share": share,
                       "bit_identical": identical[a]}
        report["workloads"][label] = rows
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()

"""Host API against device API on the C2 problem (n = 1e6, m = 3e6, nnz = 1e7; scs_b200/problems.py config()).

For each API, three alternating runs of: init, K = 200 ADMM iterations, and the whole call including the copies in
and out (scs_init + scs_solve + scs_finish on numpy arrays, against scs_b200_init_device + scs_b200_solve_device +
scs_finish on CUDA tensors already resident on the GPU). Checks that both return the same solution bit for bit, and
reads the card's name and power limit in the same run. Prints one JSON line.

    python scripts/bench_device_data.py [--scale 1.0] [--iters 200] [--runs 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi, problems, torch_solver  # noqa: E402


def card():
    """name and power limit of the library's device. nvidia-smi lists every GPU of the host whatever
    CUDA_VISIBLE_DEVICES says, so a CUDA ordinal cannot index its list: the device is found by its UUID, else by its
    PCI bus id (either may read N/A in a virtual machine), else it must be the only GPU listed."""
    p = torch.cuda.get_device_properties(torch_solver._library_device())
    keys = {f"gpu-{p.uuid}".lower(), f"{p.pci_domain_id:08x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0".lower()}
    out = subprocess.run(["nvidia-smi", "--query-gpu=uuid,pci.bus_id,name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()
    rows = [[f.strip() for f in line.split(",")] for line in out]
    for r in rows:
        if r[0].lower() in keys or r[1].lower() in keys:
            return f"{r[2]}, {r[3]}"
    if len(rows) == 1:
        return f"{rows[0][2]}, {rows[0][3]}"
    raise RuntimeError(f"cannot tell which of nvidia-smi's {len(rows)} GPUs is the library's device")


def host_run(lib, hp, iters):
    st = capi.default_settings(lib, verbose=0, max_iters=iters, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    t0 = time.perf_counter()
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    t1 = time.perf_counter()
    sol, info = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s)), capi.ScsInfo()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 0)
    t2 = time.perf_counter()
    lib.scs_finish(w)
    t3 = time.perf_counter()
    return {"init_s": t1 - t0, "solve_s": t2 - t1, "whole_s": t3 - t0}, (x, y, s)


def device_run(data, cone, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    solver = torch_solver.SCS(data, cone, verbose=0, max_iters=iters, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    r = solver.solve(warm_start=False)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    solver.close()
    t3 = time.perf_counter()
    return {"init_s": t1 - t0, "solve_s": t2 - t1, "whole_s": t3 - t0}, (r["x"], r["y"], r["s"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_device_data.py needs the H100; there is no CPU measurement")
    prob = problems.config("C2", a.scale)
    lib = capi.load()
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    dev = torch.device("cuda", torch_solver._library_device())
    Ax, Ai, Ap, shape = prob["A"]
    data = {"A": torch.sparse_csc_tensor(torch.tensor(Ap, dtype=torch.int32), torch.tensor(Ai, dtype=torch.int32),
                                         torch.tensor(Ax, dtype=torch.float64), size=shape, device=dev),
            "b": torch.tensor(prob["b"], device=dev), "c": torch.tensor(prob["c"], device=dev)}
    host_run(lib, hp, 3)  # warm-up of both paths: module load, allocator pool
    device_run(data, prob["cone"], 3)
    runs = {"host": [], "device": []}
    same = True
    for _ in range(a.runs):
        th, (xh, yh, sh) = host_run(lib, hp, a.iters)
        td, (xd, yd, sd) = device_run(data, prob["cone"], a.iters)
        runs["host"].append(th)
        runs["device"].append(td)
        same &= all(u.tobytes() == v.cpu().numpy().tobytes() for u, v in ((xh, xd), (yh, yd), (sh, sd)))
    med = {k: {f: float(np.median([r[f] for r in v])) for f in ("init_s", "solve_s", "whole_s")}
           for k, v in runs.items()}
    print(json.dumps({"card": card(), "problem": {"m": hp.m, "n": hp.n, "nnz": int(len(Ax))}, "iters": a.iters,
                      "runs": runs, "median": med, "bit_identical": bool(same)}))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench.py -- ADMM iterations/sec and time-to-eps of the SCS hot path on H100 (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config C2] [--scale f]
                  [--dump-outputs DIR]

A "step" is ONE ADMM iteration (normalise v -> indirect KKT solve by device PCG -> cone projection -> dual update,
with Anderson acceleration every 10th step and the residual / scale check every 25th) on the synthetic workload
named by `--config` (default C2: random sparse SOCP n=1e6, m=3e6, nnz=1e7, 50 SOC cones, fp64), run through the
public C ABI (scs_init / scs_solve) of scs_b200/libscs_b200.so.

BOTH ARMS TIME THE SAME WINDOW: the first K ADMM iterations of a COLD-STARTED solve with default settings and
eps = 0 (so exactly K iterations run) -- identical algorithmic work, identical `config` dict.

  value  : K / (device-resident cold solve of K iterations), problem already resident in HBM, after W untimed
           warm-up iterations on the same workspace.  CUDA events bracket the timed region; the wall clock of the
           same region is printed too (they agree: the solve synchronises at its end).
  e2e    : K / wall time of the whole host-buffer call scs() = scs_init (H2D of A, b, c; transpose, SpMV plans,
           equilibration) + scs_solve(K) + D2H of (x, y, s) + scs_finish.
  time_to_eps_1e-4 : the other half of BASELINE's metric -- a separate default-settings solve to eps_abs =
           eps_rel = 1e-4 (status, iterations, setup and solve seconds, residuals); the CPU reference needs hours
           for this, its figure is an extrapolation from its measured iterations/s and labelled so.
  roofline: the kernels of the CG loop AS THEY RUN IN THE SOLVE (spmv_flag_kernel<POST_MUL> on the solver's own p,
           <POST_FMA_DOT>+alpha hook on its tmp, k_cg_update, k_cg_pupdate), each bracketed by CUDA events inside
           genuine CG iterations; consecutive kernels stream 2 x 124 MB of matrix data, more than the 50 MB L2.
  parity : the gate of SURVEY 8(d) measured in this very run: our first ADMM iteration against the reference's
           (run beside the cpu_baseline sample), relative differences of x, y, s and the ScsInfo residuals.
  cpu_baseline: the UNMODIFIED reference CPU-indirect solver (oracle/_ref, OpenMP build) on a bounded sample (the
           first 3 iterations) of the same workload.

--impl reference times that same reference solver for the same K cold iterations as the whole arm.
--dump-outputs DIR writes what the timed solve returned in its last step -- x, y, s of the K-th iteration -- as
DIR/{x,y,s}.npy (float64) and its ScsInfo scalars as DIR/info.npy; the inputs are fixed by --config, --scale and
--seed, so two builds can be compared output for output. Beyond 64 MB in all, each vector is replaced by a fixed
seeded sample (DIR/<name>_index.npy holds the sampled positions).
N > 1: one process per GPU, ONE cooperative solve of the same workload (strong scaling): A is row-sharded across the
ranks; the CG runs in the sharded-x push mode over NVLink peer memory (DESIGN.md section 6) and the line carries the
per-phase timeline of one CG iteration (`cg_phases_us`, max over ranks).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CONFIG_DESC = {
    "C1": "random sparse SOCP n=1e3 m=4e3 nnz=3.2e4 (reference demo size)",
    "C2": "random sparse SOCP n=1e6 m=3e6 nnz=1e7, 50 SOC cones, fp64",
    "C3": "random sparse LP (box+pos cone) n=5e6 m=5e6 nnz=5e7",
    "C4": "SDP 200 PSD(100) + 1e5 linear rows, n=1e5, nnz=2e7",
    "C5": "mixed SOCP+SDP n=2e6 m=6e6 nnz=3e7, AA mem 10",
}


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons during the timed region (read-only queries)."""

    def __init__(self, gpu_index):
        super().__init__(daemon=True)
        self.gpu = gpu_index
        self.stop_flag = threading.Event()
        self.rows = []

    def run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            p = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}",
                                  "--format=csv,noheader,nounits", "-lms", "100"],
                                 stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            return
        while not self.stop_flag.is_set():
            line = p.stdout.readline()
            if not line:
                break
            self.rows.append([t.strip() for t in line.split(",")])
        p.terminate()

    def summary(self):
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx.append(float(r[1]))
            except (ValueError, IndexError):
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(max(mx)), "reasons": sorted(reasons),
                "samples": len(sm)}


def measured_peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "MEASURED_PEAKS.json hbm_gbs (measured)"
        except Exception:
            pass
    return 3350.0, "H100 SXM data-sheet HBM3 bandwidth 3.35 TB/s (not measured)"


def workload_config(name, scale, n, m, nnz, steps):
    """The `config` dict: identical in both arms (same generator, seed, sizes, settings and iteration window)."""
    return {"workload": f"{name}: {CONFIG_DESC.get(name, '')}", "scale": scale, "n": int(n), "m": int(m),
            "nnz": int(nnz), "generator": "scs_b200/problems.py config(), seed 1234",
            "settings": "SCS defaults (AA mem 10 / interval 10, adaptive scale, normalize), eps = 0 so exactly K "
                        "iterations run",
            "window": f"ADMM iterations 1..{int(steps)} of a cold-started solve",
            "l2": "working set (A and A' = 2 x 124 MB at C2, streamed alternately, + vectors) exceeds the 50 MB L2"}


def build_problem(name, scale, seed):
    from scs_b200 import problems
    t0 = time.time()
    prob = problems.config(name, scale=scale, seed=seed)
    return prob, time.time() - t0


def run_solver(lib, capi, hp, settings_over, w=None, warm=False, sol_arrays=None):
    """scs_init (if w is None) + scs_solve; returns (w, info, sol arrays)."""
    st = capi.default_settings(lib, verbose=0, **settings_over)
    if w is None:
        w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
        if not w:
            raise RuntimeError("scs_init failed")
    if sol_arrays is None:
        sol_arrays = (np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m))
    sol = capi.ScsSolution(*(capi.dptr(a) for a in sol_arrays))
    info = capi.ScsInfo()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 1 if warm else 0)
    return w, info, sol_arrays


def ref_lib_path(omp=True):
    d = os.path.join(ROOT, "oracle", "_ref")
    p = os.path.join(d, "libscsindir_ref_omp.so" if omp else "libscsindir_ref.so")
    return p if os.path.exists(p) else None


def _reference_worker():
    """Child process: run the UNMODIFIED reference for a fixed number of iterations with the thread
    environment given by the parent (thread counts must be set before the libraries load)."""
    from scs_b200 import capi
    spec = json.loads(os.environ["SCS_REF_WORKER"])
    prob, _ = build_problem(spec["config"], spec["scale"], spec["seed"])
    ref = capi.load_reference(spec["lib"])
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(ref, verbose=0, max_iters=int(spec["iters"]), eps_abs=0.0, eps_rel=0.0,
                               eps_infeas=0.0)
    x, y, s = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
    sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(s))
    info = capi.ScsInfo()
    t0 = time.time()
    w = ref.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    t_init = time.time() - t0
    if spec.get("dump"):
        # parity sample for bench.py's "parity" gate: the FIRST iteration of a cold solve (the only window two correct
        # implementations reproduce sharply, tests/test_reference_reproducibility_cpu.py); untimed
        st1 = capi.default_settings(ref, verbose=0, max_iters=1, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)
        w1 = ref.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st1))
        x1, y1, s1 = np.zeros(hp.n), np.zeros(hp.m), np.zeros(hp.m)
        sol1 = capi.ScsSolution(capi.dptr(x1), capi.dptr(y1), capi.dptr(s1))
        info1 = capi.ScsInfo()
        ref.scs_solve(w1, C.byref(sol1), C.byref(info1), 0)
        ref.scs_finish(w1)
        np.savez(spec["dump"], x=x1, y=y1, s=s1, info=np.array([info1.pobj, info1.dobj, info1.res_pri, info1.res_dual,
                                                                 info1.gap]))
    t0 = time.time()
    ref.scs_solve(w, C.byref(sol), C.byref(info), 0)
    t_solve = time.time() - t0
    ref.scs_finish(w)
    print("REFRESULT " + json.dumps({
        "iters": int(info.iter), "solve_s": t_solve, "init_s": t_init, "its_per_s": info.iter / t_solve,
        "e2e_its_per_s": info.iter / (t_solve + t_init), "lin_sys_ms": info.lin_sys_time,
        "cone_ms": info.cone_time, "accel_ms": info.accel_time, "n": prob["n"], "m": prob["m"],
        "nnz": prob["nnz"]}))


def run_reference(args, iters, lib, omp_threads, blas_threads=1, dump=None):
    env = dict(os.environ)
    env["OMP_NUM_THREADS"] = str(omp_threads)
    env["OPENBLAS_NUM_THREADS"] = str(blas_threads)
    env["SCS_REF_WORKER"] = json.dumps({"config": args.config, "scale": args.scale, "seed": args.seed,
                                        "iters": int(iters), "lib": lib, "dump": dump})
    env.pop("RANK", None)
    p = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, capture_output=True, text=True)
    for line in p.stdout.splitlines():
        if line.startswith("REFRESULT "):
            r = json.loads(line[len("REFRESULT "):])
            r.update({"lib": os.path.basename(lib), "omp_threads": omp_threads, "blas_threads": blas_threads})
            return r
    raise RuntimeError("reference worker failed: " + p.stderr[-500:])


def best_reference(args, iters, probe_iters=2, dump=None):
    """The reference with 'all the host threads it can use'. Only accum_by_atrans is parallel in the
    reference (OpenMP, linsys/scs_matrix.c:174-176); probing 1, 8, 32 and 128 threads on a 128-thread host showed
    32 threads fastest and all 128 hardware threads 6x SLOWER, so the default is min(32, cores) without probing --
    a probe costs minutes at C2 (one reference iteration takes ~10 s).
    SCS_BENCH_PROBE=1 repeats the probe."""
    d = os.path.join(ROOT, "oracle", "_ref")
    plain, omp = os.path.join(d, "libscsindir_ref.so"), os.path.join(d, "libscsindir_ref_omp.so")
    if not os.path.exists(plain):
        return None
    ncores = os.cpu_count() or 1
    if not os.environ.get("SCS_BENCH_PROBE"):
        lib, t = (omp, min(32, ncores)) if os.path.exists(omp) else (plain, 1)
        r = run_reference(args, iters, lib, t, 1, dump=dump)
        r["cores"] = t
        r["probes"] = "not probed (SCS_BENCH_PROBE=1 to probe)"
        return r
    cands = [(plain, 1, 1)]
    if os.path.exists(omp):
        for t in sorted({min(8, ncores), min(32, ncores), ncores}):
            cands.append((omp, t, 1))
    probes = []
    for lib, t, bt in cands:
        try:
            probes.append(run_reference(args, probe_iters, lib, t, bt))
        except RuntimeError:
            pass
    if not probes:
        return None
    best = max(probes, key=lambda r: r["its_per_s"])
    lib = plain if best["lib"] == os.path.basename(plain) else omp
    r = run_reference(args, iters, lib, best["omp_threads"], best["blas_threads"], dump=dump) \
        if (iters > probe_iters or dump) else best
    r["cores"] = best["omp_threads"]
    r["probes"] = [{"lib": q["lib"], "threads": q["omp_threads"], "its_per_s": q["its_per_s"]} for q in probes]
    return r


DUMP_BYTES = 64 << 20


def dump_outputs(d, arrays, info):
    """the timed solve's outputs as float64 .npy files; over DUMP_BYTES, a fixed seeded sample of each vector"""
    os.makedirs(d, exist_ok=True)
    total = sum(a.nbytes for a in arrays.values())
    for name, a in arrays.items():
        if total > DUMP_BYTES:
            k = max(1, int(a.size * (DUMP_BYTES // 2) / total))
            idx = np.sort(np.random.default_rng(len(name)).choice(a.size, min(k, a.size), replace=False))
            np.save(os.path.join(d, f"{name}_index.npy"), idx.astype(np.float64))
            a = a[idx]
        np.save(os.path.join(d, f"{name}.npy"), np.ascontiguousarray(a, dtype=np.float64))
    np.save(os.path.join(d, "info.npy"), np.array([info.iter, info.pobj, info.dobj, info.res_pri, info.res_dual,
                                                   info.gap, info.scale], dtype=np.float64))


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(1.0, float(np.abs(b).max())))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default=os.environ.get("SCS_BENCH_CONFIG", "C2"))
    ap.add_argument("--scale", type=float, default=float(os.environ.get("SCS_BENCH_SCALE", "1.0")))
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-tte", action="store_true", help="skip the time-to-eps solve")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write x, y, s of the timed solve's last step to DIR/*.npy")
    args = ap.parse_args()
    if args.warmup < 3:
        args.warmup = 3
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not os.path.exists(os.path.join(ROOT, "scs_b200", "libscs_b200.so")) and rank == 0 and world == 1:
        import __graft_entry__
        __graft_entry__.build()  # fresh checkout: the built library is git-ignored
    from scs_b200 import capi

    base = {"metric": "ADMM iters/sec", "unit": "iters/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "f64", "data": "synthetic"}

    # ------------------------------------------------------------------ reference arm
    if args.impl == "reference":
        if rank != 0:
            return 0
        # the SAME window as our arm: K cold iterations of the full workload. One reference iteration of C2 takes
        # ~10 s on this pool's hosts (32 OpenMP threads), i.e. ~3.5 min at the driver's K = 20; SCS_BENCH_REF_ITERS
        # caps K for larger requests (the line then says steps_run < steps).
        cap = int(os.environ.get("SCS_BENCH_REF_ITERS", "25"))
        big = args.scale >= 0.5 and args.config != "C1"
        k = max(2, int(min(args.steps, cap)) if big else int(args.steps))
        r = best_reference(args, k)
        if r is None:
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref not built"}))
            return 0
        out = dict(base)
        out.update({
            "impl": "reference", "value": r["its_per_s"], "ms_per_step": 1e3 / r["its_per_s"], "n_gpus": world,
            "steps": int(r["iters"]), "steps_requested": args.steps,
            "config": workload_config(args.config, args.scale, r["n"], r["m"], r["nnz"], args.steps),
            "cpu_baseline": {"value": r["its_per_s"], "unit": "iters/s", "cores": r["cores"], "kind": "reference",
                             "sample": f"{r['iters']} cold ADMM iterations of the unmodified reference CPU-indirect "
                                       f"solver ({r['lib']}, OMP_NUM_THREADS={r['cores']}; thread choice: "
                                       f"{r['probes']}) on the full workload"},
            "e2e": {"value": r["e2e_its_per_s"], "unit": "iters/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0,
            "lin_sys_ms": r["lin_sys_ms"], "cone_ms": r["cone_ms"], "accel_ms": r["accel_ms"],
            "setup_ms": 1e3 * r["init_s"],
        })
        print(json.dumps(out))
        return 0

    # ------------------------------------------------------------------ our arm
    import torch
    import torch.distributed as dist
    os.environ["SCS_B200_DEVICE"] = str(local_rank)
    if world > 1:
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    lib = capi.load()
    if not lib.scs_b200_device_ok():
        raise RuntimeError("scs_b200: no usable sm_90 device (there is no CPU fallback)")
    if world > 1:
        # row-sharded KKT solve: rank 0 creates the NCCL id, torch.distributed carries it
        idbuf = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            raw = C.create_string_buffer(128)
            assert lib.scs_b200_comm_unique_id(raw) == 0
            idbuf.copy_(torch.tensor(list(raw.raw), dtype=torch.uint8))
        dist.broadcast(idbuf, src=0)
        raw = C.create_string_buffer(bytes(idbuf.cpu().tolist()), 128)
        assert lib.scs_b200_comm_init(rank, world, raw) == 0

    # every rank holds the same problem; with N > 1 each keeps only its row block of A on its GPU
    prob, gen_s = build_problem(args.config, args.scale, args.seed)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    n, m, nnz = prob["n"], prob["m"], prob["nnz"]
    eps0 = dict(eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # one untimed short call first: CUDA lazy module loading, cuSOLVER / NCCL handles and the pinned staging
    # buffer are one-time process costs, not part of a solve (the reference arm has no such cold start)
    w0, _, _ = run_solver(lib, capi, hp, dict(max_iters=3, **eps0))
    lib.scs_finish(w0)

    # ---- e2e: whole host-buffer call (init + K cold iterations + finish), copies inside the timed region
    barrier()
    t0 = time.time()
    w, info_e, sols = run_solver(lib, capi, hp, dict(max_iters=args.steps, **eps0))
    t_fin = time.time()
    lib.scs_finish(w)
    torch.cuda.synchronize()
    t_end = time.time()
    e2e_s = t_end - t0
    e2e_parts = {"init_ms": info_e.setup_time, "solve_ms": info_e.solve_time, "finish_ms": 1e3 * (t_end - t_fin),
                 "other_ms (ctypes, result copies)": 1e3 * (t_fin - t0) - info_e.setup_time - info_e.solve_time}
    h2d = nnz * 12 + (n + 1) * 4 + (m + n) * 8          # A (vals+idx+ptr), b, c
    d2h = (n + 2 * m) * 8                                # x, y, s

    # ---- device-resident: init once, W warm-up steps, then exactly K timed steps of a COLD-STARTED solve
    st = capi.default_settings(lib, verbose=0, max_iters=args.warmup, **eps0)
    w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    if not w:
        raise RuntimeError("scs_init failed")
    sol = capi.ScsSolution(*(capi.dptr(a) for a in sols))
    info = capi.ScsInfo()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 0)          # W untimed steps
    assert lib.scs_b200_set_max_iters(w, args.steps) == 0
    sampler = ClockSampler(local_rank)
    sampler.start()
    barrier()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches0 = lib.scs_b200_launch_count()
    t0 = time.time()
    ev0.record()
    lib.scs_solve(w, C.byref(sol), C.byref(info), 0)          # cold start: the same window as the reference arm
    ev1.record()
    barrier()
    wall_s = time.time() - t0
    launches = lib.scs_b200_launch_count() - launches0
    sampler.stop_flag.set()
    stats = capi.ScsB200Stats()
    lib.scs_b200_get_stats(w, C.byref(stats))
    solve_s = info.solve_time / 1e3
    iters = int(info.iter)
    lib.scs_finish(w)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"x": sols[0], "y": sols[1], "s": sols[2]}, info)

    # ---- time to the default stopping criterion eps_abs = eps_rel = 1e-4 (second half of BASELINE's metric):
    # a separate full solve so that the K-step timing above is untouched
    tte = None
    want_tte = not args.no_tte and os.environ.get("SCS_BENCH_TTE", "1") != "0"
    if want_tte:
        t0 = time.time()
        w2, info_t, sol_t = run_solver(lib, capi, hp, dict(max_iters=100000))
        lib.scs_finish(w2)
        tte = {"status": info_t.status.decode(errors="replace"), "iters": int(info_t.iter),
               "solve_s": info_t.solve_time / 1e3, "setup_s": info_t.setup_time / 1e3,
               "wall_s_incl_init_and_copies": time.time() - t0, "pobj": info_t.pobj,
               "known_optimum": prob.get("opt"), "res_pri": info_t.res_pri, "res_dual": info_t.res_dual,
               "gap": info_t.gap, "lin_sys_s": info_t.lin_sys_time / 1e3, "cone_s": info_t.cone_time / 1e3,
               "accel_s": info_t.accel_time / 1e3}
        if world > 1:
            tm = torch.tensor([tte["solve_s"], tte["setup_s"]], device="cuda", dtype=torch.float64)
            dist.all_reduce(tm, op=dist.ReduceOp.MAX)
            tte["solve_s"], tte["setup_s"] = float(tm[0]), float(tm[1])

    # max over ranks / sum of work
    tmax = solve_s
    if world > 1:
        tm = torch.tensor([solve_s, e2e_s], device="cuda", dtype=torch.float64)
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
        tmax, e2e_s = float(tm[0]), float(tm[1])
    value = iters / tmax             # ONE cooperative solve: the job's iterations / slowest rank
    e2e_value = args.steps / e2e_s

    # ---- roofline of the in-loop kernels, timed live with CUDA events inside genuine CG iterations
    roof = None
    extra = {}
    cpu_base = None
    parity = None
    peak, peak_src = measured_peak_gbs()
    if world > 1:
        # per-phase timeline of one sharded CG iteration (all ranks take part: the kernels synchronise through peer
        # flags); max over ranks. Only the sharded-x push mode has a per-kernel breakdown.
        dr = np.empty(n + m + 1)
        z = int(prob["cone"].get("z", 0))
        dr[:n], dr[n:n + z], dr[n + z:] = 1e-6, 1.0 / 100.0, 10.0
        lw = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
        if lw:
            ab = C.c_double(0.0)
            t_it = lib.scs_b200_time_cg_iter(lw, 30, C.byref(ab))
            msv, byv = (C.c_double * 12)(), (C.c_double * 5)()
            rc = lib.scs_b200_time_cg_kernels(lw, capi.dptr(np.concatenate([prob["c"], prob["b"]])), 30, msv, byv)
            tm = torch.tensor([t_it, msv[0], msv[1], msv[2], msv[4]] if rc == 0 else [t_it, 0, 0, 0, 0],
                              device="cuda", dtype=torch.float64)
            dist.all_reduce(tm, op=dist.ReduceOp.MAX)
            extra["cg_iteration_us"] = float(tm[0]) * 1e3
            if rc == 0:
                extra["cg_phases_us"] = {"K1 local rows of A": float(tm[1]) * 1e3,
                                         "K2 local partial of A' + NVLink push + signal": float(tm[2]) * 1e3,
                                         "slice kernel: reduce, 2 scalar exchanges, K3/K4, p push, waits": float(tm[3]) * 1e3,
                                         "iteration with events between the kernels": float(tm[4]) * 1e3,
                                         "inside the slice kernel (rank 0, block 0, last iteration)": {
                                             "reduce slice (waits for rows in flight)": msv[5] * 1e3,
                                             "grid reduction + scalar exchange 1": msv[6] * 1e3,
                                             "K3 on the slice": msv[7] * 1e3,
                                             "grid reduction + scalar exchange 2": msv[8] * 1e3,
                                             "K4 on the slice + p push": msv[9] * 1e3,
                                             "unpack the peers' p slices (waits for elements in flight)": msv[10] * 1e3,
                                             "ticket + control block": msv[11] * 1e3}}
            lib.scs_free_lin_sys_work(lw)
    if world == 1:
        dr = np.empty(n + m + 1)
        z = int(prob["cone"].get("z", 0))
        dr[:n] = 1e-6
        dr[n:n + z] = 1.0 / 100.0
        dr[n + z:n + m] = 10.0
        dr[n + m] = 10.0
        lw = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
        rhs = np.concatenate([prob["c"], prob["b"]])
        ms = (C.c_double * 5)()
        by = (C.c_double * 5)()
        rc = lib.scs_b200_time_cg_kernels(lw, capi.dptr(rhs), 50, ms, by)
        lib.scs_free_lin_sys_work(lw)
        if rc == 0:
            names = ["K1 spmv_flag_kernel<POST_MUL>: tmp = R_y^-1 (A p)  [rows of A, gathers p]",
                     "K2 spmv_flag_kernel<POST_FMA_DOT>+alpha hook: Gp = R_x p + A' tmp, p'Gp  [columns of A, gathers tmp]",
                     "K3 k_cg_update: x += a p, r -= a Gp, z = M r, z'r, |r|_inf, beta",
                     "K4 k_cg_pupdate: p = z + beta p",
                     "one CG iteration (K1..K4, launch gaps included)"]
            rows = [{"kernel": names[k], "ms": ms[k], "alg_bytes": by[k], "achieved": by[k] / ms[k] / 1e6,
                     "frac": by[k] / ms[k] / 1e6 / peak} for k in range(5)]
            dom = max(rows[:4], key=lambda r: r["ms"])
            roof = {"bound": "hbm", "achieved": dom["achieved"], "peak": peak, "unit": "GB/s", "frac": dom["frac"],
                    "kernel": dom["kernel"], "ms_per_launch": dom["ms"], "alg_bytes_per_launch": dom["alg_bytes"],
                    "peak_source": peak_src,
                    "timing": "CUDA events around every launch inside 50 genuine CG iterations on the solver's own "
                              "vectors (rhs = [c; b]); K1 / K2 alternate, so each streams its 124 MB matrix after "
                              "the other's 124 MB passed through the 50 MB L2",
                    "share_of_cg_iteration": dom["ms"] / ms[4]}
            extra["roofline_all"] = rows
        if not args.no_cpu_baseline:
            try:
                k = (3 if args.config != "C1" else 40) if args.scale >= 0.5 else 40
                dump = os.path.join("/tmp", f"scs_bench_ref_{os.getpid()}.npz")
                r = best_reference(args, k, dump=dump)
                if r:
                    cpu_base = {"value": r["its_per_s"], "unit": "iters/s", "cores": r["cores"], "kind": "reference",
                                "sample": f"the first {r['iters']} cold ADMM iterations of the unmodified reference "
                                          f"CPU-indirect solver ({r['lib']}, {r['cores']} threads; thread choice: "
                                          f"{r['probes']}) on the same workload (setup {r['init_s']:.1f}s excluded)"}
                    # parity gate of SURVEY 8(d), measured in this run: our first k iterations vs the reference's
                    if os.path.exists(dump):
                        g = np.load(dump)
                        wq, iq, sq = run_solver(lib, capi, hp, dict(max_iters=1, **eps0))
                        lib.scs_finish(wq)
                        mine = [iq.pobj, iq.dobj, iq.res_pri, iq.res_dual, iq.gap]
                        parity = {"window": "the first ADMM iteration of a cold solve (equilibration, KKT solve at tol "
                                            "1e-12, cone projection, un-normalisation) vs the unmodified reference run "
                                            "on this host, max-norm relative differences; later iterations solve the "
                                            "KKT system only to 0.2 x the residual and are not reproducible even "
                                            "between the reference's own two builds "
                                            "(tests/test_reference_reproducibility_cpu.py)",
                                  "gate": "<= 1e-9 (north star 1e-10; the reference's own build-to-build spread is "
                                          "1e-11 .. 1.5e-10)",
                                  "x": rel_err(sq[0], g["x"]), "y": rel_err(sq[1], g["y"]), "s": rel_err(sq[2], g["s"])}
                        for nm, a, b in zip(("pobj", "dobj", "res_pri", "res_dual", "gap"), mine, g["info"]):
                            parity[nm] = abs(a - b) / max(1.0, abs(b))
                        parity["pass"] = bool(max(parity[k] for k in ("x", "y", "s", "pobj", "dobj", "res_pri",
                                                                         "res_dual", "gap")) <= 1e-9)
                        os.remove(dump)
            except Exception as e:  # the checker must never break the measurement
                cpu_base = {"value": None, "unit": "iters/s", "cores": 0, "kind": "reference", "sample": f"failed: {e}"}

    if rank == 0:
        out = dict(base)
        out.update({
            "value": value, "ms_per_step": 1e3 * tmax / max(iters, 1), "steps": iters,
            "config": workload_config(args.config, args.scale, n, m, nnz, args.steps),
            "parallelism": "1 GPU" if world == 1 else f"{world} GPUs, one cooperative solve: A row-sharded by nnz-balanced "
            "row blocks in both orientations; CG over NVLink peer memory (CUDA IPC) -- " +
            ("sharded-x push mode: the K2 SpMV stores its rows into the owners' inboxes, one slice kernel per rank "
             "does the reduction, both scalar exchanges, K3/K4 and stores the new p slice into every peer"
             if os.environ.get("SCS_B200_SHARD_X", "1") != "0" else
             "replicated x-space: a fused kernel sums the peers' partials in rank order") +
            "; cones, AA and the l-vectors replicated",
            "e2e": {"value": e2e_value, "unit": "iters/s", "h2d_bytes_per_step": h2d / args.steps,
                    "d2h_bytes_per_step": d2h / args.steps, "breakdown": e2e_parts,
                    "note": "whole scs() on host buffers: scs_init (transpose + SpMV plans, H2D, device equilibration) + K cold iterations + D2H; one untimed 3-iteration call ran before (process cold start)"},
            "gpu_launches": int(launches),
            "clocks": sampler.summary(),
            "cg_iters_per_step": stats.cg_iters / max(iters, 1),
            "timed_wall_s": wall_s, "timed_device_event_s": ev0.elapsed_time(ev1) / 1e3,
            "lin_sys_ms": info.lin_sys_time, "cone_ms": info.cone_time, "accel_ms": info.accel_time,
            "info_timers": "CUDA events on the solver's stream (device time per section)",
            "setup_ms": info_e.setup_time, "problem_gen_s": gen_s,
        })
        if tte:
            # the CPU reference needs hours for this: its time is extrapolated from its measured iterations/s
            if cpu_base and cpu_base.get("value"):
                tte["cpu_reference_extrapolated_s"] = tte["iters"] / cpu_base["value"]
                tte["cpu_reference_note"] = "EXTRAPOLATION: our iteration count / the reference's measured iterations/s"
            out["time_to_eps_1e-4"] = tte
        if roof:
            out["roofline"] = roof
        if cpu_base:
            out["cpu_baseline"] = cpu_base
        if parity:
            out["parity"] = parity
        out.update(extra)
        print(json.dumps(out))
    if world > 1:
        lib.scs_b200_comm_finalize()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    if os.environ.get("SCS_REF_WORKER"):
        _reference_worker()
        sys.exit(0)
    sys.exit(main())

"""Regenerates the log-det cone fixtures from the reference's USE_SPECTRAL_CONES build (oracle/spectral.mk,
oracle/logdet.mk). TEST INFRASTRUCTURE ONLY; needs the reference sources (REF, default /root/reference).

  tests/golden/problems/logdet/{exp_design, several_logdet_cones}   the reference's log-det test problems, written by
                                          its own writer from its scs() call
  tests/golden/problems/logdet/dopt_24    a seeded D-optimal design problem (order 24, 200 candidate points), written
                                          by the reference's writer
  tests/golden/problems/logdet/optima.json   their optima (the test problems' `opt`; dopt_24: -log det of the
                                          optimal design, by the multiplicative algorithm with its optimality
                                          certificate; the reference's own objective at eps 1e-7 lies 5e-6 from it)
  tests/golden/logdet_solves.npz          one-iteration x, y, s; the full solve's flag, iterations, objectives and
                                          x, y, s; the
                                          Newton columns of the first CSV trace rows; the iteration counts of ten
                                          full solves with b scaled by 1 + j 1e-15, j = -4 .. 5 (PERTURB), the
                                          spread the reference shows on these problems under rounding-sized changes
  tests/golden/logdet_cones.npz           the reference's _scs_proj_dual_cone answers, with and without r_y, on the
                                          operator inputs of tests/logdet_cases.py, and its log_cone_proj_wrapper
                                          records (status, projection, iter, newton_success, residuals) on the
                                          vector-step inputs, warm-started sequences included; on the operator
                                          inputs, its Newton_stats record after each projection (read from its
                                          ScsConeWork, NEWTON_STATS_OFFSET)

usage: python oracle/make_golden_logdet.py
"""
import csv
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from scs_b200 import capi  # noqa: E402
import logdet_cases  # noqa: E402

REF = os.environ.get("REF", "/root/reference")
OB = "/opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs"
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PROB_DIR = os.path.join(ROOT, "tests", "golden", "problems", "logdet")
PROBLEMS = ["exp_design", "several_logdet_cones", "dopt_24"]
NEWTON_COLS = ["spectral_Newton_iter", "plain_Newton_success", "res_dual_spectral", "res_pri_spectral",
               "comp_spectral"]
CSV_ROWS = 12
PERTURB = [j * 1e-15 for j in range(-4, 6)]
# offset of ScsConeWork.newton_stats in the reference's x86-64 USE_LAPACK USE_SPECTRAL_CONES build (include/cones.h:
# 11 pointers, 2 ints, a pointer, an int + padding, a double, 11 pointers, 4 ints, 3 pointers, 4 pointers, an int +
# padding, 2 pointers)
NEWTON_STATS_OFFSET = 232
PP = C.POINTER


class NewtonStats(C.Structure):
    _fields_ = [("iter", C.c_int), ("newton_success", C.c_int), ("residuals", C.c_double * 3)]


def build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "logdet.mk", "logdet", f"REF={REF}"])


def reference():
    lib = capi.load_reference(os.path.join(REF_DIR, "libscsindir_ref_spectral.so"), spectral=True)
    lib._scs_read_data.restype = C.c_int
    lib._scs_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                   PP(PP(capi.ScsSettings))]
    lib._scs_write_data.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    lib._scs_init_cone.restype = C.c_void_p
    lib._scs_init_cone.argtypes = [PP(capi.ScsConeSpectral), C.c_int]
    lib._scs_proj_dual_cone.restype = C.c_int
    lib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    lib._scs_finish_cone.argtypes = [C.c_void_p]
    lib.log_cone_proj_wrapper.restype = C.c_int
    lib.log_cone_proj_wrapper.argtypes = [C.c_double, C.c_double, capi.c_double_p, capi.c_double_p, C.c_int,
                                          capi.c_double_p, PP(NewtonStats), PP(C.c_bool)]
    return lib


def dopt(order=24, points=200, seed=24):
    """maximise log det(sum_i lam_i a_i a_i') over lam >= 0, sum lam = 1, as SCS data: x = (lam, t), minimise t,
    rows: sum lam = 1 (zero cone), lam >= 0 (lp), (t, 1, sum_i lam_i a_i a_i') in the log-det cone
    {(t, v, X) : t >= -v log det(X / v)}"""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((points, order))
    il, jl = [], []
    for j in range(order):
        for i in range(j, order):
            il.append(i)
            jl.append(j)
    il, jl = np.array(il), np.array(jl)
    scale = np.where(il == jl, 1.0, np.sqrt(2.0))
    svec = a[:, il] * a[:, jl] * scale  # points x order(order+1)/2
    nt = order * (order + 1) // 2
    m, n = 1 + points + 2 + nt, points + 1
    A = np.zeros((m, n))
    A[0, :points] = 1.0
    A[1:1 + points, :points] = -np.eye(points)
    A[1 + points, points] = -1.0
    A[3 + points:, :points] = -svec.T
    b = np.zeros(m)
    b[0] = 1.0
    b[2 + points] = 1.0
    c = np.zeros(n)
    c[points] = 1.0
    cone = {"z": 1, "l": points, "d": [order]}
    return A, b, c, cone


def dopt_optimum(order=24, points=200, seed=24, iters=100000):
    """min -log det(sum_i lam_i a_i a_i') over the simplex by the multiplicative algorithm lam_i <- lam_i g_i / order,
    g_i = a_i' X^-1 a_i. By the Kiefer-Wolfowitz theorem the design is optimal when max_i g_i = order, and
    order log(max_i g_i / order) bounds the objective's distance to the optimum."""
    a = np.random.default_rng(seed).standard_normal((points, order))
    lam = np.full(points, 1.0 / points)
    for _ in range(iters):
        g = np.einsum("ij,jk,ik->i", a, np.linalg.inv((a.T * lam) @ a), a)
        lam *= g / order
    g = np.einsum("ij,jk,ik->i", a, np.linalg.inv((a.T * lam) @ a), a)
    assert order * np.log(g.max() / order) < 1e-12
    return float(-np.linalg.slogdet((a.T * lam) @ a)[1])


def write_dopt(lib, path):
    A, b, c, cone = dopt()
    import scipy.sparse as sp
    Acsc = sp.csc_matrix(A)
    x, i, p = Acsc.data.astype(np.float64), Acsc.indices.astype(np.int32), Acsc.indptr.astype(np.int32)
    mat = capi.ScsMatrix(capi.dptr(x), capi.iptr(i), capi.iptr(p), A.shape[0], A.shape[1])
    d = capi.ScsData(A.shape[0], A.shape[1], C.pointer(mat), None, capi.dptr(b), capi.dptr(c))
    k, keep = capi.make_cone(cone, spectral=True)
    st = capi.ScsSettings()
    lib.scs_set_default_settings(C.byref(st))
    st.eps_abs = st.eps_rel = 1e-7
    st.verbose = 0
    st.write_data_filename = path.encode()
    lib._scs_write_data(C.pointer(d), C.pointer(k), C.pointer(st))


def write_problems(lib):
    os.makedirs(PROB_DIR, exist_ok=True)
    env = dict(os.environ, LD_LIBRARY_PATH=OB)
    with tempfile.TemporaryDirectory() as tmp:  # the test problems write CSV traces into the working directory
        subprocess.check_call([os.path.join(REF_DIR, "logdet_fixtures_ref"), PROB_DIR], env=env, cwd=tmp,
                              stdout=subprocess.DEVNULL)
    write_dopt(lib, os.path.join(PROB_DIR, "dopt_24"))
    optima = {}
    for name in PROBLEMS[:2]:
        src = open(os.path.join(REF, "test", "spectral_cones_problems", name + ".h")).read()
        optima[name] = float(re.search(r"scs_float opt = ([-0-9.eE+]+);", src).group(1))
    optima["dopt_24"] = dopt_optimum()
    return optima


def record_solves(lib, optima):
    out = {}
    for name in PROBLEMS:
        d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
        assert lib._scs_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
        m, n = d.contents.m, d.contents.n
        b = np.ctypeslib.as_array(d.contents.b, (m,))
        b0 = b.copy()

        def run(iters, log=None):
            st = capi.ScsSettings.from_buffer_copy(s.contents)
            st.max_iters, st.verbose = iters, 0
            if log:
                st.log_csv_filename = log.encode()
            x, y, z = np.zeros(n), np.zeros(m), np.zeros(m)
            sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(z))
            info = capi.ScsInfo()
            flag = lib.scs(d, k, C.byref(st), C.byref(sol), C.byref(info))
            return flag, info, x, y, z

        _, _, x, y, z = run(1)
        out[f"{name}/x1"], out[f"{name}/y1"], out[f"{name}/s1"] = x, y, z
        flag, info, x, y, z = run(s.contents.max_iters)
        out[f"{name}/info"] = np.array([flag, info.iter, info.pobj, info.dobj])
        out[f"{name}/xf"], out[f"{name}/yf"], out[f"{name}/sf"] = x, y, z
        # CSV logging recomputes the residuals every iteration, which moves the scale updates: a run of its own
        with tempfile.TemporaryDirectory() as tmp:
            log = os.path.join(tmp, "trace.csv")
            run(CSV_ROWS, log)
            rows = list(csv.DictReader(open(log)))[:CSV_ROWS]
            out[f"{name}/csv"] = np.array([[float(r[c]) for c in NEWTON_COLS] for r in rows])
        spread = []
        for eps in PERTURB:
            b[:] = b0 * (1 + eps)
            flag, info, _, _, _ = run(s.contents.max_iters)
            assert flag == 1, (name, eps, flag)
            spread.append(info.iter)
        b[:] = b0
        out[f"{name}/iters_spread"] = np.array(spread)
        print(name, "iterations", int(out[f"{name}/info"][1]), "under perturbations of b", spread)
    np.savez(os.path.join(ROOT, "tests", "golden", "logdet_solves.npz"), **out)
    with open(os.path.join(PROB_DIR, "optima.json"), "w") as f:
        json.dump(optima, f, indent=1, sort_keys=True)
        f.write("\n")


def proj(lib, cone, x, r_y):
    """the reference's answer and its Newton_stats record (status 0, iter, newton_success, residuals)"""
    k, keep = capi.make_cone(cone, spectral=True)
    cw = lib._scs_init_cone(C.byref(k), len(x))
    assert cw
    out = x.copy()
    ry = None if r_y is None else r_y.copy()
    assert lib._scs_proj_dual_cone(capi.dptr(out), cw, None, capi.dptr(ry)) == 0
    st = NewtonStats.from_address(cw + NEWTON_STATS_OFFSET)
    rec = np.array([0, st.iter, st.newton_success, *st.residuals])
    lib._scs_finish_cone(cw)
    return out, rec


def record_operator(lib):
    out = {}
    names = []
    for name, n, x in logdet_cases.operator_cases():
        names.append(name)
        out[f"{name}/x"] = x
        out[f"{name}/out"], out[f"{name}/rec"] = proj(lib, {"d": [n]}, x, None)
        out[f"{name}/outry"], out[f"{name}/recry"] = proj(lib, {"d": [n]}, x, logdet_cases.r_y(n))
    out["names"] = np.array(names)
    vnames = []
    for name, calls in logdet_cases.vector_cases():
        vnames.append(name)
        n = calls[0][2].size
        proj_buf = np.zeros(n + 2)
        work = np.zeros(22 * n + 122)
        warm = C.c_bool(False)
        stats = NewtonStats()
        for j, (t0, v0, e) in enumerate(calls):
            x0 = e.copy()
            status = lib.log_cone_proj_wrapper(t0, v0, capi.dptr(x0), capi.dptr(proj_buf), n, capi.dptr(work),
                                               C.byref(stats), C.byref(warm))
            out[f"v/{name}/in{j}"] = np.concatenate(([t0, v0], e))
            out[f"v/{name}/proj{j}"] = proj_buf.copy()
            out[f"v/{name}/rec{j}"] = np.array([status, stats.iter, stats.newton_success, *stats.residuals])
    out["vnames"] = np.array(vnames)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "logdet_cones.npz"), **out)


if __name__ == "__main__":
    build()
    lib = reference()
    optima = write_problems(lib)
    record_solves(lib, optima)
    record_operator(lib)
    print("log-det fixtures written")

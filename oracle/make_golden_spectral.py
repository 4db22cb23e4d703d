"""Regenerates the spectral-cone fixtures from the reference's USE_SPECTRAL_CONES build (oracle/spectral.mk).
TEST INFRASTRUCTURE ONLY; needs the reference sources (REF, default /root/reference) to build oracle/_ref/.

  tests/golden/problems/spectral/<name>   SCS problem files of the reference's spectral test problems that avoid the
                                          log-det cone, written by the reference's own writer from its scs() call
  tests/golden/problems/spectral/optima.json   their known optima (the `opt` of each problem)
  tests/golden/spectral_solves.npz        the reference's answers on those files: one-iteration x, y, s; the full
                                          solve's iteration count, status and objective
  tests/golden/spectral_cones.npz         the reference's _scs_proj_dual_cone answers, with and without r_y, on the
                                          seeded inputs of tests/spectral_cases.py (long answers sampled)

usage: python oracle/make_golden_spectral.py
"""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from scs_b200 import capi  # noqa: E402
import spectral_cases  # noqa: E402

REF = os.environ.get("REF", "/root/reference")
OB = "/opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs"
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
PROB_DIR = os.path.join(ROOT, "tests", "golden", "problems", "spectral")
PROBLEMS = ["test_ell1_cone", "test_ell1_and_nuc", "robust_pca", "several_nuc_cone", "several_sum_largest",
            "graph_partitioning"]
PP = C.POINTER


def build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "spectral.mk", f"REF={REF}"])


def write_problems():
    os.makedirs(PROB_DIR, exist_ok=True)
    env = dict(os.environ, LD_LIBRARY_PATH=OB)
    subprocess.check_call([os.path.join(REF_DIR, "spectral_fixtures_ref"), PROB_DIR], env=env,
                          stdout=subprocess.DEVNULL)
    optima = {}
    for name in PROBLEMS:
        src = open(os.path.join(REF, "test", "spectral_cones_problems", name + ".h")).read()
        optima[name] = float(re.search(r"scs_float opt = ([-0-9.eE+]+);", src).group(1))
    with open(os.path.join(PROB_DIR, "optima.json"), "w") as f:
        json.dump(optima, f, indent=1, sort_keys=True)
        f.write("\n")


def reference():
    lib = capi.load_reference(os.path.join(REF_DIR, "libscsindir_ref_spectral.so"), spectral=True)
    lib._scs_read_data.restype = C.c_int
    lib._scs_read_data.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)),
                                   PP(PP(capi.ScsSettings))]
    lib._scs_init_cone.restype = C.c_void_p
    lib._scs_init_cone.argtypes = [PP(capi.ScsConeSpectral), C.c_int]
    lib._scs_proj_dual_cone.restype = C.c_int
    lib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    lib._scs_finish_cone.argtypes = [C.c_void_p]
    return lib


def record_solves(lib):
    out = {}
    for name in PROBLEMS:
        d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
        assert lib._scs_read_data(os.path.join(PROB_DIR, name).encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
        m, n = d.contents.m, d.contents.n
        for tag, iters in (("one", 1), ("full", s.contents.max_iters)):
            st = capi.ScsSettings.from_buffer_copy(s.contents)
            st.max_iters, st.verbose = iters, 0
            x, y, z = np.zeros(n), np.zeros(m), np.zeros(m)
            sol = capi.ScsSolution(capi.dptr(x), capi.dptr(y), capi.dptr(z))
            info = capi.ScsInfo()
            flag = lib.scs(d, k, C.byref(st), C.byref(sol), C.byref(info))
            if tag == "one":
                out[f"{name}/x1"], out[f"{name}/y1"], out[f"{name}/s1"] = x, y, z
            else:
                out[f"{name}/info"] = np.array([flag, info.iter, info.pobj, info.dobj])
    np.savez(os.path.join(ROOT, "tests", "golden", "spectral_solves.npz"), **out)


def proj(lib, cone, x, r_y):
    k, keep = capi.make_cone(cone, spectral=True)
    cw = lib._scs_init_cone(C.byref(k), len(x))
    assert cw
    out = x.copy()
    ry = None if r_y is None else r_y.copy()
    assert lib._scs_proj_dual_cone(capi.dptr(out), cw, None, capi.dptr(ry)) == 0
    lib._scs_finish_cone(cw)
    return out


def record_operator(lib):
    """the reference's answers on the inputs of tests/spectral_cases.py, whole or sampled (see there)"""
    out = {"names": np.array(list(spectral_cases.CASES))}
    for name in spectral_cases.CASES:
        cone, xs = spectral_cases.inputs(name)
        ry = spectral_cases.r_y(cone)
        out[f"{name}/n"] = np.array([len(xs)])
        for i, x in enumerate(xs):
            out[f"{name}/xcheck{i}"] = x[spectral_cases.check_index(x.size)]
            for tag, r in (("", None), ("ry", ry)):
                ans = proj(lib, cone, x, r)
                idx = spectral_cases.stored_index(x.size, ans)
                out[f"{name}/idx{tag}{i}"] = idx.astype(np.int32)
                out[f"{name}/out{tag}{i}"] = ans[idx] if idx.size else ans
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "spectral_cones.npz"), **out)


if __name__ == "__main__":
    build()
    write_problems()
    lib = reference()
    record_solves(lib)
    record_operator(lib)
    print("spectral fixtures written")

"""Regenerates tests/golden/problems/long/: SCS problem files written by the reference's DLONG=1 writer (8-byte
integers; oracle/long.mk builds oracle/_ref/libscsindir_ref_long.so), so that the tests can check the DLONG reader
and writer of this library byte for byte without a reference build. TEST INFRASTRUCTURE ONLY; needs the reference
sources (REF, default /root/reference).

  tests/golden/problems/long/mixed_qp   a small QP over every cone this library projects (zero, LP, box, SOC, PSD,
                                         exponential, power), with non-default settings

usage: python oracle/make_golden_long.py
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scs_b200 import capi, problems  # noqa: E402

REF = os.environ.get("REF", "/root/reference")
REF_LONG = os.path.join(ROOT, "oracle", "_ref", "libscsindir_ref_long.so")
OUT_DIR = os.path.join(ROOT, "tests", "golden", "problems", "long")


def mixed_qp():
    """the problem of tests/golden/problems/long/mixed_qp, from fixed seeds"""
    rng = np.random.default_rng(11)
    cone = {"z": 2, "l": 4, "bl": -rng.uniform(0.5, 1.5, 3), "bu": rng.uniform(0.5, 1.5, 3), "q": [3, 5],
            "s": [2, 3], "ep": 1, "ed": 1, "p": [0.4, -0.7]}
    m, n = capi.cone_rows(cone), 9
    A = problems.random_sparse_csc(m, n, 4, rng)
    P = sp.triu(sp.random(n, n, density=0.3, random_state=np.random.RandomState(5)) + sp.identity(n), format="csc")
    P.sort_indices()
    Pt = (P.data.copy(), P.indices, P.indptr, (n, n))
    return A, rng.standard_normal(m), rng.standard_normal(n), cone, Pt


def main():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "long.mk", f"REF={REF}",
                           "_ref/libscsindir_ref_long.so"])
    ref = capi.load_reference(REF_LONG, long=True)
    write = ref._scs_write_data
    L = capi.Long
    write.argtypes = [C.POINTER(L.ScsData), C.POINTER(L.ScsCone), C.POINTER(L.ScsSettings)]
    os.makedirs(OUT_DIR, exist_ok=True)
    A, b, c, cone, Pt = mixed_qp()
    hp = capi.HostProblem(A, b, c, cone, Pt, long=True)
    st = capi.default_settings(ref, long=True, verbose=0, eps_abs=2e-6, max_iters=4321, scale=0.23,
                               acceleration_lookback=7, time_limit_secs=1.5)
    path = os.path.join(OUT_DIR, "mixed_qp")
    st.write_data_filename = path.encode()
    write(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()

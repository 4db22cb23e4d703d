"""CPU: the SCS problem-file format (scs_b200/csrc/host/rw_b200.c) against the reference's own
reader / writer (oracle/_ref: src/rw.c SCS(read_data) / SCS(write_data)) and its binary fixtures
(test/problems/{random_prob, max_ent, mpc_bug1..3}, copied to oracle/_ref/test/problems by oracle/Makefile)."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import REF_DIR, REF_LIB
from scs_b200 import capi, problems

pytestmark = pytest.mark.skipif(not os.path.exists(REF_LIB), reason="oracle/_ref not built")
PP = C.POINTER


@pytest.fixture(scope="module")
def reflib():
    """the reference build itself: files are compared byte for byte and its reader allocates the problem"""
    return capi.load_reference(REF_LIB)


def bind(lib, read, write, free=None):
    r, w = getattr(lib, read), getattr(lib, write)
    r.restype = C.c_int
    r.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsCone)), PP(PP(capi.ScsSettings))]
    w.argtypes = ([C.c_char_p] if write.startswith("scs_b200") else []) + \
                 [PP(capi.ScsData), PP(capi.ScsCone), PP(capi.ScsSettings)]
    if free:
        getattr(lib, free).argtypes = [PP(capi.ScsData), PP(capi.ScsCone), PP(capi.ScsSettings)]
    return r, w


def read_with(reader, path):
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsCone)(), PP(capi.ScsSettings)()
    assert reader(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0, path
    return d, k, s


def arr(ptr, n, dtype):
    if n <= 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    return np.ctypeslib.as_array(ptr, (n,)).copy()


def snapshot(d, k, s):
    """everything a file carries, as plain python / numpy values"""
    d, k, s = d.contents, k.contents, s.contents

    def mat(mp):
        if not mp:
            return None
        M = mp.contents
        nnz = M.p[M.n]
        return (M.m, M.n, arr(M.p, M.n + 1, np.int32), arr(M.i, nnz, np.int32), arr(M.x, nnz, np.float64))

    nbox = max(k.bsize - 1, 0)
    cone = dict(z=k.z, l=k.l, bsize=k.bsize, bl=arr(k.bl, nbox, np.float64), bu=arr(k.bu, nbox, np.float64),
                q=arr(k.q, k.qsize, np.int32), s=arr(k.s, k.ssize, np.int32), cs=arr(k.cs, k.cssize, np.int32),
                ep=k.ep, ed=k.ed, p=arr(k.p, k.psize, np.float64))
    stg = {f: getattr(s, f) for f, _ in capi.ScsSettings._fields_ if "filename" not in f and f != "warm_start"}
    return dict(m=d.m, n=d.n, b=arr(d.b, d.m, np.float64), c=arr(d.c, d.n, np.float64), A=mat(d.A), P=mat(d.P),
                cone=cone, stg=stg)


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[x], b[x]) for x in a)
    if isinstance(a, tuple):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and np.array_equal(a, b)
    return a == b or (a is None and b is None)


def test_round_trips_with_the_reference(lib, reflib, tmp_path):
    my_read, my_write = bind(lib, "scs_b200_read_data", "scs_b200_write_data", "scs_b200_free_data")
    ref_read, ref_write = bind(reflib, "_scs_read_data", "_scs_write_data")
    rng = np.random.default_rng(3)
    bl = -rng.uniform(0.5, 1.5, 7)
    bu = rng.uniform(0.5, 1.5, 7)
    cone = {"z": 3, "l": 5, "bl": bl, "bu": bu, "q": [3, 6], "s": [2, 4], "ep": 2, "ed": 1, "p": [0.3, -0.6]}
    m = capi.cone_rows(cone)
    n = 17
    A = problems.random_sparse_csc(m, n, 5, rng)
    import scipy.sparse as sp
    P = sp.triu(sp.random(n, n, density=0.2, random_state=np.random.RandomState(1)) + sp.identity(n), format="csc")
    P.sort_indices()
    for with_p in (False, True):
        Pt = (P.data.copy(), P.indices.astype(np.int32), P.indptr.astype(np.int32), (n, n)) if with_p else None
        hp = capi.HostProblem(A, rng.standard_normal(m), rng.standard_normal(n), cone, Pt)
        st = capi.default_settings(lib, verbose=0, eps_abs=3e-7, max_iters=1234, scale=0.37, adaptive_scale=0,
                                   acceleration_lookback=7, time_limit_secs=2.5)
        f_mine, f_ref = str(tmp_path / f"mine{with_p}.scs"), str(tmp_path / f"ref{with_p}.scs")
        assert my_write(f_mine.encode(), C.byref(hp.data), C.byref(hp.cone), C.byref(st)) == 0
        st.write_data_filename = f_ref.encode()
        ref_write(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
        st.write_data_filename = None
        # the two writers produce the same bytes
        assert open(f_mine, "rb").read() == open(f_ref, "rb").read()
        # each reader reads the other's file and sees what was written
        truth = snapshot(C.pointer(hp.data), C.pointer(hp.cone), C.pointer(st))
        for reader, path in ((my_read, f_ref), (ref_read, f_mine), (my_read, f_mine)):
            d, k, s = read_with(reader, path)
            got = snapshot(d, k, s)
            assert same(got, truth), (with_p, path)
            if reader is my_read:
                lib.scs_b200_free_data(d, k, s)


@pytest.mark.parametrize("name", ["random_prob", "max_ent", "mpc_bug1", "mpc_bug2", "mpc_bug3"])
def test_reference_fixtures_read_identically(lib, reflib, name):
    path = os.path.join(REF_DIR, "test", "problems", name)
    if not os.path.exists(path):
        pytest.skip("fixture not copied (oracle/Makefile copies them where /root/reference exists)")
    my_read, _ = bind(lib, "scs_b200_read_data", "scs_b200_write_data", "scs_b200_free_data")
    ref_read, _ = bind(reflib, "_scs_read_data", "_scs_write_data")
    d1, k1, s1 = read_with(my_read, path)
    d2, k2, s2 = read_with(ref_read, path)
    a, b = snapshot(d1, k1, s1), snapshot(d2, k2, s2)
    assert same(a, b)
    assert a["m"] == capi.cone_rows({**{x: a["cone"][x] for x in ("z", "l", "bsize", "ep", "ed")},
                                     "q": list(a["cone"]["q"]), "s": list(a["cone"]["s"]), "p": list(a["cone"]["p"]),
                                     "cs": list(a["cone"]["cs"])})
    lib.scs_b200_free_data(d1, k1, s1)


def test_bad_files_are_refused(lib, tmp_path):
    my_read, _ = bind(lib, "scs_b200_read_data", "scs_b200_write_data", "scs_b200_free_data")
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsCone)(), PP(capi.ScsSettings)()
    p = tmp_path / "truncated.scs"
    p.write_bytes(np.array([4, 8, 6], dtype=np.uint32).tobytes() + b"3.2.11" + np.array([1, 2], dtype=np.int32).tobytes())
    assert my_read(str(p).encode(), C.byref(d), C.byref(k), C.byref(s)) == -1
    p.write_bytes(np.array([2, 8, 6], dtype=np.uint32).tobytes() + b"3.2.11")
    assert my_read(str(p).encode(), C.byref(d), C.byref(k), C.byref(s)) == -1
    assert my_read(str(tmp_path / "missing").encode(), C.byref(d), C.byref(k), C.byref(s)) == -1

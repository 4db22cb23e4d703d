"""CPU: the DLONG flavour of the library (64-bit scs_int; include/scs_b200.h, host/abi.c): the exported symbols, the
struct layouts of the reference's headers compiled with DLONG on x86-64, the default settings, the refusals of
values above the limits of the operators (checked in 64-bit width before anything is narrowed, so they need no
GPU), the problem files with 8-byte integers, and the row partition of the multi-GPU path."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import REF_DIR, ROOT
from scs_b200 import capi, problems

L = capi.Long
PP = C.POINTER
GOLDEN_LONG = os.path.join(ROOT, "tests", "golden", "problems", "long", "mixed_qp")
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden", "problems")
SPECTRAL = ["test_ell1_cone", "test_ell1_and_nuc", "robust_pca", "several_nuc_cone", "several_sum_largest",
            "graph_partitioning"]
REF_LONG = os.path.join(REF_DIR, "libscsindir_ref_long.so")
REF_SPECTRAL_LONG = os.path.join(REF_DIR, "libscsindir_ref_spectral_long.so")
LONG_PATHS = (capi.LONG_LIB_PATH, capi.SPECTRAL_LONG_LIB_PATH, capi.LINSYS_LONG_LIB_PATH)


def ensure_built():
    """the session hook builds only when libscs_b200.so is missing: build the DLONG libraries here if need be"""
    if not all(os.path.exists(p) for p in LONG_PATHS):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "scs_b200", "csrc"), "-j", "4"])


ensure_built()


@pytest.fixture(scope="module")
def llib():
    return capi.load(long=True)


# ---------------------------------------------------------------------------------------------------- exports
def header_functions():
    text = open(os.path.join(ROOT, "include", "scs_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(scs_\w+)\s*\(", text)))


def exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return {line.split()[-1] for line in out.splitlines() if line.split()[-2] in ("T", "W")}


# the outer ABI with the workspace helpers of the ADMM driver, and the problem files: the plugin-only library leaves
# them out (host/scs_driver.c, host/rw_b200.c), since the reference tree it is linked into defines its own scs_init ...
NOT_IN_PLUGIN = {"scs_init", "scs_update", "scs_solve", "scs_finish", "scs", "scs_set_default_settings",
                 "scs_version", "scs_b200_get_stats", "scs_b200_set_max_iters", "scs_b200_launch_count",
                 "scs_b200_device_ok", "scs_b200_write_data", "scs_b200_read_data", "scs_b200_free_data"}


def test_every_header_symbol_is_exported():
    names = header_functions()
    assert len(names) > 40 and "scs_init_lin_sys_work" in names and "scs_b200_row_partition" in names
    for path in (capi.LONG_LIB_PATH, capi.SPECTRAL_LONG_LIB_PATH):
        missing = set(names) - exported(path)
        assert not missing, (path, missing)
    plugin = exported(capi.LINSYS_LONG_LIB_PATH)
    assert not (set(names) - NOT_IN_PLUGIN) - plugin
    assert not NOT_IN_PLUGIN & plugin
    assert exported(capi.LONG_LIB_PATH) == exported(capi.LIB_PATH)


# ---------------------------------------------------------------------------------------------------- layouts
def test_layouts_match_the_reference_dlong_headers():
    sizes = {"ScsMatrix": (32, 40), "ScsData": (40, 48), "ScsSettings": (136, 152), "ScsCone": (104, 120),
             "ScsConeSpectral": (184, 200), "ScsSolution": (24, 24), "AaStats": (48, 80), "ScsInfo": (448, 496)}
    for name, (int_size, long_size) in sizes.items():
        assert C.sizeof(getattr(capi, name)) == int_size, name
        assert getattr(capi, name) is getattr(capi.Int, name)
        assert C.sizeof(getattr(L, name)) == long_size, name
    assert (L.ScsSettings.write_data_filename.offset, L.ScsSettings.log_csv_filename.offset) == (136, 144)
    assert (L.ScsCone.p.offset, L.ScsCone.psize.offset) == (104, 112)
    S = L.ScsConeSpectral
    assert (S.d.offset, S.nuc_m.offset, S.ell1.offset, S.sl_n.offset, S.sl_size.offset) == (120, 136, 160, 176, 192)
    I = L.ScsInfo
    assert (I.status.offset, I.lin_sys_solver.offset, I.pobj.offset, I.aa_stats.offset, I.lin_sys_time.offset) == \
        (8, 136, 280, 392, 472)
    assert L.ScsData._fields_[2][1]._type_ is L.ScsMatrix and L.ScsInfo.aa_stats.size == 80


def test_default_settings_are_the_reference_defaults(llib):
    st = capi.default_settings(llib, long=True)
    want = dict(normalize=1, scale=0.1, adaptive_scale=1, rho_x=1e-6, max_iters=100000, eps_abs=1e-4, eps_rel=1e-4,
                eps_infeas=1e-7, alpha=1.5, time_limit_secs=0.0, verbose=1, warm_start=0, acceleration_lookback=10,
                acceleration_interval=10, acceleration_type_1=1, acceleration_regularization=1e-8,
                acceleration_relaxation=1.0, write_data_filename=None, log_csv_filename=None)
    assert {f: getattr(st, f) for f in want} == want
    if os.path.exists(REF_LONG):
        ref = capi.default_settings(capi.load_reference(REF_LONG, long=True), long=True)
        assert {f: getattr(ref, f) for f in want} == want


# ---------------------------------------------------------------------------------------------------- limits
REFUSAL_SCRIPT = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, {root!r})
from scs_b200 import capi, problems
case = sys.argv[1]
lib = capi.load(long=True)
prob = problems.make_problem(12, 5, 3, {{"l": 12}}, seed=1)
cone = dict(prob["cone"])
if case == "cone":
    cone = {{"l": 9, "s": [2 ** 32 + 2]}}   # truncates to order 2: 3 rows, as m = 12 = 9 + 3 would need
hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], cone, long=True)
st = capi.default_settings(lib, long=True, verbose=0)
if case == "m":
    hp.data.m = hp.A.m = 2 ** 30
if case == "nnz":
    Ap = np.array([0] * hp.n + [2 ** 31 + 5], dtype=np.int64)   # i and x hold far fewer entries
    hp.Ap = Ap
    hp.A.p = capi.lptr(Ap)
if case == "row":
    hp.Ai[0] = 2 ** 32 + 3                                      # truncates to the valid row 3
if case == "plugin_m":
    hp.A.m = 2 ** 30
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(np.ones(hp.n + hp.m)))
    sys.stdout.flush()
    print("RESULT", w)
    sys.exit(0)
w = lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
sys.stdout.flush()
print("RESULT", w)
"""


@pytest.mark.parametrize("case, message", [
    ("m", "m = 1073741824 exceeds the limit 2^30 - 1"),
    ("nnz", "nnz(A) = A->p[n] = 2147483653 exceeds the limit 2^31 - 129"),
    ("cone", "s[0] = 4294967298 exceeds the limit 2^30 - 1"),
    ("row", "A row index 4294967299 outside valid range [0, 11]"),
    ("plugin_m", "A->m = 1073741824 exceeds the limit 2^30 - 1"),
])
def test_values_above_the_limits_are_refused_before_narrowing(case, message):
    """each in a subprocess: a check placed after an array is read or a value narrowed fails this test (wrong message
    or a crash) instead of the session"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")  # refused before any device work
    r = subprocess.run([sys.executable, "-c", REFUSAL_SCRIPT.format(root=ROOT), case], capture_output=True, text=True,
                       env=env, timeout=120)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out
    assert message in out, out
    assert "RESULT None" in out, out


# ---------------------------------------------------------------------------------------------------- problem files
def rw(lib, long, spectral=False):
    T = capi.abi(long)
    cone = T.ScsConeSpectral if spectral else T.ScsCone
    r, w, f = lib.scs_b200_read_data, lib.scs_b200_write_data, lib.scs_b200_free_data
    r.restype = w.restype = T.int_t
    r.argtypes = [C.c_char_p, PP(PP(T.ScsData)), PP(PP(cone)), PP(PP(T.ScsSettings))]
    w.argtypes = [C.c_char_p, PP(T.ScsData), PP(cone), PP(T.ScsSettings)]
    f.argtypes = [PP(T.ScsData), PP(cone), PP(T.ScsSettings)]
    f.restype = None

    def read(path):
        d, k, s = PP(T.ScsData)(), PP(cone)(), PP(T.ScsSettings)()
        assert r(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0, path
        return d, k, s

    return read, w, f


def ref_rw(path, spectral=False):
    lib = capi.load_reference(path, spectral=spectral, long=True)
    cone = L.ScsConeSpectral if spectral else L.ScsCone
    r, w = lib._scs_read_data, lib._scs_write_data
    r.restype = C.c_int64
    r.argtypes = [C.c_char_p, PP(PP(L.ScsData)), PP(PP(cone)), PP(PP(L.ScsSettings))]
    w.argtypes = [PP(L.ScsData), PP(cone), PP(L.ScsSettings)]

    def read(p):
        d, k, s = PP(L.ScsData)(), PP(cone)(), PP(L.ScsSettings)()
        assert r(p.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0, p
        return d, k, s

    def write(path_out, d, k, s):
        s.contents.write_data_filename = path_out.encode()
        w(d, k, s)
        s.contents.write_data_filename = None

    return read, write


def arr(ptr, n, dtype):
    if n <= 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    return np.ctypeslib.as_array(ptr, (n,)).astype(dtype)


def snapshot(d, k, s, spectral=False):
    """everything a file carries, as plain python / numpy values (integers as int64 whatever the width)"""
    d, k, s = d.contents, k.contents, s.contents
    i64, f64 = np.int64, np.float64

    def mat(mp):
        if not mp:
            return None
        M = mp.contents
        nnz = M.p[M.n]
        return (M.m, M.n, arr(M.p, M.n + 1, i64), arr(M.i, nnz, i64), arr(M.x, nnz, f64))

    nbox = max(k.bsize - 1, 0)
    cone = dict(z=k.z, l=k.l, bsize=k.bsize, bl=arr(k.bl, nbox, f64), bu=arr(k.bu, nbox, f64), q=arr(k.q, k.qsize, i64),
                s=arr(k.s, k.ssize, i64), cs=arr(k.cs, k.cssize, i64), ep=k.ep, ed=k.ed, p=arr(k.p, k.psize, f64))
    if spectral:
        cone.update(d=arr(k.d, k.dsize, i64), nuc_m=arr(k.nuc_m, k.nucsize, i64), nuc_n=arr(k.nuc_n, k.nucsize, i64),
                    ell1=arr(k.ell1, k.ell1_size, i64), sl_n=arr(k.sl_n, k.sl_size, i64),
                    sl_k=arr(k.sl_k, k.sl_size, i64))
    stg = {f: getattr(s, f) for f, _ in capi.ScsSettings._fields_ if "filename" not in f and f != "warm_start"}
    return dict(m=d.m, n=d.n, b=arr(d.b, d.m, f64), c=arr(d.c, d.n, f64), A=mat(d.A), P=mat(d.P), cone=cone, stg=stg)


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[x], b[x]) for x in a)
    if isinstance(a, tuple):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and np.array_equal(a, b)
    return a == b or (a is None and b is None)


def test_golden_dlong_file_round_trips_byte_for_byte(llib, tmp_path):
    read, write, free = rw(llib, long=True)
    d, k, s = read(GOLDEN_LONG)
    assert d.contents.m == 39 and d.contents.P and k.contents.bsize == 4 and k.contents.ssize == 2
    out = str(tmp_path / "again")
    assert write(out.encode(), d, k, s) == 0
    assert open(out, "rb").read() == open(GOLDEN_LONG, "rb").read()
    assert np.frombuffer(open(out, "rb").read(4), dtype=np.uint32)[0] == 8
    free(d, k, s)


@pytest.mark.parametrize("name", ["random_prob", "mpc_bug1"])
def test_long_writer_matches_the_reference_dlong_writer(llib, tmp_path, name):
    if not os.path.exists(REF_LONG):
        pytest.skip("oracle/_ref DLONG build absent (oracle/long.mk needs the reference sources)")
    src = os.path.join(GOLDEN_DIR, name)
    read, write, free = rw(llib, long=True)
    ref_read, ref_write = ref_rw(REF_LONG)
    d, k, s = read(src)
    mine = str(tmp_path / "mine")
    assert write(mine.encode(), d, k, s) == 0
    d2, k2, s2 = ref_read(src)
    assert same(snapshot(d, k, s), snapshot(d2, k2, s2))
    ref = str(tmp_path / "ref")
    ref_write(ref, d2, k2, s2)
    assert open(mine, "rb").read() == open(ref, "rb").read()
    free(d, k, s)


def test_each_width_reads_the_others_files(lib, llib, tmp_path):
    iread, iwrite, ifree = rw(lib, long=False)
    lread, lwrite, lfree = rw(llib, long=True)
    for src in (GOLDEN_LONG, os.path.join(GOLDEN_DIR, "random_prob")):
        a = lread(src)
        b = iread(src)
        assert same(snapshot(*a), snapshot(*b)), src
        f_long, f_int = str(tmp_path / "long.scs"), str(tmp_path / "int.scs")
        assert lwrite(f_long.encode(), *a) == 0 and iwrite(f_int.encode(), *b) == 0
        assert open(f_long, "rb").read(4) != open(f_int, "rb").read(4)  # 8- and 4-byte integers
        for reader, path, release in ((iread, f_long, ifree), (lread, f_int, lfree), (lread, f_long, lfree)):
            got = reader(path)
            assert same(snapshot(*got), snapshot(*a)), (src, path)
            release(*got)
        lfree(*a)
        ifree(*b)


@pytest.mark.parametrize("name", SPECTRAL)
def test_spectral_fixtures_round_trip_through_the_spectral_dlong_library(name, tmp_path):
    slib, ilib = capi.load(spectral=True, long=True), capi.load(spectral=True)
    lread, lwrite, lfree = rw(slib, long=True, spectral=True)
    iread, _, ifree = rw(ilib, long=False, spectral=True)
    src = os.path.join(GOLDEN_DIR, "spectral", name)
    a, b = lread(src), iread(src)
    truth = snapshot(*b, spectral=True)
    assert same(snapshot(*a, spectral=True), truth)
    out = str(tmp_path / "long.scs")
    assert lwrite(out.encode(), *a) == 0
    for reader, release in ((lread, lfree), (iread, ifree)):
        got = reader(out)
        assert same(snapshot(*got, spectral=True), truth)
        release(*got)
    if os.path.exists(REF_SPECTRAL_LONG):
        ref_read, ref_write = ref_rw(REF_SPECTRAL_LONG, spectral=True)
        ref = str(tmp_path / "ref.scs")
        ref_write(ref, *ref_read(src))
        assert open(out, "rb").read() == open(ref, "rb").read()
    lfree(*a)
    ifree(*b)


# ---------------------------------------------------------------------------------------------------- row partition
def test_row_partition_matches_the_int_library(lib, llib):
    rng = np.random.default_rng(8)
    for m, n, per_col in ((50, 20, 5), (1000, 300, 12), (7, 3, 2)):
        Ax, Ai, Ap, _ = problems.random_sparse_csc(m, n, per_col, rng)
        for nranks in (1, 2, 3, 8):
            o32 = np.zeros(nranks + 1, dtype=np.int32)
            o64 = np.zeros(nranks + 1, dtype=np.int64)
            assert lib.scs_b200_row_partition(m, n, capi.iptr(np.ascontiguousarray(Ap, dtype=np.int32)),
                                              capi.iptr(np.ascontiguousarray(Ai, dtype=np.int32)), nranks,
                                              capi.iptr(o32)) == 0
            assert llib.scs_b200_row_partition(m, n, capi.lptr(np.ascontiguousarray(Ap, dtype=np.int64)),
                                               capi.lptr(np.ascontiguousarray(Ai, dtype=np.int64)), nranks,
                                               capi.lptr(o64)) == 0
            assert np.array_equal(o32, o64) and o64[0] == 0 and o64[-1] == m, (m, nranks)

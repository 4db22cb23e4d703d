"""ctypes mirror of include/scs_b200.h (and of the reference's include/scs.h layout).

This is plumbing for tests/ and bench.py: it loads the in-tree
``scs_b200/libscs_b200.so`` (hand-written sm_90a kernels behind a C ABI) and
declares argument types for every exported symbol.  There is no fallback: if the
shared library is missing, or no sm_90 device is usable, calls fail loudly.

The same struct classes are used to drive the reference build
(``oracle/_ref/libscsindir_ref.so``) in the parity tests, because the layouts
are identical by construction (reference include/scs.h:47-244).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SCS_B200_LIB", os.path.join(_HERE, "libscs_b200.so"))

c_int_p = C.POINTER(C.c_int)
c_double_p = C.POINTER(C.c_double)


class ScsMatrix(C.Structure):
    _fields_ = [("x", c_double_p), ("i", c_int_p), ("p", c_int_p), ("m", C.c_int), ("n", C.c_int)]


class ScsSettings(C.Structure):
    _fields_ = [
        ("normalize", C.c_int), ("scale", C.c_double), ("adaptive_scale", C.c_int),
        ("rho_x", C.c_double), ("max_iters", C.c_int), ("eps_abs", C.c_double),
        ("eps_rel", C.c_double), ("eps_infeas", C.c_double), ("alpha", C.c_double),
        ("time_limit_secs", C.c_double), ("verbose", C.c_int), ("warm_start", C.c_int),
        ("acceleration_lookback", C.c_int), ("acceleration_interval", C.c_int),
        ("acceleration_type_1", C.c_int), ("acceleration_regularization", C.c_double),
        ("acceleration_relaxation", C.c_double), ("write_data_filename", C.c_char_p),
        ("log_csv_filename", C.c_char_p),
    ]


class ScsData(C.Structure):
    _fields_ = [("m", C.c_int), ("n", C.c_int), ("A", C.POINTER(ScsMatrix)),
                ("P", C.POINTER(ScsMatrix)), ("b", c_double_p), ("c", c_double_p)]


class ScsCone(C.Structure):
    _fields_ = [
        ("z", C.c_int), ("l", C.c_int), ("bu", c_double_p), ("bl", c_double_p), ("bsize", C.c_int),
        ("q", c_int_p), ("qsize", C.c_int), ("s", c_int_p), ("ssize", C.c_int),
        ("cs", c_int_p), ("cssize", C.c_int), ("ep", C.c_int), ("ed", C.c_int),
        ("p", c_double_p), ("psize", C.c_int),
    ]


class ScsSolution(C.Structure):
    _fields_ = [("x", c_double_p), ("y", c_double_p), ("s", c_double_p)]


class AaStats(C.Structure):
    _fields_ = [
        ("iter", C.c_int), ("n_accept", C.c_int), ("n_reject_lapack", C.c_int),
        ("n_reject_rank0", C.c_int), ("n_reject_nonfinite", C.c_int),
        ("n_reject_weight_cap", C.c_int), ("n_safeguard_reject", C.c_int),
        ("last_rank", C.c_int), ("last_aa_norm", C.c_double), ("last_regularization", C.c_double),
    ]


class ScsInfo(C.Structure):
    _fields_ = [
        ("iter", C.c_int), ("status", C.c_char * 128), ("lin_sys_solver", C.c_char * 128),
        ("status_val", C.c_int), ("scale_updates", C.c_int), ("pobj", C.c_double),
        ("dobj", C.c_double), ("res_pri", C.c_double), ("res_dual", C.c_double),
        ("gap", C.c_double), ("res_infeas", C.c_double), ("res_unbdd_a", C.c_double),
        ("res_unbdd_p", C.c_double), ("setup_time", C.c_double), ("solve_time", C.c_double),
        ("scale", C.c_double), ("comp_slack", C.c_double), ("rejected_accel_steps", C.c_int),
        ("accepted_accel_steps", C.c_int), ("aa_stats", AaStats), ("lin_sys_time", C.c_double),
        ("cone_time", C.c_double), ("accel_time", C.c_double),
    ]


class ScsB200Stats(C.Structure):
    _fields_ = [("cg_iters", C.c_longlong), ("lin_sys_solves", C.c_longlong),
                ("kernel_launches", C.c_longlong), ("spmv_ms", C.c_double), ("n_gpus", C.c_int)]


def dptr(a):
    """float64 numpy array -> double* (no copy; the caller keeps `a` alive)."""
    if a is None:
        return c_double_p()
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_double_p)


def iptr(a):
    if a is None:
        return c_int_p()
    assert a.dtype == np.int32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_int_p)


class HostProblem:
    """Owns numpy arrays and the ctypes structs that point into them."""

    def __init__(self, A_csc, b, c, cone, P_csc=None):
        """A_csc / P_csc: (data, indices, indptr, shape) with int32 indices; cone: dict."""
        self.Ax = np.ascontiguousarray(A_csc[0], dtype=np.float64)
        self.Ai = np.ascontiguousarray(A_csc[1], dtype=np.int32)
        self.Ap = np.ascontiguousarray(A_csc[2], dtype=np.int32)
        self.m, self.n = int(A_csc[3][0]), int(A_csc[3][1])
        self.b = np.ascontiguousarray(b, dtype=np.float64)
        self.c = np.ascontiguousarray(c, dtype=np.float64)
        self.A = ScsMatrix(dptr(self.Ax), iptr(self.Ai), iptr(self.Ap), self.m, self.n)
        self.P = None
        if P_csc is not None:
            self.Px = np.ascontiguousarray(P_csc[0], dtype=np.float64)
            self.Pi = np.ascontiguousarray(P_csc[1], dtype=np.int32)
            self.Pp = np.ascontiguousarray(P_csc[2], dtype=np.int32)
            self.P = ScsMatrix(dptr(self.Px), iptr(self.Pi), iptr(self.Pp), self.n, self.n)
        self.data = ScsData(self.m, self.n, C.pointer(self.A),
                            C.pointer(self.P) if self.P is not None else C.POINTER(ScsMatrix)(),
                            dptr(self.b), dptr(self.c))
        self.cone_dict = dict(cone)
        self.cone, self._cone_keep = make_cone(cone)


def make_cone(cone):
    keep = {}
    k = ScsCone()
    k.z = int(cone.get("z", 0))
    k.l = int(cone.get("l", 0))
    bu = cone.get("bu")
    bl = cone.get("bl")
    if bu is not None and len(bu) > 0:
        keep["bu"] = np.ascontiguousarray(bu, dtype=np.float64)
        keep["bl"] = np.ascontiguousarray(bl, dtype=np.float64)
        k.bu, k.bl, k.bsize = dptr(keep["bu"]), dptr(keep["bl"]), len(keep["bu"]) + 1
    else:
        k.bsize = int(cone.get("bsize", 0))
    q = cone.get("q")
    if q is not None and len(q) > 0:
        keep["q"] = np.ascontiguousarray(q, dtype=np.int32)
        k.q, k.qsize = iptr(keep["q"]), len(keep["q"])
    s = cone.get("s")
    if s is not None and len(s) > 0:
        keep["s"] = np.ascontiguousarray(s, dtype=np.int32)
        k.s, k.ssize = iptr(keep["s"]), len(keep["s"])
    cs = cone.get("cs")
    if cs is not None and len(cs) > 0:
        keep["cs"] = np.ascontiguousarray(cs, dtype=np.int32)
        k.cs, k.cssize = iptr(keep["cs"]), len(keep["cs"])
    k.ep = int(cone.get("ep", 0))
    k.ed = int(cone.get("ed", 0))
    p = cone.get("p")
    if p is not None and len(p) > 0:
        keep["p"] = np.ascontiguousarray(p, dtype=np.float64)
        k.p, k.psize = dptr(keep["p"]), len(keep["p"])
    return k, keep


def cone_rows(cone):
    q = cone.get("q", []) or []
    s = cone.get("s", []) or []
    bs = (len(cone["bu"]) + 1) if cone.get("bu") is not None and len(cone["bu"]) else int(cone.get("bsize", 0))
    return (int(cone.get("z", 0)) + int(cone.get("l", 0)) + bs + int(sum(q)) +
            int(sum(int(k) * (int(k) + 1) // 2 for k in s)) +
            int(sum(int(k) * int(k) for k in (cone.get("cs", []) or []))) +
            3 * (int(cone.get("ep", 0)) + int(cone.get("ed", 0)) + len(cone.get("p", []) or [])))


class _Decl:
    """Attribute proxy: declaring a signature on a symbol the library does not export is a no-op
    (calling it later still raises AttributeError)."""

    class _Sink:
        restype = None
        argtypes = None

    def __init__(self, lib):
        object.__setattr__(self, "_lib", lib)

    def __getattr__(self, name):
        try:
            return getattr(self._lib, name)
        except AttributeError:
            return _Decl._Sink()


def _declare(lib, ours):
    """Declare the signatures shared by our library and the reference build."""
    lib = _Decl(lib)
    lib.scs_init.restype = C.c_void_p
    lib.scs_init.argtypes = [C.POINTER(ScsData), C.POINTER(ScsCone), C.POINTER(ScsSettings)]
    lib.scs_solve.restype = C.c_int
    lib.scs_solve.argtypes = [C.c_void_p, C.POINTER(ScsSolution), C.POINTER(ScsInfo), C.c_int]
    lib.scs_update.restype = C.c_int
    lib.scs_update.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_finish.restype = None
    lib.scs_finish.argtypes = [C.c_void_p]
    lib.scs.restype = C.c_int
    lib.scs.argtypes = [C.POINTER(ScsData), C.POINTER(ScsCone), C.POINTER(ScsSettings),
                        C.POINTER(ScsSolution), C.POINTER(ScsInfo)]
    lib.scs_set_default_settings.restype = None
    lib.scs_set_default_settings.argtypes = [C.POINTER(ScsSettings)]
    lib.scs_version.restype = C.c_char_p
    lib.scs_init_lin_sys_work.restype = C.c_void_p
    lib.scs_init_lin_sys_work.argtypes = [C.POINTER(ScsMatrix), C.POINTER(ScsMatrix), c_double_p]
    lib.scs_free_lin_sys_work.restype = None
    lib.scs_free_lin_sys_work.argtypes = [C.c_void_p]
    lib.scs_solve_lin_sys.restype = C.c_int
    lib.scs_solve_lin_sys.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_double]
    lib.scs_update_lin_sys_diag_r.restype = C.c_int
    lib.scs_update_lin_sys_diag_r.argtypes = [C.c_void_p, c_double_p]
    lib.scs_get_lin_sys_method.restype = C.c_char_p
    if not ours:
        return
    lib.scs_b200_linsys_last_cg_its.restype = C.c_int
    lib.scs_b200_linsys_last_cg_its.argtypes = [C.c_void_p]
    lib.scs_b200_linsys_total_cg_its.restype = C.c_longlong
    lib.scs_b200_linsys_total_cg_its.argtypes = [C.c_void_p]
    for f in (lib.scs_b200_accum_by_a, lib.scs_b200_accum_by_atrans):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_int]
    lib.scs_b200_time_spmv.restype = C.c_double
    lib.scs_b200_time_spmv.argtypes = [C.c_void_p, C.c_int, C.c_int, c_double_p]
    lib.scs_b200_time_cg_iter.restype = C.c_double
    lib.scs_b200_time_cg_iter.argtypes = [C.c_void_p, C.c_int, c_double_p]
    lib.scs_b200_time_cg_kernels.restype = C.c_int
    lib.scs_b200_time_cg_kernels.argtypes = [C.c_void_p, c_double_p, C.c_int, c_double_p, c_double_p]
    lib.scs_b200_init_cone.restype = C.c_void_p
    lib.scs_b200_init_cone.argtypes = [C.POINTER(ScsCone), C.c_int, c_double_p]
    lib.scs_b200_proj_dual_cone.restype = C.c_int
    lib.scs_b200_proj_dual_cone.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_finish_cone.restype = None
    lib.scs_b200_finish_cone.argtypes = [C.c_void_p]
    lib.scs_b200_aa_init.restype = C.c_void_p
    lib.scs_b200_aa_init.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double,
                                     C.c_double, C.c_double, C.c_int, C.c_int]
    lib.scs_b200_aa_apply.restype = C.c_double
    lib.scs_b200_aa_apply.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_aa_safeguard.restype = C.c_int
    lib.scs_b200_aa_safeguard.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_aa_reset.restype = None
    lib.scs_b200_aa_reset.argtypes = [C.c_void_p]
    lib.scs_b200_aa_finish.restype = None
    lib.scs_b200_aa_finish.argtypes = [C.c_void_p]
    lib.scs_b200_aa_get_stats.restype = AaStats
    lib.scs_b200_aa_get_stats.argtypes = [C.c_void_p]
    lib.scs_b200_get_stats.restype = C.c_int
    lib.scs_b200_get_stats.argtypes = [C.c_void_p, C.POINTER(ScsB200Stats)]
    lib.scs_b200_set_max_iters.restype = C.c_int
    lib.scs_b200_set_max_iters.argtypes = [C.c_void_p, C.c_int]
    lib.scs_b200_comm_unique_id.restype = C.c_int
    lib.scs_b200_comm_unique_id.argtypes = [C.c_char_p]
    lib.scs_b200_comm_init.restype = C.c_int
    lib.scs_b200_comm_init.argtypes = [C.c_int, C.c_int, C.c_char_p]
    lib.scs_b200_comm_finalize.restype = C.c_int
    lib.scs_b200_row_partition.restype = C.c_int
    lib.scs_b200_row_partition.argtypes = [C.c_int, C.c_int, c_int_p, c_int_p, C.c_int, c_int_p]
    lib.scs_b200_launch_count.restype = C.c_longlong
    lib.scs_b200_device_ok.restype = C.c_int
    lib.scs_b200_release_memory.restype = None


_lib = None


def load():
    """Load scs_b200/libscs_b200.so. Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(make -C scs_b200/csrc). There is no CPU fallback.")
        # RTLD_LOCAL: our scs_* symbols must not interpose on the reference build loaded by the tests
        lib = C.CDLL(LIB_PATH, mode=C.RTLD_LOCAL)
        _declare(lib, ours=True)
        _lib = lib
    return _lib


def load_reference(path):
    """Load a build of the UNMODIFIED reference (oracle/_ref/*.so). Test infrastructure only."""
    # the venv's OpenBLAS (the only LAPACK in this image) needs its bundled
    # libgfortran/libquadmath, which sit next to it without an rpath
    import glob
    ob = os.environ.get(
        "SCS_REF_OPENBLAS_DIR",
        "/opt/prime-rl/.venv/lib/python3.12/site-packages/opencv_python_headless.libs")
    for pat in ("libquadmath*", "libgfortran*"):
        for f in sorted(glob.glob(os.path.join(ob, pat))):
            try:
                C.CDLL(f, mode=C.RTLD_GLOBAL)
            except OSError:
                pass
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    _declare(lib, ours=False)
    return lib


def default_settings(lib, **over):
    st = ScsSettings()
    lib.scs_set_default_settings(C.byref(st))
    for k, v in over.items():
        setattr(st, k, v)
    return st

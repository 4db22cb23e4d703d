"""ctypes mirror of include/scs_b200.h (and of the reference's include/scs.h layout).

This is plumbing for tests/ and bench.py: it loads the in-tree
``scs_b200/libscs_b200.so`` (hand-written sm_90a kernels behind a C ABI) and
declares argument types for every exported symbol.  There is no fallback: if the
shared library is missing, or no sm_90 device is usable, calls fail loudly.

The same struct classes are used to drive the reference build
(``oracle/_ref/libscsindir_ref.so``) in the parity tests, because the layouts
are identical by construction (reference include/scs.h:47-244).

The module-level classes (``ScsMatrix``, ``ScsCone``, ...) are those of the
default build, where scs_int is a C int. The DLONG build's classes, with a
64-bit scs_int, are the same names under ``capi.Long`` (``capi.Long.ScsMatrix``,
...); ``load(long=True)`` loads the DLONG libraries and declares their
signatures with them, and ``HostProblem`` / ``make_cone`` build int64 inputs
with ``long=True``.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SCS_B200_LIB", os.path.join(_HERE, "libscs_b200.so"))
# the same kernels behind the reference's USE_SPECTRAL_CONES ScsCone layout (ScsConeSpectral below)
SPECTRAL_LIB_PATH = os.environ.get("SCS_B200_SPECTRAL_LIB", os.path.join(_HERE, "libscs_b200_spectral.so"))
# the DLONG flavours (64-bit scs_int): the full library, its spectral build and the plugin-only library
LONG_LIB_PATH = os.path.join(_HERE, "libscs_b200_long.so")
SPECTRAL_LONG_LIB_PATH = os.path.join(_HERE, "libscs_b200_spectral_long.so")
LINSYS_LONG_LIB_PATH = os.path.join(_HERE, "libscs_b200_linsys_long.so")

c_int_p = C.POINTER(C.c_int)
c_int64_p = C.POINTER(C.c_int64)
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


class ScsConeSpectral(ScsCone):
    """ScsCone of the reference's USE_SPECTRAL_CONES build (include/scs.h:154-171): 184 bytes, taken by
    libscs_b200_spectral.so, which projects all four spectral cones: log-det (d), nuclear-norm, l1-norm and
    sum-of-largest-eigenvalues."""
    _fields_ = [
        ("d", c_int_p), ("dsize", C.c_int), ("nuc_m", c_int_p), ("nuc_n", c_int_p), ("nucsize", C.c_int),
        ("ell1", c_int_p), ("ell1_size", C.c_int), ("sl_n", c_int_p), ("sl_k", c_int_p), ("sl_size", C.c_int),
    ]


SPECTRAL_KEYS = ("d", "nuc_m", "nuc_n", "ell1", "sl_n", "sl_k")


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


def _widened(cls, base, scope):
    """`cls` with a 64-bit scs_int: C int fields become int64, int pointers int64 pointers, and nested structs (or
    pointers to them) the widened classes already in `scope`"""
    fields = []
    for name, t in cls.__dict__["_fields_"]:
        pointee = getattr(t, "_type_", None)
        if t is C.c_int:
            t = C.c_int64
        elif t is c_int_p:
            t = c_int64_p
        elif t.__name__ in scope:
            t = scope[t.__name__]
        elif isinstance(pointee, type) and pointee.__name__ in scope:
            t = C.POINTER(scope[pointee.__name__])
        fields.append((name, t))
    return type(cls.__name__, (base,), {"_fields_": fields, "__doc__": f"{cls.__name__} of the DLONG build"})


class Long:
    """The struct classes of the DLONG build: scs_int is 64 bits (reference include/scs_types.h:14-24 on LP64)."""
    int_t = C.c_int64
    int_p = c_int64_p
    dtype = np.int64


def _make_long():
    scope = {}
    for cls in (ScsMatrix, ScsSettings, ScsData, ScsCone, ScsSolution, AaStats, ScsInfo, ScsB200Stats):
        scope[cls.__name__] = _widened(cls, C.Structure, scope)
    scope["ScsConeSpectral"] = _widened(ScsConeSpectral, scope["ScsCone"], scope)
    for name, cls in scope.items():
        setattr(Long, name, cls)


class Int:
    """The struct classes of the default build (scs_int is a C int): the module-level ones."""
    int_t = C.c_int
    int_p = c_int_p
    dtype = np.int32


for _cls in ("ScsMatrix", "ScsSettings", "ScsData", "ScsCone", "ScsSolution", "AaStats", "ScsInfo", "ScsB200Stats",
             "ScsConeSpectral"):
    setattr(Int, _cls, globals()[_cls])
_make_long()


def abi(long=False):
    """the struct classes of the default build (Int) or of the DLONG build (Long)"""
    return Long if long else Int


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


def lptr(a):
    """int64 numpy array -> scs_int* of the DLONG build (no copy)"""
    if a is None:
        return c_int64_p()
    assert a.dtype == np.int64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_int64_p)


class HostProblem:
    """Owns numpy arrays and the ctypes structs that point into them."""

    def __init__(self, A_csc, b, c, cone, P_csc=None, long=False):
        """A_csc / P_csc: (data, indices, indptr, shape); cone: dict. The structs are those of the default build with
        int32 index arrays, or with long=True those of the DLONG build (capi.Long) with int64 index arrays."""
        T = abi(long)
        ip = lptr if long else iptr
        self.Ax = np.ascontiguousarray(A_csc[0], dtype=np.float64)
        self.Ai = np.ascontiguousarray(A_csc[1], dtype=T.dtype)
        self.Ap = np.ascontiguousarray(A_csc[2], dtype=T.dtype)
        self.m, self.n = int(A_csc[3][0]), int(A_csc[3][1])
        self.b = np.ascontiguousarray(b, dtype=np.float64)
        self.c = np.ascontiguousarray(c, dtype=np.float64)
        self.A = T.ScsMatrix(dptr(self.Ax), ip(self.Ai), ip(self.Ap), self.m, self.n)
        self.P = None
        if P_csc is not None:
            self.Px = np.ascontiguousarray(P_csc[0], dtype=np.float64)
            self.Pi = np.ascontiguousarray(P_csc[1], dtype=T.dtype)
            self.Pp = np.ascontiguousarray(P_csc[2], dtype=T.dtype)
            self.P = T.ScsMatrix(dptr(self.Px), ip(self.Pi), ip(self.Pp), self.n, self.n)
        self.data = T.ScsData(self.m, self.n, C.pointer(self.A),
                              C.pointer(self.P) if self.P is not None else C.POINTER(T.ScsMatrix)(),
                              dptr(self.b), dptr(self.c))
        self.cone_dict = dict(cone)
        self.cone, self._cone_keep = make_cone(cone, long=long)


def is_spectral(cone):
    return any(cone.get(key) is not None and len(cone.get(key)) > 0 for key in SPECTRAL_KEYS)


def make_cone(cone, spectral=None, long=False):
    """ctypes cone struct + the arrays it points into. The struct is a ScsConeSpectral when `spectral` is True, or
    when it is None and the dict has spectral keys (nuc_m / nuc_n, ell1, sl_n / sl_k, d); otherwise a ScsCone.
    long=True: the DLONG build's struct (capi.Long) with int64 arrays."""
    keep = {}
    if spectral is None:
        spectral = is_spectral(cone)
    T = abi(long)
    ip = lptr if long else iptr
    k = T.ScsConeSpectral() if spectral else T.ScsCone()
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
        keep["q"] = np.ascontiguousarray(q, dtype=T.dtype)
        k.q, k.qsize = ip(keep["q"]), len(keep["q"])
    s = cone.get("s")
    if s is not None and len(s) > 0:
        keep["s"] = np.ascontiguousarray(s, dtype=T.dtype)
        k.s, k.ssize = ip(keep["s"]), len(keep["s"])
    cs = cone.get("cs")
    if cs is not None and len(cs) > 0:
        keep["cs"] = np.ascontiguousarray(cs, dtype=T.dtype)
        k.cs, k.cssize = ip(keep["cs"]), len(keep["cs"])
    k.ep = int(cone.get("ep", 0))
    k.ed = int(cone.get("ed", 0))
    p = cone.get("p")
    if p is not None and len(p) > 0:
        keep["p"] = np.ascontiguousarray(p, dtype=np.float64)
        k.p, k.psize = dptr(keep["p"]), len(keep["p"])
    if spectral:
        for key, size, names in (("d", "dsize", ("d",)), ("nuc_m", "nucsize", ("nuc_m", "nuc_n")),
                                 ("ell1", "ell1_size", ("ell1",)), ("sl_n", "sl_size", ("sl_n", "sl_k"))):
            v = cone.get(key)
            if v is None or len(v) == 0:
                continue
            for name in names:
                keep[name] = np.ascontiguousarray(cone[name], dtype=T.dtype)
                setattr(k, name, ip(keep[name]))
            setattr(k, size, len(keep[key]))
    return k, keep


def cone_rows(cone):
    q = cone.get("q", []) or []
    s = cone.get("s", []) or []
    bs = (len(cone["bu"]) + 1) if cone.get("bu") is not None and len(cone["bu"]) else int(cone.get("bsize", 0))
    return (int(cone.get("z", 0)) + int(cone.get("l", 0)) + bs + int(sum(q)) +
            int(sum(int(k) * (int(k) + 1) // 2 for k in s)) +
            int(sum(int(k) * int(k) for k in (cone.get("cs", []) or []))) +
            3 * (int(cone.get("ep", 0)) + int(cone.get("ed", 0)) + len(cone.get("p", []) or [])) +
            spectral_rows(cone))


def spectral_rows(cone):
    """rows of the spectral cones (reference cones.c:435-443); 0 for a cone without them"""
    if not is_spectral(cone):
        return 0
    rows = sum(int(d) * (int(d) + 1) // 2 + 2 for d in (cone.get("d", []) or []))
    rows += sum(int(m) * int(n) + 1 for m, n in zip(cone.get("nuc_m", []) or [], cone.get("nuc_n", []) or []))
    rows += sum(int(n) + 1 for n in (cone.get("ell1", []) or []))
    rows += sum(int(n) * (int(n) + 1) // 2 + 1 for n in (cone.get("sl_n", []) or []))
    return rows


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


def _declare(lib, ours, cone=ScsCone, T=None):
    """Declare the signatures shared by our library and the reference build (`cone`: its ScsCone layout; `T`: the
    struct classes of its integer width, Int or Long)."""
    T = T or Int
    I, IP = T.int_t, T.int_p
    ScsData, ScsSettings, ScsSolution, ScsInfo, ScsMatrix = T.ScsData, T.ScsSettings, T.ScsSolution, T.ScsInfo, T.ScsMatrix
    AaStats, ScsB200Stats = T.AaStats, T.ScsB200Stats
    lib = _Decl(lib)
    lib.scs_init.restype = C.c_void_p
    lib.scs_init.argtypes = [C.POINTER(ScsData), C.POINTER(cone), C.POINTER(ScsSettings)]
    lib.scs_solve.restype = I
    lib.scs_solve.argtypes = [C.c_void_p, C.POINTER(ScsSolution), C.POINTER(ScsInfo), I]
    lib.scs_update.restype = I
    lib.scs_update.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_finish.restype = None
    lib.scs_finish.argtypes = [C.c_void_p]
    lib.scs.restype = I
    lib.scs.argtypes = [C.POINTER(ScsData), C.POINTER(cone), C.POINTER(ScsSettings),
                        C.POINTER(ScsSolution), C.POINTER(ScsInfo)]
    lib.scs_set_default_settings.restype = None
    lib.scs_set_default_settings.argtypes = [C.POINTER(ScsSettings)]
    lib.scs_version.restype = C.c_char_p
    lib.scs_init_lin_sys_work.restype = C.c_void_p
    lib.scs_init_lin_sys_work.argtypes = [C.POINTER(ScsMatrix), C.POINTER(ScsMatrix), c_double_p]
    lib.scs_free_lin_sys_work.restype = None
    lib.scs_free_lin_sys_work.argtypes = [C.c_void_p]
    lib.scs_solve_lin_sys.restype = I
    lib.scs_solve_lin_sys.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_double]
    lib.scs_update_lin_sys_diag_r.restype = I
    lib.scs_update_lin_sys_diag_r.argtypes = [C.c_void_p, c_double_p]
    lib.scs_get_lin_sys_method.restype = C.c_char_p
    if not ours:
        return
    lib.scs_b200_linsys_last_cg_its.restype = I
    lib.scs_b200_linsys_last_cg_its.argtypes = [C.c_void_p]
    lib.scs_b200_linsys_total_cg_its.restype = C.c_longlong
    lib.scs_b200_linsys_total_cg_its.argtypes = [C.c_void_p]
    lib.scs_b200_linsys_cg_batch_solves.restype = C.c_longlong
    lib.scs_b200_linsys_cg_batch_solves.argtypes = [C.c_void_p]
    lib.scs_b200_set_cg_batch_kernel.restype = None
    lib.scs_b200_set_cg_batch_kernel.argtypes = [I]
    for f in (lib.scs_b200_accum_by_a, lib.scs_b200_accum_by_atrans):
        f.restype = I
        f.argtypes = [C.c_void_p, c_double_p, c_double_p, I]
    lib.scs_b200_time_spmv.restype = C.c_double
    lib.scs_b200_time_spmv.argtypes = [C.c_void_p, I, I, c_double_p]
    lib.scs_b200_time_cg_iter.restype = C.c_double
    lib.scs_b200_time_cg_iter.argtypes = [C.c_void_p, I, c_double_p]
    lib.scs_b200_time_cg_kernels.restype = I
    lib.scs_b200_time_cg_kernels.argtypes = [C.c_void_p, c_double_p, I, c_double_p, c_double_p]
    lib.scs_b200_time_cg_batch.restype = I
    lib.scs_b200_time_cg_batch.argtypes = [C.c_void_p, c_double_p, I, c_double_p]
    lib.scs_b200_init_cone.restype = C.c_void_p
    lib.scs_b200_init_cone.argtypes = [C.POINTER(cone), I, c_double_p]
    lib.scs_b200_proj_dual_cone.restype = I
    lib.scs_b200_proj_dual_cone.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_finish_cone.restype = None
    lib.scs_b200_finish_cone.argtypes = [C.c_void_p]
    lib.scs_b200_cone_logdet_stats.restype = I
    lib.scs_b200_cone_logdet_stats.argtypes = [C.c_void_p, IP, IP, c_double_p]
    lib.scs_b200_aa_init.restype = C.c_void_p
    lib.scs_b200_aa_init.argtypes = [I, I, I, I, C.c_double, C.c_double,
                                     C.c_double, C.c_double, I, I]
    lib.scs_b200_aa_apply.restype = C.c_double
    lib.scs_b200_aa_apply.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_aa_safeguard.restype = I
    lib.scs_b200_aa_safeguard.argtypes = [C.c_void_p, c_double_p, c_double_p]
    lib.scs_b200_aa_reset.restype = None
    lib.scs_b200_aa_reset.argtypes = [C.c_void_p]
    lib.scs_b200_aa_finish.restype = None
    lib.scs_b200_aa_finish.argtypes = [C.c_void_p]
    lib.scs_b200_aa_get_stats.restype = AaStats
    lib.scs_b200_aa_get_stats.argtypes = [C.c_void_p]
    # the device twins of the operator-level entry points (vectors in device memory, the caller's cudaStream_t last)
    for f in (lib.scs_b200_accum_by_a_device, lib.scs_b200_accum_by_atrans_device):
        f.restype = I
        f.argtypes = [C.c_void_p, c_double_p, c_double_p, I, C.c_void_p]
    lib.scs_b200_init_lin_sys_work_device.restype = C.c_void_p
    lib.scs_b200_init_lin_sys_work_device.argtypes = [C.POINTER(ScsMatrix), C.POINTER(ScsMatrix), c_double_p,
                                                      C.c_void_p]
    lib.scs_b200_solve_lin_sys_device.restype = I
    lib.scs_b200_solve_lin_sys_device.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_double, C.c_void_p]
    lib.scs_b200_update_lin_sys_diag_r_device.restype = I
    lib.scs_b200_update_lin_sys_diag_r_device.argtypes = [C.c_void_p, c_double_p, C.c_void_p]
    lib.scs_b200_proj_dual_cone_device.restype = I
    lib.scs_b200_proj_dual_cone_device.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_void_p]
    lib.scs_b200_aa_apply_device.restype = C.c_double
    lib.scs_b200_aa_apply_device.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_void_p]
    lib.scs_b200_aa_safeguard_device.restype = I
    lib.scs_b200_aa_safeguard_device.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_void_p]
    lib.scs_b200_get_stats.restype = I
    lib.scs_b200_get_stats.argtypes = [C.c_void_p, C.POINTER(ScsB200Stats)]
    lib.scs_b200_set_max_iters.restype = I
    lib.scs_b200_set_max_iters.argtypes = [C.c_void_p, I]
    lib.scs_b200_g_reuse.restype = I
    lib.scs_b200_g_reuse.argtypes = []
    lib.scs_b200_comm_unique_id.restype = I
    lib.scs_b200_comm_unique_id.argtypes = [C.c_char_p]
    lib.scs_b200_comm_init.restype = I
    lib.scs_b200_comm_init.argtypes = [I, I, C.c_char_p]
    lib.scs_b200_comm_finalize.restype = I
    lib.scs_b200_row_partition.restype = I
    lib.scs_b200_row_partition.argtypes = [I, I, IP, IP, I, IP]
    lib.scs_b200_init_device.restype = C.c_void_p
    lib.scs_b200_init_device.argtypes = [C.POINTER(ScsData), C.POINTER(cone), C.POINTER(ScsSettings), C.c_void_p]
    lib.scs_b200_update_device.restype = I
    lib.scs_b200_update_device.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_void_p]
    lib.scs_b200_update_matrix_device.restype = I
    lib.scs_b200_update_matrix_device.argtypes = [C.c_void_p, C.POINTER(ScsMatrix), C.POINTER(ScsMatrix), C.c_void_p]
    lib.scs_b200_solve_device.restype = I
    lib.scs_b200_solve_device.argtypes = [C.c_void_p, C.POINTER(ScsSolution), C.POINTER(ScsInfo), I, C.c_void_p]
    lib.scs_b200_transfer_stats.restype = None
    lib.scs_b200_transfer_stats.argtypes = [C.POINTER(C.c_longlong)]
    lib.scs_b200_transfer_stats_reset.restype = None
    lib.scs_b200_cg_k34_paths.restype = I
    lib.scs_b200_cg_k34_paths.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
    lib.scs_b200_launch_count.restype = C.c_longlong
    lib.scs_b200_device_ok.restype = I
    lib.scs_b200_release_memory.restype = None


_libs = {}


def load(spectral=False, long=False, linsys=False):
    """Load scs_b200/libscs_b200.so, or with spectral=True scs_b200/libscs_b200_spectral.so (ScsConeSpectral
    layout, nuclear-norm / l1 / sum-of-largest cones). long=True loads the DLONG flavour (64-bit scs_int; declared
    with the classes of capi.Long): libscs_b200_long.so, libscs_b200_spectral_long.so, or with linsys=True the
    plugin-only libscs_b200_linsys_long.so. Raises if it has not been built."""
    if linsys and not long:
        raise ValueError("the plugin-only library is loaded with long=True (its int flavour links into a reference tree)")
    key = (spectral, long, linsys)
    if long:
        path = LINSYS_LONG_LIB_PATH if linsys else SPECTRAL_LONG_LIB_PATH if spectral else LONG_LIB_PATH
    else:
        path = SPECTRAL_LIB_PATH if spectral else LIB_PATH
    if key not in _libs:
        if not os.path.exists(path):
            raise RuntimeError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(make -C scs_b200/csrc). There is no CPU fallback.")
        # RTLD_LOCAL: our scs_* symbols must not interpose on the reference build loaded by the tests
        lib = C.CDLL(path, mode=C.RTLD_LOCAL)
        T = abi(long)
        _declare(lib, ours=True, cone=T.ScsConeSpectral if spectral else T.ScsCone, T=T)
        _libs[key] = lib
    return _libs[key]


def load_reference(path, spectral=False, long=False):
    """Load a build of the UNMODIFIED reference (oracle/_ref/*.so; long=True: a DLONG=1 build). Test infrastructure
    only."""
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
    T = abi(long)
    _declare(lib, ours=False, cone=T.ScsConeSpectral if spectral else T.ScsCone, T=T)
    return lib


def default_settings(lib, long=False, **over):
    st = abi(long).ScsSettings()
    lib.scs_set_default_settings(C.byref(st))
    for k, v in over.items():
        setattr(st, k, v)
    return st

"""PyTorch front end of the operator-level device entry points (include/scs_b200.h group (3)): the cone projection,
the KKT solve with its SpMV pair, and Anderson acceleration on CUDA tensors, with no copy through host memory::

    proj = ConeProjector({"l": 100, "q": [50], "s": [10]})
    y = proj.project_dual(x)                      # Pi_{K*}(x), a new tensor
    z = proj.project(x)                           # Pi_K(x) = x + Pi_{K*}(-x)

    kkt = LinSys(A, diag_r)                       # [[R_x + P, A'], [A, -R_y]]
    xy = kkt.solve(rhs, warm=x0, tol=1e-6)        # [x; y]
    Ax = kkt.A_mul(x)

    aa = Anderson(dim, mem=10)
    aa.apply(f, x)                                # f updated in place

Vectors are 1-D CUDA float64 tensors on the library's device (``SCS_B200_DEVICE`` / ``LOCAL_RANK``); ``A`` (m x n)
and ``P`` (n x n, its upper triangle) are CUDA ``torch.sparse_csc_tensor``s, as for ``torch_solver.SCS``. int32
indices go to libscs_b200.so and int64 indices to the DLONG library; a cone with spectral keys selects the spectral
library. Every call is ordered on ``torch.cuda.current_stream()``. One object per thread is supported, as for ``SCS``.
Every argument is checked with a Python error before the library is loaded or called; the cone and AA workspaces are
made at their first call.
"""
import ctypes as C

import numpy as np
import torch

from . import capi
from .torch_solver import _check_csc, _check_device, _check_vector, _dptr, _library_device, _matrix


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _vector(name, t, length, device, out=False):
    """t checked as a CUDA float64 vector of `length` on `device`; an input is made contiguous, an output (written in
    place) must already be"""
    _check_vector(name, t, length)
    _check_device(name, t, device)
    if t.is_contiguous():
        return t
    if out:
        raise ValueError(f"{name} is written in place and must be contiguous")
    return t.contiguous()


class ConeProjector:
    """The cone operator (scs_b200_init_cone / scs_b200_proj_dual_cone_device) on CUDA tensors. `cone` is a dict as
    for ``SCS``; D (length m, numpy or a tensor on any device) is the row scaling the box bounds follow, read on the
    host here and not kept."""

    def __init__(self, cone, D=None):
        self.cone = dict(cone)
        self.m = capi.cone_rows(self.cone)
        self._device = _library_device()
        self._D = None
        if D is not None:
            if isinstance(D, torch.Tensor):
                if D.dtype != torch.float64:
                    raise ValueError(f"D must be float64, got {D.dtype}")
                D = D.detach().cpu().numpy()
            D = np.ascontiguousarray(D, dtype=np.float64)
            if D.shape != (self.m,):
                raise ValueError(f"D must have shape ({self.m},), got {D.shape}")
            self._D = D
        self._lib = self._work = None

    def _workspace(self):
        if self._work is None:
            spectral = capi.is_spectral(self.cone)
            lib = capi.load(spectral=spectral)
            k, _keep = capi.make_cone(self.cone, spectral=spectral)
            work = lib.scs_b200_init_cone(C.byref(k), self.m, capi.dptr(self._D))
            if not work:
                raise ValueError("scs_b200_init_cone refused the cone (its message is printed above)")
            self._lib, self._work = lib, work
        return self._lib, self._work

    def project_dual_(self, x, r_y=None):
        """x := Pi_{K*}(x) under the R_y metric when r_y (length m) is given, in place; returns x"""
        _vector("x", x, self.m, self._device, out=True)
        if r_y is not None:
            r_y = _vector("r_y", r_y, self.m, self._device)
        lib, work = self._workspace()
        rc = lib.scs_b200_proj_dual_cone_device(work, _dptr(x), _dptr(r_y) if r_y is not None else None,
                                                _stream(self._device))
        if rc != 0:
            raise RuntimeError("scs_b200_proj_dual_cone_device failed (its message is printed above)")
        return x

    def project_dual(self, x, r_y=None):
        """Pi_{K*}(x) (under the R_y metric when r_y is given), a new tensor"""
        _vector("x", x, self.m, self._device)
        return self.project_dual_(x.clone(memory_format=torch.contiguous_format), r_y)

    def project(self, x):
        """Pi_K(x) = x + Pi_{K*}(-x) (Moreau), a new tensor"""
        _vector("x", x, self.m, self._device)
        return x + self.project_dual_(-x)

    def logdet_stats(self):
        """(iter, newton_success, (three residuals)) of the last log-det cone the last projection handled, or None
        when the cone has no log-det cones"""
        lib, work = self._workspace()
        T = capi.abi(False)
        it, ok, res = T.int_t(), T.int_t(), (C.c_double * 3)()
        if lib.scs_b200_cone_logdet_stats(work, C.byref(it), C.byref(ok), res) != 0:
            return None
        return it.value, ok.value, tuple(res)

    def close(self):
        if self._work:
            torch.cuda.current_stream(self._device).synchronize()
            self._lib.scs_b200_finish_cone(self._work)
            self._work = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LinSys:
    """SCS's KKT system [[R_x + P, A'], [A, -R_y]] on the device (scs_b200_init_lin_sys_work_device), with the SpMV
    pair of its A. diag_r = [R_x; R_y] (n + m)."""

    def __init__(self, A, diag_r, P=None):
        _check_csc("A", A, None)
        m, n = A.shape
        if P is not None:
            _check_csc("P", P, (n, n))
            if P.ccol_indices().dtype != A.ccol_indices().dtype:
                raise ValueError("A and P must have the same index dtype")
        _check_vector("diag_r", diag_r, n + m)
        device = _library_device()
        _check_device("A", A, device)
        if P is not None:
            _check_device("P", P, device)
        diag_r = _vector("diag_r", diag_r, n + m, device)
        self.m, self.n, self._device = m, n, device
        self._long = A.ccol_indices().dtype == torch.int64
        self._lib = capi.load(long=self._long)
        T = capi.abi(self._long)
        keep = []
        Am = _matrix(A, T, keep)
        Pm = _matrix(P, T, keep) if P is not None else None
        self._work = self._lib.scs_b200_init_lin_sys_work_device(C.byref(Am), C.byref(Pm) if Pm is not None else None,
                                                                 _dptr(diag_r), _stream(device))
        if not self._work:
            raise ValueError("scs_b200_init_lin_sys_work_device refused the system (its message is printed above)")

    def solve(self, rhs, warm=None, tol=1e-12):
        """[x; y] solving the KKT system for rhs (n + m), a new tensor; warm (n) is the CG warm start"""
        rhs = _vector("rhs", rhs, self.n + self.m, self._device)
        if warm is not None:
            warm = _vector("warm", warm, self.n, self._device)
        out = rhs.clone()  # a fresh block: the CG loop reads x two entries at a time and needs it 16-byte aligned
        rc = self._lib.scs_b200_solve_lin_sys_device(self._work, _dptr(out), _dptr(warm) if warm is not None else None,
                                                     float(tol), _stream(self._device))
        if rc != 0:
            raise RuntimeError("scs_b200_solve_lin_sys_device failed (its message is printed above)")
        return out

    @property
    def last_cg_its(self):
        """CG iterations of the last solve"""
        return int(self._lib.scs_b200_linsys_last_cg_its(self._work))

    def update_diag_r(self, diag_r):
        """new [R_x; R_y] (n + m)"""
        diag_r = _vector("diag_r", diag_r, self.n + self.m, self._device)
        if self._lib.scs_b200_update_lin_sys_diag_r_device(self._work, _dptr(diag_r), _stream(self._device)) != 0:
            raise RuntimeError("scs_b200_update_lin_sys_diag_r_device failed (its message is printed above)")

    def _mul(self, f, xname, x, xlen, yname, y, ylen):
        x = _vector(xname, x, xlen, self._device)
        accumulate = y is not None
        if accumulate:
            _vector(yname, y, ylen, self._device, out=True)
        else:
            y = torch.empty(ylen, dtype=torch.float64, device=x.device)
        if f(self._work, _dptr(x), _dptr(y), int(accumulate), _stream(self._device)) != 0:
            raise RuntimeError("the device SpMV refused its arguments (its message is printed above)")
        return y

    def A_mul(self, x, y=None):
        """A x, a new tensor; with y given, y += A x in place, returned"""
        return self._mul(self._lib.scs_b200_accum_by_a_device, "x", x, self.n, "y", y, self.m)

    def At_mul(self, y, x=None):
        """A' y, a new tensor; with x given, x += A' y in place, returned"""
        return self._mul(self._lib.scs_b200_accum_by_atrans_device, "y", y, self.m, "x", x, self.n)

    def close(self):
        if getattr(self, "_work", None):
            torch.cuda.current_stream(self._device).synchronize()
            self._lib.scs_free_lin_sys_work(self._work)
            self._work = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_AA_STATS = ("iter", "n_accept", "n_reject_lapack", "n_reject_rank0", "n_reject_nonfinite", "n_reject_weight_cap",
             "n_safeguard_reject", "last_rank", "last_aa_norm", "last_regularization")


class Anderson:
    """Anderson acceleration of a fixed-point map x -> f(x) in `dim` entries (scs_b200_aa_init with min_len = mem, as
    SCS runs it), used as the reference's aa.h documents: after each map application, apply(f, x) with x the input
    of the map and f its output, then safeguard with the next pair."""

    def __init__(self, dim, mem=10, type1=True, regularization=1e-8, relaxation=1.0, safeguard_factor=1.0,
                 max_weight_norm=1e10, ir_max_steps=5):
        self.dim = int(dim)
        if self.dim <= 0:
            raise ValueError(f"dim must be positive, got {dim}")
        self._args = (self.dim, int(mem), int(mem), int(bool(type1)), float(regularization), float(relaxation),
                      float(safeguard_factor), float(max_weight_norm), int(ir_max_steps), 0)
        self._device = _library_device()
        self._lib = self._work = None

    def _workspace(self):
        if self._work is None:
            lib = capi.load()
            work = lib.scs_b200_aa_init(*self._args)
            if not work:
                raise ValueError("scs_b200_aa_init refused its arguments")
            self._lib, self._work = lib, work
        return self._lib, self._work

    def apply(self, f, x):
        """f := the accelerated iterate, in place; returns aa_norm (> 0 accepted, <= 0 not, as the reference)"""
        _vector("f", f, self.dim, self._device, out=True)
        x = _vector("x", x, self.dim, self._device)
        lib, work = self._workspace()
        nrm = lib.scs_b200_aa_apply_device(work, _dptr(f), _dptr(x), _stream(self._device))
        if nrm != nrm:
            raise RuntimeError("scs_b200_aa_apply_device refused its arguments (its message is printed above)")
        return nrm

    def safeguard(self, f_new, x_new):
        """0, or -1 when the step is rejected: f_new and x_new are then restored in place"""
        _vector("f_new", f_new, self.dim, self._device, out=True)
        _vector("x_new", x_new, self.dim, self._device, out=True)
        lib, work = self._workspace()
        return int(lib.scs_b200_aa_safeguard_device(work, _dptr(f_new), _dptr(x_new), _stream(self._device)))

    def reset(self):
        """forget the history (the next apply starts a new one)"""
        lib, work = self._workspace()
        lib.scs_b200_aa_reset(work)

    def stats(self):
        lib, work = self._workspace()
        st = lib.scs_b200_aa_get_stats(work)
        return {key: getattr(st, key) for key in _AA_STATS}

    def close(self):
        if self._work:
            torch.cuda.current_stream(self._device).synchronize()
            self._lib.scs_b200_aa_finish(self._work)
            self._work = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

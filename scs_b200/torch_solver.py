"""PyTorch front end of the device-data entry points (include/scs_b200.h): the problem goes in as CUDA tensors and the
solution comes back as CUDA tensors, with no copy through host memory. The interface mirrors the ``scs`` Python
package::

    solver = SCS({"A": A, "P": P, "b": b, "c": c}, cone, eps_abs=1e-6, verbose=0)
    sol = solver.solve()                    # {"x", "y", "s", "info"}
    solver.update(b=b2)
    sol = solver.solve(warm_start=True)

``A`` (m x n) and ``P`` (n x n, its upper triangle; optional) are CUDA ``torch.sparse_csc_tensor``s with float64
values, ``b`` (m) and ``c`` (n) CUDA float64 tensors, all on the library's device (``SCS_B200_DEVICE`` /
``LOCAL_RANK``). int32 indices go to libscs_b200.so and int64 indices to the DLONG library, without a conversion; a
cone with spectral keys selects the spectral flavour. Work is ordered with ``torch.cuda.current_stream()``.

One ``SCS`` object per thread is supported: threads solve their own problems at the same time, each on its own
stream inside the library, ordered with that thread's current stream (PyTorch's current stream is per thread).
"""
import ctypes as C
import os

import torch

from . import capi

_INFO_KEYS = ("iter", "status_val", "scale_updates", "pobj", "dobj", "res_pri", "res_dual", "gap", "res_infeas",
              "res_unbdd_a", "res_unbdd_p", "setup_time", "solve_time", "scale", "comp_slack",
              "rejected_accel_steps", "accepted_accel_steps", "lin_sys_time", "cone_time", "accel_time")


def _library_device():
    """the CUDA device index the library drives (kernels/runtime.cu: SCS_B200_DEVICE, else LOCAL_RANK, else 0)"""
    e = os.environ.get("SCS_B200_DEVICE", os.environ.get("LOCAL_RANK", "0"))
    return int(e) % max(1, torch.cuda.device_count())


def _check_device(name, t, device):
    if t.device.type != "cuda":
        raise ValueError(f"{name} must be a CUDA tensor, got one on {t.device}")
    if device is not None and t.device.index != device:
        raise ValueError(f"{name} is on cuda:{t.device.index}; the library drives cuda:{device}")


def _check_vector(name, t, length):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if t.layout != torch.strided:
        raise ValueError(f"{name} must be a dense tensor, got layout {t.layout}")
    if t.dtype != torch.float64:
        raise ValueError(f"{name} must be float64, got {t.dtype}")
    if tuple(t.shape) != (length,):
        raise ValueError(f"{name} must have shape ({length},), got {tuple(t.shape)}")


def _check_csc(name, t, shape):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if t.layout != torch.sparse_csc:
        raise ValueError(f"{name} must be a torch.sparse_csc_tensor, got layout {t.layout}")
    if t.dtype != torch.float64:
        raise ValueError(f"{name} must have float64 values, got {t.dtype}")
    if t.ccol_indices().dtype not in (torch.int32, torch.int64):
        raise ValueError(f"{name} must have int32 or int64 indices, got {t.ccol_indices().dtype}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")


def check_args(data, device=None):
    """Every argument check of SCS, raised as a Python error before the library is loaded or called. Returns
    (m, n, the index dtype)."""
    A = data.get("A")
    _check_csc("A", A, None)
    m, n = A.shape
    P = data.get("P")
    if P is not None:
        _check_csc("P", P, (n, n))
        if P.ccol_indices().dtype != A.ccol_indices().dtype:
            raise ValueError("A and P must have the same index dtype")
    _check_vector("b", data.get("b"), m)
    _check_vector("c", data.get("c"), n)
    if device is None:
        device = _library_device()
    for name, t in (("A", A), ("P", P), ("b", data["b"]), ("c", data["c"])):
        if t is not None:
            _check_device(name, t, device)
    return m, n, A.ccol_indices().dtype


def _dptr(t):
    return C.cast(C.c_void_p(t.data_ptr()), capi.c_double_p)


def _iptr(t, T):
    return C.cast(C.c_void_p(t.data_ptr()), T.int_p)


def _matrix(M, T, keep):
    """the ScsMatrix (struct classes T) of a CUDA sparse-CSC tensor, pointing into its arrays; the contiguous arrays
    are appended to `keep`, which must outlive the call that reads them"""
    p, i, x = M.ccol_indices().contiguous(), M.row_indices().contiguous(), M.values().contiguous()
    keep.extend((p, i, x))
    return T.ScsMatrix(_dptr(x), _iptr(i, T), _iptr(p, T), M.shape[0], M.shape[1])


class SCS:
    """A problem resident on the GPU (scs_b200_init_device), solved and updated in place there."""

    def __init__(self, data, cone, **settings):
        self.m, self.n, idx = check_args(data)
        self.device = data["A"].device
        self._long = idx == torch.int64
        self._has_P = data.get("P") is not None
        spectral = capi.is_spectral(cone)
        self._lib = capi.load(spectral=spectral, long=self._long)
        T = capi.abi(self._long)
        self._T = T
        self._keep = []  # the tensors the structs point into, alive as long as the call needs them
        A = _matrix(data["A"], T, self._keep)
        P = _matrix(data["P"], T, self._keep) if data.get("P") is not None else None
        b, c = data["b"].contiguous(), data["c"].contiguous()
        self._keep += [b, c]
        d = T.ScsData(self.m, self.n, C.pointer(A), C.pointer(P) if P is not None else C.POINTER(T.ScsMatrix)(),
                      _dptr(b), _dptr(c))
        k, _cone_keep = capi.make_cone(cone, spectral=spectral, long=self._long)
        st = capi.default_settings(self._lib, long=self._long, **settings)
        self._work = self._lib.scs_b200_init_device(C.byref(d), C.byref(k), C.byref(st), self._stream())
        self._keep = []
        if not self._work:
            raise ValueError("scs_b200_init_device refused the problem (its message is printed above)")
        self._sol = None

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def update(self, b=None, c=None, A=None, P=None):
        """new b and / or c (CUDA float64) and / or new values of A and P (CUDA sparse-CSC tensors with the pattern the
        solver was built with: scs_b200_update_matrix_device); None keeps the current one. A solver built with P takes
        P with every A, and P only with A. The matrices are updated first, then b and c; the previous solution stays
        the warm start."""
        if b is not None:
            _check_vector("b", b, self.m)
            _check_device("b", b, self.device.index)
            b = b.contiguous()
        if c is not None:
            _check_vector("c", c, self.n)
            _check_device("c", c, self.device.index)
            c = c.contiguous()
        if P is not None and A is None:
            raise ValueError("P is updated together with A: pass A as well")
        if A is not None:
            if P is None and self._has_P:
                raise ValueError("this solver was built with P: pass P together with A")
            if P is not None and not self._has_P:
                raise ValueError("this solver was built without P; P cannot be added by an update")
            idx = torch.int64 if self._long else torch.int32
            for name, M, shape in (("A", A, (self.m, self.n)), ("P", P, (self.n, self.n))):
                if M is None:
                    continue
                _check_csc(name, M, shape)
                if M.ccol_indices().dtype != idx:
                    raise ValueError(f"{name} must have {idx} indices, as the solver was built with, "
                                     f"got {M.ccol_indices().dtype}")
                _check_device(name, M, self.device.index)
            keep = []
            Am = _matrix(A, self._T, keep)
            Pm = _matrix(P, self._T, keep) if P is not None else None
            rc = self._lib.scs_b200_update_matrix_device(self._work, C.byref(Am),
                                                         C.byref(Pm) if Pm is not None else None, self._stream())
            if rc != 0:
                raise RuntimeError("scs_b200_update_matrix_device refused the matrices (its message is printed above)")
        if A is not None and b is None and c is None:
            return
        rc = self._lib.scs_b200_update_device(self._work, _dptr(b) if b is not None else None,
                                              _dptr(c) if c is not None else None, self._stream())
        if rc != 0:
            raise RuntimeError("scs_b200_update_device failed")

    def solve(self, warm_start=True, x=None, y=None, s=None):
        """{"x", "y", "s": new CUDA tensors, "info": dict}. With warm_start, the start is x, y, s where given, else
        the previous solution (a cold start when there is none)."""
        prev = self._sol
        out = []
        for name, v, length, i in (("x", x, self.n, 0), ("y", y, self.m, 1), ("s", s, self.m, 2)):
            if v is not None:
                _check_vector(name, v, length)
                _check_device(name, v, self.device.index)
                out.append(v.clone())
            elif prev is not None:
                out.append(prev[i].clone())
            else:
                out.append(torch.zeros(length, dtype=torch.float64, device=self.device))
        warm = bool(warm_start) and (prev is not None or x is not None or y is not None or s is not None)
        sol = self._T.ScsSolution(_dptr(out[0]), _dptr(out[1]), _dptr(out[2]))
        info = self._T.ScsInfo()
        rc = self._lib.scs_b200_solve_device(self._work, C.byref(sol), C.byref(info), int(warm), self._stream())
        if rc == -1 and not info.lin_sys_solver:  # refused before the solve started (-1 is also SCS_UNBOUNDED)
            raise RuntimeError("scs_b200_solve_device refused the call (its message is printed above)")
        self._sol = tuple(out)
        d = {key: getattr(info, key) for key in _INFO_KEYS}
        d["status"] = info.status.decode()
        return {"x": out[0], "y": out[1], "s": out[2], "info": d}

    def close(self):
        if getattr(self, "_work", None):
            torch.cuda.current_stream(self.device).synchronize()
            self._lib.scs_finish(self._work)
            self._work = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

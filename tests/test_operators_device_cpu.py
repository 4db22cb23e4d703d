"""The operator-level device twins without a GPU: every library flavour that exports a host twin exports its device
twin, and the PyTorch operator classes refuse bad arguments with a Python error before they load the library."""
import ctypes as C
import os
import re

import pytest
import torch

from scs_b200 import capi, torch_ops

TWINS = {
    "scs_b200_proj_dual_cone": "scs_b200_proj_dual_cone_device",
    "scs_b200_accum_by_a": "scs_b200_accum_by_a_device",
    "scs_b200_accum_by_atrans": "scs_b200_accum_by_atrans_device",
    "scs_init_lin_sys_work": "scs_b200_init_lin_sys_work_device",
    "scs_solve_lin_sys": "scs_b200_solve_lin_sys_device",
    "scs_update_lin_sys_diag_r": "scs_b200_update_lin_sys_diag_r_device",
    "scs_b200_aa_apply": "scs_b200_aa_apply_device",
    "scs_b200_aa_safeguard": "scs_b200_aa_safeguard_device",
}
LIBS = [capi.LIB_PATH, capi.SPECTRAL_LIB_PATH, capi.LONG_LIB_PATH, capi.SPECTRAL_LONG_LIB_PATH,
        capi.LINSYS_LONG_LIB_PATH, os.path.join(os.path.dirname(capi.LIB_PATH), "libscs_b200_linsys.so")]


@pytest.mark.parametrize("path", LIBS, ids=os.path.basename)
def test_every_host_twin_has_its_device_twin(path):
    if not os.path.exists(path) and path == LIBS[-1]:
        pytest.skip("the int plugin-only library is built on request (make -C scs_b200/csrc linsys)")
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    for host, device in TWINS.items():
        assert hasattr(lib, host), (os.path.basename(path), host)
        assert hasattr(lib, device), (os.path.basename(path), device)


@pytest.fixture
def no_library(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(capi, "load", refuse)


def _A(idx=torch.int32, dense=False):
    A = torch.sparse_csc_tensor(torch.tensor([0, 1, 2], dtype=idx), torch.tensor([0, 2], dtype=idx),
                                torch.tensor([1.0, 2.0], dtype=torch.float64), size=(3, 2))
    return A.to_dense() if dense else A


def _P(idx=torch.int32):
    return torch.sparse_csc_tensor(torch.tensor([0, 1, 2], dtype=idx), torch.tensor([0, 1], dtype=idx),
                                   torch.tensor([1.0, 1.0], dtype=torch.float64), size=(2, 2))


def _v(n, **kw):
    return torch.ones(n, dtype=torch.float64, **kw)


LINSYS_BAD = {
    "cpu tensors": (lambda: (_A(), _v(5), None), "must be a CUDA tensor"),
    "dense A": (lambda: (_A(dense=True), _v(5), None), "sparse_csc"),
    "csr A": (lambda: (_A().to_sparse_csr(), _v(5), None), "sparse_csc"),
    "float32 A": (lambda: (_A().to(torch.float32), _v(5), None), "float64"),
    "float32 diag_r": (lambda: (_A(), _v(5).float(), None), "float64"),
    "short diag_r": (lambda: (_A(), _v(4), None), "shape (5,)"),
    "2-d diag_r": (lambda: (_A(), _v(5).reshape(5, 1), None), "shape (5,)"),
    "P not square": (lambda: (_A(), _v(5), _A()), "shape (2, 2)"),
    "P of another index dtype": (lambda: (_A(), _v(5), _P(torch.int64)), "same index dtype"),
    "numpy diag_r": (lambda: (_A(), _v(5).numpy(), None), "torch.Tensor"),
}


@pytest.mark.parametrize("case", sorted(LINSYS_BAD))
def test_linsys_refuses_bad_arguments_before_the_library(no_library, case):
    make, message = LINSYS_BAD[case]
    A, diag_r, P = make()
    with pytest.raises((ValueError, TypeError), match=re.escape(message)):
        torch_ops.LinSys(A, diag_r, P=P)


CONE = {"z": 1, "l": 2, "q": [3]}  # m = 6
CONE_BAD = {
    "cpu x": (lambda p: p.project_dual(_v(6)), "must be a CUDA tensor"),
    "cpu x in place": (lambda p: p.project_dual_(_v(6)), "must be a CUDA tensor"),
    "cpu x primal": (lambda p: p.project(_v(6)), "must be a CUDA tensor"),
    "float32 x": (lambda p: p.project_dual(_v(6).float()), "float64"),
    "short x": (lambda p: p.project_dual(_v(5)), "shape (6,)"),
    "batched x": (lambda p: p.project(_v(12).reshape(2, 6)), "shape (6,)"),
    "numpy x": (lambda p: p.project_dual(_v(6).numpy()), "torch.Tensor"),
    "r_y to project": (lambda p: p.project(_v(6), r_y=_v(6)), "r_y"),
}


@pytest.mark.parametrize("case", sorted(CONE_BAD))
def test_cone_projector_refuses_bad_arguments_before_the_library(no_library, case):
    make, message = CONE_BAD[case]
    with pytest.raises((ValueError, TypeError), match=re.escape(message)):
        make(torch_ops.ConeProjector(CONE))


def test_cone_projector_checks_D(no_library):
    with pytest.raises(ValueError, match=re.escape("shape (6,)")):
        torch_ops.ConeProjector(CONE, D=_v(5))
    with pytest.raises(ValueError, match="float64"):
        torch_ops.ConeProjector(CONE, D=_v(6).float())


AA_BAD = {
    "cpu f": (lambda a: a.apply(_v(4), _v(4)), "must be a CUDA tensor"),
    "float32 f": (lambda a: a.apply(_v(4).float(), _v(4)), "float64"),
    "cpu f_new": (lambda a: a.safeguard(_v(4), _v(4)), "must be a CUDA tensor"),
    "wrong shape": (lambda a: a.apply(_v(3), _v(4)), "shape (4,)"),
}


@pytest.mark.parametrize("case", sorted(AA_BAD))
def test_anderson_refuses_bad_arguments_before_the_library(no_library, case):
    make, message = AA_BAD[case]
    with pytest.raises((ValueError, TypeError), match=re.escape(message)):
        make(torch_ops.Anderson(4, mem=3))

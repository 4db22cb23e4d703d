"""The device-data entry points without a GPU: the four full libraries export them (the linsys-only ones do not), and
the PyTorch front end refuses bad arguments with a Python error before it loads or calls the library."""
import ctypes as C
import os
import re

import pytest
import torch

from scs_b200 import capi, torch_solver

SYMBOLS = ("scs_b200_init_device", "scs_b200_update_device", "scs_b200_solve_device", "scs_b200_transfer_stats",
           "scs_b200_transfer_stats_reset")


@pytest.mark.parametrize("path", [capi.LIB_PATH, capi.SPECTRAL_LIB_PATH, capi.LONG_LIB_PATH,
                                  capi.SPECTRAL_LONG_LIB_PATH])
def test_full_libraries_export_the_device_entry_points(path):
    lib = C.CDLL(path, mode=C.RTLD_LOCAL)
    for name in SYMBOLS:
        assert hasattr(lib, name), (os.path.basename(path), name)


def test_linsys_library_has_no_device_data_entry_points():
    lib = C.CDLL(capi.LINSYS_LONG_LIB_PATH, mode=C.RTLD_LOCAL)
    assert not hasattr(lib, "scs_b200_init_device")


def _data(idx=torch.int32):
    A = torch.sparse_csc_tensor(torch.tensor([0, 1, 2], dtype=idx), torch.tensor([0, 1], dtype=idx),
                                torch.tensor([1.0, 2.0], dtype=torch.float64), size=(3, 2))
    return {"A": A, "b": torch.ones(3, dtype=torch.float64), "c": torch.ones(2, dtype=torch.float64)}


BAD = {
    "cpu tensors": (lambda d: d, "must be a CUDA tensor"),
    "dense A": (lambda d: {**d, "A": d["A"].to_dense()}, "sparse_csc"),
    "csr A": (lambda d: {**d, "A": d["A"].to_sparse_csr()}, "sparse_csc"),
    "float32 A": (lambda d: {**d, "A": d["A"].to(torch.float32)}, "float64"),
    "int16 indices": (lambda d: {**d, "A": torch.sparse_csc_tensor(d["A"].ccol_indices().to(torch.int16),
                                                                   d["A"].row_indices().to(torch.int16),
                                                                   d["A"].values(), size=(3, 2))}, "int32 or int64"),
    "float32 b": (lambda d: {**d, "b": d["b"].float()}, "float64"),
    "short b": (lambda d: {**d, "b": d["b"][:2]}, "shape (3,)"),
    "2-d c": (lambda d: {**d, "c": d["c"].reshape(2, 1)}, "shape (2,)"),
    "P not square": (lambda d: {**d, "P": d["A"]}, "shape (2, 2)"),
    "P of another index dtype": (lambda d: {**d, "P": torch.sparse_csc_tensor(
        torch.tensor([0, 1, 2]), torch.tensor([0, 1]), torch.tensor([1.0, 1.0], dtype=torch.float64), size=(2, 2))},
        "same index dtype"),
    "numpy b": (lambda d: {**d, "b": d["b"].numpy()}, "torch.Tensor"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_front_end_refuses_bad_arguments_before_the_library(monkeypatch, case):
    def no_library(*a, **k):
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(capi, "load", no_library)
    make, message = BAD[case]
    with pytest.raises((ValueError, TypeError), match=re.escape(message)):
        torch_solver.SCS(make(_data()), {"l": 3})

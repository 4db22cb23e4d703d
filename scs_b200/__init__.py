"""scs_b200 -- H100-native (sm_90a) ADMM hot path for SCS behind SCS's own C ABI.

The product is the shared library ``scs_b200/libscs_b200.so`` (C ABI declared in
``include/scs_b200.h``). This Python package only holds the ctypes mirror used
by the tests and the benchmark, and the synthetic problem generators.
"""
from . import capi  # noqa: F401

__all__ = ["capi"]
__version__ = "0.1.0"

"""scs_b200_update_matrix_device without a GPU: declared in include/scs_b200_device.h (not in scs_b200.h, whose
functions the plugin-only library must export) and exported by the four full libraries."""
import ctypes as C
import os
import re

import pytest

from scs_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "scs_b200_update_matrix_device"


def test_declared_in_the_device_header_only():
    with open(os.path.join(ROOT, "include", "scs_b200_device.h")) as f:
        dev = f.read()
    with open(os.path.join(ROOT, "include", "scs_b200.h")) as f:
        main = f.read()
    assert re.search(r"scs_int\s+scs_b200_update_matrix_device\s*\(\s*ScsWork\s*\*\s*w\s*,\s*const ScsMatrix\s*\*\s*A"
                     r"\s*,\s*const ScsMatrix\s*\*\s*P\s*,\s*void\s*\*\s*stream\s*\)\s*;", dev)
    assert NAME not in main


@pytest.mark.parametrize("path", [capi.LIB_PATH, capi.SPECTRAL_LIB_PATH, capi.LONG_LIB_PATH,
                                  capi.SPECTRAL_LONG_LIB_PATH])
def test_full_libraries_export_it(path):
    assert hasattr(C.CDLL(path, mode=C.RTLD_LOCAL), NAME), os.path.basename(path)


def test_linsys_library_does_not():
    assert not hasattr(C.CDLL(capi.LINSYS_LONG_LIB_PATH, mode=C.RTLD_LOCAL), NAME)

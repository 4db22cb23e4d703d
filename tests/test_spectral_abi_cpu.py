"""CPU: the spectral build's ABI. libscs_b200_spectral.so takes the reference's USE_SPECTRAL_CONES ScsCone
(include/scs.h:154-171: 184 bytes) and exports the same symbols as libscs_b200.so, whose ScsCone stays 104 bytes."""
import ctypes as C
import os
import subprocess

from scs_b200 import capi


def test_spectral_cone_layout():
    assert C.sizeof(capi.ScsCone) == 104
    S = capi.ScsConeSpectral
    assert C.sizeof(S) == 184
    assert (S.d.offset, S.dsize.offset, S.nuc_m.offset, S.nuc_n.offset, S.nucsize.offset) == (104, 112, 120, 128, 136)
    assert (S.ell1.offset, S.ell1_size.offset, S.sl_n.offset, S.sl_k.offset, S.sl_size.offset) == (144, 152, 160, 168, 176)


def test_make_cone_without_spectral_keys_is_unchanged():
    cone = {"z": 3, "l": 4, "q": [3, 5], "s": [2], "ep": 1, "p": [0.5]}
    k, _ = capi.make_cone(cone)
    assert type(k) is capi.ScsCone and C.sizeof(k) == 104
    assert capi.cone_rows(cone) == 3 + 4 + 8 + 3 + 3 + 3
    k2, _ = capi.make_cone({"l": 2, "ell1": [4], "nuc_m": [3], "nuc_n": [2], "sl_n": [3], "sl_k": [1]})
    assert type(k2) is capi.ScsConeSpectral
    assert (k2.ell1_size, k2.nucsize, k2.sl_size, k2.dsize) == (1, 1, 1, 0)
    assert capi.cone_rows({"l": 2, "ell1": [4], "nuc_m": [3], "nuc_n": [2], "sl_n": [3], "sl_k": [1]}) == \
        2 + 5 + 7 + 7


def exported(path):
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True, check=True).stdout
    return sorted(line.split()[-1] for line in out.splitlines() if line.split()[-2] in ("T", "W"))


def test_spectral_library_exports_the_same_symbols():
    assert os.path.exists(capi.SPECTRAL_LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    assert exported(capi.SPECTRAL_LIB_PATH) == exported(capi.LIB_PATH)
    assert capi.load(spectral=True).scs_version().decode().endswith("b200")

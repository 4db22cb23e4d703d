"""CPU: the spectral cones without a GPU.

* tests/spectral_numpy.py (the projections restated from the math) agrees with the reference spectral build's
  answers recorded in tests/golden/spectral_cones.npz (on the inputs of tests/spectral_cases.py) to 1e-13, and with
  the live build where oracle/_ref has it;
* problem files with spectral cones round-trip through scs_b200_read_data / scs_b200_write_data of the spectral
  library, byte for byte, and match the reference spectral writer where it is built;
* a file with log-det cones is read, then refused by scs_init with a message naming the log-det cone."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import spectral_cases
import spectral_numpy
from conftest import REF_DIR, ROOT
from scs_b200 import capi

GOLD = os.path.join(ROOT, "tests", "golden")
PROB_DIR = os.path.join(GOLD, "problems", "spectral")
OPS = np.load(os.path.join(GOLD, "spectral_cones.npz"))
REF_SPECTRAL = os.path.join(REF_DIR, "libscsindir_ref_spectral.so")
PP = C.POINTER


def numpy_proj_dual(cone, x):
    """the Moreau wrapper with r_y = NULL on a cone of spectral rows only (plus zero / LP / SOC / PSD rows)"""
    return spectral_numpy.proj_dual_cone(x, cone)


@pytest.mark.parametrize("name", [str(n) for n in OPS["names"]])
def test_numpy_restatement_matches_reference(name):
    cone, xs = spectral_cases.inputs(name)
    assert len(xs) == int(OPS[f"{name}/n"][0])
    for i, x in enumerate(xs):
        spectral_cases.check_regenerated(OPS, name, i, x)
        idx, ref = spectral_cases.recorded(OPS, name, i, False)
        mine = numpy_proj_dual(cone, x)[idx]
        err = np.abs(mine - ref).max() / max(np.abs(ref).max(), np.abs(x).max(), 1e-300)
        assert err <= 1e-13, (name, i, err)


@pytest.mark.skipif(not os.path.exists(REF_SPECTRAL), reason="oracle/_ref spectral build not built")
def test_numpy_restatement_matches_live_reference():
    lib = capi.load_reference(REF_SPECTRAL, spectral=True)
    lib._scs_init_cone.restype = C.c_void_p
    lib._scs_init_cone.argtypes = [PP(capi.ScsConeSpectral), C.c_int]
    lib._scs_proj_dual_cone.argtypes = [capi.c_double_p, C.c_void_p, C.c_void_p, capi.c_double_p]
    lib._scs_finish_cone.argtypes = [C.c_void_p]
    rng = np.random.default_rng(77)
    cone = {"nuc_m": [6, 4], "nuc_n": [3, 4], "ell1": [1, 7, 50], "sl_n": [5, 8], "sl_k": [2, 7]}
    m = capi.cone_rows(cone)
    for trial in range(5):
        x = rng.standard_normal(m) * 10.0 ** rng.integers(-2, 3)
        k, keep = capi.make_cone(cone)
        cw = lib._scs_init_cone(C.byref(k), m)
        ref = x.copy()
        assert lib._scs_proj_dual_cone(capi.dptr(ref), cw, None, None) == 0
        lib._scs_finish_cone(cw)
        mine = numpy_proj_dual(cone, x)
        assert np.abs(mine - ref).max() / max(np.abs(ref).max(), np.abs(x).max()) <= 1e-13


def bind(lib, prefix):
    r, w = getattr(lib, prefix + "read_data"), getattr(lib, prefix + "write_data")
    r.restype = C.c_int
    r.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)), PP(PP(capi.ScsSettings))]
    w.argtypes = ([C.c_char_p] if prefix.startswith("scs_b200") else []) + \
                 [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    return r, w


def read(reader, path):
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert reader(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0, path
    return d, k, s


@pytest.mark.parametrize("name", sorted(json.load(open(os.path.join(PROB_DIR, "optima.json")))))
def test_problem_files_round_trip(name, tmp_path):
    lib = capi.load(spectral=True)
    r, w = bind(lib, "scs_b200_")
    src = os.path.join(PROB_DIR, name)
    d, k, s = read(r, src)
    K = k.contents
    assert K.nucsize + K.ell1_size + K.sl_size > 0 and K.dsize == 0
    out = str(tmp_path / "rt")
    assert w(out.encode(), d, k, s) == 0
    # the fixture was written by the reference spectral build's writer: byte-identical
    assert open(out, "rb").read() == open(src, "rb").read()
    if os.path.exists(REF_SPECTRAL):
        ref = capi.load_reference(REF_SPECTRAL, spectral=True)
        rr, rw = bind(ref, "_scs_")
        d2, k2, s2 = read(rr, out)
        # the reference's writer takes the file name from the settings it is given
        ref_out = str(tmp_path / "ref").encode()
        s2.contents.write_data_filename = ref_out
        rw(d2, k2, s2)
        assert open(ref_out, "rb").read() == open(out, "rb").read()


def test_logdet_cone_is_read_then_refused(tmp_path, capfd):
    lib = capi.load(spectral=True)
    r, w = bind(lib, "scs_b200_")
    d, k, s = read(r, os.path.join(PROB_DIR, "test_ell1_cone"))
    # add one log-det cone of order 2 (4 rows) to a copy of the problem, through the file format
    K = k.contents
    dd = np.array([2], dtype=np.int32)
    K.d, K.dsize = capi.iptr(dd), 1
    path = str(tmp_path / "logdet")
    assert w(path.encode(), d, k, s) == 0
    K.d, K.dsize = capi.c_int_p(), 0
    d2, k2, s2 = read(r, path)
    assert k2.contents.dsize == 1 and k2.contents.d[0] == 2
    lib.scs_init.restype = C.c_void_p
    capfd.readouterr()
    assert not lib.scs_init(d2, k2, s2)
    out = capfd.readouterr().out
    assert "log-det" in out, out

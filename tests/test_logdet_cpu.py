"""CPU: the log-det cone's host side and its numpy restatement.

* every operator input of tests/logdet_cases.py takes the branch it is named after in the reference's projection;
* tests/logdet_numpy.py reproduces the reference's recorded branch, newton_success and iteration count on every
  vector-step input of tests/golden/logdet_cones.npz, and its answers lie within a measured spread of the reference's
  (printed: the GPU tests hold the device to 10x that spread);
* the log-det problem files round-trip byte-identically through our writer and the reference's;
* the DLONG ABI narrows d and refuses an order beyond the limits with a message;
* the spectral build's cone-dimension mismatch message names the log-det rows."""
import ctypes as C
import os

import numpy as np
import pytest

import logdet_cases
import logdet_numpy as ln
from conftest import REF_DIR, ROOT
from scs_b200 import capi

GOLD = os.path.join(ROOT, "tests", "golden")
OPS = np.load(os.path.join(GOLD, "logdet_cones.npz"))
PROB_DIR = os.path.join(GOLD, "problems", "logdet")
REF_SPECTRAL = os.path.join(REF_DIR, "libscsindir_ref_spectral.so")
PP = C.POINTER


def test_cases_regenerate():
    names = [str(s) for s in OPS["names"]]
    cases = logdet_cases.operator_cases()
    assert [c[0] for c in cases] == names
    for name, _, x in cases:
        np.testing.assert_array_equal(x, OPS[f"{name}/x"])
    vc = logdet_cases.vector_cases()
    assert [c[0] for c in vc] == [str(s) for s in OPS["vnames"]]
    for name, calls in vc:
        for j, (t0, v0, e) in enumerate(calls):
            np.testing.assert_array_equal(np.concatenate(([t0, v0], e)), OPS[f"v/{name}/in{j}"])
    kinds = {n.rsplit("_", 1)[0] for n, _ in vc}
    assert kinds == {"cold", "warm", "ipm"}


def test_numpy_restatement_reproduces_the_reference_vector_step():
    spread = 0.0
    branches = set()
    for name, seq in logdet_cases.replay(logdet_cases.vector_cases()).items():
        for j, (status, proj, stats) in enumerate(seq):
            rec = OPS[f"v/{name}/rec{j}"]
            assert status == int(rec[0]), (name, j)
            assert stats["iter"] == int(rec[1]) and stats["newton_success"] == int(rec[2]), (name, j, stats, rec)
            ref = OPS[f"v/{name}/proj{j}"]
            spread = max(spread, np.abs(proj - ref).max() / max(np.abs(ref).max(), 1.0))
            branches.add(int(rec[2]))
    assert branches == {ln.NEWTON_SUCCESS, ln.IPM0_SUCCESS}
    print(f"vector step: numpy vs reference spread {spread:.3e}")
    assert spread < 1e-9


def test_operator_inputs_take_their_named_branch_in_the_reference():
    """each operator input reaches the branch it is named after in the reference's own projection (its Newton record),
    and the numpy restatement reproduces the reference's record with and without r_y"""
    for name, n, x in logdet_cases.operator_cases():
        kind = name.rsplit("_", 1)[0]
        rec, recry = OPS[f"{name}/rec"], OPS[f"{name}/recry"]
        t0, v0, e = logdet_cases._step_input(-x, n)
        assert logdet_cases.BRANCH[kind]((int(rec[2]), int(rec[1])), v0), (name, rec)
        assert logdet_cases.robust_record(t0, v0, e) == (int(rec[2]), int(rec[1])), (name, rec)
        t0, v0, e = logdet_cases._step_input(-logdet_cases.r_y(n) * x, n)
        assert logdet_cases.robust_record(t0, v0, e) == (int(recry[2]), int(recry[1])), (name, recry)


def test_numpy_restatement_matches_the_reference_operator():
    spread = 0.0
    for name, n, x in logdet_cases.operator_cases():
        mine = ln.proj_dual_cone(x, {"d": [n]})
        ref = OPS[f"{name}/out"]
        spread = max(spread, np.abs(mine - ref).max() / max(np.abs(ref).max(), np.abs(x).max()))
    spread_ry = 0.0
    for name, n, x in logdet_cases.operator_cases():
        r = logdet_cases.r_y(n)
        _, p, _ = ln.proj_logdet(-r * x, n, ln.State(n))
        ref = OPS[f"{name}/outry"]
        spread_ry = max(spread_ry, np.abs(x + p / r - ref).max() / max(np.abs(ref).max(), np.abs(x).max()))
    print(f"operator: numpy vs reference spread {spread:.3e}, with r_y {spread_ry:.3e} "
          f"(the GPU gates are max(5e-13, 10x these))")
    assert spread < 1e-11 and spread_ry < 1e-9


def _bind(lib, prefix):
    r = getattr(lib, prefix + "read_data")
    r.restype = C.c_int
    r.argtypes = [C.c_char_p, PP(PP(capi.ScsData)), PP(PP(capi.ScsConeSpectral)), PP(PP(capi.ScsSettings))]
    w = getattr(lib, prefix + "write_data")
    return r, w


def _read(r, path):
    d, k, s = PP(capi.ScsData)(), PP(capi.ScsConeSpectral)(), PP(capi.ScsSettings)()
    assert r(path.encode(), C.byref(d), C.byref(k), C.byref(s)) == 0
    return d, k, s


@pytest.mark.parametrize("name", ["exp_design", "several_logdet_cones", "dopt_24"])
def test_problem_files_round_trip(name, tmp_path):
    lib = capi.load(spectral=True)
    r, w = _bind(lib, "scs_b200_")
    w.argtypes = [C.c_char_p, PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    src = os.path.join(PROB_DIR, name)
    d, k, s = _read(r, src)
    assert k.contents.dsize > 0
    out = str(tmp_path / "ours")
    assert w(out.encode(), d, k, s) == 0
    assert open(out, "rb").read() == open(src, "rb").read()
    if not os.path.exists(REF_SPECTRAL):
        pytest.skip("the reference's spectral build is not built")
    ref = capi.load_reference(REF_SPECTRAL, spectral=True)
    rr, rw = _bind(ref, "_scs_")
    rw.argtypes = [PP(capi.ScsData), PP(capi.ScsConeSpectral), PP(capi.ScsSettings)]
    d2, k2, s2 = _read(rr, out)
    ref_out = str(tmp_path / "ref").encode()
    s2.contents.write_data_filename = ref_out
    rw(d2, k2, s2)
    assert open(ref_out, "rb").read() == open(src, "rb").read()


def test_mismatch_message_names_the_logdet_rows(capfd):
    lib = capi.load(spectral=True)
    lib.scs_init.restype = C.c_void_p
    m, n = 10, 2
    A = np.ones(m * n)
    rows = np.tile(np.arange(m, dtype=np.int32), n)
    cols = np.arange(0, m * n + 1, m, dtype=np.int32)
    hp = capi.HostProblem((A, rows, cols, (m, n)), np.zeros(m), np.zeros(n), {"l": 10})
    k, keep = capi.make_cone({"l": 10, "d": [2]}, spectral=True)
    st = capi.default_settings(lib, verbose=0)
    capfd.readouterr()
    assert not lib.scs_init(C.pointer(hp.data), C.byref(k), C.byref(st))
    out = capfd.readouterr().out
    assert "Error: Cone dims 15 != rows in A 10 (spectral: 5 rows in 1 log-det cone)" in out, out


def test_dlong_abi_narrows_d_and_refuses_an_order_beyond_the_limit(capfd):
    lib = capi.load(spectral=True, long=True)
    T = capi.abi(True)
    lib.scs_b200_init_cone.restype = C.c_void_p
    lib.scs_b200_init_cone.argtypes = [PP(T.ScsConeSpectral), T.int_t, capi.c_double_p]
    k, keep = capi.make_cone({"d": [3]}, spectral=True, long=True)
    assert keep["d"].dtype == np.int64
    capfd.readouterr()
    k.d[0] = 1 << 32 | 3  # a 64-bit order whose low 32 bits would pass as 3
    assert not lib.scs_b200_init_cone(C.byref(k), logdet_cases.rows(3), None)
    out = capfd.readouterr().out
    assert "d[0] = 4294967299 exceeds the limit" in out, out

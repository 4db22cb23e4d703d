"""CPU tests (no GPU): the C-ABI library loads and exports every symbol that
include/scs_b200.h declares; struct layouts match the reference's; the library
fails loudly (no CPU fallback) when there is no sm_90 device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from scs_b200 import capi, problems


def declared_functions():
    src = open(os.path.join(ROOT, "include", "scs_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b([a-z_0-9A-Z]+)\s*\([^;{]*\)\s*;", src)
    return sorted(set(n for n in names if n.startswith("scs")))


def test_library_exports_every_declared_symbol():
    assert os.path.exists(capi.LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    raw = C.CDLL(capi.LIB_PATH, mode=C.RTLD_LOCAL)
    names = declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(raw, n), f"{n} declared in include/scs_b200.h but not exported"


def test_struct_layouts_match_reference_abi():
    # reference include/scs.h with DLONG=0, SFLOAT=0 on LP64
    assert C.sizeof(capi.ScsMatrix) == 32
    assert C.sizeof(capi.ScsSettings) == 136
    assert C.sizeof(capi.ScsData) == 40
    assert C.sizeof(capi.ScsCone) == 104
    assert C.sizeof(capi.ScsSolution) == 24
    assert C.sizeof(capi.AaStats) == 48
    assert capi.ScsInfo.status.offset == 4 and capi.ScsInfo.lin_sys_solver.offset == 132
    assert capi.ScsInfo.pobj.offset == 272


def test_default_settings_match_reference_defaults():
    lib = capi.load()
    st = capi.default_settings(lib)
    assert (st.normalize, st.scale, st.adaptive_scale, st.rho_x, st.max_iters) == (1, 0.1, 1, 1e-6, 100000)
    assert (st.eps_abs, st.eps_rel, st.eps_infeas, st.alpha) == (1e-4, 1e-4, 1e-7, 1.5)
    assert (st.acceleration_lookback, st.acceleration_interval, st.acceleration_type_1) == (10, 10, 1)
    assert (st.acceleration_regularization, st.acceleration_relaxation) == (1e-8, 1.0)
    assert lib.scs_get_lin_sys_method().decode().startswith("sparse-indirect-b200")


@pytest.mark.skipif(os.path.exists("/dev/nvidia0"), reason="needs a box WITHOUT a GPU")
def test_no_cpu_fallback_without_gpu():
    lib = capi.load()
    assert lib.scs_b200_device_ok() == 0
    prob = problems.make_problem(30, 10, 3, {"l": 30}, 0)
    hp = capi.HostProblem(prob["A"], prob["b"], prob["c"], prob["cone"])
    st = capi.default_settings(lib, verbose=0)
    assert not lib.scs_init(C.byref(hp.data), C.byref(hp.cone), C.byref(st))
    dr = np.ones(41)
    assert not lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))


def test_generator_known_optimum():
    prob = problems.make_problem(120, 40, 5, {"z": 10, "l": 40, "q": [30, 40]}, 3)
    A = prob["A"]
    # primal/dual feasibility and complementary slackness by construction (problem_utils.h:22-81)
    assert np.abs(problems.csc_matvec(A, prob["x_opt"]) + prob["s_opt"] - prob["b"]).max() < 1e-12
    assert np.abs(problems.csc_rmatvec(A, prob["y_opt"]) + prob["c"]).max() < 1e-12
    assert abs(prob["s_opt"] @ prob["y_opt"]) < 1e-10
    assert abs(prob["c"] @ prob["x_opt"] + prob["b"] @ prob["y_opt"]) < 1e-10

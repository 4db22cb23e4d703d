"""The CG loop's fused K3 + K4 (kernels/cg.cu k_cg_update_p): which path a problem size takes, run-to-run bit identity
of a KKT solve on the fused path, including a size whose every thread holds the most elements and the odd tail, and
the bits of x, y, s after 1 and 20 ADMM iterations against those the K3 / K4 pair computed before the fusion."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

from scs_b200 import capi, problems
from test_device_data_gpu import host_solve, read_fixture
from test_linsys_gpu import diag_r_for, kkt_reduced_residual

pytestmark = pytest.mark.gpu

# SHA-256 of x, y, s (float64 bytes) after K ADMM iterations with eps = 0, recorded on an H100 80GB HBM3 from commit
# 8000646, whose CG loop ran every iteration as the K3 / K4 pair
PAIR_HASHES = {
    ("random_prob", 1): {"x": "3cb5b0368972611f16494d254c7b7b5e70d36002d1407061920d66291762b80a",
                         "y": "8773ac319bf67e8d52d3250c706fdbf74c8e76851eaf769e018c7ad50bfb62c1",
                         "s": "468450ccbf4c05488d5de17f76f2f06cdd56c69228aae0cdbc65cfd38e85ec29"},
    ("random_prob", 20): {"x": "f83ade00aaee7beef538487977f154ce38b83d7e1f115758a424d549ce1f839a",
                          "y": "d68dd87e8fbf695c2b0812747ace65f3af816a80a1b8ea9cffa2f03a2aa02dee",
                          "s": "dbe59e08f51948be9653af5baf42980bf0978d15d826281786066adf6aa18a74"},
    ("C2x0.01", 1): {"x": "136322821942187e7ced5f17aede8737114212dcaa560708fb3c859ae6107707",
                     "y": "6ff056e77ba005855f9bb6b0ca49c34b5a95e19129bea1afee055a7306722e92",
                     "s": "a9fb5e402644c01175e73cd1be4b9281b913d94e9bfc36600e3343bcab593edd"},
    ("C2x0.01", 20): {"x": "23eeab7cdcd8690ba27567888bd8b424acace594e38bb3d76bf63c1ec8e09de5",
                      "y": "63fa47257b67beca52a72cac7c15b83a7dc8d0900867ecfec72d50e423283bc2",
                      "s": "f9a63419ce04edb2c9fa6e90645f8f5edad358e9a52ec43d3e2f190694cc50fd"},
}


def fused_limit():
    """largest n the fused kernel takes: K3's grid of 2 blocks of 512 threads per SM, 4 double2 per thread"""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 4096


def admm_problem(name):
    if name == "random_prob":
        return read_fixture("random_prob")
    import scipy.sparse as sp
    prob = problems.config("C2", scale=0.01, seed=1234)
    A = sp.csc_matrix((prob["A"][0], prob["A"][1], prob["A"][2]), shape=prob["A"][3])
    return A, None, prob["b"], prob["c"], prob["cone"]


def solution_hashes():
    """{(problem, K): {"x", "y", "s": SHA-256 hex}} for every key of PAIR_HASHES"""
    out = {}
    for name, k in PAIR_HASHES:
        x, y, s, info = host_solve(*admm_problem(name), max_iters=k, eps_abs=0.0, eps_rel=0.0, eps_infeas=0.0)[0]
        assert info["iter"] == k
        out[(name, k)] = {v: hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()
                          for v, a in (("x", x), ("y", y), ("s", s))}
    return out


def linsys(lib, n, m, col_nnz, seed):
    A = problems.random_sparse_csc(m, n, col_nnz, np.random.default_rng(seed))
    hp = capi.HostProblem(A, np.zeros(m), np.zeros(n), {"l": m})
    dr = diag_r_for(n, m, m // 10)
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    assert w, "scs_init_lin_sys_work failed"
    return w, A, dr, hp


def launches_per_cg_iteration(lib, w):
    """launches of R more CG iterations through scs_b200_time_cg_iter (the same start-up for both counts)"""
    ab = C.c_double()
    counts = []
    for reps in (5, 15):
        l0 = lib.scs_b200_launch_count()
        assert lib.scs_b200_time_cg_iter(w, reps, C.byref(ab)) > 0
        counts.append(lib.scs_b200_launch_count() - l0)
    return (counts[1] - counts[0]) / 10


@pytest.mark.parametrize("where", ["small", "limit-1", "limit", "limit+1"])
def test_path_choice_by_size(lib, where):
    """3 launches per CG iteration (K1, K2, fused K3 + K4) up to 2 SMs x 4096 columns, the pair (4) above"""
    lim = fused_limit()
    n = {"small": 10_000, "limit-1": lim - 1, "limit": lim, "limit+1": lim + 1}[where]
    w, _, _, _ = linsys(lib, n, n, 2, 11)
    try:
        assert launches_per_cg_iteration(lib, w) == (4 if where == "limit+1" else 3)
    finally:
        lib.scs_free_lin_sys_work(w)


@pytest.mark.parametrize("n,col_nnz", [(10_000, 10), (None, 3)])
def test_kkt_solve_repeats_bit_for_bit(lib, n, col_nnz):
    """the same KKT solve twice on one workspace (m = 3 n): identical bits and CG counts, and a converged answer;
    n = None is the largest odd n on the fused path (every thread holds 4 double2, block 0's thread 0 also the last
    element)"""
    n = fused_limit() - 1 if n is None else n
    m = 3 * n
    w, A, dr, _ = linsys(lib, n, m, col_nnz, 5)
    try:
        rhs = np.random.default_rng(6).standard_normal(n + m)
        sols, its = [], []
        for _ in range(2):
            sol = rhs.copy()
            assert lib.scs_solve_lin_sys(w, capi.dptr(sol), None, 1e-10) == 0
            sols.append(sol)
            its.append(lib.scs_b200_linsys_last_cg_its(w))
        assert its[0] == its[1] and its[0] > 1
        assert sols[0].tobytes() == sols[1].tobytes()
        rx, ry = kkt_reduced_residual(A, dr, rhs, sols[0])
        assert rx <= 1e-7 and ry <= 1e-7, (rx, ry)
    finally:
        lib.scs_free_lin_sys_work(w)


def test_admm_bits_equal_the_pair():
    """x, y, s after 1 and 20 ADMM iterations of random_prob and of C2 x 0.01 are the bits the K3 / K4 pair gave"""
    got = solution_hashes()
    for key, want in PAIR_HASHES.items():
        assert got[key] == want, key

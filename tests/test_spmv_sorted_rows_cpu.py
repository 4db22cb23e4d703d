"""CPU checks of the v3 SpMV plan on the shape of the CG operator's copy of A (host/linsys_b200.c cg_ops_build,
kernels/spmv.cu b200_spmv_permuted_rows): the rows of a random matrix sorted by their smallest column, empty rows left
out, every row placed so that the kernel cuts it into the same lane pieces as in the original stream. The kernel's lane
algorithm, re-executed in numpy, must then give bit-for-bit the row sums of the original operator. No GPU needed."""
import numpy as np
import pytest
import scipy.sparse as sp

from scs_b200 import problems
from test_spmv_plan_cpu import WT, build_plan, check_invariants, emulate_kernel


def c2_like(m, n, per_col, seed):
    data, indices, indptr, _ = problems.random_sparse_csc(m, n, per_col, np.random.default_rng(seed))
    R = sp.csc_matrix((data, indices, indptr), shape=(m, n)).tocsr()
    R.sort_indices()
    return R


def min_col_order(R):
    """stable order of the rows by smallest column, empty rows (last) left out -- b200_perm_rows_by_min_col"""
    m, n = R.shape
    lens = np.diff(R.indptr)
    key = np.full(m, n, dtype=np.int64)
    key[lens > 0] = R.indices[R.indptr[:-1][lens > 0]]
    return np.argsort(key, kind="stable")[:int((lens > 0).sum())]


def lane_preserving_csr(R, perm):
    """the permuted copy with its leading explicit zeros, as b200_spmv_permuted_rows lays it out; the zeros are stored
    here as entries of column 0 with value 0 (the kernel stores them as SKIP entries: product 0 either way)"""
    lens = np.diff(R.indptr)
    old_sp = np.concatenate([[0], np.cumsum(np.maximum(lens, 1))])  # stored positions in the flagged stream of R
    rows_i, rows_v, ptr, pos = [], [], [0], 0
    for o in perm:
        a, ln = int(old_sp[o]), int(lens[o])
        phase, c = a & 3, pos & 3
        if phase + ln <= 4:
            lead = 0 if c + ln <= 4 else 4 - c
        else:
            lead = (phase - c) & 3
        if c + lead + ln > WT:
            lead = 0
        seg_i = R.indices[R.indptr[o]:R.indptr[o + 1]]
        rows_i.append(np.concatenate([np.zeros(lead, np.int32), seg_i]))
        rows_v.append(np.concatenate([np.zeros(lead), R.data[R.indptr[o]:R.indptr[o + 1]]]))
        pos += lead + ln
        ptr.append(pos)
    return (np.array(ptr, np.int32), np.concatenate(rows_i).astype(np.int32), np.concatenate(rows_v), pos - lens[perm].sum())


@pytest.mark.parametrize("grid_cap", [3, 132])
def test_row_sorted_copy_reproduces_the_row_sums_bit_for_bit(lib, grid_cap):
    R = c2_like(15000, 5000, 10, 11)
    m, n = R.shape
    rng = np.random.default_rng(grid_cap)
    x = rng.standard_normal(n)
    x[0] = 1.0  # the explicit zeros of the copy multiply x[0]: keep their products +0.0, as the kernel's SKIP entries
    rp, ci = R.indptr.astype(np.int32), R.indices.astype(np.int32)
    base = build_plan(lib, m, n, rp, ci, R.data, grid_cap)
    y = emulate_kernel(base, m, x, rng)

    perm = min_col_order(R)
    prp, pci, pva, zeros = lane_preserving_csr(R, perm)
    assert zeros < 1.5 * len(perm)  # at most 3 per row, about one on average
    plan = build_plan(lib, len(perm), n, prp, pci, pva, grid_cap)
    check_invariants(plan, len(perm), prp, pci, pva)
    y_copy = emulate_kernel(plan, len(perm), x, rng)
    assert np.array_equal(y_copy, y[perm])

    # the same rows packed back to back are cut into other lane pieces: their sums differ in the last bits
    Rp = R[perm, :]
    packed = build_plan(lib, len(perm), n, Rp.indptr.astype(np.int32), Rp.indices.astype(np.int32), Rp.data, grid_cap)
    y_packed = emulate_kernel(packed, len(perm), x, rng)
    assert not np.array_equal(y_packed, y[perm])
    assert np.abs(y_packed - y[perm]).max() <= 1e-14 * np.abs(y).max()

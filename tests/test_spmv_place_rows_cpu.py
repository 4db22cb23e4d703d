"""CPU checks of the placement of the CG operator's row-sorted copy of A (kernels/spmv.cu `b200_spmv_place_rows`,
called by `b200_spmv_permuted_rows`): rows taken from a window of the next 32 in smallest-column order, so that each
starts at a phase (position modulo 4) where the kernel sums it as in A, with explicit zeros only where no row fits.
The kernel's lane algorithm, re-executed in numpy, must give bit-for-bit the row sums of the original operator. No GPU
needed: the placement is host code exported by the library."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from scs_b200 import problems
from test_spmv_plan_cpu import MAXROW, WT, build_plan, check_invariants, emulate_kernel

WINDOW = 32


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


def place_rows(lib, sp_old, perm):
    """b200_spmv_place_rows: (placed order, stored row pointers of the copy, stored count)"""
    ip = C.POINTER(C.c_int)
    lib.b200_spmv_place_rows.restype = C.c_longlong
    lib.b200_spmv_place_rows.argtypes = [C.c_int, ip, ip, ip]
    sp_old = np.ascontiguousarray(sp_old, dtype=np.int32)
    placed = np.ascontiguousarray(perm, dtype=np.int32).copy()
    sp_new = np.zeros(len(placed) + 1, dtype=np.int32)
    stored = lib.b200_spmv_place_rows(len(placed), sp_old.ctypes.data_as(ip), placed.ctypes.data_as(ip),
                                      sp_new.ctypes.data_as(ip))
    return placed, sp_new, int(stored)


def stored_rowptr(R):
    """stored row pointers of R's flagged stream (one explicit zero per empty row)"""
    return np.concatenate([[0], np.cumsum(np.maximum(np.diff(R.indptr), 1))]).astype(np.int32)


def copy_csr(R, placed, sp_new):
    """the copy as a CSR: each segment's leading zeros are stored as entries of column 0 with value 0 (the kernel
    stores them as SKIP entries: product +0.0 either way as long as x[0] is finite and positive)"""
    lens = np.diff(R.indptr)[placed]
    lead = np.diff(sp_new) - lens
    ci, va = [], []
    for o, z in zip(placed, lead):
        a, b = R.indptr[o], R.indptr[o + 1]
        ci.append(np.zeros(z, np.int32))
        ci.append(R.indices[a:b].astype(np.int32))
        va.append(np.zeros(z))
        va.append(R.data[a:b])
    return np.concatenate(ci), np.concatenate(va)


def check_placement(lib, R, perm, placed, sp_new, stored):
    """a permutation of the kept rows, each within the window of its sorted slot, at a phase where it sums as in R"""
    lens = np.diff(R.indptr)
    assert np.array_equal(np.sort(placed), np.sort(perm))
    slot = np.empty(R.shape[0], dtype=np.int64)
    slot[perm] = np.arange(len(perm))
    assert np.abs(slot[placed] - np.arange(len(placed))).max() < WINDOW
    assert stored == sp_new[-1] and (np.diff(sp_new) >= lens[placed]).all()
    lead = np.diff(sp_new) - lens[placed]
    assert lead.max() <= 3
    ln = lens[placed]
    assert ln.max() <= MAXROW
    table = np.array([[sum(1 << q for q in admitted_phases(lib, L, p)) if L else 0 for p in range(4)]
                      for L in range(ln.max() + 1)])
    phase_old = stored_rowptr(R)[placed] & 3
    phase_new = (sp_new[:-1] + lead) & 3
    assert ((table[ln, phase_old] >> phase_new) & 1).all()
    return int(lead.sum())


def test_c2_shaped_placement_needs_almost_no_zeros(lib):
    R = c2_like(600000, 200000, 10, 1)
    perm = min_col_order(R)
    placed, sp_new, stored = place_rows(lib, stored_rowptr(R), perm)
    zeros = check_placement(lib, R, perm, placed, sp_new, stored)
    assert zeros <= 0.01 * R.nnz, zeros / R.nnz
    # the order refines the sort: a row's smallest column moves by less than one column on average
    key = R.indices[R.indptr[:-1]]
    assert np.abs(key[placed].astype(np.int64) - key[perm]).mean() < 1.0
    # the placement is a function of A alone
    again = place_rows(lib, stored_rowptr(R), perm)
    assert np.array_equal(again[0], placed) and np.array_equal(again[1], sp_new)


@pytest.mark.parametrize("grid_cap", [3, 132])
def test_placed_copy_reproduces_the_row_sums_bit_for_bit(lib, grid_cap):
    R = c2_like(15000, 5000, 10, 11)
    m, n = R.shape
    rng = np.random.default_rng(grid_cap)
    x = rng.standard_normal(n)
    x[0] = 1.0  # the explicit zeros of the copy multiply x[0]: keep their products +0.0, as the kernel's SKIP entries
    base = build_plan(lib, m, n, R.indptr.astype(np.int32), R.indices.astype(np.int32), R.data, grid_cap)
    y = emulate_kernel(base, m, x, rng)

    perm = min_col_order(R)
    placed, sp_new, stored = place_rows(lib, stored_rowptr(R), perm)
    zeros = check_placement(lib, R, perm, placed, sp_new, stored)
    assert zeros <= 0.01 * R.nnz
    pci, pva = copy_csr(R, placed, sp_new)
    plan = build_plan(lib, len(placed), n, sp_new, pci, pva, grid_cap)
    check_invariants(plan, len(placed), sp_new, pci, pva)
    y_copy = emulate_kernel(plan, len(placed), x, rng)
    assert np.array_equal(y_copy, y[placed])

    # the same rows packed back to back are cut into other lane pieces: their sums differ in the last bits
    Rp = R[placed, :]
    packed = build_plan(lib, len(placed), n, Rp.indptr.astype(np.int32), Rp.indices.astype(np.int32), Rp.data,
                        grid_cap)
    y_packed = emulate_kernel(packed, len(placed), x, rng)
    assert not np.array_equal(y_packed, y[placed])
    assert np.abs(y_packed - y[placed]).max() <= 1e-14 * np.abs(y).max()


def test_long_rows_keep_their_segment_in_one_warp_tile(lib):
    """rows of up to MAXROW entries: every segment (leading zeros + row) fits one warp-tile's aligned span, and only a
    row whose zeros would not fit may start at a phase it does not sum the same at"""
    rng = np.random.default_rng(3)
    m = 3000
    lens = np.where(rng.random(m) < 0.3, rng.integers(100, MAXROW + 1, m), rng.integers(0, 8, m))
    sp_old = np.concatenate([[0], np.cumsum(np.maximum(lens, 1))]).astype(np.int32)
    perm = rng.permutation(np.nonzero(lens > 0)[0]).astype(np.int32)
    placed, sp_new, stored = place_rows(lib, sp_old, perm)
    assert np.array_equal(np.sort(placed), np.sort(perm)) and stored == sp_new[-1]
    slot = np.empty(m, dtype=np.int64)
    slot[perm] = np.arange(len(perm))
    assert np.abs(slot[placed] - np.arange(len(placed))).max() < WINDOW
    seg = np.diff(sp_new)
    ln = lens[placed]
    lead = seg - ln
    assert lead.min() >= 0 and lead.max() <= 3
    assert ((sp_new[:-1] & 3) + seg <= WT).all()
    mask = np.array([sum(1 << q for q in admitted_phases(lib, int(L), int(p))) for L, p in zip(ln, sp_old[placed] & 3)])
    ok = (mask >> ((sp_new[:-1] + lead) & 3)) & 1 == 1
    assert (ln[~ok] > WT - 6).all() and (lead[~ok] == 0).all()


def admitted_phases(lib, length, phase):
    """spmv3_same_sum_phases: the phases at which a row of `length` entries sums as it does at `phase`"""
    lib.b200_spmv3_phase_mask.restype = C.c_uint
    lib.b200_spmv3_phase_mask.argtypes = [C.c_int, C.c_int]
    mask = lib.b200_spmv3_phase_mask(length, phase)
    assert 0 < mask < 16
    return {q for q in range(4) if mask >> q & 1}


def phase_sums(lib, length, rng, draws):
    """row sums of `draws` rows of `length` products of large dynamic range, each row alone at phase q (preceded by a
    filler row), for q = 0..3, by the numpy re-execution of the kernel's lane algorithm. Returns [4, draws]."""
    ncols = length * draws + 1
    cols = np.arange(1, ncols).reshape(draws, length).astype(np.int32)
    vals = rng.standard_normal((draws, length)) * 10.0 ** rng.uniform(-12, 12, (draws, length))
    x = np.ones(ncols)
    x[1:] = rng.standard_normal(ncols - 1) * 10.0 ** rng.uniform(-6, 6, ncols - 1)
    out = np.empty((4, draws))
    for q in range(4):
        rp, ci, va, rows, pos = [0], [], [], [], 0
        for i in range(draws):
            f = (q - pos) & 3 or 4  # filler: puts the next row's first entry at phase q
            ci.append(np.zeros(f, np.int32))
            va.append(np.ones(f))
            pos += f
            rp.append(pos)
            ci.append(cols[i])
            va.append(vals[i])
            pos += length
            rp.append(pos)
            rows.append(2 * i + 1)
        rp = np.array(rp, np.int32)
        plan = build_plan(lib, len(rp) - 1, ncols, rp, np.concatenate(ci), np.concatenate(va), 4)
        out[q] = emulate_kernel(plan, len(rp) - 1, x, rng)[rows]
    return out


def test_admitted_phases_give_the_same_sum(lib):
    rng = np.random.default_rng(5)
    for length in range(1, MAXROW + 1):
        adm = {phase: admitted_phases(lib, length, phase) for phase in range(4)}
        for phase in range(4):
            assert phase in adm[phase]
            # every phase the lane-preserving rule admitted (same phase, or one lane to one lane) is still admitted
            old = {q for q in range(4) if q + length <= 4} if phase + length <= 4 else {phase}
            assert old <= adm[phase], (length, phase, adm[phase])
        s = phase_sums(lib, length, rng, 200 if length <= 8 else 16)
        for phase in range(4):
            for q in range(4):
                if q in adm[phase]:
                    assert np.array_equal(s[q], s[phase]), (length, phase, q)
                else:  # the rule is exact: a phase left out sums differently on some draw
                    assert not np.array_equal(s[q], s[phase]), (length, phase, q)

"""CPU checks of the v3 "flagged stream" SpMV plan (scs_b200/csrc/kernels/spmv.cu, test export
`b200_spmv3_plan_build`: the stream as the device builder fills it, by the same per-row fill `spmv3_fill_row` run on the
host, and the virtual rows, warp-tiles and CTA partition of `spmv3_finish`): format invariants, and a numpy
re-execution of the kernel's LANE algorithm (`spmv_flag_kernel`: 4 entries per lane, END ballots -> row numbers,
in-lane sequential sums, segmented Hillis-Steele scan of the open tails, staging through a garbage-filled stage buffer
exactly as the TMA producer cuts it) against a plain CSR product. No GPU needed (operator: reference
linsys/scs_matrix.c:161-186)."""
import ctypes as C

import numpy as np
import pytest

from scs_b200 import capi

END = 0x80000000
SKIP = 0x40000000
COLMASK = 0x3FFFFFFF
WT = 128
MAXROW = 124


def random_csr(nrows, ncols, rng, lens):
    rp = np.zeros(nrows + 1, dtype=np.int32)
    rp[1:] = np.cumsum(lens)
    ci = np.concatenate([np.sort(rng.choice(ncols, size=int(l), replace=False)) for l in lens] + [np.zeros(0, int)])
    va = rng.standard_normal(int(rp[-1]))
    return rp, ci.astype(np.int32), va


def build_plan(lib, nrows, ncols, rp, ci, va, grid_cap):
    ip = C.POINTER(C.c_int)
    dp = C.POINTER(C.c_double)
    lib.b200_spmv3_plan_build.restype = C.c_void_p
    lib.b200_spmv3_plan_build.argtypes = [C.c_int, C.c_int, ip, ip, dp, C.c_int]
    for name, rt in (("rowptr", ip), ("idx", ip), ("vals", dp), ("desc", ip), ("cta_begin", ip)):
        f = getattr(lib, "b200_spmv3_plan_" + name)
        f.restype = rt
        f.argtypes = [C.c_void_p]
    lib.b200_spmv3_plan_free.argtypes = [C.c_void_p]
    lib.b200_spmv3_plan_info.argtypes = [C.c_void_p] + [ip] * 5
    ci_ = np.ascontiguousarray(ci if len(ci) else np.zeros(1, np.int32))
    va_ = np.ascontiguousarray(va if len(va) else np.zeros(1))
    h = lib.b200_spmv3_plan_build(nrows, ncols, rp.ctypes.data_as(ip), ci_.ctypes.data_as(ip),
                                  va_.ctypes.data_as(dp), grid_cap)
    if not h:
        return None
    vals = [C.c_int() for _ in range(5)]
    lib.b200_spmv3_plan_info(h, *[C.byref(v) for v in vals])
    stored, nwt, ndesc, grid, ncw = [v.value for v in vals]
    plan = {
        "stored": stored, "nwt": nwt, "ndesc": ndesc, "grid": grid, "ncw": ncw,
        "rowptr": np.ctypeslib.as_array(lib.b200_spmv3_plan_rowptr(h), (nrows + 1,)).copy(),
        "idx": np.ctypeslib.as_array(lib.b200_spmv3_plan_idx(h), (stored,)).copy().view(np.uint32),
        "vals": np.ctypeslib.as_array(lib.b200_spmv3_plan_vals(h), (stored,)).copy(),
        "desc": np.ctypeslib.as_array(lib.b200_spmv3_plan_desc(h), (ndesc * 4,)).copy().reshape(ndesc, 4),
        "cta_begin": np.ctypeslib.as_array(lib.b200_spmv3_plan_cta_begin(h), (grid + 1,)).copy(),
    }
    lib.b200_spmv3_plan_free(h)
    return plan


def emulate_kernel(plan, nrows, x, rng):
    """numpy restatement of spmv_flag_kernel<POST_NONE> (no init): lanes are vectors of 32."""
    ncw = plan["ncw"]
    cap = ncw * WT + 8
    idx, vals, desc = plan["idx"], plan["vals"], plan["desc"]
    stored = plan["stored"]
    pad = ((stored + 3) & ~3) + 8
    g_idx = np.zeros(pad, dtype=np.uint32)
    g_val = np.zeros(pad)
    g_idx[:stored] = idx
    g_val[:stored] = vals
    y = np.full(nrows, np.nan)
    written = np.zeros(nrows, dtype=int)
    lane = np.arange(32)
    for c in range(plan["grid"]):
        for g in range(plan["cta_begin"][c], plan["cta_begin"][c + 1]):
            grp = desc[g * ncw:(g + 1) * ncw]
            # producer: extent of the group, staged into a stage buffer full of garbage
            ka = int(grp[0][1]) & ~3
            kend_g = int(grp[-1][1] + grp[-1][2])
            cnt = (kend_g - ka + 3) & ~3
            assert 0 < cnt <= cap, (cnt, cap)
            s_idx = rng.integers(0, 2**32, size=cap, dtype=np.uint64).astype(np.uint32)
            s_val = np.full(cap, np.inf)
            s_idx[:cnt] = g_idx[ka:ka + cnt]
            s_val[:cnt] = g_val[ka:ka + cnt]
            for cw in range(ncw):
                row0, k0, cn, _ = [int(t) for t in grp[cw]]
                kend = k0 + cn
                kb = (k0 & ~3) + 4 * lane
                anyl = (kb < kend) & (kb + 4 > k0)
                e = kb - ka
                iv = np.zeros((32, 4), dtype=np.uint32)
                av = np.zeros((32, 4))
                for l in np.nonzero(anyl)[0]:
                    assert 0 <= e[l] and e[l] + 4 <= cnt
                    iv[l] = s_idx[e[l]:e[l] + 4]
                    av[l] = s_val[e[l]:e[l] + 4]
                if cn == 0:
                    continue
                k = kb[:, None] + np.arange(4)[None, :]
                v = anyl[:, None] & (k >= k0) & (k < kend)
                gth = v & ((iv & SKIP) == 0)
                xs = np.where(gth, x[(iv & COLMASK).astype(np.int64) % len(x)], 0.0)
                with np.errstate(invalid="ignore"):
                    p = np.where(gth, av * xs, 0.0)
                en = v & ((iv & END) != 0)
                ends_lane = en.any(axis=1)
                before = np.concatenate([[0], np.cumsum(en.sum(axis=1))[:-1]])  # popc(b_u & lt) summed
                # in-lane sums
                o = np.zeros((32, 4))
                acc = np.zeros(32)
                for u in range(4):
                    acc = acc + p[:, u]
                    o[:, u] = acc
                    acc = np.where(en[:, u], 0.0, acc)
                tail = acc
                # h = last lane <= me with an END, else 0
                h = np.zeros(32, dtype=int)
                last = 0
                for l in range(32):
                    if ends_lane[l]:
                        last = l
                    h[l] = last if ends_lane[:l + 1].any() else 0
                maxdist = int((lane - h).max())
                I = tail.copy()
                dd = 1
                while dd <= maxdist:
                    up = np.concatenate([I[:dd], I[:-dd]])  # shfl_up keeps own value for lane < dd
                    I = np.where(lane - dd >= h, up + I, I)
                    dd <<= 1
                carry = np.concatenate([[0.0], I[:-1]])
                for l in range(32):
                    r = row0 + before[l]
                    first = True
                    for u in range(4):
                        if en[l, u]:
                            s = o[l, u]
                            if first:
                                s = carry[l] + s
                                first = False
                            y[r] = s
                            written[r] += 1
                            r += 1
    assert (written == 1).all(), "every row must be written exactly once"
    return y


def check_invariants(plan, nrows, rp, ci, va):
    prp, idx, vals, desc = plan["rowptr"], plan["idx"], plan["vals"], plan["desc"]
    ncw = plan["ncw"]
    lens = np.diff(rp)
    assert plan["stored"] == rp[-1] + (lens == 0).sum()
    assert (np.diff(prp) == np.maximum(lens, 1)).all()
    # END exactly on the last stored entry of each row, SKIP exactly on the explicit zeros
    endpos = prp[1:] - 1
    is_end = (idx & END) != 0
    assert is_end.sum() == nrows and is_end[endpos].all()
    is_skip = (idx & SKIP) != 0
    assert (is_skip[prp[:-1]] == (lens == 0)).all() and is_skip.sum() == (lens == 0).sum()
    assert (vals[is_skip] == 0).all()
    keep = ~is_skip
    assert np.array_equal((idx[keep] & COLMASK).astype(np.int32), ci) and np.array_equal(vals[keep], va)
    # real warp-tiles tile the rows and the entries; aligned span <= 128; groups are contiguous in entries
    real = desc[desc[:, 2] > 0]
    assert len(real) == plan["nwt"]
    assert real[0, 0] == 0 and real[0, 1] == 0
    assert (real[1:, 0] == real[:-1, 0] + real[:-1, 3]).all() and real[-1, 0] + real[-1, 3] == nrows
    assert (real[1:, 1] == real[:-1, 1] + real[:-1, 2]).all() and real[-1, 1] + real[-1, 2] == plan["stored"]
    assert (real[:, 1] == prp[real[:, 0]]).all()
    assert ((real[:, 1] + real[:, 2]) - (real[:, 1] & ~3) <= WT).all()
    assert plan["ndesc"] % ncw == 0 and plan["cta_begin"][-1] * ncw == plan["ndesc"]
    for c in range(plan["grid"]):
        a, b = plan["cta_begin"][c] * ncw, plan["cta_begin"][c + 1] * ncw
        d = desc[a:b]
        assert b > a and d[0, 2] > 0
        assert (d[1:, 1] == d[:-1, 1] + d[:-1, 2]).all(), "padding descriptors must continue the entry range"


CASES = [
    # (nrows, ncols, row-length sampler, grid_cap)
    (1, 5, lambda rng, n: np.array([3]), 4),
    (1, 5, lambda rng, n: np.array([0]), 4),
    (7, 3, lambda rng, n: np.zeros(n, int), 2),
    (300, 1000, lambda rng, n: rng.poisson(3.3, n), 3),
    (300, 1000, lambda rng, n: rng.poisson(3.3, n), 296),
    (2000, 50000, lambda rng, n: np.full(n, 10), 2),
    (500, 400, lambda rng, n: rng.integers(0, MAXROW + 1, n), 5),
    (64, 200, lambda rng, n: np.full(n, MAXROW), 1),
    (5000, 300, lambda rng, n: (rng.random(n) < 0.5).astype(int), 7),
    (777, 999, lambda rng, n: np.where(rng.random(n) < 0.1, 100, rng.poisson(2, n)), 4),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_plan_and_lane_algorithm(lib, case):
    nrows, ncols, sampler, grid_cap = CASES[case]
    rng = np.random.default_rng(100 + case)
    lens = np.minimum(sampler(rng, nrows), min(ncols, MAXROW))
    if case == 3:
        lens[0] = 0
        lens[-1] = 0
    rp, ci, va = random_csr(nrows, ncols, rng, lens)
    plan = build_plan(lib, nrows, ncols, rp, ci, va, grid_cap)
    assert plan is not None
    check_invariants(plan, nrows, rp, ci, va)
    x = rng.standard_normal(ncols)
    y = emulate_kernel(plan, nrows, x, rng)
    ref = np.zeros(nrows)
    for r in range(nrows):
        ref[r] = np.dot(va[rp[r]:rp[r + 1]], x[ci[rp[r]:rp[r + 1]]])
    scale = np.abs(ref).max() + 1e-300
    assert np.abs(y - ref).max() / scale <= 1e-14


def test_plan_property_random_shapes(lib):
    """hypothesis: arbitrary row-length patterns (runs of empty rows, rows of exactly 124 entries, single
    rows, tiny column spaces) -> plan invariants hold and the lane algorithm reproduces the CSR product"""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=60, deadline=None)
    @given(st.lists(st.one_of(st.integers(0, 6), st.sampled_from([0, 1, 2, 123, MAXROW])), min_size=1, max_size=400),
           st.integers(1, 7), st.integers(0, 2**31 - 1))
    def check(lens, grid_cap, seed):
        rng = np.random.default_rng(seed)
        ncols = max(MAXROW, 130)
        lens_a = np.asarray(lens)
        rp, ci, va = random_csr(len(lens), ncols, rng, lens_a)
        plan = build_plan(lib, len(lens), ncols, rp, ci, va, grid_cap)
        assert plan is not None
        check_invariants(plan, len(lens), rp, ci, va)
        x = rng.standard_normal(ncols)
        y = emulate_kernel(plan, len(lens), x, rng)
        ref = np.array([np.dot(va[rp[r]:rp[r + 1]], x[ci[rp[r]:rp[r + 1]]]) for r in range(len(lens))])
        assert np.abs(y - ref).max() <= 1e-13 * (np.abs(ref).max() + 1.0)

    check()


def test_long_rows_as_virtual_rows(lib):
    """long-row mode (the default): rows longer than 124 entries are cut into balanced pieces
    (an END flag per piece = one "virtual row"); the lane algorithm produces one sum per virtual row and the combine
    pass (spmv_combine_kernel) adds the pieces of each true row in order."""
    lib.b200_spmv3_plan_nvrows.restype = C.c_int
    lib.b200_spmv3_plan_nvrows.argtypes = [C.c_void_p]
    lib.b200_spmv3_plan_vptr.restype = C.POINTER(C.c_int)
    lib.b200_spmv3_plan_vptr.argtypes = [C.c_void_p]
    rng = np.random.default_rng(321)
    for trial, (nrows, ncols, sampler) in enumerate([
        (40, 3000, lambda: rng.choice([0, 3, 124, 125, 200, 248, 249, 700, 1500], 40)),
        (300, 900, lambda: np.where(rng.random(300) < 0.1, rng.integers(125, 900, 300), rng.poisson(4, 300))),
        (3, 2000, lambda: np.array([2000, 0, 1999])),
    ]):
        lens = np.minimum(sampler(), ncols)
        rp, ci, va = random_csr(nrows, ncols, rng, lens)
        ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
        lib.b200_spmv3_plan_build.restype = C.c_void_p
        lib.b200_spmv3_plan_build.argtypes = [C.c_int, C.c_int, ip, ip, dp, C.c_int]
        h = lib.b200_spmv3_plan_build(nrows, ncols, rp.ctypes.data_as(ip), ci.ctypes.data_as(ip), va.ctypes.data_as(dp), 5)
        assert h
        nv = lib.b200_spmv3_plan_nvrows(h)
        vp = lib.b200_spmv3_plan_vptr(h)
        pieces = np.maximum(1, -(-lens // MAXROW))
        assert nv == pieces.sum()
        vptr = np.ctypeslib.as_array(vp, (nrows + 1,)).copy() if (lens > MAXROW).any() else np.arange(nrows + 1)
        assert np.array_equal(np.diff(vptr), pieces)
        lib.b200_spmv3_plan_free(h)
        plan = build_plan(lib, nrows, ncols, rp, ci, va, 5)
        # format: CSR view unchanged, one END per virtual row, every piece <= 124 entries, pieces of a row balanced
        is_end = (plan["idx"] & END) != 0
        assert is_end.sum() == nv
        assert np.array_equal(plan["rowptr"][1:] - plan["rowptr"][:-1], np.maximum(lens, 1))
        ends = np.nonzero(is_end)[0]
        plen = np.diff(np.concatenate([[-1], ends]))
        assert plen.max() <= MAXROW
        for r in np.nonzero(lens > MAXROW)[0]:
            pl = plen[vptr[r]:vptr[r + 1]]
            assert pl.sum() == lens[r] and pl.max() - pl.min() <= 1
        real = plan["desc"][plan["desc"][:, 2] > 0]
        assert real[-1, 0] + real[-1, 3] == nv and ((real[:, 1] + real[:, 2]) - (real[:, 1] & ~3) <= WT).all()
        # lane algorithm on the virtual rows + combine
        x = rng.standard_normal(ncols)
        yv = emulate_kernel(plan, nv, x, rng)
        y = np.array([yv[vptr[r]:vptr[r + 1]].sum() for r in range(nrows)])
        ref = np.array([np.dot(va[rp[r]:rp[r + 1]], x[ci[rp[r]:rp[r + 1]]]) for r in range(nrows)])
        assert np.abs(y - ref).max() <= 1e-12 * (np.abs(ref).max() + 1.0), trial


def device_fill_restated(rp, ci, va):
    """numpy restatement of k_fill_flagged (kernels/spmv.cu, the device builder's fill kernel): one stored entry per
    nonzero, one SKIP|END zero per empty row, an END at the end of every balanced piece of a long row."""
    idx, vals = [], []
    for r in range(len(rp) - 1):
        a, b = int(rp[r]), int(rp[r + 1])
        ln = b - a
        if ln == 0:
            idx.append(END | SKIP)
            vals.append(0.0)
            continue
        if ln <= MAXROW:
            ends = {ln - 1}
        else:
            pieces = -(-ln // MAXROW)
            small, big = divmod(ln, pieces)
            left, q, ends = small + (1 if big > 0 else 0), 0, set()
            for j in range(ln):
                left -= 1
                if left == 0:
                    ends.add(j)
                    q += 1
                    left = small + (1 if q < big else 0)
        for j in range(ln):
            idx.append(int(ci[a + j]) | (END if j in ends else 0))
            vals.append(va[a + j])
    return np.array(idx, dtype=np.uint32), np.array(vals)


def test_device_fill_rule_equals_host_plan_stream(lib):
    """The rule restated above gives exactly the stream of the library's fill (spmv3_fill_row, run on the host by the
    plan export); tests/test_linsys_gpu.py::test_operator_stream_from_host_csr checks the fill kernel on the device
    against the same restatement."""
    rng = np.random.default_rng(77)
    for nrows, ncols, sampler in [
        (40, 3000, lambda: rng.choice([0, 1, 3, 124, 125, 200, 248, 249, 373, 700, 1500], 40)),
        (500, 900, lambda: np.where(rng.random(500) < 0.1, rng.integers(125, 900, 500), rng.poisson(4, 500))),
        (3, 2000, lambda: np.array([2000, 0, 1999])),
        (200, 50, lambda: rng.poisson(3, 200)),
    ]:
        lens = np.minimum(sampler(), ncols)
        rp, ci, va = random_csr(nrows, ncols, rng, lens)
        plan = build_plan(lib, nrows, ncols, rp, ci, va, 7)
        idx, vals = device_fill_restated(rp, ci, va)
        assert np.array_equal(idx, plan["idx"])
        assert np.array_equal(vals, plan["vals"])

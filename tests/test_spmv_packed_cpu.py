"""CPU checks of the packed index stream of the CG loop's operators (kernels/spmv.cu `spmv3_idx24_*`): 3 bytes per
entry, column in bits 0..21, END in bit 22, SKIP in bit 23. The encode / decode helper and the producer's aligned
bulk-copy slice are host code exported by the library; the kernel's lane algorithm, re-executed in numpy on the decoded
stream, must give the row sums of the int32 stream bit for bit."""
import ctypes as C

import numpy as np
import pytest

from test_spmv_plan_cpu import WT, build_plan, emulate_kernel
from test_spmv_place_rows_cpu import c2_like

END, SKIP = 1 << 31, 1 << 30


def helpers(lib):
    lib.b200_spmv3_idx24_encode.restype = C.c_uint
    lib.b200_spmv3_idx24_encode.argtypes = [C.c_int]
    lib.b200_spmv3_idx24_decode.restype = C.c_int
    lib.b200_spmv3_idx24_decode.argtypes = [C.c_uint]
    lib.b200_spmv3_idx24_slice_bytes.restype = C.c_uint
    lib.b200_spmv3_idx24_slice_bytes.argtypes = [C.c_int, C.c_int]
    return lib.b200_spmv3_idx24_encode, lib.b200_spmv3_idx24_decode, lib.b200_spmv3_idx24_slice_bytes


def signed(v):
    return v - (1 << 32) if v >= 1 << 31 else v


def test_round_trip_every_flag_combination(lib):
    enc, dec, _ = helpers(lib)
    for col in (0, 1, 12345, (1 << 21) + 7, (1 << 22) - 1):
        for flags in (0, END, SKIP, END | SKIP):
            v = signed(col | flags)
            e = enc(v)
            assert e < 1 << 24
            assert e & ((1 << 22) - 1) == col
            assert dec(e) == v


def pack_bytes(enc, idx):
    """the device layout: entry k in bytes [3k, 3k + 3), little endian"""
    e = np.array([enc(signed(int(v))) for v in idx], dtype=np.uint32)
    return np.stack([e & 0xFF, (e >> 8) & 0xFF, (e >> 16) & 0xFF], axis=1).astype(np.uint8).ravel()


def lane_decode(dec, b, k):
    """what lane l reads for entries [k, k + 4): three 32-bit words from byte 3k, then the four 24-bit fields"""
    w = b[3 * k:3 * k + 12].view("<u4").astype(np.uint64)
    f = [w[0] & 0xFFFFFF, (w[0] >> 24) | ((w[1] & 0xFFFF) << 8), (w[1] >> 16) | ((w[2] & 0xFF) << 16), w[2] >> 8]
    return [dec(int(x)) & 0xFFFFFFFF for x in f]


@pytest.mark.parametrize("grid_cap", [3, 132])
def test_slices_cover_each_stage_and_decode_to_the_same_row_sums(lib, grid_cap):
    enc, dec, slice_bytes = helpers(lib)
    R = c2_like(6000, 2000, 10, 5 + grid_cap)
    m, n = R.shape
    plan = build_plan(lib, m, n, R.indptr.astype(np.int32), R.indices.astype(np.int32), R.data, grid_cap)
    ncw, stored = plan["ncw"], plan["stored"]
    cap_bytes = 4 * (ncw * WT + 8)
    pad = ((stored + 3) & ~3) + 8
    g_idx = np.zeros(pad, dtype=np.uint32)
    g_idx[:stored] = plan["idx"]
    b = np.concatenate([pack_bytes(enc, g_idx), np.zeros(16, np.uint8)])  # the allocation's 16 spare bytes
    desc = plan["desc"]
    for c in range(plan["grid"]):
        for g in range(plan["cta_begin"][c], plan["cta_begin"][c + 1]):
            grp = desc[g * ncw:(g + 1) * ncw]
            ka = int(grp[0][1]) & ~3
            cnt = (int(grp[-1][1] + grp[-1][2]) - ka + 3) & ~3
            start, nb = 3 * (ka & ~15), int(slice_bytes(ka, cnt))
            assert start % 16 == 0 and nb % 16 == 0
            assert start + nb >= 3 * (ka + cnt)  # covers every entry of the stage
            assert nb <= cap_bytes               # fits the stage's index area
            assert start + nb <= len(b)          # stays inside the allocation
            for kb in range(ka, ka + cnt, 4):    # every lane's 12 bytes lie in the slice and decode exactly
                assert 3 * kb + 12 <= start + nb
                assert lane_decode(dec, b, kb) == [int(v) for v in g_idx[kb:kb + 4]]
    rng = np.random.default_rng(grid_cap)
    x = rng.standard_normal(n)
    y = emulate_kernel(plan, m, x, rng)
    decoded = dict(plan)
    decoded["idx"] = np.array([dec(enc(signed(int(v)))) for v in plan["idx"]], dtype=np.int64).astype(np.uint32)
    assert np.array_equal(emulate_kernel(decoded, m, x, rng), y)

"""The update phase of the CG loop's batch kernel (kernels/cg.cu k_cg_batch) restated in numpy: k34_grid(n) virtual
blocks of 512 threads on a grid of G CTAs (CTA c runs virtual blocks c and c + G, virtual warp w of a CTA on real warp
w % 24) give z'r and ||r||_inf the bits of k_cg_update_p's grid-stride schedule (one real block per virtual block):
the same elements per thread in the same order, the same xor-shuffle warp trees, the same block and grid stages."""
import numpy as np
import pytest

VEC = 512      # threads per (virtual) block
V2 = 4         # double2 per thread (CG_FUSED_V2)
WARPS = 24     # real warps of a batch-kernel CTA (768 threads)


def k34_grid(n, sms):
    return max(1, min((n + VEC * 8 - 1) // (VEC * 8), 2 * sms))


def warp_tree(v, op):
    """common.cuh warp_sum / warp_max: xor shuffles 16, 8, 4, 2, 1 over 32 lanes; returns lane 0's value"""
    v = list(v)
    for o in (16, 8, 4, 2, 1):
        v = [op(v[l], v[l ^ o]) for l in range(32)]
    return v[0]


def add(a, b):
    return np.float64(a) + np.float64(b)


def thread_acc(n, g, v, t, z_r, r):
    """k_cg_update_p's thread t of block v: the chain acc0 += z r (rounded twice here, an fma on the device: both
    schedules share it, only the order is under test) and the running max of |r| over its elements in order"""
    acc0, acc1 = np.float64(0.0), np.float64(0.0)
    n2, stride = n >> 1, g * VEC
    idx = []
    for k in range(V2):
        i = v * VEC + t + k * stride
        if i < n2:
            idx += [2 * i, 2 * i + 1]
    if n & 1 and v == 0 and t == 0:
        idx.append(n - 1)
    for e in idx:
        acc0 = acc0 + np.float64(z_r[e][0]) * np.float64(z_r[e][1])
        acc1 = max(acc1, abs(r[e]))
    return acc0, acc1, idx


def block_stage(warp_vals, op):
    """second stage of block_sum / block_max: warp 0 reduces the per-warp values, lanes >= #warps hold 0"""
    lanes = [warp_vals[l] if l < len(warp_vals) else np.float64(0.0) for l in range(32)]
    return warp_tree(lanes, op)


def grid_stage(slots, op, threads):
    """grid_finish: thread t takes slot t (0 op slot), then a block reduction over `threads` threads"""
    per_thread = [op(np.float64(0.0), slots[t]) if t < len(slots) else np.float64(0.0) for t in range(threads)]
    warps = [warp_tree(per_thread[w * 32:(w + 1) * 32], op) for w in range(threads // 32)]
    return block_stage(warps, op)


def pairs(n, seed):
    rng = np.random.default_rng(seed)
    r = rng.standard_normal(n) * np.exp(rng.uniform(-20, 20, n))
    z = r * rng.uniform(0.1, 10.0, n)
    return list(zip(z, r)), r


def fused_schedule(n, sms, zr, r):
    g = k34_grid(n, sms)
    s_slots, m_slots, seen = [], [], []
    for v in range(g):
        accs = [thread_acc(n, g, v, t, zr, r) for t in range(VEC)]
        for a in accs:
            seen += a[2]
        ws = [warp_tree([a[0] for a in accs[w * 32:(w + 1) * 32]], add) for w in range(VEC // 32)]
        wm = [warp_tree([a[1] for a in accs[w * 32:(w + 1) * 32]], max) for w in range(VEC // 32)]
        s_slots.append(block_stage(ws, add))
        m_slots.append(block_stage(wm, max))
    return grid_stage(s_slots, add, VEC), grid_stage(m_slots, max, VEC), sorted(seen)


def batch_schedule(n, sms, grid, zr, r):
    """CTA c, real warp w, rounds: virtual warp vw = w + 24 round < 32 of virtual block c + (vw // 16) grid"""
    g = k34_grid(n, sms)
    assert g <= 2 * grid
    s_slots, m_slots, seen = [None] * g, [None] * g, []
    for c in range(grid):
        s_ws, s_wm = [np.float64(0.0)] * 32, [np.float64(0.0)] * 32
        for w in range(WARPS):
            for vw in range(w, 32, WARPS):
                v = c + (vw >> 4) * grid
                lanes = [thread_acc(n, g, v, (vw & 15) * 32 + l, zr, r) if v < g else (0.0, 0.0, [])
                         for l in range(32)]
                for a in lanes:
                    seen += a[2]
                s_ws[vw] = warp_tree([np.float64(a[0]) for a in lanes], add)
                s_wm[vw] = warp_tree([np.float64(a[1]) for a in lanes], max)
        for slot in range(2):
            v = c + slot * grid
            if v < g:
                s_slots[v] = block_stage(s_ws[slot * 16:slot * 16 + 16], add)
                m_slots[v] = block_stage(s_wm[slot * 16:slot * 16 + 16], max)
    # the finishing CTA has 768 threads; those beyond 512 hold exact zeros
    return grid_stage(s_slots, add, 768), grid_stage(m_slots, max, 768), sorted(seen)


@pytest.mark.parametrize("n,sms,grid", [
    (1, 4, 4), (2, 4, 4), (7, 4, 2),            # a grid smaller than the SM count
    (4096 * 3 + 1, 4, 4),                       # odd n, one virtual block per CTA
    (4096 * 5 + 3, 4, 4),                       # 5 virtual blocks on 4 CTAs: 1 or 2 per CTA
    (2 * 4 * 4096, 4, 4),                       # the fused limit of 4 SMs: 2 virtual blocks on every CTA
    (2 * 4 * 4096 - 1, 4, 4),                   # the largest odd n there
])
def test_virtual_blocks_reduce_like_real_blocks(n, sms, grid):
    zr, r = pairs(n, n)
    a = fused_schedule(n, sms, zr, r)
    b = batch_schedule(n, sms, grid, zr, r)
    assert a[2] == list(range(n)) and b[2] == a[2]
    assert a[0].tobytes() == b[0].tobytes()
    assert a[1].tobytes() == b[1].tobytes()

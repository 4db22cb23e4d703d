"""Experiment: how much does an m-space / n-space REORDERING of the C2 matrix buy the SpMV?
The SpMV is bound by L2->SM sector traffic (32 B per random 8-byte gather, DESIGN.md section 3.1); the
m-space ordering inside the CG operator is free (tmp = R_y^-1 A p never leaves it), so rows can be
sorted to make one gather per row sequential. Times the unchanged kernels on permuted copies."""
import ctypes as C
import os
import sys
import time

import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import reverse_cuthill_mckee

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scs_b200 import capi, problems

scale = float(os.environ.get("SCALE", "1.0"))
rng = np.random.default_rng(1234)
n = int(1_000_000 * scale)
m = 3 * n
data, indices, indptr, _ = problems.random_sparse_csc(m, n, 10, rng)
A = sp.csc_matrix((data, indices, indptr), shape=(m, n))
lib = capi.load()
reps = int(os.environ.get("REPS", "20"))


def bench(name, M):
    M = sp.csc_matrix(M)
    M.sort_indices()
    tup = (np.ascontiguousarray(M.data), np.ascontiguousarray(M.indices.astype(np.int32)),
           np.ascontiguousarray(M.indptr.astype(np.int32)), M.shape)
    hp = capi.HostProblem(tup, np.zeros(M.shape[0]), np.zeros(M.shape[1]), {"l": M.shape[0]})
    dr = np.empty(M.shape[1] + M.shape[0] + 1)
    dr[:M.shape[1]] = 1e-6
    dr[M.shape[1]:] = 10.0
    w = lib.scs_init_lin_sys_work(C.byref(hp.A), None, capi.dptr(dr))
    ab = C.c_double()
    out = []
    for op in (0, 1):
        ms = lib.scs_b200_time_spmv(w, op, reps, C.byref(ab))
        out.append(ms * 1e3)
    ms = lib.scs_b200_time_cg_iter(w, reps, C.byref(ab))
    print(f"REORDER {name:28s} A x {out[0]:6.1f} us   A'y {out[1]:6.1f} us   cg iter {ms*1e3:6.1f} us", flush=True)
    lib.scs_free_lin_sys_work(w)


bench("original", A)

t0 = time.time()
R = A.tocsr()
R.sort_indices()
lens = np.diff(R.indptr)
mincol = np.full(m, n, dtype=np.int64)
ne = lens > 0
mincol[ne] = R.indices[R.indptr[:-1][ne]]
perm = np.argsort(mincol, kind="stable")
print(f"rows by min col: {time.time()-t0:.1f}s", flush=True)
bench("rows sorted by min col", R[perm, :])

# second smallest column as tie-breaker does nothing; try: rows by min col, THEN columns by min (new) row
Rp = R[perm, :].tocsc()
Rp.sort_indices()
clen = np.diff(Rp.indptr)
minrow = np.full(n, m, dtype=np.int64)
nz = clen > 0
minrow[nz] = Rp.indices[Rp.indptr[:-1][nz]]
cperm = np.argsort(minrow, kind="stable")
bench("+ cols sorted by min row", Rp[:, cperm])

t0 = time.time()
G = sp.bmat([[None, A], [A.T, None]], format="csr")
order = reverse_cuthill_mckee(G, symmetric_mode=True)
rows = order[order < m]
cols = order[order >= m] - m
print(f"RCM on the bipartite graph: {time.time()-t0:.1f}s", flush=True)
bench("RCM rows+cols", A.tocsr()[rows, :][:, cols])
bench("RCM rows only", A.tocsr()[rows, :])

// setup.cu -- device-side construction of the two resident orientations of A at scs_init_lin_sys_work time.
//
// Replaces the host transpose of the reference (linsys/cpu/indirect/private.c:7-46: a stable counting sort that leaves
// the entries of every row in ascending source-column order): the caller's CSC arrays are copied ONCE into the
// builder's int32 / fp64 arrays by the validating copy below, the CSR of A is produced on the device by a STABLE radix sort of the entries by row index (stability = ascending column order inside
// each row, exactly the reference's order), and both flagged-stream operators are built from device data
// (b200_spmv_create_dev, kernels/spmv.cu, the builder of every operator). A host transpose took 0.8 s on 8 cores for C2.
//
// CUB (ships with the CUDA toolkit) provides the scan and the radix sort: this is setup plumbing, not the hot path.
#include "../common.cuh"
#include "../dev_api.h"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <stdio.h>
#include <stdlib.h>

extern "C" B200Spmv *b200_spmv_create_dev(int nrows, int ncols, long long nnz, const int *d_rp, const int *d_ci,
                                          const double *d_va);

#include <time.h>
// SCS_B200_SETUP_TIMING=1: wall-clock marks inside the device builder (syncs at every mark)
static double setup_now_ms() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec;
}
static void dev_mark(const char *what, double *t_last) {
  if (!getenv("SCS_B200_SETUP_TIMING")) return;
  b200_sync();
  const double t = setup_now_ms();
  fprintf(stderr, "scs_b200 setup:     device builder: %-28s %8.1f ms\n", what, t - *t_last);
  *t_last = t;
}

extern "C" int b200_dev_exclusive_scan_int(const int *d_in, int *d_out, int count) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  size_t tmp_bytes = 0;
  CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_in, d_out, count, st));
  void *tmp = b200_malloc(tmp_bytes ? tmp_bytes : 16);
  if (!tmp) return -1;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, d_in, d_out, count, st);
  // the temporary storage must outlive the kernels: the stream is synchronised before it is freed
  cudaError_t e2 = cudaStreamSynchronize(st);
  b200_free(tmp);
  if (e != cudaSuccess || e2 != cudaSuccess) {
    b200_set_error("cub::DeviceScan::ExclusiveSum", e != cudaSuccess ? e : e2, __FILE__, __LINE__);
    return -1;
  }
  return 0;
}

// rows[k] of the CSC entry k is given; cols[k] = the column whose pointer range holds k
__global__ void k_expand_cols(int n, const int *__restrict__ Ap, int *__restrict__ cols) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    for (int k = Ap[j]; k < Ap[j + 1]; ++k) cols[k] = j;
}
__global__ void k_iota(long long n, int *__restrict__ v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    v[i] = (int)i;
}
__global__ void k_count_rows(long long nnz, const int *__restrict__ Ai, int *__restrict__ cnt) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < nnz; k += (long long)gridDim.x * blockDim.x)
    atomicAdd(&cnt[Ai[k]], 1);  // integer counts: order-independent, deterministic
}
__global__ void k_gather_transposed(long long nnz, const int *__restrict__ perm, const int *__restrict__ cols,
                                    const double *__restrict__ Ax, int *__restrict__ Ti, double *__restrict__ Tx) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < nnz; q += (long long)gridDim.x * blockDim.x) {
    const int k = perm[q];
    Ti[q] = cols[k];
    Tx[q] = Ax[k];
  }
}

// The validating copy of a CSC in device memory (the caller's, or a host CSC staged there) into the builder's int32 /
// fp64 arrays,
// in two grid-stride passes templated on the index width (int, or the 64-bit indices of the DLONG ABI, narrowed as they are copied). The first pass copies the
// column pointers and sets B200_CSC_BAD_P0 (p[0] != 0) or B200_CSC_BAD_PTR (a pointer decreases or leaves [0, nnz]).
// The second runs only once the host has read a clean flag, so it may find an entry's column by bisection of the
// copied pointers: it copies the row indices (and the values, when given) and records in *d_first the smallest
// (k << 2 | code) of an entry that fails, code = B200_CSC_BAD_ROW (row outside [0, rows)), B200_CSC_BAD_UPPER (for P,
// a row below the diagonal) or B200_CSC_BAD_VAL (a non-finite value), in the order the host checks each entry.
// A truncated index (2^32 + 3 -> 3) is checked in its own width and would look valid if narrowed first.
template <typename IdxT>
__global__ void k_csc_copy_ptrs(int n, long long nnz, const IdxT *__restrict__ p, int *__restrict__ Ap,
                                unsigned *__restrict__ d_bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned bad = 0;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j <= n; j += stride) {
    const long long v = (long long)p[j];
    if (j == 0 && v != 0) bad |= B200_CSC_BAD_P0;
    if (v < 0 || v > nnz || (j < n && (long long)p[j + 1] < v)) bad |= B200_CSC_BAD_PTR;
    Ap[j] = (int)v;
  }
  if (bad) atomicOr(d_bad, bad);
}
template <typename IdxT>
__global__ void k_csc_copy_entries(int rows, int n, long long nnz, const IdxT *__restrict__ pi,
                                   const double *__restrict__ px, const int *__restrict__ Ap, int upper,
                                   int *__restrict__ Ai, double *__restrict__ Ax,
                                   unsigned long long *__restrict__ d_first, unsigned long long *__restrict__ d_ndiag) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned long long first = ~0ULL, ndiag = 0;
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < nnz; k += stride) {
    const long long r = (long long)pi[k];
    int code = -1;
    if (r < 0 || r >= rows) code = B200_CSC_BAD_ROW;
    if (upper && code < 0) {
      int lo = 0, hi = n;  // the column j with Ap[j] <= k < Ap[j + 1]: the last pointer <= k
      while (hi - lo > 1) {
        const int mid = lo + (hi - lo) / 2;
        if (Ap[mid] <= k) lo = mid; else hi = mid;
      }
      if (r > lo) code = B200_CSC_BAD_UPPER;
      ndiag += r == lo;
    }
    if (px) {
      const double v = px[k];
      if (code < 0 && !isfinite(v)) code = B200_CSC_BAD_VAL;
      Ax[k] = v;
    }
    if (code >= 0 && ((unsigned long long)k << 2 | (unsigned)code) < first) first = (unsigned long long)k << 2 | code;
    Ai[k] = (int)r;
  }
  if (first != ~0ULL) atomicMin(d_first, first);
  if (ndiag) atomicAdd(d_ndiag, ndiag);
}

static int csc_grid(long long work) {
  const long long g = (work + 255) / 256, cap = 8LL * b200_num_sms();
  return (int)(g < 1 ? 1 : g > cap ? cap : g);
}
// the pointer pass: *flags receives the B200_CSC_BAD_* bits of the pointers (one 4-byte read-back)
extern "C" int b200_csc_check_ptrs(int n, long long nnz, const void *d_p, int idx64, int *d_Ap, unsigned *flags) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  unsigned *d_bad = (unsigned *)b200_malloc(4);
  int rc = -1;
  *flags = 0;
  if (d_bad && b200_memset0(d_bad, 4) == 0) {
    if (idx64) k_csc_copy_ptrs<<<csc_grid((long long)n + 1), 256, 0, st>>>(n, nnz, (const long long *)d_p, d_Ap, d_bad);
    else k_csc_copy_ptrs<<<csc_grid((long long)n + 1), 256, 0, st>>>(n, nnz, (const int *)d_p, d_Ap, d_bad);
    b200_count_launch(1);
    if (cudaGetLastError() == cudaSuccess && b200_d2h(flags, d_bad, 4) == 0 && b200_sync() == 0) rc = 0;
  }
  b200_free(d_bad);
  return rc;
}
// the entry pass, after a clean pointer pass: *first = ~0 when every entry is valid, else the smallest k << 2 | code;
// *ndiag = the diagonal entries (upper != 0). d_x / d_Ax may be NULL (indices only). One 16-byte read-back.
extern "C" int b200_csc_copy_entries(int rows, int n, long long nnz, const void *d_i, const double *d_x, int idx64,
                                     const int *d_Ap, int upper, int *d_Ai, double *d_Ax, unsigned long long *first,
                                     long long *ndiag) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  unsigned long long *d_out = (unsigned long long *)b200_malloc(16), h[2] = {~0ULL, 0};
  int rc = -1;
  if (d_out && cudaMemsetAsync(d_out, 0xff, 8, st) == cudaSuccess && b200_memset0(d_out + 1, 8) == 0) {
    if (nnz > 0) {
      if (idx64)
        k_csc_copy_entries<<<csc_grid(nnz), 256, 0, st>>>(rows, n, nnz, (const long long *)d_i, d_x, d_Ap, upper,
                                                          d_Ai, d_Ax, d_out, d_out + 1);
      else
        k_csc_copy_entries<<<csc_grid(nnz), 256, 0, st>>>(rows, n, nnz, (const int *)d_i, d_x, d_Ap, upper, d_Ai,
                                                          d_Ax, d_out, d_out + 1);
      b200_count_launch(1);
    }
    if (cudaGetLastError() == cudaSuccess && b200_d2h(h, d_out, 16) == 0 && b200_sync() == 0) rc = 0;
  }
  b200_free(d_out);
  *first = h[0];
  *ndiag = (long long)h[1];
  return rc;
}

// The transpose of the builder's device CSC of A (m x n, int32 indices, validated): d_Tp (m + 1), d_Ti, d_Tx (nnz) =
// the CSR of A, the entries of each row by ascending column. Row counts, scan, then a stable radix sort of (row, entry
// id): stability keeps the column order of the reference's counting sort. The one transpose of the builder
// (b200_setup_ops_from_dev) and of the matrix update (scs_b200_update_matrix_device); its temporaries are freed here.
extern "C" int b200_csc_transpose(int m, int n, long long nnz, const int *d_Ap, const int *d_Ai, const double *d_Ax,
                                  int *d_Tp, int *d_Ti, double *d_Tx) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  int *d_cnt = (int *)b200_malloc((size_t)(m + 2) * 4);
  int *d_cols = (int *)b200_malloc((size_t)nnz * 4), *d_iota = (int *)b200_malloc((size_t)nnz * 4);
  int *d_keys = (int *)b200_malloc((size_t)nnz * 4), *d_perm = (int *)b200_malloc((size_t)nnz * 4);
  void *d_tmp = nullptr;
  const int nsm = b200_num_sms();
  int rc = -1;
  do {
    if (!d_cnt || !d_cols || !d_iota || !d_keys || !d_perm) break;
    if (b200_memset0(d_cnt, (size_t)(m + 2) * 4) != 0) break;
    k_count_rows<<<8 * nsm, 256, 0, st>>>(nnz, d_Ai, d_cnt);
    if (b200_dev_exclusive_scan_int(d_cnt, d_Tp, m + 1) != 0) break;
    k_expand_cols<<<8 * nsm, 256, 0, st>>>(n, d_Ap, d_cols);
    k_iota<<<8 * nsm, 256, 0, st>>>(nnz, d_iota);
    int bits = 1;
    while ((1LL << bits) < (long long)m) ++bits;
    size_t tmp_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_Ai, d_keys, d_iota, d_perm, (int)nnz, 0, bits, st) !=
        cudaSuccess)
      break;
    d_tmp = b200_malloc(tmp_bytes ? tmp_bytes : 16);
    if (!d_tmp) break;
    if (cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_Ai, d_keys, d_iota, d_perm, (int)nnz, 0, bits, st) !=
        cudaSuccess)
      break;
    k_gather_transposed<<<8 * nsm, 256, 0, st>>>(nnz, d_perm, d_cols, d_Ax, d_Ti, d_Tx);
    b200_count_launch(4);
    if (cudaGetLastError() != cudaSuccess || b200_sync() != 0) break;
    rc = 0;
  } while (0);
  b200_sync();
  b200_free(d_cnt); b200_free(d_cols); b200_free(d_iota); b200_free(d_keys); b200_free(d_perm); b200_free(d_tmp);
  return rc;
}

// Both operators from the builder's device CSC of A (m x n; m, n or nnz may be 0; int32 indices, already validated).
// Returns 0 and sets *A_out (CSR of A) / *At_out (CSR of A' = the CSC arrays); < 0 on failure. The arrays are read
// only, and may be freed in stream order once this returns.
extern "C" int b200_setup_ops_from_dev(int m, int n, long long nnz, const int *d_Ap, const int *d_Ai,
                                       const double *d_Ax, B200Spmv **A_out, B200Spmv **At_out) {
  *A_out = *At_out = nullptr;
  if (b200_runtime_init() != 0) return -1;
  int *d_Tp = (int *)b200_malloc((size_t)(m + 2) * 4);
  int *d_Ti = (int *)b200_malloc((size_t)nnz * 4);
  double *d_Tx = (double *)b200_malloc((size_t)nnz * 8);
  int rc = -1;
  B200Spmv *A = nullptr, *At = nullptr;
  double t_mark = setup_now_ms();
  dev_mark("allocations", &t_mark);
  do {
    if (!d_Tp || !d_Ti || !d_Tx) break;
    // A' first: its CSR is the CSC as given
    At = b200_spmv_create_dev(n, m, nnz, d_Ap, d_Ai, d_Ax);
    if (!At) break;
    dev_mark("operator A' (stream + tiles)", &t_mark);
    if (b200_csc_transpose(m, n, nnz, d_Ap, d_Ai, d_Ax, d_Tp, d_Ti, d_Tx) != 0) break;
    dev_mark("transpose (count, scan, sort)", &t_mark);
    A = b200_spmv_create_dev(m, n, nnz, d_Tp, d_Ti, d_Tx);
    if (!A) break;
    dev_mark("operator A (stream + tiles)", &t_mark);
    rc = 0;
  } while (0);
  b200_sync();
  b200_free(d_Tp); b200_free(d_Ti); b200_free(d_Tx);
  dev_mark("frees", &t_mark);
  if (rc != 0) {
    b200_spmv_destroy(A);
    b200_spmv_destroy(At);
    // a pending CUDA error names the failure; else the failing step has set its own message (e.g. a size limit)
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) b200_set_error("b200_setup_ops_from_dev", e, __FILE__, __LINE__);
    return rc;
  }
  *A_out = A;
  *At_out = At;
  return 0;
}
// ---------------------------------------------------------------------------------------------
// Row order for the CG-internal copy of A: rows by their smallest column index (stable, so equal keys keep the
// original order; empty rows go last). perm[new] = old row; b200_spmv_permuted_rows refines the order and inverts it.
__global__ void k_min_col_key(int nrows, int ncols, const int *__restrict__ sp, const int *__restrict__ ci,
                              int *__restrict__ key) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    const unsigned v = (unsigned)ci[sp[r]];  // first stored entry of the row: its smallest column (rows are sorted)
    key[r] = (v & B200_FLAG_SKIP) ? ncols : (int)(v & B200_COLMASK);
  }
}
extern "C" int b200_perm_rows_by_min_col(const B200Spmv *A, int *d_perm) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int nrows = b200_spmv_nrows(A), ncols = b200_spmv_ncols(A);
  int *d_key = (int *)b200_malloc((size_t)nrows * 4), *d_key2 = (int *)b200_malloc((size_t)nrows * 4);
  int *d_iota = (int *)b200_malloc((size_t)nrows * 4);
  void *d_tmp = nullptr;
  int rc = -1;
  do {
    if (!d_key || !d_key2 || !d_iota) break;
    const int g = 8 * b200_num_sms();
    k_min_col_key<<<g, 256, 0, st>>>(nrows, ncols, b200_spmv_rowptr(A), b200_spmv_colidx(A), d_key);
    k_iota<<<g, 256, 0, st>>>(nrows, d_iota);
    int bits = 1;
    while ((1LL << bits) < (long long)ncols + 1) ++bits;
    size_t tmp_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_key, d_key2, d_iota, d_perm, nrows, 0, bits, st) != cudaSuccess)
      break;
    d_tmp = b200_malloc(tmp_bytes ? tmp_bytes : 16);
    if (!d_tmp) break;
    if (cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_key, d_key2, d_iota, d_perm, nrows, 0, bits, st) != cudaSuccess)
      break;
    b200_count_launch(3);
    if (cudaGetLastError() != cudaSuccess || b200_sync() != 0) break;
    rc = 0;
  } while (0);
  b200_sync();
  b200_free(d_key); b200_free(d_key2); b200_free(d_iota); b200_free(d_tmp);
  return rc;
}
__global__ void k_gather_vec(int n, const int *__restrict__ perm, const double *__restrict__ src, double *__restrict__ dst) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[perm[i]];
}
extern "C" int b200_gather_vec(int n, const int *d_perm, const double *d_src, double *d_dst) {
  k_gather_vec<<<8 * b200_num_sms(), 256, 0, (cudaStream_t)b200_stream()>>>(n, d_perm, d_src, d_dst);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// The full symmetric P from its upper-triangular CSC on the device, in CSR: row r holds first the mirrors of column r's strict-upper entries in k order, then its
// direct entries (r, j), j >= r, by ascending j. A stable radix sort by row of the list [every entry's mirror in (j, k)
// order, then every direct entry in (j, k) order] gives that order; the mirror of a diagonal entry is keyed to row n,
// which sorts last and is dropped. The structure is built first, with d_Fsrc[q] = the CSC entry that full entry q
// copies, so that the values can be taken after the upper CSC has been equilibrated in place.
__global__ void k_sym_items(int n, long long nnz, const int *__restrict__ Pi, const int *__restrict__ cols,
                            int *__restrict__ keys) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nnz; t += (long long)gridDim.x * blockDim.x) {
    const int i = Pi[t], j = cols[t];
    keys[t] = i != j ? j : n;  // mirror (j, i): row j
    keys[nnz + t] = i;         // direct (i, j): row i
  }
}
__global__ void k_sym_gather(long long full, long long nnz, const int *__restrict__ item, const int *__restrict__ Pi,
                             const int *__restrict__ cols, int *__restrict__ Fi, int *__restrict__ Fsrc) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < full; q += (long long)gridDim.x * blockDim.x) {
    const long long t = item[q];
    const long long k = t < nnz ? t : t - nnz;
    Fi[q] = t < nnz ? Pi[k] : cols[k];
    Fsrc[q] = (int)k;
  }
}
// n x n upper CSC (d_Pp, d_Pi, nnz entries, `full` entries in the symmetric form) -> d_Fp (n + 1), d_Fi, d_Fsrc (full)
extern "C" int b200_sym_expand_structure(int n, long long nnz, long long full, const int *d_Pp, const int *d_Pi,
                                         int *d_Fp, int *d_Fi, int *d_Fsrc) {
  if (2 * nnz > 2147483647LL) {
    b200_set_error("b200_sym_expand_structure: 2 nnz(P) must fit in an int", cudaErrorInvalidValue, __FILE__, __LINE__);
    return -1;
  }
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int items = (int)(2 * nnz), g = csc_grid(items);
  int *d_cols = (int *)b200_malloc((size_t)nnz * 4), *d_keys = (int *)b200_malloc((size_t)items * 4);
  int *d_keys2 = (int *)b200_malloc((size_t)items * 4), *d_iota = (int *)b200_malloc((size_t)items * 4);
  int *d_item = (int *)b200_malloc((size_t)items * 4), *d_cnt = (int *)b200_malloc((size_t)(n + 1) * 4);
  void *d_tmp = nullptr;
  int rc = -1;
  do {
    if (!d_cols || !d_keys || !d_keys2 || !d_iota || !d_item || !d_cnt) break;
    if (b200_memset0(d_cnt, (size_t)(n + 1) * 4) != 0) break;
    k_expand_cols<<<g, 256, 0, st>>>(n, d_Pp, d_cols);
    k_sym_items<<<g, 256, 0, st>>>(n, nnz, d_Pi, d_cols, d_keys);
    k_iota<<<g, 256, 0, st>>>(items, d_iota);
    int bits = 1;
    while ((1LL << bits) < (long long)n + 1) ++bits;
    size_t tmp_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_keys, d_keys2, d_iota, d_item, items, 0, bits, st) !=
        cudaSuccess)
      break;
    d_tmp = b200_malloc(tmp_bytes ? tmp_bytes : 16);
    if (!d_tmp) break;
    if (cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_keys, d_keys2, d_iota, d_item, items, 0, bits, st) !=
        cudaSuccess)
      break;
    k_count_rows<<<g, 256, 0, st>>>(full, d_keys2, d_cnt);
    k_sym_gather<<<g, 256, 0, st>>>(full, nnz, d_item, d_Pi, d_cols, d_Fi, d_Fsrc);
    b200_count_launch(6);
    if (cudaGetLastError() != cudaSuccess || b200_dev_exclusive_scan_int(d_cnt, d_Fp, n + 1) != 0) break;
    rc = 0;
  } while (0);
  b200_sync();
  b200_free(d_cols); b200_free(d_keys); b200_free(d_keys2); b200_free(d_iota); b200_free(d_item); b200_free(d_cnt);
  b200_free(d_tmp);
  return rc;
}
// d_Fx[q] = d_Px[d_Fsrc[q]]; d_diag[r] = the sum of row r's diagonal entries in row order
__global__ void k_sym_values(int n, const int *__restrict__ Fp, const int *__restrict__ Fi,
                             const int *__restrict__ Fsrc, const double *__restrict__ Px, double *__restrict__ Fx,
                             double *__restrict__ diag) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    double d = 0.0;
    for (int q = Fp[r]; q < Fp[r + 1]; ++q) {
      const double v = Px[Fsrc[q]];
      Fx[q] = v;
      if (Fi[q] == r) d += v;
    }
    diag[r] = d;
  }
}
// the values of the full symmetric P (d_Fx, `full`) and its diagonal (d_diag, n) from the structure above and the
// values of the upper CSC: what b200_sym_build builds P's operator from, and what the matrix update scatters into it
extern "C" int b200_sym_values(int n, const int *d_Fp, const int *d_Fi, const int *d_Fsrc, const double *d_Px,
                               double *d_Fx, double *d_diag) {
  k_sym_values<<<csc_grid(n), 256, 0, (cudaStream_t)b200_stream()>>>(n, d_Fp, d_Fi, d_Fsrc, d_Px, d_Fx, d_diag);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}
// the operator of the full symmetric P (*P_out) and its diagonal (d_diag, n) from the structure above and the values
// of the upper CSC
extern "C" int b200_sym_build(int n, long long full, const int *d_Fp, const int *d_Fi, const int *d_Fsrc,
                              const double *d_Px, double *d_diag, B200Spmv **P_out) {
  double *d_Fx = (double *)b200_malloc((size_t)full * 8);
  *P_out = nullptr;
  if (!d_Fx) return -1;
  if (b200_sym_values(n, d_Fp, d_Fi, d_Fsrc, d_Px, d_Fx, d_diag) == 0)
    *P_out = b200_spmv_create_dev(n, n, full, d_Fp, d_Fi, d_Fx);
  b200_sync();
  b200_free(d_Fx);
  return *P_out ? 0 : -1;
}

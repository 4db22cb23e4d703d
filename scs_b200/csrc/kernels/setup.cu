// setup.cu -- device-side construction of the two resident orientations of A at scs_init_lin_sys_work time.
//
// Replaces, for the single-GPU path, the host transpose (reference linsys/cpu/indirect/private.c:7-46: a stable
// counting sort that leaves the entries of every row in ascending source-column order) and the host SpMV plan
// builder: the user's CSC arrays are uploaded ONCE, the CSR of A is produced on the device by a STABLE radix sort
// of the entries by row index (stability = ascending column order inside each row, exactly the reference's
// order), and both flagged-stream operators are built from device data (b200_spmv_create_dev, kernels/spmv.cu).
// VERDICT r01 item 7: the host transpose alone took 0.8 s on 8 cores for C2.
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

// Both operators from the host CSC of A (m x n). Returns 0 and sets *A_out (CSR of A) / *At_out (CSR of A' = the CSC
// arrays); returns 1 when the device path declines (the caller then uses the host builders); < 0 on a CUDA error.
extern "C" int b200_setup_ops_from_csc(int m, int n, const int *h_Ap, const int *h_Ai, const double *h_Ax,
                                       B200Spmv **A_out, B200Spmv **At_out) {
  *A_out = *At_out = nullptr;
  if (b200_runtime_init() != 0) return -1;
  {
    const char *e = getenv("SCS_B200_HOST_SETUP");
    if (e && atoi(e) != 0) return 1;
  }
  const long long nnz = h_Ap[n];
  if (nnz <= 0 || m <= 0 || n <= 0 || nnz > 2000000000LL) return 1;
  cudaStream_t st = (cudaStream_t)b200_stream();
  int *d_Ap = (int *)b200_malloc((size_t)(n + 1) * 4), *d_Ai = (int *)b200_malloc((size_t)nnz * 4);
  double *d_Ax = (double *)b200_malloc((size_t)nnz * 8);
  int *d_Tp = (int *)b200_malloc((size_t)(m + 2) * 4), *d_cnt = (int *)b200_malloc((size_t)(m + 2) * 4);
  int *d_Ti = (int *)b200_malloc((size_t)nnz * 4);
  double *d_Tx = (double *)b200_malloc((size_t)nnz * 8);
  int *d_cols = (int *)b200_malloc((size_t)nnz * 4), *d_iota = (int *)b200_malloc((size_t)nnz * 4);
  int *d_keys = (int *)b200_malloc((size_t)nnz * 4), *d_perm = (int *)b200_malloc((size_t)nnz * 4);
  void *d_tmp = nullptr;
  int rc = -1;
  B200Spmv *A = nullptr, *At = nullptr;
  const int nsm = b200_num_sms();
  double t_mark = setup_now_ms();
  dev_mark("allocations", &t_mark);
  do {
    if (!d_Ap || !d_Ai || !d_Ax || !d_Tp || !d_cnt || !d_Ti || !d_Tx || !d_cols || !d_iota || !d_keys || !d_perm) break;
    if (b200_h2d(d_Ap, h_Ap, (size_t)(n + 1) * 4) != 0 || b200_h2d(d_Ai, h_Ai, (size_t)nnz * 4) != 0 ||
        b200_h2d(d_Ax, h_Ax, (size_t)nnz * 8) != 0)
      break;
    dev_mark("H2D of the CSC arrays", &t_mark);
    // A' first: its CSR is the CSC as given
    At = b200_spmv_create_dev(n, m, nnz, d_Ap, d_Ai, d_Ax);
    if (!At) { rc = 1; break; }
    dev_mark("operator A' (stream + tiles)", &t_mark);
    // transpose: row counts -> row pointers; stable sort of (row, entry id) -> entries of each row by ascending column
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
    dev_mark("transpose (count, scan, sort)", &t_mark);
    A = b200_spmv_create_dev(m, n, nnz, d_Tp, d_Ti, d_Tx);
    if (!A) { rc = 1; break; }
    dev_mark("operator A (stream + tiles)", &t_mark);
    rc = 0;
  } while (0);
  b200_sync();
  b200_free(d_Ap); b200_free(d_Ai); b200_free(d_Ax); b200_free(d_Tp); b200_free(d_cnt); b200_free(d_Ti);
  b200_free(d_Tx); b200_free(d_cols); b200_free(d_iota); b200_free(d_keys); b200_free(d_perm); b200_free(d_tmp);
  dev_mark("frees", &t_mark);
  if (rc != 0) {
    b200_spmv_destroy(A);
    b200_spmv_destroy(At);
    if (rc < 0) b200_set_error("b200_setup_ops_from_csc", cudaGetLastError(), __FILE__, __LINE__);
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

// equil.cu -- Ruiz + L2 equilibration of A on the device (P = 0 case), in place on BOTH
// resident orientations of the matrix (CSR of A and CSR of A'), producing D (rows) and E (cols).
//
// Replaces reference linsys/scs_matrix.c:229-496 (compute_ruiz_mats / compute_l2_mats /
// rescale / normalize_a_p: 25 Ruiz passes + 1 L2 pass, limits 1e-4 / 1e4, D constant inside
// every cone of size > 1 via enforce_cone_boundaries, src/cones.c:366-379).  This is setup, not
// the per-iteration hot loop; SURVEY.md 8(f)-2 lists it as the second "next" item because the
// 26 x 2 sweeps over nnz dominate setup_time (hence e2e) at nnz >= 1e7 when done on the host.
//
// Row norms come from the row-major copy and column norms from the column-major copy, so every
// reduction is a sequential loop over one stored row: no atomics, bit-reproducible; the sums of
// squares run in ascending column (resp. row) order like the reference's scatter loops. Both
// copies are rescaled by the same factor Dt[i]*Et[j], so they stay bit-identical.
#include "../common.cuh"
#include "../admm_api.h"
#include <math.h>
#include <stdlib.h>
#include <vector>

#define MIN_NORM_FACTOR (1e-4)
#define MAX_NORM_FACTOR (1e4)
#define DIV_EPS (1e-18)

__device__ __forceinline__ double eq_limit(double x) {
  x = x < MIN_NORM_FACTOR ? 1.0 : x;
  return x > MAX_NORM_FACTOR ? MAX_NORM_FACTOR : x;
}
// out[r] = max_k |v_k| (l2 == 0) or sqrt(sum_k v_k^2) (l2 == 1) over stored row r
__global__ void k_eq_rownorm(int nrows, const int *__restrict__ rowptr, const double *__restrict__ vals,
                             int l2, double *__restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    double acc = 0.0;
    const int a = rowptr[r], b = rowptr[r + 1];
    if (l2) {
      for (int k = a; k < b; ++k) acc += vals[k] * vals[k];
      acc = sqrt(acc);
    } else {
      for (int k = a; k < b; ++k) acc = fmax(acc, fabs(vals[k]));
    }
    out[r] = acc;
  }
}
// one block per cone block: v[off .. off+len) := max (mean == 0) or mean (mean == 1) of the block
__global__ void __launch_bounds__(256)
k_eq_cone_aggregate(const int *__restrict__ off, int mean, double *__restrict__ v) {
  __shared__ double s_red[32];
  __shared__ double s_out;
  const int o = off[blockIdx.x], len = off[blockIdx.x + 1] - o;
  double a[1] = {0.0};
  if (mean) {
    for (int i = threadIdx.x; i < len; i += blockDim.x) a[0] += v[o + i];
    block_sum<1>(a, s_red);
  } else {
    for (int i = threadIdx.x; i < len; i += blockDim.x) a[0] = fmax(a[0], fabs(v[o + i]));
    block_max<1>(a, s_red);
  }
  if (threadIdx.x == 0) s_out = mean ? (len > 0 ? a[0] / len : 0.0) : a[0];
  __syncthreads();
  const double w = s_out;
  for (int i = threadIdx.x; i < len; i += blockDim.x) v[o + i] = w;
}
// t = 1 / sqrt(limit(t)) ; acc *= t
__global__ void k_eq_finish(long long len, double *__restrict__ t, double *__restrict__ acc) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len;
       i += (long long)gridDim.x * blockDim.x) {
    double x = sqrt(eq_limit(t[i]));
    x = (x < DIV_EPS) ? (1.0 / DIV_EPS) : 1.0 / x;
    t[i] = x;
    acc[i] *= x;
  }
}
// vals[k] *= rowscale[r] * colscale[colidx[k]]   (row-major copy: rowscale = Dt, colscale = Et;
// column-major copy: rowscale = Et, colscale = Dt -- the product is the same number)
__global__ void k_eq_rescale(int nrows, const int *__restrict__ rowptr, const int *__restrict__ colidx,
                             double *__restrict__ vals, const double *__restrict__ rowscale,
                             const double *__restrict__ colscale, int row_is_d) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    const double rs = rowscale[r];
    const int a = rowptr[r], b = rowptr[r + 1];
    for (int k = a; k < b; ++k) {
      const double cs = colscale[colidx[k] & B200_COLMASK];  // flags in the top bits (spmv.cu v3)
      // reference: A->x[j] *= Dt[A->i[j]] * ei  -> always D * E in this order
      vals[k] *= row_is_d ? (rs * cs) : (cs * rs);
    }
  }
}

static int eq_grid(long long n) {
  long long g = (n + 255) / 256, cap = 16LL * b200_num_sms();
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

// A_rows: CSR of A (m rows), A_cols: CSR of A' (n rows). bnd[0] = rows before the first cone that
// must share one D (z + l + bsize); bnd[1..nbnd) = sizes of those cones. d_D (m), d_E (n): outputs.
extern "C" int b200_equilibrate_dev(B200Spmv *A_rows, B200Spmv *A_cols, const int *bnd, int nbnd,
                                    double *d_D, double *d_E) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int m = b200_spmv_nrows(A_rows), n = b200_spmv_nrows(A_cols);
  double *d_Dt = (double *)b200_malloc((size_t)m * 8);
  double *d_Et = (double *)b200_malloc((size_t)n * 8);
  int *d_off = nullptr;
  int rc = -1;
  const int ncones = nbnd - 1;
  if (!d_Dt || !d_Et) goto out;
  if (ncones > 0) {
    std::vector<int> off(ncones + 1);
    off[0] = bnd[0];
    for (int i = 0; i < ncones; ++i) off[i + 1] = off[i] + bnd[i + 1];
    d_off = (int *)b200_malloc((size_t)(ncones + 1) * 4);
    if (!d_off || b200_h2d(d_off, off.data(), (size_t)(ncones + 1) * 4) != 0 || b200_sync() != 0) goto out;
  }
  if (b200_vec_fill(m, d_D, 1.0) != 0 || b200_vec_fill(n, d_E, 1.0) != 0) goto out;
  {
    double *vr = const_cast<double *>(b200_spmv_vals(A_rows));
    double *vc = const_cast<double *>(b200_spmv_vals(A_cols));
    for (int pass = 0; pass < 26; ++pass) {
      const int l2 = pass == 25;  // 25 Ruiz passes then one L2 pass
      k_eq_rownorm<<<eq_grid(m), 256, 0, st>>>(m, b200_spmv_rowptr(A_rows), vr, l2, d_Dt);
      k_eq_rownorm<<<eq_grid(n), 256, 0, st>>>(n, b200_spmv_rowptr(A_cols), vc, l2, d_Et);
      if (ncones > 0) k_eq_cone_aggregate<<<ncones, 256, 0, st>>>(d_off, l2, d_Dt);
      k_eq_finish<<<eq_grid(m), 256, 0, st>>>(m, d_Dt, d_D);
      k_eq_finish<<<eq_grid(n), 256, 0, st>>>(n, d_Et, d_E);
      k_eq_rescale<<<eq_grid(m), 256, 0, st>>>(m, b200_spmv_rowptr(A_rows), b200_spmv_colidx(A_rows), vr,
                                               d_Dt, d_Et, 1);
      k_eq_rescale<<<eq_grid(n), 256, 0, st>>>(n, b200_spmv_rowptr(A_cols), b200_spmv_colidx(A_cols), vc,
                                               d_Et, d_Dt, 0);
      b200_count_launch(ncones > 0 ? 7 : 6);
    }
  }
  if (cudaGetLastError() != cudaSuccess) goto out;
  if (b200_sync() != 0) goto out;
  rc = 0;
out:
  b200_free(d_Dt);
  b200_free(d_Et);
  b200_free(d_off);
  return rc;
}

// vals[k] *= D[row] * E[col] once, with the accumulated D, E (row-sharded path: the local blocks
// of A are scaled after D, E were computed from the full matrix).
extern "C" int b200_rescale_dev(B200Spmv *M, const double *d_rowscale, const double *d_colscale,
                                int row_is_d) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int nr = b200_spmv_nrows(M);
  if (nr <= 0) return 0;
  k_eq_rescale<<<eq_grid(nr), 256, 0, st>>>(nr, b200_spmv_rowptr(M), b200_spmv_colidx(M),
                                            const_cast<double *>(b200_spmv_vals(M)), d_rowscale,
                                            d_colscale, row_is_d);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Ruiz + L2 equilibration with P != 0 on the device, bit for bit host/equilibrate.c: A in place on both resident
// orientations, P in place on its upper CSC (d_Pp, d_Pi, d_Px). The row pass of the symmetric P reads the structure of
// the full P (b200_sym_expand_structure: d_Fp, d_Fi, d_Fsrc = the CSC entry of every full entry). Every sum runs in the
// host's order with rounded products and sums (__dmul_rn / __dadd_rn: no contraction into an FMA), and the cone-block
// mean is a sequential sum in row order, as enforce_boundaries takes it.
// out[r] = sqrt(sum_k v_k^2) over stored row r, in row order
__global__ void k_eq_rownorm_l2_rn(int nrows, const int *__restrict__ rowptr, const double *__restrict__ vals,
                                   double *__restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int k = rowptr[r]; k < rowptr[r + 1]; ++k) acc = __dadd_rn(acc, __dmul_rn(vals[k], vals[k]));
    out[r] = sqrt(acc);
  }
}
// one thread per cone block: v[off .. off+len) := the mean of the block, summed in row order
__global__ void k_eq_cone_mean_seq(int ncones, const int *__restrict__ off, double *__restrict__ v) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ncones; c += gridDim.x * blockDim.x) {
    const int o = off[c], len = off[c + 1] - o;
    double w = 0.0;
    for (int i = 0; i < len; ++i) w += v[o + i];
    w = len > 0 ? w / len : 0.0;
    for (int i = 0; i < len; ++i) v[o + i] = w;
  }
}
// Et[x] before the limit: Ruiz (l2 == 0): max(|P| over row x of the full P, |A| over column x); L2: sqrt(the P squares
// in the host's scatter order -- column x of the upper CSC in k order, then the row-x entries of columns j > x by
// ascending j -- plus A's column-x sum of squares)
__global__ void k_eq_col_qp(int n, int l2, const int *__restrict__ Acp, const double *__restrict__ Acx,
                            const int *__restrict__ Pp, const double *__restrict__ Px, const int *__restrict__ Fp,
                            const int *__restrict__ Fi, const int *__restrict__ Fsrc, double *__restrict__ Et) {
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    double t = 0.0, a = 0.0;
    if (l2) {
      for (int k = Pp[x]; k < Pp[x + 1]; ++k) t = __dadd_rn(t, __dmul_rn(Px[k], Px[k]));
      for (int q = Fp[x]; q < Fp[x + 1]; ++q)
        if (Fi[q] > x) { const double v = Px[Fsrc[q]]; t = __dadd_rn(t, __dmul_rn(v, v)); }
      for (int k = Acp[x]; k < Acp[x + 1]; ++k) a = __dadd_rn(a, __dmul_rn(Acx[k], Acx[k]));
      Et[x] = sqrt(__dadd_rn(t, a));
    } else {
      for (int q = Fp[x]; q < Fp[x + 1]; ++q) t = fmax(t, fabs(Px[Fsrc[q]]));
      for (int k = Acp[x]; k < Acp[x + 1]; ++k) a = fmax(a, fabs(Acx[k]));
      Et[x] = a > t ? a : t;
    }
  }
}
// Px[k] *= Et[row] * Et[col] on the upper CSC
__global__ void k_eq_rescale_p(int n, const int *__restrict__ Pp, const int *__restrict__ Pi, double *__restrict__ Px,
                               const double *__restrict__ Et) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
    const double ec = Et[c];
    for (int k = Pp[c]; k < Pp[c + 1]; ++k) Px[k] *= Et[Pi[k]] * ec;
  }
}

extern "C" int b200_equilibrate_qp_dev(B200Spmv *A_rows, B200Spmv *A_cols, const int *d_Pp, const int *d_Pi,
                                       double *d_Px, const int *d_Fp, const int *d_Fi, const int *d_Fsrc,
                                       const int *bnd, int nbnd, double *d_D, double *d_E) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int m = b200_spmv_nrows(A_rows), n = b200_spmv_nrows(A_cols);
  double *d_Dt = (double *)b200_malloc((size_t)m * 8);
  double *d_Et = (double *)b200_malloc((size_t)n * 8);
  int *d_off = nullptr;
  int rc = -1;
  const int ncones = nbnd - 1;
  if (!d_Dt || !d_Et) goto out;
  if (ncones > 0) {
    std::vector<int> off(ncones + 1);
    off[0] = bnd[0];
    for (int i = 0; i < ncones; ++i) off[i + 1] = off[i] + bnd[i + 1];
    d_off = (int *)b200_malloc((size_t)(ncones + 1) * 4);
    if (!d_off || b200_h2d(d_off, off.data(), (size_t)(ncones + 1) * 4) != 0 || b200_sync() != 0) goto out;
  }
  if (b200_vec_fill(m, d_D, 1.0) != 0 || b200_vec_fill(n, d_E, 1.0) != 0) goto out;
  {
    double *vr = const_cast<double *>(b200_spmv_vals(A_rows));
    double *vc = const_cast<double *>(b200_spmv_vals(A_cols));
    for (int pass = 0; pass < 26; ++pass) {
      const int l2 = pass == 25;  // 25 Ruiz passes then one L2 pass
      if (l2) k_eq_rownorm_l2_rn<<<eq_grid(m), 256, 0, st>>>(m, b200_spmv_rowptr(A_rows), vr, d_Dt);
      else k_eq_rownorm<<<eq_grid(m), 256, 0, st>>>(m, b200_spmv_rowptr(A_rows), vr, 0, d_Dt);
      k_eq_col_qp<<<eq_grid(n), 256, 0, st>>>(n, l2, b200_spmv_rowptr(A_cols), vc, d_Pp, d_Px, d_Fp, d_Fi, d_Fsrc,
                                               d_Et);
      if (ncones > 0) {
        if (l2) k_eq_cone_mean_seq<<<eq_grid(ncones), 256, 0, st>>>(ncones, d_off, d_Dt);
        else k_eq_cone_aggregate<<<ncones, 256, 0, st>>>(d_off, 0, d_Dt);
      }
      k_eq_finish<<<eq_grid(m), 256, 0, st>>>(m, d_Dt, d_D);
      k_eq_finish<<<eq_grid(n), 256, 0, st>>>(n, d_Et, d_E);
      k_eq_rescale<<<eq_grid(m), 256, 0, st>>>(m, b200_spmv_rowptr(A_rows), b200_spmv_colidx(A_rows), vr,
                                               d_Dt, d_Et, 1);
      k_eq_rescale<<<eq_grid(n), 256, 0, st>>>(n, b200_spmv_rowptr(A_cols), b200_spmv_colidx(A_cols), vc,
                                               d_Et, d_Dt, 0);
      k_eq_rescale_p<<<eq_grid(n), 256, 0, st>>>(n, d_Pp, d_Pi, d_Px, d_Et);
      b200_count_launch(ncones > 0 ? 8 : 7);
    }
  }
  if (cudaGetLastError() != cudaSuccess) goto out;
  if (b200_sync() != 0) goto out;
  rc = 0;
out:
  b200_free(d_Dt);
  b200_free(d_Et);
  b200_free(d_off);
  return rc;
}

// ---------------------------------------------------------------------------------------------
// b and c from their device originals (every door): out = orig * scale (scale NULL: a copy), with max |orig| and
// max |out| into d_max[0], d_max[1]. A maximum does not depend on the order it is taken in, and the products are
// elementwise, so the result is the reference's normalize_b_c bit for bit. Non-negative doubles order like their bit
// patterns, so the maxima are taken with an integer atomicMax, and a NaN entry is skipped, as the reference's norm_inf
// (src/linalg.c:71-79) skips it.
__device__ __forceinline__ void bc_atomic_max(double *d_max, double v) {
  for (int o = 16; o > 0; o >>= 1) {
    const double w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  if ((threadIdx.x & 31) == 0 && v > 0.0)
    atomicMax((unsigned long long *)d_max, (unsigned long long)__double_as_longlong(v));
}
__global__ void k_bc_scale_max(long long len, const double *__restrict__ orig, const double *__restrict__ scale,
                               double *__restrict__ out, double *__restrict__ d_max) {
  double mo = 0.0, mx = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  // every thread of the warp runs the same number of rounds of the shuffle below
  for (long long base = blockIdx.x * (long long)blockDim.x; base < len; base += stride) {
    const long long i = base + threadIdx.x;
    if (i < len) {
      const double o = orig[i], v = scale ? o * scale[i] : o;
      out[i] = v;
      if (fabs(o) > mo) mo = fabs(o);
      if (fabs(v) > mx) mx = fabs(v);
    }
  }
  bc_atomic_max(d_max, mo);
  bc_atomic_max(d_max + 1, mx);
}
__global__ void k_bc_sigma(long long m, long long n, double *__restrict__ b, double *__restrict__ c, double sigma) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m + n; i += stride) {
    if (i < n) c[i] *= sigma;
    else b[i - n] *= sigma;
  }
}
// h_max (host, 4): max |b_orig|, max |b|, max |c_orig|, max |c|; one 32-byte read-back
extern "C" int b200_normalize_b_c_dev(int m, int n, const double *d_b_orig, const double *d_c_orig, const double *d_D,
                                      const double *d_E, double *d_b, double *d_c, double *h_max) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  double *d_mx = (double *)b200_malloc(4 * 8);
  int rc = -1;
  if (d_mx && b200_memset0(d_mx, 4 * 8) == 0) {
    k_bc_scale_max<<<eq_grid(m), 256, 0, st>>>(m, d_b_orig, d_D, d_b, d_mx);
    k_bc_scale_max<<<eq_grid(n), 256, 0, st>>>(n, d_c_orig, d_E, d_c, d_mx + 2);
    b200_count_launch(2);
    if (cudaGetLastError() == cudaSuccess && b200_d2h(h_max, d_mx, 4 * 8) == 0 && b200_sync() == 0) rc = 0;
  }
  b200_free(d_mx);
  return rc;
}
extern "C" int b200_scale_b_c(int m, int n, double *d_b, double *d_c, double sigma) {
  k_bc_sigma<<<eq_grid((long long)m + n), 256, 0, (cudaStream_t)b200_stream()>>>(m, n, d_b, d_c, sigma);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// aa.cu -- Anderson acceleration of the ADMM fixed-point map on the device.
//
// Replaces reference src/aa.c: init_accel_params :310-324, update_accel_params
// :340-390, solve :422-652, relax :393-408, aa_apply :822-854, aa_safeguard
// :856-901, aa_reset :934-964, aa_get_stats :966-979.
//
// The reference factors the tall augmented matrix [A; sqrt(r) I] ((dim+mem) x mem,
// dim = n+m+1 up to millions) with LAPACK geqp3 and applies Q' to [g;0] and to
// [Y; sqrt(r) I] with ormqr.  Here the dim-sized part is reduced ONCE on the GPU by
// a Householder TSQR of the panel [A | Y | g] (dim x (2 len + 1)): every CTA
// streams 128-row tiles through shared memory and keeps a running len x NC
// triangle; a second single-CTA pass combines the per-CTA triangles in index
// order (bit-reproducible).  What is left -- the (2 len) x (2 len + 1) stack
// [[R0 | Q0'Y | Q0'g]; [sqrt(r) I | sqrt(r) I | 0]] -- is finished on the host with
// the same algorithm as the reference (column-pivoted Householder QR, rank
// truncation at len*eps*|R11|, LU solve + iterative refinement for type-I,
// triangular solve + refinement for type-II).  In exact arithmetic the result is
// identical to geqp3/ormqr on the full matrix.  f -= D gamma is a fused GEMV.
#include "../common.cuh"
#include "../admm_api.h"
#include <float.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define AA_MAX_MEM 31
#define AA_TILE_ROWS 128
#define AA_THREADS 256
#define AA_EPS DBL_EPSILON

struct B200Aa {
  int type1, mem, min_len, dim, iter, verbosity, success, ir_max_steps;
  double relaxation, regularization, safeguard_factor, max_weight_norm;
  double *d_x, *d_f, *d_g, *d_g_prev, *d_Y, *d_S, *d_D, *d_work;
  double norm_g;
  double nrm_s_col[AA_MAX_MEM + 1], nrm_y_col[AA_MAX_MEM + 1];
  // TSQR
  int grid;
  double *d_cta_R;    // grid * len * NC
  double *d_final_R;  // len * NC
  double *h_final_R;  // pinned
  double *d_sc3, *h_sc3;  // 3 reductions
  double *d_part;
  unsigned int *d_cnt;
  // stats
  int n_accept, n_reject_lapack, n_reject_rank0, n_reject_nonfinite, n_reject_weight_cap,
      n_safeguard_reject, last_rank;
  double last_aa_norm, last_regularization;
};

struct GammaArg { double g[AA_MAX_MEM + 1]; };

#define GSL(i, n)                                                                    \
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n);     \
       i += (long long)gridDim.x * blockDim.x)

// ------------------------------------------------------------------ vector kernels
__global__ void k_aa_seed(long long dim, const double *__restrict__ x, const double *__restrict__ f,
                          double *__restrict__ ax, double *__restrict__ af,
                          double *__restrict__ g_prev) {
  GSL(i, dim) {
    const double xi = x[i], fi = f[i];
    ax[i] = xi;
    af[i] = fi;
    g_prev[i] = xi - fi;
  }
}
__global__ void __launch_bounds__(B200_RED_THREADS)
k_aa_update(long long dim, const double *__restrict__ x, const double *__restrict__ f,
            double *__restrict__ ax, double *__restrict__ af, double *__restrict__ g,
            double *__restrict__ g_prev, double *__restrict__ s_col, double *__restrict__ d_col,
            double *__restrict__ y_col, double *out3, double *partials, unsigned int *counter) {
  __shared__ double s_red[3 * 32];
  double a[3] = {0, 0, 0};
  GSL(i, dim) {
    const double xi = x[i], fi = f[i];
    const double s = xi - ax[i];
    const double d = fi - af[i];
    const double gi = xi - fi;
    const double y = gi - g_prev[i];
    s_col[i] = s;
    d_col[i] = d;
    y_col[i] = y;
    g[i] = gi;
    ax[i] = xi;
    af[i] = fi;
    g_prev[i] = gi;
    a[0] = fma(s, s, a[0]);
    a[1] = fma(y, y, a[1]);
    a[2] = fma(gi, gi, a[2]);
  }
  block_sum<3>(a, s_red);
  if (grid_finish<3>(a, partials, counter, 0u, s_red))
    if (threadIdx.x == 0) { out3[0] = a[0]; out3[1] = a[1]; out3[2] = a[2]; }
}
// f -= D gamma ; optional relaxation: f = beta f + (1-beta) (x_prev_input - S gamma)
__global__ void k_aa_combine(long long dim, int len, GammaArg ga, const double *__restrict__ Dm,
                             const double *__restrict__ Sm, const double *__restrict__ xw,
                             double relaxation, double *__restrict__ f) {
  GSL(i, dim) {
    double acc = f[i];
    for (int c = 0; c < len; ++c) acc = fma(-ga.g[c], Dm[(size_t)c * dim + i], acc);
    if (relaxation != 1.0) {
      double xa = xw[i];
      for (int c = 0; c < len; ++c) xa = fma(-ga.g[c], Sm[(size_t)c * dim + i], xa);
      acc = relaxation * acc + (1.0 - relaxation) * xa;
    }
    f[i] = acc;
  }
}
__global__ void __launch_bounds__(B200_RED_THREADS)
k_aa_diffnorm(long long dim, const double *__restrict__ a, const double *__restrict__ b,
              double *out, double *partials, unsigned int *counter) {
  __shared__ double s_red[32];
  double acc[1] = {0.0};
  GSL(i, dim) {
    const double d = a[i] - b[i];
    acc[0] = fma(d, d, acc[0]);
  }
  block_sum<1>(acc, s_red);
  if (grid_finish<1>(acc, partials, counter, 0u, s_red))
    if (threadIdx.x == 0) out[0] = acc[0];
}

// ------------------------------------------------------------------ TSQR
// Shared panel P (ld = len + AA_TILE_ROWS), column-major, NC columns. Rows [0,len) hold the
// running triangle [R | Z]; rows [len, ld) the fresh tile. Eliminates the tile rows
// below the triangle with `len` Householder reflectors whose support is {j} U tile rows.
// The elimination is BLOCKED (compact WY, blocks of 4 reflectors) so that the trailing update is two small
// GEMMs on the fp64 tensor-core path (mma.sync.aligned.m8n8k4.f64, SASS DMMA) -- north_star "small tensor-core QR".
// Reflector j of this TSQR step has support {row j of the triangle} U {tile rows}: the top parts of the block's
// reflectors are distinct unit vectors, so with V = the 128 x nb matrix of their (normalised) tile parts
//   T (larft, forward):  T_kk = tau_k,  T_{0:k,k} = -tau_k T_{0:k,0:k} (V_{:,0:k}' v_k)
//   W = C_top + V' C_tile   [DMMA: M = nb (padded to 8), N = trailing columns, K = 128 tile rows]
//   W = T' W
//   C_top -= W ;  C_tile -= V W   [DMMA: M = 128 tile rows, N = trailing columns, K = 4 = the m8n8k4 depth]
// Inside a block the reflectors are still generated and applied one at a time (to the <= 3 later columns of the
// block). Checked against a reflector-at-a-time elimination in numpy (1e-16) and by the AA parity tests. Tile rows
// beyond `rows` are zero-filled by the callers, so the block always works on all AA_TILE_ROWS rows.
#define AA_BLK 4
// W = V'C_tile is staged as AA_BLK rows of stride AA_WPAD, one column per trailing column of the panel. The trailing
// block is widest right after the first reflector block: NC - 1 <= 2 AA_MAX_MEM columns, which C1 covers with one warp
// per 8 columns. The stride is that width rounded up to 8 plus 8 doubles: 8 (mod 16) doubles, so the 4 rows x 8
// columns C2 reads per mma fall on alternate halves of the banks.
#define AA_NCT_MAX (2 * AA_MAX_MEM)
#define AA_WPAD (8 * ((AA_NCT_MAX + 7) / 8) + 8)
static_assert(8 * ((AA_NCT_MAX + 7) / 8) <= AA_WPAD, "W staging narrower than the widest trailing block");
static_assert((AA_NCT_MAX + 7) / 8 <= AA_THREADS / 32, "C1 needs one warp per 8 trailing columns");
static_assert(AA_WPAD % 16 == 8, "W row stride: rows on alternate bank halves");
__device__ void tsqr_eliminate_blocked(double *P, int ld, int len, int NC, double *s_tmp, double *Vt /*[4][128]*/,
                                       double *Tm /*[16]*/, double *Wm /*[4][AA_WPAD]*/) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  for (int jb = 0; jb < len; jb += AA_BLK) {
    const int nb = (len - jb) < AA_BLK ? (len - jb) : AA_BLK;
    // ---- A: reflectors of the block, applied to the later columns of the block only
    for (int k = 0; k < nb; ++k) {
      const int j = jb + k;
      double *cj = P + (size_t)j * ld;
      if (wid == 0) {
        double sg = 0.0;
        for (int i = lane; i < AA_TILE_ROWS; i += 32) {
          const double v = cj[len + i];
          sg = fma(v, v, sg);
        }
        sg = warp_sum(sg);
        if (lane == 0) {
          const double alpha = cj[j];
          double tau = 0.0, scale = 0.0, beta = alpha;
          if (sg != 0.0) {
            const double nrm = sqrt(fma(alpha, alpha, sg));
            beta = (alpha >= 0.0) ? -nrm : nrm;
            tau = (beta - alpha) / beta;
            scale = 1.0 / (alpha - beta);
          }
          s_tmp[0] = tau;
          s_tmp[1] = scale;
          s_tmp[2] = beta;
          Tm[k * AA_BLK + k] = tau;
        }
      }
      __syncthreads();
      const double tau = s_tmp[0], scale = s_tmp[1];
      for (int i = tid; i < AA_TILE_ROWS; i += blockDim.x) Vt[k * AA_TILE_ROWS + i] = cj[len + i] * scale;
      __syncthreads();
      if (tau != 0.0) {
        for (int c = j + 1 + wid; c < jb + nb; c += nw) {
          double *cc = P + (size_t)c * ld;
          double w = 0.0;
          for (int i = lane; i < AA_TILE_ROWS; i += 32) w = fma(Vt[k * AA_TILE_ROWS + i], cc[len + i], w);
          w = warp_sum(w);
          w = tau * (cc[j] + w);
          for (int i = lane; i < AA_TILE_ROWS; i += 32) cc[len + i] = fma(-w, Vt[k * AA_TILE_ROWS + i], cc[len + i]);
          if (lane == 0) cc[j] -= w;
        }
      }
      __syncthreads();
      if (tid == 0 && tau != 0.0) cj[j] = s_tmp[2];
      __syncthreads();
    }
    const int c0 = jb + nb, nct = NC - c0;
    if (nct <= 0) continue;  // uniform
    // ---- B: T (warp 0)
    if (wid == 0) {
      for (int k = 1; k < nb; ++k) {
        double z[AA_BLK - 1];
        for (int i = 0; i < k; ++i) {
          double acc = 0.0;
          for (int r = lane; r < AA_TILE_ROWS; r += 32) acc = fma(Vt[i * AA_TILE_ROWS + r], Vt[k * AA_TILE_ROWS + r], acc);
          z[i] = warp_sum(acc);
        }
        if (lane == 0) {
          const double tk = Tm[k * AA_BLK + k];
          for (int i = 0; i < k; ++i) {
            double acc = 0.0;
            for (int q = i; q < k; ++q) acc = fma(Tm[i * AA_BLK + q], z[q], acc);  // T upper triangular
            Tm[i * AA_BLK + k] = -tk * acc;
          }
        }
        __syncwarp();
      }
    }
    // ---- C1: W = V' C_tile on the tensor pipe, one warp per 8 trailing columns
    const int ntl = (nct + 7) / 8;
    if (wid < ntl) {
      double a0 = 0.0, a1 = 0.0;
      const int col = c0 + 8 * wid + g;
      const double *bc = P + (size_t)(col < NC ? col : 0) * ld + len;
      for (int k0 = 0; k0 < AA_TILE_ROWS; k0 += 4) {
        const double a = (g < nb) ? Vt[g * AA_TILE_ROWS + k0 + t] : 0.0;
        const double b = (col < NC) ? bc[k0 + t] : 0.0;
        dmma_m8n8k4(a0, a1, a, b);
      }
      if (g < nb) {
        Wm[g * AA_WPAD + 8 * wid + 2 * t] = a0;
        Wm[g * AA_WPAD + 8 * wid + 2 * t + 1] = a1;
      }
    }
    __syncthreads();
    // ---- W = T'(C_top + W); C_top -= W; keep -W (zero-padded) for the second GEMM
    if (tid < 8 * ntl) {
      const int c = c0 + tid;
      double w[AA_BLK], o[AA_BLK];
      for (int k = 0; k < AA_BLK; ++k) w[k] = (k < nb && c < NC) ? P[(size_t)c * ld + jb + k] + Wm[k * AA_WPAD + tid] : 0.0;
      for (int k = 0; k < AA_BLK; ++k) {
        double acc = 0.0;
        for (int i = 0; i <= k; ++i) acc = fma((i < nb && k < nb) ? Tm[i * AA_BLK + k] : 0.0, w[i], acc);
        o[k] = acc;
      }
      for (int k = 0; k < AA_BLK; ++k) {
        if (k < nb && c < NC) P[(size_t)c * ld + jb + k] -= o[k];
        Wm[k * AA_WPAD + tid] = (k < nb && c < NC) ? -o[k] : 0.0;
      }
    }
    __syncthreads();
    // ---- C2: C_tile += V (-W) on the tensor pipe: 16 row tiles x ntl column tiles, K = 4 in one mma each
    for (int id = wid; id < (AA_TILE_ROWS / 8) * ntl; id += nw) {
      const int mt = id % (AA_TILE_ROWS / 8), nt = id / (AA_TILE_ROWS / 8);
      const double a = (t < nb) ? Vt[t * AA_TILE_ROWS + 8 * mt + g] : 0.0;
      const double b = Wm[t * AA_WPAD + 8 * nt + g];
      const int ca = c0 + 8 * nt + 2 * t, cb = ca + 1;
      double *pa = P + (size_t)(ca < NC ? ca : 0) * ld + len + 8 * mt + g;
      double *pb = P + (size_t)(cb < NC ? cb : 0) * ld + len + 8 * mt + g;
      double x0 = (ca < NC) ? *pa : 0.0, x1 = (cb < NC) ? *pb : 0.0;
      dmma_m8n8k4(x0, x1, a, b);
      if (ca < NC) *pa = x0;
      if (cb < NC) *pb = x1;
    }
    __syncthreads();
  }
}

// src columns: column c < len -> A_src[:,c]; len <= c < 2 len -> Y[:, c-len] (type-I only); last -> g
__device__ __forceinline__ const double *aa_col(int c, int len, int type1, const double *A_src,
                                                const double *Y, const double *g, long long dim) {
  if (c < len) return A_src + (size_t)c * dim;
  if (type1 && c < 2 * len) return Y + (size_t)(c - len) * dim;
  return g;
}

__global__ void __launch_bounds__(AA_THREADS)
k_aa_tsqr_local(long long dim, int len, int type1, const double *__restrict__ A_src,
                const double *__restrict__ Y, const double *__restrict__ g,
                double *__restrict__ cta_R) {
  extern __shared__ double P[];
  __shared__ double s_tmp[4];
  __shared__ double s_Vt[AA_BLK * AA_TILE_ROWS], s_Tm[AA_BLK * AA_BLK], s_Wm[AA_BLK * AA_WPAD];
  const int NC = (type1 ? 2 * len : len) + 1;
  const int ld = len + AA_TILE_ROWS;
  for (int e = threadIdx.x; e < ld * NC; e += blockDim.x) P[e] = 0.0;
  __syncthreads();
  const long long ntiles = (dim + AA_TILE_ROWS - 1) / AA_TILE_ROWS;
  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const long long r0 = t * AA_TILE_ROWS;
    const int rows = (int)((dim - r0) < AA_TILE_ROWS ? (dim - r0) : AA_TILE_ROWS);
    for (int e = threadIdx.x; e < AA_TILE_ROWS * NC; e += blockDim.x) {
      const int i = e % AA_TILE_ROWS, c = e / AA_TILE_ROWS;
      const double *col = aa_col(c, len, type1, A_src, Y, g, dim);
      P[(size_t)c * ld + len + i] = (i < rows) ? col[r0 + i] : 0.0;
    }
    __syncthreads();
    tsqr_eliminate_blocked(P, ld, len, NC, s_tmp, s_Vt, s_Tm, s_Wm);
  }
  for (int e = threadIdx.x; e < len * NC; e += blockDim.x) {
    const int i = e % len, c = e / len;
    cta_R[(size_t)blockIdx.x * len * NC + e] = P[(size_t)c * ld + i];
  }
}
// single CTA: combine `nblk` triangles (each len x NC, column-major, ld = len)
__global__ void __launch_bounds__(AA_THREADS)
k_aa_tsqr_combine(int nblk, int len, int NC, const double *__restrict__ cta_R,
                  double *__restrict__ out) {
  extern __shared__ double P[];
  __shared__ double s_tmp[4];
  __shared__ double s_Vt[AA_BLK * AA_TILE_ROWS], s_Tm[AA_BLK * AA_BLK], s_Wm[AA_BLK * AA_WPAD];
  const int ld = len + AA_TILE_ROWS;
  for (int e = threadIdx.x; e < ld * NC; e += blockDim.x) P[e] = 0.0;
  __syncthreads();
  const int per = AA_TILE_ROWS / len;  // triangles stacked per pass
  for (int b0 = 0; b0 < nblk; b0 += per) {
    const int nb = (nblk - b0) < per ? (nblk - b0) : per;
    const int rows = nb * len;
    for (int e = threadIdx.x; e < AA_TILE_ROWS * NC; e += blockDim.x) {
      const int i = e % AA_TILE_ROWS, c = e / AA_TILE_ROWS;
      double v = 0.0;
      if (i < rows) {
        const int b = b0 + i / len, ii = i % len;
        v = cta_R[(size_t)b * len * NC + (size_t)c * len + ii];
      }
      P[(size_t)c * ld + len + i] = v;
    }
    __syncthreads();
    tsqr_eliminate_blocked(P, ld, len, NC, s_tmp, s_Vt, s_Tm, s_Wm);
  }
  for (int e = threadIdx.x; e < len * NC; e += blockDim.x) {
    const int i = e % len, c = e / len;
    out[e] = P[(size_t)c * ld + i];
  }
}

// ------------------------------------------------------------------ host: small dense algebra
// Column-pivoted Householder QR of the first `len` columns of H (rows x ncols, column-major,
// ld = rows), reflectors applied to ALL columns. jpvt (0-based) records the pivot order of
// the first len columns; the remaining columns are not permuted. Mirrors geqp3 + ormqr.
static void host_pivoted_qr(double *H, int rows, int ncols, int len, int *jpvt) {
  for (int j = 0; j < len; ++j) jpvt[j] = j;
  for (int j = 0; j < len && j < rows; ++j) {
    // pivot: remaining column with the largest norm over rows j..rows-1 (first on ties)
    int best = j;
    double bestn = -1.0;
    for (int c = j; c < len; ++c) {
      double s = 0.0;
      for (int i = j; i < rows; ++i) s += H[(size_t)c * rows + i] * H[(size_t)c * rows + i];
      if (s > bestn) { bestn = s; best = c; }
    }
    if (best != j) {
      for (int i = 0; i < rows; ++i) {
        double t = H[(size_t)j * rows + i];
        H[(size_t)j * rows + i] = H[(size_t)best * rows + i];
        H[(size_t)best * rows + i] = t;
      }
      int t = jpvt[j]; jpvt[j] = jpvt[best]; jpvt[best] = t;
    }
    double *cj = H + (size_t)j * rows;
    double sg = 0.0;
    for (int i = j + 1; i < rows; ++i) sg += cj[i] * cj[i];
    if (sg == 0.0) continue;
    const double alpha = cj[j];
    const double nrm = sqrt(alpha * alpha + sg);
    const double beta = alpha >= 0.0 ? -nrm : nrm;
    const double tau = (beta - alpha) / beta;
    const double scale = 1.0 / (alpha - beta);
    for (int i = j + 1; i < rows; ++i) cj[i] *= scale;  // v (v_j = 1 implicit)
    for (int c = j + 1; c < ncols; ++c) {
      double *cc = H + (size_t)c * rows;
      double w = cc[j];
      for (int i = j + 1; i < rows; ++i) w += cj[i] * cc[i];
      w *= tau;
      cc[j] -= w;
      for (int i = j + 1; i < rows; ++i) cc[i] -= w * cj[i];
    }
    cj[j] = beta;
    for (int i = j + 1; i < rows; ++i) cj[i] = 0.0;
  }
}
// LU with partial pivoting, in place (n x n, ld); returns 0 or k+1 if singular
static int host_getrf(double *A, int n, int ld, int *ipiv) {
  for (int k = 0; k < n; ++k) {
    int p = k;
    double mx = fabs(A[(size_t)k * ld + k]);
    for (int i = k + 1; i < n; ++i)
      if (fabs(A[(size_t)k * ld + i]) > mx) { mx = fabs(A[(size_t)k * ld + i]); p = i; }
    ipiv[k] = p;
    if (mx == 0.0) return k + 1;
    if (p != k)
      for (int c = 0; c < n; ++c) {
        double t = A[(size_t)c * ld + k];
        A[(size_t)c * ld + k] = A[(size_t)c * ld + p];
        A[(size_t)c * ld + p] = t;
      }
    const double piv = A[(size_t)k * ld + k];
    for (int i = k + 1; i < n; ++i) A[(size_t)k * ld + i] /= piv;
    for (int c = k + 1; c < n; ++c) {
      const double akc = A[(size_t)c * ld + k];
      for (int i = k + 1; i < n; ++i) A[(size_t)c * ld + i] -= A[(size_t)k * ld + i] * akc;
    }
  }
  return 0;
}
static void host_getrs(const double *LU, int n, int ld, const int *ipiv, double *b) {
  for (int k = 0; k < n; ++k) {
    if (ipiv[k] != k) { double t = b[k]; b[k] = b[ipiv[k]]; b[ipiv[k]] = t; }
    for (int i = k + 1; i < n; ++i) b[i] -= LU[(size_t)k * ld + i] * b[k];
  }
  for (int k = n - 1; k >= 0; --k) {
    b[k] /= LU[(size_t)k * ld + k];
    for (int i = 0; i < k; ++i) b[i] -= LU[(size_t)k * ld + i] * b[k];
  }
}
static double frob_from_col_norms(const double *nrm, int mem) {
  double m = 0;
  for (int i = 0; i < mem; ++i) if (nrm[i] > m) m = nrm[i];
  if (m == 0) return 0;
  double ss = 0;
  for (int i = 0; i < mem; ++i) { double t = nrm[i] / m; ss += t * t; }
  return m * sqrt(ss);
}
static double nrm2_small(const double *v, int n) {
  double s = 0;
  for (int i = 0; i < n; ++i) s += v[i] * v[i];
  return sqrt(s);
}

// ------------------------------------------------------------------ API
#define ST ((cudaStream_t)b200_stream())
static int vgrid(long long n) {
  long long g = (n + 2047) / 2048, cap = 4LL * b200_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" B200Aa *b200_aa_create(int dim, int mem, int min_len, int type1, double regularization,
                                  double relaxation, double safeguard_factor,
                                  double max_weight_norm, int ir_max_steps, int verbosity) {
  int mem_c = mem < dim ? mem : dim;
  if (dim <= 0 || mem < 0 || !isfinite(regularization) || relaxation < 0 || relaxation > 2 ||
      safeguard_factor < 0 || max_weight_norm <= 0 || ir_max_steps < 0 ||
      (mem_c > 0 && min_len < 1)) {
    fprintf(stderr, "Invalid AA parameters.\n");
    return nullptr;
  }
  if (mem_c > AA_MAX_MEM) {
    fprintf(stderr, "scs_b200: AA memory %d exceeds the device limit %d\n", mem_c, AA_MAX_MEM);
    return nullptr;
  }
  if (b200_runtime_init() != 0) return nullptr;
  B200Aa *a = (B200Aa *)calloc(1, sizeof(B200Aa));
  if (!a) return nullptr;
  a->type1 = type1; a->dim = dim; a->mem = mem_c;
  a->min_len = mem_c > 0 ? (min_len < mem_c ? min_len : mem_c) : 0;
  a->regularization = regularization; a->relaxation = relaxation;
  a->safeguard_factor = safeguard_factor; a->max_weight_norm = max_weight_norm;
  a->ir_max_steps = ir_max_steps; a->verbosity = verbosity;
  a->last_aa_norm = NAN;
  if (a->mem <= 0) return a;
  const size_t d8 = (size_t)dim * 8;
  a->d_x = (double *)b200_malloc(d8);
  a->d_f = (double *)b200_malloc(d8);
  a->d_g = (double *)b200_malloc(d8);
  a->d_g_prev = (double *)b200_malloc(d8);
  a->d_work = (double *)b200_malloc(d8);
  a->d_Y = (double *)b200_malloc(d8 * a->mem);
  a->d_S = (double *)b200_malloc(d8 * a->mem);
  a->d_D = (double *)b200_malloc(d8 * a->mem);
  const int NCmax = 2 * a->mem + 1;
  long long ntiles = ((long long)dim + AA_TILE_ROWS - 1) / AA_TILE_ROWS;
  a->grid = 2 * b200_num_sms();
  if (a->grid > ntiles) a->grid = (int)ntiles;
  if (a->grid < 1) a->grid = 1;
  a->d_cta_R = (double *)b200_malloc((size_t)a->grid * a->mem * NCmax * 8);
  a->d_final_R = (double *)b200_malloc((size_t)a->mem * NCmax * 8);
  a->h_final_R = (double *)b200_host_alloc((size_t)a->mem * NCmax * 8);
  a->d_sc3 = (double *)b200_malloc(64);
  a->h_sc3 = (double *)b200_host_alloc(64);
  a->d_part = (double *)b200_malloc(4 * 2048 * 8);
  a->d_cnt = (unsigned int *)b200_malloc(64);
  if (!a->d_x || !a->d_f || !a->d_g || !a->d_g_prev || !a->d_work || !a->d_Y || !a->d_S ||
      !a->d_D || !a->d_cta_R || !a->d_final_R || !a->h_final_R || !a->d_sc3 || !a->h_sc3 ||
      !a->d_part || !a->d_cnt) {
    fprintf(stderr, "Failed to allocate memory for AA.\n");
    b200_aa_destroy(a);
    return nullptr;
  }
  b200_memset0(a->d_cnt, 64);
  const int smem = (a->mem + AA_TILE_ROWS) * NCmax * 8;
  cudaFuncSetAttribute(k_aa_tsqr_local, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaFuncSetAttribute(k_aa_tsqr_combine, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  b200_sync();
  return a;
}

extern "C" void b200_aa_destroy(B200Aa *a) {
  if (!a) return;
  b200_sync();
  b200_free(a->d_x); b200_free(a->d_f); b200_free(a->d_g); b200_free(a->d_g_prev);
  b200_free(a->d_work); b200_free(a->d_Y); b200_free(a->d_S); b200_free(a->d_D);
  b200_free(a->d_cta_R); b200_free(a->d_final_R); b200_host_free(a->h_final_R);
  b200_free(a->d_sc3); b200_host_free(a->h_sc3); b200_free(a->d_part); b200_free(a->d_cnt);
  free(a);
}

extern "C" void b200_aa_reset_dev(B200Aa *a) {
  if (!a) return;
  if (a->verbosity > 0) printf("AA reset.\n");
  a->iter = 0;
  a->success = 0;
  a->norm_g = 0;
  memset(a->nrm_s_col, 0, sizeof(a->nrm_s_col));
  memset(a->nrm_y_col, 0, sizeof(a->nrm_y_col));
}

// the state of b200_aa_create: b200_aa_reset_dev and the statistics (ScsInfo.aa_stats) back to zero
extern "C" void b200_aa_restart_dev(B200Aa *a) {
  if (!a) return;
  b200_aa_reset_dev(a);
  a->n_accept = a->n_reject_lapack = a->n_reject_rank0 = a->n_reject_nonfinite = a->n_reject_weight_cap = 0;
  a->n_safeguard_reject = a->last_rank = 0;
  a->last_aa_norm = NAN;
  a->last_regularization = 0;
}

// reference solve(), aa.c:422-652
static double aa_solve(B200Aa *a, double *d_f, int len) {
  const int dim = a->dim;
  const int type1 = a->type1;
  const int NC = (type1 ? 2 * len : len) + 1;
  double r;
  if (a->regularization > 0) {
    const double nrm_y = frob_from_col_norms(a->nrm_y_col, a->mem);
    const double nrm_a = type1 ? frob_from_col_norms(a->nrm_s_col, a->mem) : nrm_y;
    r = a->regularization * nrm_a * nrm_y;
  } else if (a->regularization < 0) {
    r = -a->regularization;
  } else {
    r = 0.0;
  }
  const double sqrt_r = r > 0 ? sqrt(r) : 0.0;
  int info = 0, rank = 0;

  // 1. device TSQR of [A | Y | g]
  const double *A_src = type1 ? a->d_S : a->d_Y;
  const size_t smem = (size_t)(len + AA_TILE_ROWS) * NC * 8;
  k_aa_tsqr_local<<<a->grid, AA_THREADS, smem, ST>>>((long long)dim, len, type1, A_src, a->d_Y,
                                                      a->d_g, a->d_cta_R);
  k_aa_tsqr_combine<<<1, AA_THREADS, smem, ST>>>(a->grid, len, NC, a->d_cta_R, a->d_final_R);
  b200_count_launch(2);
  if (cudaGetLastError() != cudaSuccess) info = -1;
  if (info == 0 && (b200_d2h(a->h_final_R, a->d_final_R, (size_t)len * NC * 8) != 0 || b200_sync() != 0))
    info = -1;
  const int lapack_info = info;

  std::vector<double> H, W, W_orig, gamma_red(len), c_top(len), ir_res(len), gamma(len, 0.0);
  std::vector<int> jpvt(len), ipiv(len);
  const int rows = 2 * len;
  if (info == 0) {
    // 2. stack the regularisation rows and finish with the pivoted QR
    H.assign((size_t)rows * NC, 0.0);
    for (int c = 0; c < NC; ++c)
      for (int i = 0; i < len; ++i) H[(size_t)c * rows + i] = a->h_final_R[(size_t)c * len + i];
    for (int c = 0; c < len; ++c) {
      H[(size_t)c * rows + len + c] = sqrt_r;                     // [A; sqrt(r) I]
      if (type1) H[(size_t)(len + c) * rows + len + c] = sqrt_r;  // [Y; sqrt(r) I]
    }
    for (size_t e = 0; e < H.size(); ++e)
      if (!isfinite(H[e])) { info = 2; break; }
  }
  if (info == 0) {
    host_pivoted_qr(H.data(), rows, NC, len, jpvt.data());
    const double r11 = fabs(H[0]);
    if (r11 > 0) {
      const double tol = r11 * (double)len * AA_EPS;
      for (rank = 0; rank < len; ++rank)
        if (fabs(H[(size_t)rank * rows + rank]) < tol) break;
    }
    if (rank == 0) info = 1;
  }
  if (info == 0) {
    for (int i = 0; i < rank; ++i) c_top[i] = H[(size_t)(NC - 1) * rows + i];
    if (type1) {
      W.assign((size_t)len * len, 0.0);
      for (int i = 0; i < rank; ++i)    // column i of the permuted B = Y column jpvt[i]
        for (int k = 0; k < rank; ++k) W[(size_t)i * len + k] = H[(size_t)(len + jpvt[i]) * rows + k];
      W_orig = W;
      for (int i = 0; i < rank; ++i) gamma_red[i] = c_top[i];
      info = host_getrf(W.data(), rank, len, ipiv.data());
      if (info == 0) {
        host_getrs(W.data(), rank, len, ipiv.data(), gamma_red.data());
        double prev = 0.0;
        for (int k = 0; k < a->ir_max_steps; ++k) {
          for (int i = 0; i < rank; ++i) {
            double s = c_top[i];
            for (int c = 0; c < rank; ++c) s -= W_orig[(size_t)c * len + i] * gamma_red[c];
            ir_res[i] = s;
          }
          host_getrs(W.data(), rank, len, ipiv.data(), ir_res.data());
          const double dn = nrm2_small(ir_res.data(), rank);
          for (int i = 0; i < rank; ++i) gamma_red[i] += ir_res[i];
          if (k > 0 && dn >= 0.5 * prev) break;
          prev = dn;
        }
      }
    } else {
      auto trsv = [&](double *b) {
        for (int k = rank - 1; k >= 0; --k) {
          b[k] /= H[(size_t)k * rows + k];
          for (int i = 0; i < k; ++i) b[i] -= H[(size_t)k * rows + i] * b[k];
        }
      };
      for (int i = 0; i < rank; ++i) gamma_red[i] = c_top[i];
      trsv(gamma_red.data());
      double prev = 0.0;
      for (int k = 0; k < a->ir_max_steps; ++k) {
        for (int i = 0; i < rank; ++i) {
          double s = 0.0;
          for (int c = i; c < rank; ++c) s += H[(size_t)c * rows + i] * gamma_red[c];
          ir_res[i] = c_top[i] - s;
        }
        trsv(ir_res.data());
        const double dn = nrm2_small(ir_res.data(), rank);
        for (int i = 0; i < rank; ++i) gamma_red[i] += ir_res[i];
        if (k > 0 && dn >= 0.5 * prev) break;
        prev = dn;
      }
    }
    if (info == 0)
      for (int i = 0; i < rank; ++i) gamma[jpvt[i]] = gamma_red[i];
  }
  double aa_norm = (info == 0) ? nrm2_small(gamma.data(), len) : -1.0;
  a->last_rank = rank;
  a->last_regularization = r;
  a->last_aa_norm = (info == 0 && isfinite(aa_norm)) ? aa_norm : NAN;
  if (a->verbosity > 1)
    printf("AA type %i, iter: %i, len %i, rank %i, info: %i, aa_norm %.2e\n", type1 ? 1 : 2, a->iter,
           len, rank, info, aa_norm);
  if (info != 0 || !isfinite(aa_norm) || aa_norm >= a->max_weight_norm) {
    if (lapack_info != 0) a->n_reject_lapack++;
    else if (rank == 0) a->n_reject_rank0++;
    else if (!isfinite(aa_norm)) a->n_reject_nonfinite++;
    else a->n_reject_weight_cap++;
    a->success = 0;
    b200_aa_reset_dev(a);
    if (!isfinite(aa_norm)) aa_norm = -1.0;
    return aa_norm < 0 ? aa_norm : -aa_norm;
  }
  GammaArg ga;
  memset(&ga, 0, sizeof(ga));
  for (int i = 0; i < len; ++i) ga.g[i] = gamma[i];
  // x_work (= x of this call) is a->d_x after the state advance
  k_aa_combine<<<vgrid(dim), 256, 0, ST>>>((long long)dim, len, ga, a->d_D, a->d_S, a->d_x,
                                           a->relaxation, d_f);
  b200_count_launch(1);
  a->success = 1;
  return aa_norm;
}

extern "C" double b200_aa_apply_dev(B200Aa *a, double *d_f, const double *d_x) {
  double aa_norm = 0;
  const int len = a->iter < a->mem ? a->iter : a->mem;
  a->success = 0;
  if (a->mem <= 0) return 0;
  const long long dim = a->dim;
  if (a->iter == 0) {
    k_aa_seed<<<vgrid(dim), 256, 0, ST>>>(dim, d_x, d_f, a->d_x, a->d_f, a->d_g_prev);
    b200_count_launch(1);
    a->iter++;
    return 0;
  }
  const int idx = (a->iter - 1) % a->mem;
  k_aa_update<<<vgrid(dim), B200_RED_THREADS, 0, ST>>>(
      dim, d_x, d_f, a->d_x, a->d_f, a->d_g, a->d_g_prev, a->d_S + (size_t)idx * dim,
      a->d_D + (size_t)idx * dim, a->d_Y + (size_t)idx * dim, a->d_sc3, a->d_part, a->d_cnt);
  b200_count_launch(1);
  if (b200_d2h(a->h_sc3, a->d_sc3, 24) != 0 || b200_sync() != 0) return -1.0;
  a->nrm_s_col[idx] = sqrt(a->h_sc3[0]);
  a->nrm_y_col[idx] = sqrt(a->h_sc3[1]);
  a->norm_g = sqrt(a->h_sc3[2]);
  if (a->iter >= a->min_len) {
    aa_norm = aa_solve(a, d_f, len);
    if (aa_norm > 0) a->n_accept++;
  }
  a->iter++;
  return aa_norm;
}

extern "C" int b200_aa_safeguard_dev(B200Aa *a, double *d_f_new, double *d_x_new) {
  if (a->mem <= 0) return 0;
  if (!a->success) return 0;
  a->success = 0;
  const long long dim = a->dim;
  k_aa_diffnorm<<<vgrid(dim), B200_RED_THREADS, 0, ST>>>(dim, d_x_new, d_f_new, a->d_sc3, a->d_part,
                                                         a->d_cnt);
  b200_count_launch(1);
  if (b200_d2h(a->h_sc3, a->d_sc3, 8) != 0 || b200_sync() != 0) return 0;
  const double norm_diff = sqrt(a->h_sc3[0]);
  if (norm_diff > a->safeguard_factor * a->norm_g) {
    b200_d2d(d_f_new, a->d_f, (size_t)dim * 8);
    b200_d2d(d_x_new, a->d_x, (size_t)dim * 8);
    if (a->verbosity > 0)
      printf("AA rejection, iter: %i, norm_diff %.4e, prev_norm_diff %.4e\n", a->iter, norm_diff,
             a->norm_g);
    a->n_safeguard_reject++;
    b200_aa_reset_dev(a);
    return -1;
  }
  return 0;
}

extern "C" void b200_aa_stats(const B200Aa *a, int *o, double *d) {
  o[0] = a->iter; o[1] = a->n_accept; o[2] = a->n_reject_lapack; o[3] = a->n_reject_rank0;
  o[4] = a->n_reject_nonfinite; o[5] = a->n_reject_weight_cap; o[6] = a->n_safeguard_reject;
  o[7] = a->last_rank;
  d[0] = a->last_aa_norm; d[1] = a->last_regularization;
}

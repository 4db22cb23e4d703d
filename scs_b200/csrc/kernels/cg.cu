// cg.cu -- device-resident Jacobi-preconditioned conjugate gradient for the SCS
// reduced KKT system  (R_x + P + A' R_y^{-1} A) x = r_x + A' R_y^{-1} r_y,
// y = R_y^{-1}(A x - r_y).
//
// Replaces reference linsys/cpu/indirect/private.c:50-82 (set_preconditioner),
// :106-119 (mat_vec), :133-217 (pcg), :284-324 (scs_solve_lin_sys) and the
// cuBLAS/cuSPARSE composition of linsys/gpu/indirect/private.c:364-527.
//
// The scalars alpha, beta, z'r, ||r||_inf and the stop decision never leave the
// GPU: a control block (B200CgCtl) lives in device memory, the last block of
// each reduction-carrying kernel updates it, and every kernel of the loop
// returns at once when ctl->done is set.  The host enqueues CG iterations in
// batches and polls `done` with one small async copy per batch.
//
// One CG iteration = 4 kernels:
//   K1  tmp = R_y^{-1} (A p)                         spmv (CSR of A), POST_DIV
//   K2  Gp  = R_x p + [P p] + A' tmp ;  p'Gp ; alpha spmv (CSR of A'), POST_FMA_DOT + hook
//   K3  x += alpha p; r -= alpha Gp; z = M r; z'r, ||r||_inf; stop test; beta
//   K4  p = z + beta p
// Algorithmic bytes: 24 nnz + 4 (m+n+2) + 24 m + 120 n   (DESIGN.md).
#include "../common.cuh"
#include "../dev_api.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define VEC_THREADS B200_RED_THREADS

static inline int vec_grid(long long n) {
  long long g = (n + (long long)VEC_THREADS * 4 - 1) / ((long long)VEC_THREADS * 4);
  long long cap = 4LL * b200_num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// ---------------------------------------------------------------------------
// M_j = 1 / (R_x,j + sum_k A_kj^2 / R_y,row(k) + P_jj), same accumulation order
// as the reference loop (private.c:61-78). One thread per column of A.
__global__ void k_set_preconditioner(int n, const int *__restrict__ colptr,
                                     const int *__restrict__ rowidx, const double *__restrict__ vals,
                                     const double *__restrict__ rx, const double *__restrict__ ry,
                                     const double *__restrict__ pdiag, double *__restrict__ M) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    double acc = rx[j];
    const int a = colptr[j], b = colptr[j + 1];
    for (int k = a; k < b; ++k) {
      const double v = vals[k];
      acc += v * v / ry[rowidx[k] & B200_COLMASK];  // top bits of stored indices are flags (spmv.cu v3)
    }
    if (pdiag != nullptr) acc += pdiag[j];
    M[j] = 1.0 / acc;
  }
}

// ---------------------------------------------------------------------------
// Prologue: bnorm = ||b||_inf over n+m, tmp = r_y ./ R_y, control block reset.
// (private.c:296-303)
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_prepare(int n, int m, const double *__restrict__ b, const double *__restrict__ ry,
             double *__restrict__ tmp, B200CgCtl *ctl, double tol, const double *d_tol, int max_its,
             double *partials, unsigned int *counter) {
  __shared__ double s_red[64];
  double mx[1] = {0.0};
  const long long tot = (long long)n + m;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < tot;
       i += (long long)gridDim.x * blockDim.x) {
    const double v = b[i];
    mx[0] = fmax(mx[0], fabs(v));
    if (i >= n) tmp[i - n] = v / ry[i - n];
  }
  block_max<1>(mx, s_red);
  if (grid_finish<1>(mx, partials, counter, 1u, s_red)) {
    if (threadIdx.x == 0) {
      const double t = (d_tol != nullptr) ? *d_tol : tol;
      ctl->bnorm = mx[0];
      ctl->tol = t;
      ctl->skip = (mx[0] <= 1e-12) ? 1 : 0;  // NaN compares false -> not skipped, like the reference
      ctl->done = ctl->skip;
      ctl->iters = 0;
      ctl->max_its = max_its;
      ctl->ztr = 0.0;
      ctl->ztr_prev = 0.0;
      ctl->alpha = 0.0;
      ctl->beta = 0.0;
      ctl->rnorm = 0.0;
    }
  }
}

// ---------------------------------------------------------------------------
// CG start (private.c:145-172). warm==0: r = b, x = 0.  warm==1: Gs is in r;
// r = -(Gs - b) ; x = s.  Then ||r||_inf test, z = M r, ztr = z'r, p = z.
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_init(int n, int warm, double *__restrict__ x /* b[0:n] */, const double *__restrict__ s,
          double *__restrict__ r, const double *__restrict__ M, double *__restrict__ z,
          double *__restrict__ p, B200CgCtl *ctl, double *partials, unsigned int *counter) {
  if (ctl->skip) return;
  __shared__ double s_red[128];
  double acc[2] = {0.0, 0.0};  // [0] = z'r (sum), [1] = ||r||_inf (max)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double ri;
    if (warm) {
      double t = r[i];
      t += -1.0 * x[i];
      ri = -t;
      x[i] = s[i];
    } else {
      ri = x[i];
      x[i] = 0.0;
    }
    r[i] = ri;
    const double zi = ri * M[i];
    z[i] = zi;
    p[i] = zi;
    acc[0] = fma(zi, ri, acc[0]);
    acc[1] = fmax(acc[1], fabs(ri));
  }
  double sm[1] = {acc[0]}, mx[1] = {acc[1]};
  block_sum<1>(sm, s_red);
  block_max<1>(mx, s_red + 64);
  double both[2] = {sm[0], mx[0]};
  if (grid_finish<2>(both, partials, counter, 2u, s_red)) {
    if (threadIdx.x == 0) {
      ctl->ztr = both[0];
      ctl->rnorm = both[1];
      if (both[1] < fmax(ctl->tol, 1e-12)) ctl->done = 1;
      if (ctl->max_its <= 0) ctl->done = 1;
    }
  }
}

// ---------------------------------------------------------------------------
// K3 (private.c:181-211): x += alpha p; r -= alpha Gp; z = M r; reductions.
// 128-bit loads/stores (double2), 2 independent double2 per thread per trip.
__device__ __forceinline__ void cg_update_elem(double alpha, double nalpha, double &x, double &r,
                                               double p, double gp, double m, double &z,
                                               double &acc0, double &acc1) {
  x = fma(alpha, p, x);
  r = fma(nalpha, gp, r);
  z = r * m;
  acc0 = fma(z, r, acc0);
  acc1 = fmax(acc1, fabs(r));
}
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_update(int n, double *__restrict__ x, double *__restrict__ r, const double *__restrict__ p,
            const double *__restrict__ Gp, const double *__restrict__ M, double *__restrict__ z,
            B200CgCtl *ctl, double *partials, unsigned int *counter) {
  pdl_launch_dependents();  // K4's CTAs may become resident now; they wait for this grid in their own pdl_wait()
  pdl_wait();               // K2 (Gp, alpha) complete and visible
  if (ctl->done) return;
  __shared__ double s_red[128];
  const double alpha = ctl->alpha;
  const double nalpha = -alpha;
  double acc0 = 0.0, acc1 = 0.0;
  const int n2 = n >> 1;
  double2 *x2 = reinterpret_cast<double2 *>(x), *r2 = reinterpret_cast<double2 *>(r),
          *z2 = reinterpret_cast<double2 *>(z);
  const double2 *p2 = reinterpret_cast<const double2 *>(p), *g2 = reinterpret_cast<const double2 *>(Gp),
                *m2 = reinterpret_cast<const double2 *>(M);
  const int stride = gridDim.x * blockDim.x;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + stride < n2; i += 2 * stride) {
    double2 xa = x2[i], ra = r2[i], pa = p2[i], ga = g2[i], ma = m2[i], za;
    double2 xb = x2[i + stride], rb = r2[i + stride], pb = p2[i + stride], gb = g2[i + stride],
            mb = m2[i + stride], zb;
    cg_update_elem(alpha, nalpha, xa.x, ra.x, pa.x, ga.x, ma.x, za.x, acc0, acc1);
    cg_update_elem(alpha, nalpha, xa.y, ra.y, pa.y, ga.y, ma.y, za.y, acc0, acc1);
    cg_update_elem(alpha, nalpha, xb.x, rb.x, pb.x, gb.x, mb.x, zb.x, acc0, acc1);
    cg_update_elem(alpha, nalpha, xb.y, rb.y, pb.y, gb.y, mb.y, zb.y, acc0, acc1);
    x2[i] = xa; r2[i] = ra; z2[i] = za;
    x2[i + stride] = xb; r2[i + stride] = rb; z2[i + stride] = zb;
  }
  for (; i < n2; i += stride) {
    double2 xa = x2[i], ra = r2[i], pa = p2[i], ga = g2[i], ma = m2[i], za;
    cg_update_elem(alpha, nalpha, xa.x, ra.x, pa.x, ga.x, ma.x, za.x, acc0, acc1);
    cg_update_elem(alpha, nalpha, xa.y, ra.y, pa.y, ga.y, ma.y, za.y, acc0, acc1);
    x2[i] = xa; r2[i] = ra; z2[i] = za;
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
    const int k = n - 1;
    double xv = x[k], rv = r[k], zv;
    cg_update_elem(alpha, nalpha, xv, rv, p[k], Gp[k], M[k], zv, acc0, acc1);
    x[k] = xv; r[k] = rv; z[k] = zv;
  }
  double sm[1] = {acc0}, mx[1] = {acc1};
  block_sum<1>(sm, s_red);
  block_max<1>(mx, s_red + 64);
  double both[2] = {sm[0], mx[0]};
  if (grid_finish<2>(both, partials, counter, 2u, s_red)) {
    if (threadIdx.x == 0) {
      const double ztr_prev = ctl->ztr;
      ctl->ztr_prev = ztr_prev;
      ctl->ztr = both[0];
      ctl->rnorm = both[1];
      ctl->iters += 1;
      if (both[1] < ctl->tol) {
        ctl->done = 1;
      } else if (ztr_prev == 0.0) {
        ctl->done = 1;
      } else {
        ctl->beta = both[0] / ztr_prev;
        if (ctl->iters >= ctl->max_its) ctl->done = 1;
      }
    }
  }
}

// K4 (private.c:212-214): p = z + beta p
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_pupdate(int n, double *__restrict__ p, const double *__restrict__ z, const B200CgCtl *ctl) {
  pdl_launch_dependents();  // the next iteration's K1 may start its prologue (barrier init, first matrix stages)
  pdl_wait();               // K3 (z, beta, done) complete and visible
  if (ctl->done) return;
  const double beta = ctl->beta;
  const int n2 = n >> 1;
  double2 *p2 = reinterpret_cast<double2 *>(p);
  const double2 *z2 = reinterpret_cast<const double2 *>(z);
  const int stride = gridDim.x * blockDim.x;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + stride < n2; i += 2 * stride) {
    double2 pa = p2[i], za = z2[i], pb = p2[i + stride], zb = z2[i + stride];
    pa.x = fma(beta, pa.x, za.x); pa.y = fma(beta, pa.y, za.y);
    pb.x = fma(beta, pb.x, zb.x); pb.y = fma(beta, pb.y, zb.y);
    p2[i] = pa; p2[i + stride] = pb;
  }
  for (; i < n2; i += stride) {
    double2 pa = p2[i], za = z2[i];
    pa.x = fma(beta, pa.x, za.x); pa.y = fma(beta, pa.y, za.y);
    p2[i] = pa;
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) p[n - 1] = fma(beta, p[n - 1], z[n - 1]);
}


__global__ void k_zero_if(long long len, double *__restrict__ v, const int *flag) {
  if (!*flag) return;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len;
       i += (long long)gridDim.x * blockDim.x)
    v[i] = 0.0;
}

// ---------------------------------------------------------------------------
// Row-sharded mode (SURVEY 8e): every rank holds rows [row0, row0+mloc) of A in both
// orientations; x-space vectors are replicated. A' R_y^-1 A p is the sum over ranks of the
// local partial products -> one all-reduce of an n-vector per CG iteration; every other
// quantity (dots, alpha, beta, stop test) is then computed redundantly and bit-identically
// on every rank, so no scalar collective is needed.
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_finish_mv(int n, double *__restrict__ y, const double *__restrict__ red, int y_has_px,
               const double *__restrict__ rx, const double *__restrict__ x, int with_dot,
               B200CgCtl *ctl, const int *skip, double *partials, unsigned int *counter) {
  if (skip != nullptr && *skip) return;
  __shared__ double s_red[64];
  double acc[1] = {0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double base = y_has_px ? y[i] + red[i] : red[i];
    const double xi = x[i];
    const double out = fma(rx[i], xi, base);
    y[i] = out;
    acc[0] = fma(xi, out, acc[0]);
  }
  if (!with_dot) return;
  block_sum<1>(acc, s_red);
  if (grid_finish<1>(acc, partials, counter, 0u, s_red)) {
    if (threadIdx.x == 0) {
      ctl->pGp = acc[0];
      ctl->alpha = ctl->ztr / acc[0];
    }
  }
}
// Fused "all-reduce + finish" over NVLink peer memory: every rank has written its partial
// A_g' z into its own exchange buffer (slot seq & 1); this kernel (i) publishes "my partial of
// step seq is ready" into every peer's flag line, (ii) waits until every peer has published the
// same step, (iii) reads all partials -- the remote ones straight through the mapped peer
// pointers -- adds them IN RANK ORDER (so every rank gets the same bits), applies R_x p (+ P p)
// and reduces p'Gp. No NCCL call, no separate finish pass.
struct P2pView {
  int nranks, rank, stride;
  const double *base[8];
  unsigned long long *flags[8];
};
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_finish_p2p(int n, double *__restrict__ y, P2pView pv, unsigned long long seq, int do_signal,
                int y_has_px, const double *__restrict__ rx, const double *__restrict__ x,
                int with_dot, B200CgCtl *ctl, const int *skip, double *partials,
                unsigned int *counter) {
  if (skip != nullptr && *skip) return;
  __shared__ double s_red[64];
  if (threadIdx.x == 0) {
    if (do_signal && blockIdx.x == 0) {  // only when the producing SpMV did not signal itself
      __threadfence_system();
      for (int r = 0; r < pv.nranks; ++r)
        if (r != pv.rank) *((volatile unsigned long long *)(pv.flags[r] + pv.rank)) = seq;
    }
    volatile unsigned long long *mine = pv.flags[pv.rank];
    const long long t0 = clock64();
    for (int r = 0; r < pv.nranks; ++r) {
      if (r == pv.rank) continue;
      while (mine[r] < seq) {
        // never hang the GPU: after ~10 s (2e10 cycles) flag an error and go on (the host aborts the solve)
        if (clock64() - t0 > 20000000000LL) { ctl->pad[0] = 1; break; }
      }
    }
    __threadfence_system();
  }
  __syncthreads();
  const size_t slot = (size_t)(seq & 1ull) * pv.stride;
  double acc[1] = {0.0};
  constexpr int U = 4;  // independent remote loads in flight per thread and rank
  const int stride = gridDim.x * blockDim.x;
  for (int i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += U * stride) {
    double sum[U];
#pragma unroll
    for (int u = 0; u < U; ++u) sum[u] = 0.0;
    for (int r = 0; r < pv.nranks; ++r) {  // rank order => identical bits on every rank
      const double *src = pv.base[r] + slot;
      double t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * stride;
        t[u] = (i < n) ? __ldcg(src + i) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) sum[u] += t[u];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * stride;
      if (i < n) {
        const double base = y_has_px ? y[i] + sum[u] : sum[u];
        const double xi = x[i];
        const double out = fma(rx[i], xi, base);
        y[i] = out;
        acc[0] = fma(xi, out, acc[0]);
      }
    }
  }
  if (!with_dot) return;
  block_sum<1>(acc, s_red);
  if (grid_finish<1>(acc, partials, counter, 0u, s_red)) {
    if (threadIdx.x == 0) {
      ctl->pGp = acc[0];
      ctl->alpha = ctl->ztr / acc[0];
    }
  }
}

// Two-phase variant for G >= 3 ranks: a reduce-scatter and an all-gather over peer memory instead of
// every rank reading every partial in full -- 2 (G-1)/G n remote doubles per rank and CG iteration instead
// of (G-1) n (G = 8: 1.75 n instead of 7 n).
//   phase 1  rank g sums slice [n g/G, n (g+1)/G) of all partials in rank order into its own `rs` buffer;
//            the last block to finish publishes "slice ready" (flag slots 8..15) to every rank, itself included;
//   phase 2  every rank reads the reduced slices of all owners (remote for G-1 of them), applies R_x p (+ P p)
//            and reduces p'Gp.
// Every element is summed by exactly one rank in rank order, so all ranks still hold identical bits.
// `rs` = doubles [2 n, 4 n) of each rank's exchange allocation, double-buffered by seq like the partials.
__global__ void __launch_bounds__(VEC_THREADS)
k_cg_finish_p2p2(int n, double *__restrict__ y, P2pView pv, unsigned long long seq, int do_signal,
                 int y_has_px, const double *__restrict__ rx, const double *__restrict__ x,
                 int with_dot, B200CgCtl *ctl, const int *skip, double *partials,
                 unsigned int *counter) {
  if (skip != nullptr && *skip) return;
  __shared__ double s_red[64];
  const int G = pv.nranks, me = pv.rank;
  const size_t slot = (size_t)(seq & 1ull) * pv.stride;
  const size_t rs_base = (size_t)2 * pv.stride + slot;
  if (threadIdx.x == 0) {
    if (do_signal && blockIdx.x == 0) {
      __threadfence_system();
      for (int r = 0; r < G; ++r)
        if (r != me) *((volatile unsigned long long *)(pv.flags[r] + me)) = seq;
    }
    volatile unsigned long long *mine = pv.flags[me];
    const long long t0 = clock64();
    for (int r = 0; r < G; ++r) {
      if (r == me) continue;
      while (mine[r] < seq) {
        if (clock64() - t0 > 20000000000LL) { ctl->pad[0] = 1; break; }
      }
    }
    __threadfence_system();
  }
  __syncthreads();
  // ---- phase 1: my slice of the sum
  {
    const long long lo = (long long)n * me / G, hi = (long long)n * (me + 1) / G;
    double *dst = const_cast<double *>(pv.base[me]) + rs_base;
    constexpr int U = 4;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i0 = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x; i0 < hi; i0 += U * stride) {
      double sum[U];
#pragma unroll
      for (int u = 0; u < U; ++u) sum[u] = 0.0;
      for (int r = 0; r < G; ++r) {  // rank order
        const double *src = pv.base[r] + slot;
        double t[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long i = i0 + u * stride;
          t[u] = (i < hi) ? __ldcg(src + i) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) sum[u] += t[u];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long i = i0 + u * stride;
        if (i < hi) dst[i] = sum[u];
      }
    }
  }
  // the last block to finish its part publishes "slice of step seq ready" to everybody
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const unsigned tk = atomicAdd(counter, 1u);
    if (tk == gridDim.x - 1) {
      *counter = 0u;  // grid_finish below reuses the ticket counter
      __threadfence_system();
      for (int r = 0; r < G; ++r) *((volatile unsigned long long *)(pv.flags[r] + 8 + me)) = seq;
    }
    volatile unsigned long long *mine = pv.flags[me] + 8;
    const long long t0 = clock64();
    for (int r = 0; r < G; ++r) {
      while (mine[r] < seq) {
        if (clock64() - t0 > 20000000000LL) { ctl->pad[0] = 1; break; }
      }
    }
    __threadfence_system();
  }
  __syncthreads();
  // ---- phase 2: gather the reduced slices, finish G p and reduce p'Gp
  double acc[1] = {0.0};
  {
    constexpr int U = 4;
    const int stride = gridDim.x * blockDim.x;
    for (int i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += U * stride) {
      double t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * stride;
        if (i < n) {
          int owner = (int)(((long long)i * G) / n);  // slice g holds [n g/G, n (g+1)/G)
          while (owner + 1 < G && (long long)n * (owner + 1) / G <= i) ++owner;
          while (owner > 0 && (long long)n * owner / G > i) --owner;
          t[u] = __ldcg(pv.base[owner] + rs_base + i);
        } else {
          t[u] = 0.0;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * stride;
        if (i < n) {
          const double base = y_has_px ? y[i] + t[u] : t[u];
          const double xi = x[i];
          const double out = fma(rx[i], xi, base);
          y[i] = out;
          acc[0] = fma(xi, out, acc[0]);
        }
      }
    }
  }
  if (!with_dot) return;
  block_sum<1>(acc, s_red);
  if (grid_finish<1>(acc, partials, counter, 0u, s_red)) {
    if (threadIdx.x == 0) {
      ctl->pGp = acc[0];
      ctl->alpha = ctl->ztr / acc[0];
    }
  }
}


// ---------------------------------------------------------------------------------------------
// "Sharded-x" CG iteration for G >= 2 ranks, PUSH-based (the default multi-GPU mode; SCS_B200_SHARD_X=0 /
// scs_b200_set_shard_x(0) select the replicated modes above).
// p stays replicated (it is the SpMV gather vector) but lives in the peer-mapped exchange allocation; x, r, z and
// Gp are owned by n-slices [n g/G, n (g+1)/G). Data only ever moves by STORES into peer memory (NVLink writes
// pipeline; remote loads pay the full round trip), synchronisation is by sequence-numbered flags:
//   K1  tmp_g = R_g^-1 A_g p                                   local SpMV
//   K2  partial_g = A_g' tmp_g, every output row pushed into the inbox of the rank that owns it by the SpMV
//       epilogue itself (B200_HOOK_P2P_ROUTE = the reduce-scatter send) as a SELF-VALIDATING 16-byte element (value
//       halves + sequence number, common.cuh ll_store): no fence, no "ready" flag, no end-of-kernel signal
//   K34 ONE kernel per rank (this one):
//       1  sum MY slice from the LOCAL inbox in rank order, waiting per element for rows still in flight,
//          Gp = R_x p (+ P p) + sum, block-reduce p'Gp over the slice; the last block sends the slice's p'Gp to every
//          rank as a self-validating scalar message;
//       2  collect the G partial scalars, add them in rank order => p'Gp and alpha, identical bits everywhere;
//       3  K3 on the slice (x, r, z; z'r and ||r||_inf partials), pushed the same way;
//       4  wait, combine => z'r, ||r||_inf, the stop decision and beta, identical everywhere;
//       5  K4 on the slice: p = z + beta p into the local p and, as self-validating elements, into every peer's p-box
//          (the all-gather is G-1 remote 16-byte stores per element);
//       6  unpack the peers' slices from my p-box into p, waiting per element (the next K1 gathers from all of p).
// There is NO fence and NO flag anywhere in the protocol, and no buffer is double-buffered: a rank can overwrite a peer's
// inbox / message slot / p-box element of iteration k only after it has consumed data that peer sent AFTER reading them
// (rows of k+1 are sent after the peer's p slice of k arrived, which the peer sends after its reduction of k; messages
// and p elements of k+1 are sent after the peer's rows / round-2 message of k+1 arrived): the data flow itself orders
// the accesses (tests/test_shardx_protocol_cpu.py emulates the protocol with threads, split pushes and random delays).
// Remote volume per rank and iteration: 2 (G-1)/G n doubles OUT; K3 / K4 shrink by G. All blocks spin on flags, so
// the grid must be co-resident (<= #SMs blocks).
// Exchange allocation (comm.cu): [0, 4n) buffers of the replicated modes, [4n, 5n) p, [5n, 7n+32) inbox
// [G][S][2 words] with S = ceil(n / G), [7n+32, 9n+64) p-box [n][2 words], then the flag line (replicated modes only)
// and 64 words of scalar messages [round][from rank][4].
struct P2pViewX {
  int nranks, rank, S;
  const unsigned long long *inbox;  // local: element (q * S + i - lo) = rank q's partial for my element i (16 bytes)
  unsigned long long *peer_pbox[8];  // peer_pbox[q]: rank q's p-box as mapped here (element i = 2 words)
  const unsigned long long *pbox;    // local p-box: the peers' slices of the new p arrive here
  unsigned long long *flags[8];
  unsigned long long *dbg;          // optional: 8 globaltimer stamps (ns) of block 0 at the phase boundaries, or NULL
};
__device__ __forceinline__ void px_stamp(const P2pViewX &pv, int k) {
  if (pv.dbg != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    pv.dbg[k] = t;
  }
}
// scalar messages: after the 64 flags of every rank's line, 64 words = [round 0..1][from rank 0..7][4 words]
// (a double = 2 self-validating words; round 0 carries 1 double, round 1 carries 2)
__device__ __forceinline__ unsigned long long *px_msg(const P2pViewX &pv, int r, int round, int from) {
  return pv.flags[r] + 64 + (round * 8 + from) * 4;
}
// spin until the self-validating element carries seq32; gives up after ~1.5 s and raises the sticky error flag
__device__ __forceinline__ double ll_wait(const unsigned long long *src2, unsigned seq32, B200CgCtl *ctl) {
  double v = 0.0;
  if (ll_try_load(src2, seq32, v)) return v;
  const long long t0 = clock64();
  while (!ll_try_load(src2, seq32, v)) {
    if (*((volatile int *)&ctl->pad[0])) return 0.0;
    if (clock64() - t0 > 3000000000LL) { ctl->pad[0] = 1; return 0.0; }
  }
  return v;
}
__device__ __forceinline__ void px_wait(volatile unsigned long long *line, int first, int G, int skip_rank,
                                        unsigned long long seq, B200CgCtl *ctl) {
  // never hang the GPU: a wait gives up after ~1.5 s (3e9 cycles) and raises the error flag; once the flag is up every
  // later wait of this and the following iterations returns at once (the host aborts the solve when it sees it)
  if (*((volatile int *)&ctl->pad[0])) return;
  const long long t0 = clock64();
  for (int r = 0; r < G; ++r) {
    if (r == skip_rank) continue;
    while (line[first + r] < seq) {
      if (clock64() - t0 > 3000000000LL) { ctl->pad[0] = 1; return; }
    }
  }
  asm volatile("fence.acq_rel.sys;" ::: "memory");  // acquire side: the peer's data stores precede its flag store
}

__global__ void __launch_bounds__(VEC_THREADS)
k_cgx_iteration(int n, P2pViewX pv, unsigned long long seq, int y_has_px,
                const double *__restrict__ rx, const double *__restrict__ M, double *p,
                double *__restrict__ Gp, double *__restrict__ x, double *__restrict__ r,
                double *__restrict__ z, B200CgCtl *ctl, double *partials, unsigned int *counters) {
  pdl_launch_dependents();  // the next K1 may start its prologue; it waits for this grid before it gathers from p
  pdl_wait();               // K2 (this rank's pushes) complete
  if (ctl->done || ctl->pad[0]) return;
  __shared__ double s_red[192];
  __shared__ double s_bc[4];
  const int G = pv.nranks, me = pv.rank;
  const unsigned seq32 = (unsigned)seq;
  const long long lo = (long long)n * me / G, hi = (long long)n * (me + 1) / G;
  const long long gstride = (long long)gridDim.x * blockDim.x;
  const long long gtid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  volatile unsigned long long *myflags = pv.flags[me];
  // values of the control block as of the start of the iteration (the last block rewrites it at the end)
  const double ztr_old = ctl->ztr, tol = ctl->tol;
  const int iters_old = ctl->iters, max_its = ctl->max_its;

  px_stamp(pv, 0);
  // ---- 1: my slice of G p from the self-validating rows in my inbox (rank order; a row that has not arrived yet is
  // simply waited for -- the reduction overlaps the tail of the peers' K2), partial p'Gp
  double acc = 0.0;
  for (long long i = lo + gtid; i < hi; i += gstride) {
    // all G reads are issued before any is looked at (they are independent); only a row that has not arrived is polled
    unsigned long long w0[8], w1[8];
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (q < G) ll_load_raw(pv.inbox + 2 * ((size_t)q * pv.S + (size_t)(i - lo)), w0[q], w1[q]);
    double sum = 0.0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      if (q < G) {
        const double vq = ll_valid(w0[q], w1[q], seq32)
                              ? ll_value(w0[q], w1[q])
                              : ll_wait(pv.inbox + 2 * ((size_t)q * pv.S + (size_t)(i - lo)), seq32, ctl);
        sum += vq;  // rank order
      }
    }
    const double base = y_has_px ? Gp[i] + sum : sum;
    const double pi = p[i];
    const double out = fma(rx[i], pi, base);
    Gp[i] = out;
    acc = fma(pi, out, acc);
  }
  px_stamp(pv, 1);
  {
    // slice total: every block publishes its partial as a self-validating element (local memory), block 0 collects
    // them in a fixed order (slot t -> thread t, then the fixed block_sum tree) and sends ONE message to every rank --
    // no atomic ticket, no fence, no last-block serialisation on the critical path
    double a[1] = {acc};
    block_sum<1>(a, s_red);
    unsigned long long *slots = reinterpret_cast<unsigned long long *>(partials + 2048);  // [2048, 4096): only this kernel
    if (threadIdx.x == 0) ll_store(slots + 2 * blockIdx.x, a[0], seq32);
    if (blockIdx.x == 0) {
      double t[1] = {0.0};
      for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) t[0] += ll_wait(slots + 2 * b, seq32, ctl);
      block_sum<1>(t, s_red);
      if (threadIdx.x == 0)
        for (int q = 0; q < G; ++q) ll_store(px_msg(pv, q, 0, me), t[0], seq32);
    }
    if (threadIdx.x == 0) {
      // ---- 2: all partial scalars -> alpha (rank order: identical bits on every rank)
      double pGp = 0.0;
      for (int q = 0; q < G; ++q) pGp += ll_wait(px_msg(pv, me, 0, q), seq32, ctl);
      s_bc[0] = pGp;
      s_bc[1] = ztr_old / pGp;
    }
  }
  __syncthreads();
  px_stamp(pv, 2);
  const double pGp = s_bc[0], alpha = s_bc[1], nalpha = -alpha;

  // ---- 3: K3 on the slice
  double acc0 = 0.0, acc1 = 0.0;
  for (long long i = lo + gtid; i < hi; i += gstride) {
    const double pi = p[i];
    const double xi = fma(alpha, pi, x[i]);
    const double ri = fma(nalpha, Gp[i], r[i]);
    const double zi = ri * M[i];
    x[i] = xi;
    r[i] = ri;
    z[i] = zi;
    acc0 = fma(zi, ri, acc0);
    acc1 = fmax(acc1, fabs(ri));
  }
  px_stamp(pv, 3);
  {
    double sm[1] = {acc0}, mx[1] = {acc1};
    block_sum<1>(sm, s_red);
    block_max<1>(mx, s_red + 64);
    unsigned long long *slots = reinterpret_cast<unsigned long long *>(partials + 3072);
    if (threadIdx.x == 0) {
      ll_store(slots + 4 * blockIdx.x, sm[0], seq32);
      ll_store(slots + 4 * blockIdx.x + 2, mx[0], seq32);
    }
    if (blockIdx.x == 0) {
      double t[1] = {0.0}, u[1] = {0.0};
      for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) {
        t[0] += ll_wait(slots + 4 * b, seq32, ctl);
        u[0] = fmax(u[0], ll_wait(slots + 4 * b + 2, seq32, ctl));
      }
      block_sum<1>(t, s_red);
      block_max<1>(u, s_red + 64);
      if (threadIdx.x == 0)
        for (int q = 0; q < G; ++q) {
          ll_store(px_msg(pv, q, 1, me), t[0], seq32);
          ll_store(px_msg(pv, q, 1, me) + 2, u[0], seq32);
        }
    }
    if (threadIdx.x == 0) {
      // ---- 4: z'r, ||r||_inf, stop decision, beta (same arithmetic as k_cg_update's last block)
      double ztr = 0.0, rn = 0.0;
      for (int q = 0; q < G; ++q) {
        ztr += ll_wait(px_msg(pv, me, 1, q), seq32, ctl);
        rn = fmax(rn, ll_wait(px_msg(pv, me, 1, q) + 2, seq32, ctl));
      }
      int done = 0;
      double beta = 0.0;
      if (rn < tol) done = 1;
      else if (ztr_old == 0.0) done = 1;
      else {
        beta = ztr / ztr_old;
        if (iters_old + 1 >= max_its) done = 1;
      }
      s_bc[0] = ztr;
      s_bc[1] = rn;
      s_bc[2] = beta;
      s_bc[3] = (double)done;
    }
  }
  __syncthreads();
  px_stamp(pv, 4);
  const double ztr_new = s_bc[0], rnorm = s_bc[1], beta = s_bc[2];
  const int done = s_bc[3] != 0.0;

  // ---- 5: K4 on the slice (skipped once the stop test fired, like k_cg_pupdate): the new p goes into the local p and,
  // as self-validating elements, into every peer's p-box (the all-gather is G-1 remote 16-byte stores per element)
  if (!done) {
    for (long long i = lo + gtid; i < hi; i += gstride) {
      const double pn = fma(beta, p[i], z[i]);
      p[i] = pn;
      for (int q = 0; q < G; ++q)
        if (q != me) ll_store(pv.peer_pbox[q] + 2 * (size_t)i, pn, seq32);
    }
  }
  px_stamp(pv, 5);
  // ---- 6: unpack the peers' slices from my p-box into p, waiting per element for what is still in flight (the next K1
  // gathers from all of p). No fence, no flag: the elements validate themselves.
  if (!done) {
    for (int q = 0; q < G; ++q) {
      if (q == me) continue;
      const long long qlo = (long long)n * q / G, qhi = (long long)n * (q + 1) / G;
      for (long long i = qlo + gtid; i < qhi; i += gstride) p[i] = ll_wait(pv.pbox + 2 * (size_t)i, seq32, ctl);
    }
  }
  px_stamp(pv, 6);
  __syncthreads();
  if (threadIdx.x == 0) {
    // the last block to arrive records the iteration in the control block: every block read its start values long ago
    __threadfence();
    if (atomicAdd(&counters[6], 1u) == gridDim.x - 1) {
      counters[6] = 0u;
      ctl->ztr_prev = ztr_old;
      ctl->ztr = ztr_new;
      ctl->rnorm = rnorm;
      ctl->pGp = pGp;
      ctl->alpha = alpha;
      ctl->iters = iters_old + 1;
      if (!done) ctl->beta = beta;
      if (done) ctl->done = 1;
    }
    px_stamp(pv, 7);
  }
}

__global__ void k_add_if_not(int n, double *__restrict__ a, const double *__restrict__ b, const int *skip) {
  if (skip != nullptr && *skip) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) a[i] += b[i];
}
// M = 1 / (R_x + P_jj + sum over ALL ranks of the local column sums)
__global__ void k_precond_partial(int n, const int *__restrict__ colptr, const int *__restrict__ rowidx,
                                  const double *__restrict__ vals, const double *__restrict__ ry_loc,
                                  double *__restrict__ out) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int k = colptr[j]; k < colptr[j + 1]; ++k) {
      const double v = vals[k];
      acc += v * v / ry_loc[rowidx[k] & B200_COLMASK];
    }
    out[j] = acc;
  }
}
__global__ void k_precond_finish(int n, const double *__restrict__ rx, const double *__restrict__ sum,
                                 const double *__restrict__ pdiag, double *__restrict__ M) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    double acc = rx[j] + sum[j];
    if (pdiag != nullptr) acc += pdiag[j];
    M[j] = 1.0 / acc;
  }
}

__global__ void k_recip(long long len, const double *__restrict__ v, double *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < len; i += (long long)gridDim.x * blockDim.x)
    out[i] = 1.0 / v[i];
}
// ---------------------------------------------------------------------------
extern "C" int b200_cg_set_preconditioner(const B200Cg *cg, const double *d_Pdiag) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  // R_y^-1 for K1 (reference linsys/gpu/indirect/private.c:75-80 keeps the same inverse)
  k_recip<<<vec_grid(cg->m), 256, 0, st>>>(cg->m, cg->d_ry, cg->d_ry_inv);
  b200_count_launch(1);
  if (cg->nranks > 1) {
    k_precond_partial<<<vec_grid(cg->n), 256, 0, st>>>(cg->n, b200_spmv_rowptr(cg->At),
                                                      b200_spmv_colidx(cg->At), b200_spmv_vals(cg->At),
                                                      cg->d_ry + cg->row0, cg->d_red);
    if (b200_allreduce_sum(cg->d_red, (size_t)cg->n) != 0) return -1;
    k_precond_finish<<<vec_grid(cg->n), 256, 0, st>>>(cg->n, cg->d_rx, cg->d_red, d_Pdiag, cg->d_M);
    b200_count_launch(2);
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  // CSR of A' == CSC of A: rowptr = column pointers, colidx = row indices
  k_set_preconditioner<<<vec_grid(cg->n), 256, 0, st>>>(
      cg->n, b200_spmv_rowptr(cg->At), b200_spmv_colidx(cg->At), b200_spmv_vals(cg->At), cg->d_rx,
      cg->d_ry, d_Pdiag, cg->d_M);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// programmatic dependent launch of the CG loop's kernels (SCS_B200_PDL=0 turns it off for A/B measurements)
static int g_pdl = -1;
static bool cg_pdl_enabled() {
  if (g_pdl < 0) {
    const char *e = getenv("SCS_B200_PDL");
    g_pdl = (e && atoi(e) == 0) ? 0 : 1;
  }
  return g_pdl == 1;
}

// peer-memory reduction: 0 = automatic (one pass for 2 ranks, two-phase for more), 1 = one pass, 2 = two-phase
static int g_p2p_mode = -1;
extern "C" void scs_b200_set_p2p_mode(int mode) { g_p2p_mode = mode; }

// y = (R_x + P + A' R_y^-1 A) x   (private.c:106-119); dot/hook optional
static int mat_vec_sharded(B200Cg *cg, const double *d_x, double *d_y, int with_dot,
                           const int *d_skip) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  B200SpmvArgs a;
  memset(&a, 0, sizeof(a));
  // K1 (local rows): tmp[row0:row0+mloc] = (A_g x) ./ R_y
  a.d_x = d_x; a.d_y = cg->d_tmp + cg->row0; a.init_sign = 1.0; a.post = B200_POST_MUL;
  a.d_d = cg->d_ry_inv + cg->row0; a.d_skip = d_skip;
  if (b200_spmv(cg->A, &a) != 0) return -1;
  // local partial  red = A_g' tmp_g ; sum over ranks
  unsigned long long seq = 0;
  double *red = cg->d_red;
  if (cg->use_p2p) {
    seq = b200_p2p_next_seq();
    red = b200_p2p_base(b200_comm_rank()) + (size_t)(seq & 1ull) * b200_p2p_stride();
  }
  a.d_x = cg->d_tmp + cg->row0; a.d_y = red; a.post = B200_POST_NONE; a.d_d = nullptr;
  if (cg->use_p2p && cg->d_p2p_sig) {  // the SpMV's last block publishes "partial ready" to the peers
    a.hook = B200_HOOK_P2P_SIGNAL; a.d_hook_arg = cg->d_p2p_sig; a.hook_val = seq;
  }
  if (b200_spmv(cg->At, &a) != 0) return -1;
  a.hook = B200_HOOK_NONE; a.d_hook_arg = nullptr; a.hook_val = 0;
  if (!cg->use_p2p && b200_allreduce_sum(cg->d_red, (size_t)cg->n) != 0) return -1;
  if (cg->P) {  // P is replicated
    a.d_x = d_x; a.d_y = d_y;
    if (b200_spmv(cg->P, &a) != 0) return -1;
  }
  int g = (cg->n + VEC_THREADS * 4 - 1) / (VEC_THREADS * 4);
  if (g > 2 * b200_num_sms()) g = 2 * b200_num_sms();
  if (cg->use_p2p) {
    P2pView pv;
    pv.nranks = cg->nranks; pv.rank = b200_comm_rank(); pv.stride = b200_p2p_stride();
    for (int r = 0; r < 8; ++r) {
      pv.base[r] = r < cg->nranks ? b200_p2p_base(r) : nullptr;
      pv.flags[r] = r < cg->nranks ? b200_p2p_flags(r) : nullptr;
    }
    if (g > b200_num_sms()) g = b200_num_sms();  // all blocks spin on the flags: keep them co-resident
    // two ranks: one pass (same remote volume, one synchronisation less); more: reduce-scatter + all-gather
    if (g_p2p_mode < 0) {
      const char *e = getenv("SCS_B200_P2P_MODE");
      g_p2p_mode = e ? atoi(e) : 0;
    }
    const bool two_phase = g_p2p_mode == 2 || (g_p2p_mode != 1 && cg->nranks >= 3);
    if (two_phase)
      k_cg_finish_p2p2<<<g, VEC_THREADS, 0, st>>>(cg->n, d_y, pv, seq, cg->d_p2p_sig == nullptr,
                                                  cg->P != nullptr, cg->d_rx, d_x, with_dot, cg->d_ctl,
                                                  d_skip, cg->d_partials, cg->d_counter);
    else
      k_cg_finish_p2p<<<g, VEC_THREADS, 0, st>>>(cg->n, d_y, pv, seq, cg->d_p2p_sig == nullptr,
                                                 cg->P != nullptr, cg->d_rx, d_x,
                                                 with_dot, cg->d_ctl, d_skip, cg->d_partials,
                                                 cg->d_counter);
    b200_count_launch(1);
    return 0;
  }
  k_cg_finish_mv<<<g, VEC_THREADS, 0, st>>>(cg->n, d_y, cg->d_red, cg->P != nullptr, cg->d_rx, d_x,
                                            with_dot, cg->d_ctl, d_skip, cg->d_partials, cg->d_counter);
  b200_count_launch(1);
  return 0;
}

static int mat_vec(B200Cg *cg, const double *d_x, double *d_y, int with_dot, const int *d_skip) {
  if (cg->nranks > 1) return mat_vec_sharded(cg, d_x, d_y, with_dot, d_skip);
  // the m-space-reordered pair when present: tmp is internal to the operator, so its ordering is free
  const bool re = cg->A_cg != nullptr && cg->At_cg != nullptr && cg->d_ry_cg != nullptr;
  const B200Spmv *A = re ? cg->A_cg : cg->A, *At = re ? cg->At_cg : cg->At;
  B200SpmvArgs a;
  memset(&a, 0, sizeof(a));
  // K1: tmp = (A x) ./ R_y
  a.pdl = cg_pdl_enabled() ? 1 : 0;
  a.d_x = d_x; a.d_y = cg->d_tmp; a.d_init = nullptr; a.init_sign = 1.0;
  a.post = B200_POST_MUL; a.d_d = re ? cg->d_ry_cg : cg->d_ry_inv; a.d_v = nullptr; a.d_dot = nullptr;
  a.hook = B200_HOOK_NONE; a.d_hook_arg = nullptr; a.d_skip = d_skip;
  if (b200_spmv(A, &a) != 0) return -1;
  const double *init = nullptr;
  if (cg->P) {
    // y = P x first (reference accumulates P x before A' z)
    a.d_x = d_x; a.d_y = d_y; a.d_init = nullptr; a.post = B200_POST_NONE;
    a.d_d = nullptr; a.d_v = nullptr;
    if (b200_spmv(cg->P, &a) != 0) return -1;
    init = d_y;
  }
  // K2: y = fma(R_x, x, init + A' tmp)
  a.d_x = cg->d_tmp; a.d_y = d_y; a.d_init = init; a.init_sign = 1.0;
  a.post = with_dot ? B200_POST_FMA_DOT : B200_POST_FMA;
  a.d_d = cg->d_rx; a.d_v = d_x; a.d_dot = with_dot ? &cg->d_ctl->pGp : nullptr;
  a.hook = with_dot ? B200_HOOK_CG_ALPHA : B200_HOOK_NONE;
  a.d_hook_arg = cg->d_ctl; a.d_skip = d_skip;
  return b200_spmv(At, &a);
}

// sharded-x push mode (see k_cgx_iteration): -1 = read SCS_B200_SHARD_X once (default ON; =0 selects the replicated
// modes), 0 = off, 1 = on
static int g_shard_x = -1;
extern "C" void scs_b200_set_shard_x(int on) { g_shard_x = on ? 1 : 0; }
static int shard_x_active(const B200Cg *cg) {
  if (g_shard_x < 0) {
    const char *e = getenv("SCS_B200_SHARD_X");
    g_shard_x = (e && atoi(e) == 0) ? 0 : 1;
  }
  return g_shard_x == 1 && cg->nranks > 1 && cg->use_p2p && cg->d_p2p_route != nullptr;
}

static int cg_iteration_shard_x(B200Cg *cg, double *d_x, cudaEvent_t *ev = nullptr) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int *d_skip = &cg->d_ctl->done;
  if (ev) cudaEventRecord(ev[0], st);
  B200SpmvArgs a;
  memset(&a, 0, sizeof(a));
  // K1 (local rows): tmp_g = (A_g p) ./ R_g
  a.pdl = cg_pdl_enabled() ? 1 : 0;
  a.d_x = cg->d_p; a.d_y = cg->d_tmp + cg->row0; a.init_sign = 1.0; a.post = B200_POST_MUL;
  a.d_d = cg->d_ry_inv + cg->row0; a.d_skip = d_skip;
  if (b200_spmv(cg->A, &a) != 0) return -1;
  if (ev) cudaEventRecord(ev[1], st);
  // K2: partial A_g' tmp_g, every row pushed to its owner's inbox; the last block signals "partial ready"
  const unsigned long long seq = b200_p2p_next_seq();
  a.d_x = cg->d_tmp + cg->row0;
  a.d_y = cg->d_red;  // not written in routed mode
  a.post = B200_POST_NONE; a.d_d = nullptr;
  a.hook = B200_HOOK_P2P_ROUTE; a.d_hook_arg = cg->d_p2p_route; a.hook_val = seq;
  if (b200_spmv(cg->At, &a) != 0) return -1;
  if (cg->P) {  // P is replicated: Gp = P p on every rank, the slice kernel adds the rest
    memset(&a, 0, sizeof(a));
    a.d_x = cg->d_p; a.d_y = cg->d_Gp; a.init_sign = 1.0; a.post = B200_POST_NONE; a.d_skip = d_skip;
    if (b200_spmv(cg->P, &a) != 0) return -1;
  }
  if (ev) cudaEventRecord(ev[2], st);
  const int G = cg->nranks, me = b200_comm_rank();
  P2pViewX pv;
  pv.nranks = G; pv.rank = me; pv.S = (cg->n + G - 1) / G;
  pv.inbox = (const unsigned long long *)b200_p2p_inbox(me);
  pv.pbox = (const unsigned long long *)b200_p2p_pbox(me);
  for (int r = 0; r < 8; ++r) {
    pv.peer_pbox[r] = r < G ? (unsigned long long *)b200_p2p_pbox(r) : nullptr;
    pv.flags[r] = r < G ? b200_p2p_flags(r) : nullptr;
  }
  pv.dbg = ev ? reinterpret_cast<unsigned long long *>(cg->d_partials + 3 * 2048) : nullptr;  // timing runs only
  int g = b200_num_sms();  // every block spins on flags: one block per SM, co-resident
  const long long slice = ((long long)cg->n + G - 1) / G;
  const long long want = (slice + VEC_THREADS - 1) / VEC_THREADS;
  if (want < g) g = (int)(want < 1 ? 1 : want);
  CUDA_OK(b200_launch(k_cgx_iteration, dim3(g), dim3(VEC_THREADS), 0, st, cg_pdl_enabled(), cg->n, pv, seq,
                      (int)(cg->P != nullptr), (const double *)cg->d_rx, (const double *)cg->d_M, cg->d_p, cg->d_Gp,
                      d_x, cg->d_r, cg->d_z, cg->d_ctl, cg->d_partials, cg->d_counter));
  if (ev) cudaEventRecord(ev[3], st);
  b200_count_launch(1);
  return 0;
}

static int cg_iteration(B200Cg *cg, double *d_x) {
  if (shard_x_active(cg)) return cg_iteration_shard_x(cg, d_x);
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int n = cg->n;
  int g = (n + VEC_THREADS * 8 - 1) / (VEC_THREADS * 8);
  if (g > 2 * b200_num_sms()) g = 2 * b200_num_sms();
  if (g < 1) g = 1;
  if (mat_vec(cg, cg->d_p, cg->d_Gp, 1, &cg->d_ctl->done) != 0) return -1;
  const bool pdl = cg_pdl_enabled();
  CUDA_OK(b200_launch(k_cg_update, dim3(g), dim3(VEC_THREADS), 0, st, pdl, n, d_x, cg->d_r, (const double *)cg->d_p,
                      (const double *)cg->d_Gp, (const double *)cg->d_M, cg->d_z, cg->d_ctl, cg->d_partials,
                      cg->d_counter));
  CUDA_OK(b200_launch(k_cg_pupdate, dim3(g), dim3(VEC_THREADS), 0, st, pdl, n, cg->d_p, (const double *)cg->d_z,
                      (const B200CgCtl *)cg->d_ctl));
  b200_count_launch(2);
  return 0;
}

extern "C" int b200_cg_one_iteration(B200Cg *cg, double *d_x) { return cg_iteration(cg, d_x); }

// Per-kernel device times of the CG loop AS IT RUNS IN A SOLVE (bench.py roofline): `reps` genuine iterations on
// the solver's own p / tmp / r, every kernel bracketed by CUDA events on the library stream. out_ms[0..3] = average
// per launch of K1 (tmp = R_y^-1 A p, spmv POST_MUL), K2 (Gp = R_x p + A' tmp, p'Gp, alpha: spmv POST_FMA_DOT + hook),
// K3 (k_cg_update), K4 (k_cg_pupdate); out_ms[4] = whole iteration (first event to last, launch gaps included).
// Single-GPU, P = NULL path only (the configuration the roofline is quoted on).
extern "C" int b200_cg_time_kernels(B200Cg *cg, double *d_x, int reps, double *out_ms) {
  if (cg->nranks > 1 && shard_x_active(cg) && !cg->P && reps > 0) {
    // sharded-x push mode: K1 (local rows), K2 (local partial + pushes + signal), K34 (the slice kernel incl. all waits
    // on the peers); out_ms[3] = 0. Every rank runs this together (the kernels synchronise through the peer flags).
    cudaStream_t st = (cudaStream_t)b200_stream();
    std::vector<cudaEvent_t> ev((size_t)reps * 4);
    for (auto &e : ev) cudaEventCreate(&e);
    int rc = 0;
    for (int r = 0; r < reps && rc == 0; ++r) rc = cg_iteration_shard_x(cg, d_x, &ev[(size_t)r * 4]);
    if (cudaStreamSynchronize(st) != cudaSuccess) rc = -1;
    if (rc == 0) {
      for (int k = 0; k < 5; ++k) out_ms[k] = 0.0;
      for (int r = 0; r < reps; ++r) {
        float ms;
        for (int k = 0; k < 3; ++k) {
          cudaEventElapsedTime(&ms, ev[(size_t)r * 4 + k], ev[(size_t)r * 4 + k + 1]);
          out_ms[k] += ms;
        }
        cudaEventElapsedTime(&ms, ev[(size_t)r * 4], ev[(size_t)r * 4 + 3]);
        out_ms[4] += ms;
      }
      for (int k = 0; k < 5; ++k) out_ms[k] /= reps;
      // phase boundaries inside the slice kernel of the LAST timed iteration (block 0, globaltimer ns)
      unsigned long long h[8];
      if (cudaMemcpy(h, cg->d_partials + 3 * 2048, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess)
        for (int k = 0; k < 7; ++k) out_ms[5 + k] = (double)(long long)(h[k + 1] - h[k]) * 1e-6;
    }
    for (auto &e : ev) cudaEventDestroy(e);
    return rc;
  }
  if (cg->nranks > 1 || cg->P || reps <= 0) return -1;
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int n = cg->n;
  int g = (n + VEC_THREADS * 8 - 1) / (VEC_THREADS * 8);
  if (g > 2 * b200_num_sms()) g = 2 * b200_num_sms();
  if (g < 1) g = 1;
  std::vector<cudaEvent_t> ev((size_t)reps * 5);
  for (auto &e : ev) e = nullptr;
  int rc = -1;
  bool ok = true;
  for (auto &e : ev)
    if (cudaEventCreate(&e) != cudaSuccess) ok = false;
  if (ok) {
    const int *d_skip = &cg->d_ctl->done;
    for (int r = 0; r < reps && ok; ++r) {
      B200SpmvArgs a;
      memset(&a, 0, sizeof(a));
      cudaEventRecord(ev[(size_t)r * 5 + 0], st);
      const bool re = cg->A_cg != nullptr && cg->At_cg != nullptr && cg->d_ry_cg != nullptr;
      a.d_x = cg->d_p; a.d_y = cg->d_tmp; a.init_sign = 1.0; a.post = B200_POST_MUL;
      a.d_d = re ? cg->d_ry_cg : cg->d_ry_inv;
      a.d_skip = d_skip;
      if (b200_spmv(re ? cg->A_cg : cg->A, &a) != 0) ok = false;
      cudaEventRecord(ev[(size_t)r * 5 + 1], st);
      a.d_x = cg->d_tmp; a.d_y = cg->d_Gp; a.post = B200_POST_FMA_DOT; a.d_d = cg->d_rx; a.d_v = cg->d_p;
      a.d_dot = &cg->d_ctl->pGp; a.hook = B200_HOOK_CG_ALPHA; a.d_hook_arg = cg->d_ctl;
      if (b200_spmv(re ? cg->At_cg : cg->At, &a) != 0) ok = false;
      cudaEventRecord(ev[(size_t)r * 5 + 2], st);
      k_cg_update<<<g, VEC_THREADS, 0, st>>>(n, d_x, cg->d_r, cg->d_p, cg->d_Gp, cg->d_M, cg->d_z, cg->d_ctl,
                                             cg->d_partials, cg->d_counter);
      cudaEventRecord(ev[(size_t)r * 5 + 3], st);
      k_cg_pupdate<<<g, VEC_THREADS, 0, st>>>(n, cg->d_p, cg->d_z, cg->d_ctl);
      cudaEventRecord(ev[(size_t)r * 5 + 4], st);
      b200_count_launch(2);
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) ok = false;
  }
  if (ok) {
    for (int k = 0; k < 5; ++k) out_ms[k] = 0.0;
    for (int r = 0; r < reps; ++r) {
      for (int k = 0; k < 4; ++k) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[(size_t)r * 5 + k], ev[(size_t)r * 5 + k + 1]);
        out_ms[k] += ms;
      }
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[(size_t)r * 5], ev[(size_t)r * 5 + 4]);
      out_ms[4] += ms;
    }
    for (int k = 0; k < 5; ++k) out_ms[k] /= reps;
    rc = 0;
  }
  for (auto &e : ev)
    if (e) cudaEventDestroy(e);
  return rc;
}

extern "C" double b200_cg_iter_alg_bytes(const B200Cg *cg) {
  const double nnz = (double)b200_spmv_nnz(cg->A);
  return 24.0 * nnz + 4.0 * (cg->m + cg->n + 2.0) + 24.0 * cg->m + 120.0 * cg->n;
}

extern "C" int b200_cg_solve(B200Cg *cg, double *d_b, const double *d_s, double tol, int max_its,
                             int its_hint, const double *d_tol) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int n = cg->n, m = cg->m;
  const int g = vec_grid(n);
  const int *d_skip = &cg->d_ctl->skip;

  // prologue: ||b||, tmp = r_y / R_y
  k_cg_prepare<<<vec_grid((long long)n + m), VEC_THREADS, 0, st>>>(
      n, m, d_b, cg->d_ry, cg->d_tmp, cg->d_ctl, tol, d_tol, max_its, cg->d_partials,
      cg->d_counter);
  b200_count_launch(1);
  // b[0:n] += A' tmp   (private.c:305)
  if (cg->nranks > 1) {
    B200SpmvArgs a;
    memset(&a, 0, sizeof(a));
    a.d_x = cg->d_tmp + cg->row0; a.d_y = cg->d_red; a.init_sign = 1.0; a.post = B200_POST_NONE;
    a.d_skip = d_skip;
    if (b200_spmv(cg->At, &a) != 0) return -1;
    if (b200_allreduce_sum(cg->d_red, (size_t)n) != 0) return -1;
    k_add_if_not<<<g, VEC_THREADS, 0, st>>>(n, d_b, cg->d_red, d_skip);
    b200_count_launch(1);
  } else {
    B200SpmvArgs a;
    memset(&a, 0, sizeof(a));
    a.d_x = cg->d_tmp; a.d_y = d_b; a.d_init = d_b; a.init_sign = 1.0; a.post = B200_POST_NONE;
    a.d_d = nullptr; a.d_v = nullptr; a.d_dot = nullptr; a.hook = B200_HOOK_NONE;
    a.d_hook_arg = nullptr; a.d_skip = d_skip;
    if (b200_spmv(cg->At, &a) != 0) return -1;
  }
  // r = G s (warm) ; start
  if (d_s != nullptr) {
    if (mat_vec(cg, d_s, cg->d_r, 0, d_skip) != 0) return -1;
  }
  k_cg_init<<<g, VEC_THREADS, 0, st>>>(n, d_s != nullptr ? 1 : 0, d_b, d_s, cg->d_r, cg->d_M,
                                       cg->d_z, cg->d_p, cg->d_ctl, cg->d_partials, cg->d_counter);
  b200_count_launch(1);
  CUDA_OK(cudaGetLastError());

  // main loop in batches. An iteration enqueued after `done` costs 4 empty launches (~12 us), a
  // host poll costs a ~40 us bubble: the first batch is the previous solve's count plus a 6 % margin
  // (consecutive ADMM iterations need nearly the same number of CG steps), later batches are small.
  int batch = its_hint + (its_hint / 16 > 2 ? its_hint / 16 : 2);
  if (batch < 4) batch = 4;
  if (batch > 512) batch = 512;  // a sharp drop of the CG count between two solves wastes at most 512 empty iterations
  const int follow = its_hint / 8 > 8 ? (its_hint / 8 < 256 ? its_hint / 8 : 256) : 8;
  long long enq = 0;
  int polls = 0;
  for (;;) {
    for (int i = 0; i < batch; ++i)
      if (cg_iteration(cg, d_b) != 0) return -1;
    enq += batch;
    CUDA_OK(cudaMemcpyAsync(cg->h_ctl, cg->d_ctl, sizeof(B200CgCtl), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (cg->h_ctl->pad[0]) {
      b200_set_error("peer-memory wait timed out in k_cg_finish_p2p", cudaErrorUnknown, __FILE__, __LINE__);
      return -1;
    }
    if (cg->h_ctl->done) break;
    if (enq >= (long long)max_its + 1) break;  // safety; device sets done at max_its
    // after a miss: a small batch first (the hint is usually only slightly short), then geometric growth up
    // to 256 per poll (cold solves, or a solve that needs many more iterations than the previous one)
    ++polls;
    if (its_hint > 0 && polls == 1) batch = follow;
    else batch = batch < 128 ? batch * 2 : 256;
  }
  if (shard_x_active(cg) && !cg->h_ctl->skip) {
    // sharded-x mode: every rank owns a slice of x; all ranks need all of it for the back-substitution
    std::vector<int> xoff((size_t)cg->nranks + 1);
    for (int q = 0; q <= cg->nranks; ++q) xoff[(size_t)q] = (int)((long long)n * q / cg->nranks);
    if (b200_allgatherv(d_b, xoff.data()) != 0) return -1;
  }
  // y = R_y^{-1} (A x - r_y)   (private.c:313-317)
  if (cg->nranks > 1) {
    B200SpmvArgs a;
    memset(&a, 0, sizeof(a));
    double *yl = d_b + n + cg->row0;
    a.d_x = d_b; a.d_y = yl; a.d_init = yl; a.init_sign = -1.0; a.post = B200_POST_DIV;
    a.d_d = cg->d_ry + cg->row0; a.d_skip = d_skip;
    if (b200_spmv(cg->A, &a) != 0) return -1;
    if (b200_allgatherv(d_b + n, cg->offsets) != 0) return -1;
  } else {
    B200SpmvArgs a;
    memset(&a, 0, sizeof(a));
    a.d_x = d_b; a.d_y = d_b + n; a.d_init = d_b + n; a.init_sign = -1.0; a.post = B200_POST_DIV;
    a.d_d = cg->d_ry; a.d_v = nullptr; a.d_dot = nullptr; a.hook = B200_HOOK_NONE;
    a.d_hook_arg = nullptr; a.d_skip = d_skip;
    if (b200_spmv(cg->A, &a) != 0) return -1;
  }
  if (cg->h_ctl->skip) {
    k_zero_if<<<vec_grid((long long)n + m), 256, 0, st>>>((long long)n + m, d_b, d_skip);
    b200_count_launch(1);
  }
  CUDA_OK(cudaGetLastError());
  return cg->h_ctl->iters;
}

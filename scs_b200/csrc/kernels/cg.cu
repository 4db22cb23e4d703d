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
// Up to n = 2 SMs * 4096 (single GPU), K3 and K4 run as one kernel, k_cg_update_p, that keeps z and p in registers
// across a grid barrier: 3 kernels per iteration, z never stored. There, with the reordered pair and P = 0, a whole
// batch of iterations runs as one cooperative kernel, k_cg_batch, with the three as phases behind grid barriers.
// Algorithmic bytes: 24 nnz + 4 (m+n+2) + 24 m + 120 n; 96 n instead of 120 n fused   (DESIGN.md).
#include "../common.cuh"
#include "../dev_api.h"
#include "../spmv_flag.cuh"
#include <atomic>
#include <mutex>
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

// K3 + K4 as one pass, for n <= 2 SMs * 4096 (cg_plan_k34): K3's grid is then not capped, so every thread of it
// covers at most CG_FUSED_V2 double2 elements and can keep their z and p in registers across the beta dependency.
//   phase 1  k_cg_update over the same grid: the same elements in the same order, the same cg_update_elem, the same
//            block_sum / block_max / grid_finish slots and ticket, so z'r, ||r||_inf and beta are the same bits. z is
//            never stored. The last block writes the control block as K3 does, then releases a grid barrier by storing
//            ctl->iters last; every other block spins on iters (read before its ticket, so it cannot see the new value
//            too early).
//   phase 2  k_cg_pupdate from the registers: p = z + beta p unless the stop test fired.
// The barrier needs every block resident at once (checked at setup). The next K1 may take SM resources only after
// the barrier has released: pdl_launch_dependents() before it could hand a block's SM slot to K1 while that block is
// still to be scheduled, and the resident blocks would spin for ever. The spin gives up after ~1.5 s and raises the
// sticky ctl->pad[0] (the host fails the solve). stamps (timing runs only, else NULL): block 0's %globaltimer at entry
// and at the release, and the latest block end (atomicMax), in ns.
#define CG_FUSED_V2 4
__device__ __forceinline__ unsigned long long cg_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__global__ void __launch_bounds__(VEC_THREADS, 2)
k_cg_update_p(int n, double *__restrict__ x, double *__restrict__ r, double *__restrict__ p,
              const double *__restrict__ Gp, const double *__restrict__ M, B200CgCtl *ctl, double *partials,
              unsigned int *counter, unsigned long long *stamps) {
  if (stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0) stamps[0] = cg_globaltimer();
  pdl_wait();  // K2 (Gp, alpha) complete and visible
  if (ctl->done) return;
  __shared__ double s_red[128];
  __shared__ double s_beta;
  __shared__ int s_done;
  const double alpha = ctl->alpha;
  const double nalpha = -alpha;
  const int iters0 = *((volatile int *)&ctl->iters);  // before this block's ticket: the last block bumps it after
  double acc0 = 0.0, acc1 = 0.0;
  const int n2 = n >> 1;
  double2 *x2 = reinterpret_cast<double2 *>(x), *r2 = reinterpret_cast<double2 *>(r),
          *p2 = reinterpret_cast<double2 *>(p);
  const double2 *g2 = reinterpret_cast<const double2 *>(Gp), *m2 = reinterpret_cast<const double2 *>(M);
  const int stride = gridDim.x * blockDim.x;
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x;
  // K3 visits i0, i0 + stride, ... in increasing order (pairs, then the remainder): so does this loop
  double2 zk[CG_FUSED_V2], pk[CG_FUSED_V2];
#pragma unroll
  for (int k = 0; k < CG_FUSED_V2; ++k) {
    const int i = i0 + k * stride;
    if (i < n2) {
      double2 xa = x2[i], ra = r2[i], pa = p2[i], ga = g2[i], ma = m2[i], za;
      cg_update_elem(alpha, nalpha, xa.x, ra.x, pa.x, ga.x, ma.x, za.x, acc0, acc1);
      cg_update_elem(alpha, nalpha, xa.y, ra.y, pa.y, ga.y, ma.y, za.y, acc0, acc1);
      x2[i] = xa; r2[i] = ra;
      zk[k] = za; pk[k] = pa;
    }
  }
  const bool tail = (n & 1) && blockIdx.x == 0 && threadIdx.x == 0;
  double zt = 0.0, pt = 0.0;
  if (tail) {
    const int k = n - 1;
    double xv = x[k], rv = r[k];
    pt = p[k];
    cg_update_elem(alpha, nalpha, xv, rv, pt, Gp[k], M[k], zt, acc0, acc1);
    x[k] = xv; r[k] = rv;
  }
  double sm[1] = {acc0}, mx[1] = {acc1};
  block_sum<1>(sm, s_red);
  block_max<1>(mx, s_red + 64);
  double both[2] = {sm[0], mx[0]};
  if (grid_finish<2>(both, partials, counter, 2u, s_red)) {
    if (threadIdx.x == 0) {
      // k_cg_update's last block, with iters stored last: it releases the barrier
      const double ztr_prev = ctl->ztr;
      const int iters = iters0 + 1;
      int done = 0;
      double beta = 0.0;
      ctl->ztr_prev = ztr_prev;
      ctl->ztr = both[0];
      ctl->rnorm = both[1];
      if (both[1] < ctl->tol) {
        done = 1;
      } else if (ztr_prev == 0.0) {
        done = 1;
      } else {
        beta = both[0] / ztr_prev;
        ctl->beta = beta;
        if (iters >= ctl->max_its) done = 1;
      }
      if (done) ctl->done = 1;
      __threadfence();
      *((volatile int *)&ctl->iters) = iters;
      s_done = done;
      s_beta = beta;
    }
  } else if (threadIdx.x == 0) {
    const volatile int *vit = (const volatile int *)&ctl->iters;
    const long long t0 = clock64();
    bool released = true;
    while (*vit == iters0) {
      if (*((volatile int *)&ctl->pad[0]) || clock64() - t0 > 3000000000LL) {
        ctl->pad[0] = 1;
        released = false;
        break;
      }
    }
    __threadfence();  // acquire side: the last block's control-block stores precede its store of iters
    s_done = released ? *((volatile int *)&ctl->done) : 1;  // after a timeout p is left alone
    s_beta = *((volatile double *)&ctl->beta);
  }
  __syncthreads();
  pdl_launch_dependents();  // every block has arrived: the next K1 may take SM resources now
  if (stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0) stamps[1] = cg_globaltimer();
  if (!s_done) {
    const double beta = s_beta;
#pragma unroll
    for (int k = 0; k < CG_FUSED_V2; ++k) {
      const int i = i0 + k * stride;
      if (i < n2) {
        double2 pa = pk[k];
        pa.x = fma(beta, pa.x, zk[k].x); pa.y = fma(beta, pa.y, zk[k].y);
        p2[i] = pa;
      }
    }
    if (tail) p[n - 1] = fma(beta, pt, zt);
  }
  if (stamps != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(stamps + 2, cg_globaltimer());
  }
}


// ---------------------------------------------------------------------------
// A batch of CG iterations as ONE cooperative kernel (single GPU, the reordered pair, P = 0): k_cg_batch runs up to
// `iters` iterations, each as three phases behind grid barriers instead of three launches:
//   K1      tmp = R_y^-1 A_cg p    A_cg's partition, warp-tiles and lanes (spmv3_consume_stage): the same row sums
//   K2      Gp = R_x p + At_cg' tmp, p'Gp over At_cg's CTAs with its slots and ticket, the last one writes alpha
//   update  k_cg_update_p on k34_grid(n) VIRTUAL blocks of VEC_THREADS threads: CTA c runs virtual blocks c and c + G,
//           virtual warp w of them (w < 32) on real warp w % 24, lane for lane. The same elements in the same order,
//           cg_update_elem, the warp trees of block_sum / block_max, the slots and the finish of grid_finish over the
//           virtual grid: z'r, ||r||_inf and beta are the same bits. z and p wait for beta in the ring's shared
//           memory (CG_BATCH_ZP_BYTES; k34_fused bounds n so that they fit).
// A grid barrier (cg_grid_sync) follows K1 and another the p update. After K2 and after the update's reductions the
// CTAs wait instead for the release of the last one to finish the reduction (cg_flag_wait): it stores a new value into
// a word every CTA read at the start of the iteration, after alpha, resp. the control block, so one round of atomics
// (the tickets) serves both the reduction and the synchronisation. Every CTA reads `done` after the wait that follows
// the update's finish and leaves the loop when it is set, so iterations past the stop cost nothing. Within one launch p and tmp are rewritten between phases: every read of them is a weak load after the
// acquire that precedes the phase (spmv3_consume_stage<.., NC = false>), never the non-coherent path. The first ring stages of K2
// and of the next iteration's K1 are issued before the barrier that precedes them (matrix streams are never written). The grid is co-resident (cooperative
// launch, checked at setup) and runs only under the K34 token. stamps (timing runs only, else NULL): block 0's
// %globaltimer at the start of every iteration and after each of its four barriers or waits, 5 per iteration.
#define CG_BATCH_VW (2 * VEC_THREADS / 32)  // virtual warps per CTA
#define CG_BATCH_ZP_BYTES (2 * CG_BATCH_VW * CG_FUSED_V2 * 32 * 16)
struct B200CgBatchArgs {
  double *x, *r, *p, *Gp, *tmp;
  const double *M;
  const double *d1;       // K1's 1 / R_y (vector or table), dmask1 its row mask for B200_D_TWO
  const unsigned *dmask1;
  int dform1;
  const double *d2;       // K2's R_x (vector or table)
  int dform2;
  B200CgCtl *ctl;
  double *partials;       // the update's slots and ticket
  unsigned *counter;
  unsigned *bar;          // the grid barrier's word
  int *seq;               // released by K2's finish (a new value every iteration)
  int g34;                // virtual blocks of the update
  unsigned long long *stamps;
};

// grid barrier over the co-resident grid: block 0 adds 2^31 - (G - 1), every other block 1, so the top bit flips once
// all have arrived and the low bits are 0 again (the word needs no reset between barriers or launches). The arrival is
// a release at gpu scope (after __syncthreads, so it orders the whole CTA's stores), the spin an acquire (which also
// invalidates the SM's L1; __syncthreads then orders the CTA's later loads after it). Gives up after ~1.5 s and raises
// the sticky ctl->pad[0]; returns 0 then (uniform over the CTA). `between` runs in thread 0 after its arrival, before
// it waits: work that must follow the CTA's __syncthreads but need not delay the other CTAs.
struct CgNothing {
  __device__ void operator()() const {}
};
template <typename F = CgNothing>
__device__ __forceinline__ int cg_grid_sync(unsigned *bar, B200CgCtl *ctl, int *s_ok, F between = F()) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned add = blockIdx.x == 0 ? 0x80000000u - (gridDim.x - 1) : 1u;
    unsigned old;
    asm volatile("atom.add.release.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(bar), "r"(add) : "memory");
    between();
    const long long t0 = clock64();
    int ok = 1;
    for (;;) {
      unsigned cur;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(cur) : "l"(bar) : "memory");
      if ((cur ^ old) & 0x80000000u) break;
      if (*((volatile int *)&ctl->pad[0]) || clock64() - t0 > 3000000000LL) {
        ctl->pad[0] = 1;
        ok = 0;
        break;
      }
    }
    *s_ok = ok;
  }
  __syncthreads();
  return *s_ok;
}
// the release side of cg_flag_wait: the finishing CTA's thread 0, after its stores of the results
__device__ __forceinline__ void cg_flag_release(int *word, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(word), "r"(v) : "memory");
}
__device__ __forceinline__ int cg_flag_load(const int *word) {
  int v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(word) : "memory");
  return v;
}
// thread 0 spins (acquire) until *word is no longer `old`, the value it read before the grid barrier that precedes
// the release (so it cannot see the new value too early, nor miss it: the next release needs this CTA at that barrier
// again). Same timeout as cg_grid_sync.
__device__ __forceinline__ int cg_flag_wait(const int *word, int old, B200CgCtl *ctl, int *s_ok) {
  if (threadIdx.x == 0) {
    const long long t0 = clock64();
    int ok = 1;
    for (;;) {
      int cur;
      asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(cur) : "l"(word) : "memory");
      if (cur != old) break;
      if (*((volatile int *)&ctl->pad[0]) || clock64() - t0 > 3000000000LL) {
        ctl->pad[0] = 1;
        ok = 0;
        break;
      }
    }
    *s_ok = ok;
  }
  __syncthreads();
  return *s_ok;
}

// producer: stages [from, to) of this CTA's share of op, stage i at ring position ring + i
template <bool IDX24>
__device__ __forceinline__ void cg_batch_produce(const B200FlagView &op, const Spmv3Ring &R, int ring, int from, int to,
                                                 uint64_t pol) {
  if (from >= to) return;
  const int4 *g = op.wt + (size_t)op.cta_begin[blockIdx.x] * SPMV3_NCW;
  for (int i = from; i < to; ++i) {
    const int q = ring + i, st = q % SPMV3_STAGES, use = q / SPMV3_STAGES;
    const int ka = __ldg(&g[(size_t)i * SPMV3_NCW].y) & ~3;
    const int4 l = __ldg(&g[(size_t)(i + 1) * SPMV3_NCW - 1]);
    const int cnt = (l.y + l.z - ka + 3) & ~3;
    if (use > 0) mbar_wait(&R.empty[st], (unsigned)((use - 1) & 1));
    spmv3_issue_stage<IDX24>(R, st, g, i, ka, cnt, op.idx, op.vals, pol);
  }
}
// one product as a phase: this CTA's nt stages of op from ring position `ring` (the first `pre` of them were issued by
// the previous phase), then the first ring round of the next phase (nt_next stages of next)
template <int POST, bool IDX24, bool NEXT_IDX24>
__device__ __forceinline__ void cg_batch_spmv(const B200FlagView &op, int nt, int pre, const B200FlagView &next,
                                              int nt_next, int &ring, const Spmv3Ring &R, const Spmv3Epi &E,
                                              double &dot_acc) {
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (wid == 0) {
    if (lane == 0) {
      const uint64_t pol = l2_policy_evict_first();
      cg_batch_produce<IDX24>(op, R, ring, pre, nt, pol);
      cg_batch_produce<NEXT_IDX24>(next, R, ring + nt, 0, nt_next < SPMV3_STAGES ? nt_next : SPMV3_STAGES, pol);
    }
  } else {
    for (int i = 0; i < nt; ++i) {
      const int q = ring + i;
      spmv3_consume_stage<POST, IDX24, false>(R, q % SPMV3_STAGES, (unsigned)((q / SPMV3_STAGES) & 1), wid - 1, lane,
                                              E, dot_acc);
    }
  }
  ring += nt;
}

template <bool PK1, bool PK2>
__global__ void __launch_bounds__(SPMV3_THREADS, 1)
k_cg_batch(int n, int iters, B200FlagView A, B200FlagView At, B200CgBatchArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t s_mbar[2 * SPMV3_STAGES];
  __shared__ double s_red[64];
  __shared__ double s_ws[CG_BATCH_VW], s_wm[CG_BATCH_VW];  // per virtual warp: warp_sum of z'r, warp_max of |r|
  __shared__ double s_tail[2], s_beta;
  __shared__ int s_ok, s_flag;
  double *s_vals = reinterpret_cast<double *>(smem_raw);
  int *s_idx = reinterpret_cast<int *>(s_vals + SPMV3_STAGES * SPMV3_CAP);
  int4 *s_desc = reinterpret_cast<int4 *>(s_idx + SPMV3_STAGES * SPMV3_CAP);
  double *s_out = reinterpret_cast<double *>(s_desc + SPMV3_STAGES * SPMV3_NCW);
  const Spmv3Ring R = {s_vals, s_idx, s_desc, s_mbar, s_mbar + SPMV3_STAGES, s_out};
  // the update's z and p, [virtual warp][k][lane], over the ring (every stage has been consumed by then)
  double2 *s_z = reinterpret_cast<double2 *>(smem_raw);
  double2 *s_p = s_z + CG_BATCH_VW * CG_FUSED_V2 * 32;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, b = blockIdx.x, G = gridDim.x;
  volatile B200CgCtl *c = a.ctl;
  if (tid == 0) {
    for (int s = 0; s < SPMV3_STAGES; ++s) {
      mbar_init(&R.full[s], 1);
      mbar_init(&R.empty[s], SPMV3_NCW);
    }
    mbar_fence_init();
    s_flag = c->done;
  }
  __syncthreads();
  if (s_flag) return;
  const int nt1 = b < A.grid ? A.cta_begin[b + 1] - A.cta_begin[b] : 0;
  const int nt2 = b < At.grid ? At.cta_begin[b + 1] - At.cta_begin[b] : 0;
  Spmv3Epi E1 = {a.p, a.tmp, nullptr, 1.0, a.d1, a.dmask1, a.dform1, 0.0, 0.0, nullptr, false, nullptr, nullptr, 0ull};
  Spmv3Epi E2 = {a.tmp, a.Gp, nullptr, 1.0, a.d2, nullptr, a.dform2, 0.0, 0.0, a.p, false, nullptr, nullptr, 0ull};
  if (a.dform1 != B200_D_VEC) {
    E1.dt0 = a.d1[0];
    E1.dt1 = a.dform1 == B200_D_TWO ? a.d1[1] : E1.dt0;
  }
  if (a.dform2 != B200_D_VEC) E2.dt0 = E2.dt1 = a.d2[0];
  const int g34 = a.g34, n2 = n >> 1, stride = g34 * VEC_THREADS;
  double2 *x2 = reinterpret_cast<double2 *>(a.x), *r2 = reinterpret_cast<double2 *>(a.r),
          *p2 = reinterpret_cast<double2 *>(a.p);
  const double2 *g2 = reinterpret_cast<const double2 *>(a.Gp), *m2 = reinterpret_cast<const double2 *>(a.M);
  unsigned long long *stamp = (a.stamps != nullptr && b == 0 && tid == 0) ? a.stamps : nullptr;
  int ring = 0;
  for (int it = 0; it < iters; ++it) {
    if (stamp) stamp[5 * it] = cg_globaltimer();
    // the words the two finishes release this iteration, as they are before the K1 -> K2 barrier (thread 0 only)
    const int seq0 = tid == 0 ? cg_flag_load(a.seq) : 0;
    const int its0 = tid == 0 ? cg_flag_load(&a.ctl->iters) : 0;
    double dot = 0.0;
    // ---- K1, then K2's first ring round
    const int pre1 = it > 0 ? (nt1 < SPMV3_STAGES ? nt1 : SPMV3_STAGES) : 0;  // issued before the last barrier
    cg_batch_spmv<B200_POST_MUL, PK1, PK2>(A, nt1, pre1, At, nt2, ring, R, E1, dot);
    if (!cg_grid_sync(a.bar, a.ctl, &s_ok)) return;
    if (stamp) stamp[5 * it + 1] = cg_globaltimer();
    // ---- K2 and its dot product; the last of At's CTAs writes alpha (spmv_tail, B200_HOOK_CG_ALPHA)
    cg_batch_spmv<B200_POST_FMA_DOT, PK2, PK2>(At, nt2, nt2 < SPMV3_STAGES ? nt2 : SPMV3_STAGES, At, 0, ring, R, E2,
                                               dot);
    if (b < At.grid) {
      double acc[1] = {dot};
      block_sum<1>(acc, s_red);
      if (grid_finish_of<1>(acc, At.partials, At.counter, 0u, s_red, (unsigned)At.grid, (unsigned)b)) {
        if (tid == 0) {
          c->pGp = acc[0];
          c->alpha = c->ztr / acc[0];
          cg_flag_release(a.seq, seq0 + 1);
        }
      }
    }
    // At's CTAs stored Gp and took their tickets before the release; the update reads Gp and alpha after it
    if (!cg_flag_wait(a.seq, seq0, a.ctl, &s_ok)) return;
    if (stamp) stamp[5 * it + 2] = cg_globaltimer();
    // ---- update, first half (k_cg_update_p up to its barrier) on the virtual blocks
    const double alpha = c->alpha, nalpha = -alpha;
    for (int vw = wid; vw < CG_BATCH_VW; vw += SPMV3_THREADS / 32) {
      const int v = b + (vw >> 4) * G;
      double acc0 = 0.0, acc1 = 0.0;
      if (v < g34) {
        const int i0 = v * VEC_THREADS + (vw & 15) * 32 + lane;
#pragma unroll
        for (int k = 0; k < CG_FUSED_V2; ++k) {
          const int i = i0 + k * stride;
          if (i < n2) {
            double2 xa = x2[i], ra = r2[i], pa = p2[i], ga = g2[i], ma = m2[i], za;
            cg_update_elem(alpha, nalpha, xa.x, ra.x, pa.x, ga.x, ma.x, za.x, acc0, acc1);
            cg_update_elem(alpha, nalpha, xa.y, ra.y, pa.y, ga.y, ma.y, za.y, acc0, acc1);
            x2[i] = xa; r2[i] = ra;
            s_z[(vw * CG_FUSED_V2 + k) * 32 + lane] = za;
            s_p[(vw * CG_FUSED_V2 + k) * 32 + lane] = pa;
          }
        }
        if ((n & 1) && v == 0 && vw == 0 && lane == 0) {  // k_cg_update_p's tail: block 0, thread 0, last
          const int k = n - 1;
          double xv = a.x[k], rv = a.r[k], zt;
          const double pt = a.p[k];
          cg_update_elem(alpha, nalpha, xv, rv, pt, a.Gp[k], a.M[k], zt, acc0, acc1);
          a.x[k] = xv; a.r[k] = rv;
          s_tail[0] = zt;
          s_tail[1] = pt;
        }
      }
      acc0 = warp_sum(acc0);
      acc1 = warp_max(acc1);
      if (lane == 0) {
        s_ws[vw] = acc0;
        s_wm[vw] = acc1;
      }
    }
    __syncthreads();
    // block_sum / block_max's second stage for each virtual block (16 warps), into its slots of grid_finish<2>
    if (wid < 2 && b + wid * G < g34) {
      const double t = warp_sum(lane < 16 ? s_ws[wid * 16 + lane] : 0.0);
      const double u = warp_max(lane < 16 ? s_wm[wid * 16 + lane] : 0.0);
      if (lane == 0) {
        a.partials[b + wid * G] = t;
        a.partials[g34 + b + wid * G] = u;
      }
    }
    __syncthreads();
    if (tid == 0) {
      const unsigned mine = (unsigned)(b < g34) + (unsigned)(b + G < g34);
      int last = 0;
      if (mine) {  // release of this CTA's slots, acquire of the others' for the finish
        unsigned t;
        asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(t) : "l"(a.counter), "r"(mine) : "memory");
        last = t + mine == (unsigned)g34;
      }
      s_flag = last;
    }
    __syncthreads();
    if (s_flag) {
      // grid_finish<2> over the g34 virtual blocks: thread t < VEC_THREADS takes slot t; the threads beyond a virtual
      // block's VEC_THREADS hold exact zeros, which leave block_sum's and block_max's trees as they are
      double s[1] = {0.0}, m[1] = {0.0};
      if (tid < g34) {
        s[0] = s[0] + __ldcg(&a.partials[tid]);
        m[0] = fmax(m[0], __ldcg(&a.partials[g34 + tid]));
      }
      block_sum<1>(s, s_red);
      block_max<1>(m, s_red);
      if (tid == 0) {
        // k_cg_update_p's last block
        const double ztr_prev = c->ztr;
        const int its = its0 + 1;
        int done = 0;
        c->ztr_prev = ztr_prev;
        c->ztr = s[0];
        c->rnorm = m[0];
        if (m[0] < c->tol) {
          done = 1;
        } else if (ztr_prev == 0.0) {
          done = 1;
        } else {
          c->beta = s[0] / ztr_prev;
          if (its >= c->max_its) done = 1;
        }
        if (done) c->done = 1;
        *a.counter = 0u;
        cg_flag_release(&a.ctl->iters, its);  // last: it releases the other CTAs (k_cg_update_p stores iters last too)
      }
    }
    if (!cg_flag_wait(&a.ctl->iters, its0, a.ctl, &s_ok)) return;
    if (stamp) stamp[5 * it + 3] = cg_globaltimer();
    // ---- update, second half: p = z + beta p unless the stop test fired
    if (tid == 0) {
      s_flag = c->done;
      s_beta = c->beta;
    }
    __syncthreads();
    if (s_flag) return;
    const double beta = s_beta;
    for (int vw = wid; vw < CG_BATCH_VW; vw += SPMV3_THREADS / 32) {
      const int v = b + (vw >> 4) * G;
      if (v >= g34) continue;
      const int i0 = v * VEC_THREADS + (vw & 15) * 32 + lane;
#pragma unroll
      for (int k = 0; k < CG_FUSED_V2; ++k) {
        const int i = i0 + k * stride;
        if (i < n2) {
          double2 pa = s_p[(vw * CG_FUSED_V2 + k) * 32 + lane];
          const double2 za = s_z[(vw * CG_FUSED_V2 + k) * 32 + lane];
          pa.x = fma(beta, pa.x, za.x); pa.y = fma(beta, pa.y, za.y);
          p2[i] = pa;
        }
      }
      if ((n & 1) && v == 0 && vw == 0 && lane == 0) a.p[n - 1] = fma(beta, s_tail[1], s_tail[0]);
    }
    // the next K1's first ring round overwrites what z and p occupied in this CTA: after every thread's last read of
    // them, a proxy fence and the barrier's __syncthreads, thread 0 issues it between its arrival and its wait (A_cg's
    // stream is never written)
    fence_proxy_async();
    const int pre_next = it + 1 < iters ? (nt1 < SPMV3_STAGES ? nt1 : SPMV3_STAGES) : 0;
    const int ring_now = ring;
    auto prefetch = [&] {
      if (pre_next > 0) cg_batch_produce<PK1>(A, R, ring_now, 0, pre_next, l2_policy_evict_first());
    };
    if (!cg_grid_sync(a.bar, a.ctl, &s_ok, prefetch)) {
      if (tid == 0)  // the stages in flight land before the CTA exits
        for (int i = 0; i < pre_next; ++i) mbar_wait(&R.full[(ring + i) % SPMV3_STAGES], ((ring + i) / SPMV3_STAGES) & 1);
      return;
    }
    if (stamp) stamp[5 * it + 4] = cg_globaltimer();
  }
}
// dynamic shared memory: the ring (stages, descriptors, warp scratch; its barriers are static) or z and p, the larger
#define CG_BATCH_RING_BYTES \
  ((size_t)SPMV3_STAGES * (SPMV3_CAP * 12 + SPMV3_NCW * 16) + (size_t)SPMV3_NCW * SPMV3_WT * 8)
#define CG_BATCH_SMEM (CG_BATCH_RING_BYTES > CG_BATCH_ZP_BYTES ? CG_BATCH_RING_BYTES : CG_BATCH_ZP_BYTES)
typedef void (*CgBatchFn)(int, int, B200FlagView, B200FlagView, B200CgBatchArgs);
static CgBatchFn cg_batch_fn(bool packed1, bool packed2) {
  return packed1 ? (packed2 ? k_cg_batch<true, true> : k_cg_batch<true, false>)
                 : (packed2 ? k_cg_batch<false, true> : k_cg_batch<false, false>);
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
// Row operands of the reordered pair as tables. SCS sets R_y to two values (zero-cone rows and the rest) and R_x to
// one, so K1 and K2 need not stream a row vector for them. The table holds k_recip's own results, so the products
// are the same bits as with d_ry_cg / d_rx. Values are compared by their bits.
__global__ void k_diag_tab_init(const int *__restrict__ perm, const double *__restrict__ ry_inv,
                                const double *__restrict__ rx, double *__restrict__ tab, unsigned *mixed) {
  tab[0] = tab[1] = ry_inv[perm[0]];
  tab[2] = rx[0];
  *mixed = 0u;
}
// bit r of mask: 1/R_y of row r of A_cg is not tab[0]. The first other value claims tab[1]; a third one sets bit 0 of
// *mixed, an R_x that is not tab[2] bit 1.
__global__ void k_diag_tab_classify(int kept, int n, const int *__restrict__ perm, const double *__restrict__ ry_inv,
                                    const double *__restrict__ rx, double *tab, unsigned *mask, unsigned *mixed) {
  const unsigned FULL = 0xffffffffu;
  const unsigned long long b0 = (unsigned long long)__double_as_longlong(tab[0]);
  const unsigned long long x0 = (unsigned long long)__double_as_longlong(tab[2]);
  unsigned long long *b1 = reinterpret_cast<unsigned long long *>(tab + 1);
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  unsigned mx = 0u;
  for (long long base = warp * 32; base < kept; base += nwarps * 32) {  // warp-uniform
    const long long r = base + lane;
    const unsigned long long b = r < kept ? (unsigned long long)__double_as_longlong(ry_inv[perm[r]]) : b0;
    const unsigned w = __ballot_sync(FULL, b != b0);
    if (lane == 0) mask[base >> 5] = w;
    if (w != 0u) {
      const unsigned long long bl = __shfl_sync(FULL, b, __ffs(w) - 1);
      if (b != b0 && b != bl) mx |= 1u;
      if (lane == 0) {
        unsigned long long cur = *(volatile unsigned long long *)b1;
        if (cur == b0) {
          cur = atomicCAS(b1, b0, bl);
          if (cur == b0) cur = bl;
        }
        if (cur != bl) mx |= 1u;
      }
    }
  }
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x)
    if ((unsigned long long)__double_as_longlong(rx[j]) != x0) mx |= 2u;
  if (mx) atomicOr(mixed, mx);
}

extern "C" int b200_cg_classify_diag(B200Cg *cg, const int *d_perm) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int kept = b200_spmv_nrows(cg->A_cg);
  unsigned mixed = 3u;
  k_diag_tab_init<<<1, 1, 0, st>>>(d_perm, cg->d_ry_inv, cg->d_rx, cg->d_diag_tab, cg->d_diag_mixed);
  k_diag_tab_classify<<<vec_grid((long long)kept + cg->n), 256, 0, st>>>(kept, cg->n, d_perm, cg->d_ry_inv, cg->d_rx,
                                                                        cg->d_diag_tab, cg->d_ry_mask,
                                                                        cg->d_diag_mixed);
  b200_count_launch(2);
  if (b200_d2h(&mixed, cg->d_diag_mixed, 4) != 0 || b200_sync() != 0) return -1;
  cg->ry_form = (mixed & 1u) ? B200_D_VEC : B200_D_TWO;
  cg->rx_form = (mixed & 2u) ? B200_D_VEC : B200_D_ONE;
  return 0;
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

// peer-memory reduction: 0 = automatic (one pass for 2 ranks, two-phase for more), 1 = one pass, 2 = two-phase
static std::atomic<int> g_p2p_mode{-1};  // read by every solving thread: atomic
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

// K1's and K2's row operands: 1 / R_y and R_x, from the tables when the reordered pair has them (the plain pair: the
// vectors). Sets d_d / dform / d_dmask.
static void k1_operand(const B200Cg *cg, bool re, B200SpmvArgs &a) {
  a.dform = re ? cg->ry_form : B200_D_VEC;
  a.d_d = a.dform == B200_D_TWO ? cg->d_diag_tab : re ? cg->d_ry_cg : cg->d_ry_inv;
  a.d_dmask = a.dform == B200_D_TWO ? cg->d_ry_mask : nullptr;
}
static void k2_operand(const B200Cg *cg, bool re, B200SpmvArgs &a) {
  a.dform = re ? cg->rx_form : B200_D_VEC;
  a.d_d = a.dform == B200_D_ONE ? cg->d_diag_tab + 2 : cg->d_rx;
  a.d_dmask = nullptr;
}

static int mat_vec(B200Cg *cg, const double *d_x, double *d_y, int with_dot, const int *d_skip) {
  if (cg->nranks > 1) return mat_vec_sharded(cg, d_x, d_y, with_dot, d_skip);
  // the m-space-reordered pair when present: tmp is internal to the operator, so its ordering is free
  const bool re = cg->A_cg != nullptr && cg->At_cg != nullptr && cg->d_ry_cg != nullptr;
  const B200Spmv *A = re ? cg->A_cg : cg->A, *At = re ? cg->At_cg : cg->At;
  B200SpmvArgs a;
  memset(&a, 0, sizeof(a));
  // K1: tmp = (A x) ./ R_y; every kernel of the CG loop is a programmatic dependent of its predecessor
  a.pdl = 1;
  a.d_x = d_x; a.d_y = cg->d_tmp; a.d_init = nullptr; a.init_sign = 1.0;
  a.post = B200_POST_MUL; a.d_v = nullptr; a.d_dot = nullptr;
  k1_operand(cg, re, a);
  a.hook = B200_HOOK_NONE; a.d_hook_arg = nullptr; a.d_skip = d_skip;
  if (b200_spmv(A, &a) != 0) return -1;
  const double *init = nullptr;
  if (cg->P) {
    // y = P x first (reference accumulates P x before A' z)
    a.d_x = d_x; a.d_y = d_y; a.d_init = nullptr; a.post = B200_POST_NONE;
    a.d_d = nullptr; a.dform = B200_D_VEC; a.d_dmask = nullptr; a.d_v = nullptr;
    if (b200_spmv(cg->P, &a) != 0) return -1;
    init = d_y;
  }
  // K2: y = fma(R_x, x, init + A' tmp)
  a.d_x = cg->d_tmp; a.d_y = d_y; a.d_init = init; a.init_sign = 1.0;
  a.post = with_dot ? B200_POST_FMA_DOT : B200_POST_FMA;
  k2_operand(cg, re, a);
  a.d_v = d_x; a.d_dot = with_dot ? &cg->d_ctl->pGp : nullptr;
  a.hook = with_dot ? B200_HOOK_CG_ALPHA : B200_HOOK_NONE;
  a.d_hook_arg = cg->d_ctl; a.d_skip = d_skip;
  return b200_spmv(At, &a);
}

// sharded-x push mode (see k_cgx_iteration): -1 = read SCS_B200_SHARD_X once (default ON; =0 selects the replicated
// modes), 0 = off, 1 = on
static std::atomic<int> g_shard_x{-1};
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
  a.pdl = 1;
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
  CUDA_OK(b200_launch(k_cgx_iteration, dim3(g), dim3(VEC_THREADS), 0, st, true, cg->n, pv, seq,
                      (int)(cg->P != nullptr), (const double *)cg->d_rx, (const double *)cg->d_M, cg->d_p, cg->d_Gp,
                      d_x, cg->d_r, cg->d_z, cg->d_ctl, cg->d_partials, cg->d_counter));
  if (ev) cudaEventRecord(ev[3], st);
  b200_count_launch(1);
  return 0;
}

// K3 / K4 grid (also the fused kernel's): 8 doubles per thread, at most 2 blocks of VEC_THREADS per SM
static int k34_grid(int n) {
  int g = (n + VEC_THREADS * 8 - 1) / (VEC_THREADS * 8);
  if (g > 2 * b200_num_sms()) g = 2 * b200_num_sms();
  if (g < 1) g = 1;
  return g;
}

extern "C" int b200_cg_plan_k34(B200Cg *cg) {
  cg->k34_fused = 0;
  if (cg->nranks > 1) return 0;
  // uncapped grid: each thread holds at most CG_FUSED_V2 double2 of z and p
  if ((long long)cg->n > 2LL * b200_num_sms() * VEC_THREADS * 2 * CG_FUSED_V2) return 0;
  int per_sm = 0;
  CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cg_update_p, VEC_THREADS, 0));
  cg->k34_fused = (long long)per_sm * b200_num_sms() >= k34_grid(cg->n) ? 1 : 0;
  // the batch kernel: one CTA per SM must fit, and the device must take cooperative launches
  cg->k34_batch = 0;
  if (!cg->k34_fused) return 0;
  static std::once_flag once;
  std::call_once(once, [] {
    for (int k = 0; k < 4; ++k)
      cudaFuncSetAttribute(cg_batch_fn(k & 1, k & 2), cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)CG_BATCH_SMEM);
  });
  int dev = 0, coop = 0;
  CUDA_OK(cudaGetDevice(&dev));
  CUDA_OK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  int fit = coop;
  for (int k = 0; k < 4 && fit; ++k) {
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cg_batch_fn(k & 1, k & 2), SPMV3_THREADS,
                                                          CG_BATCH_SMEM));
    fit = per_sm >= 1;
  }
  cg->k34_batch = fit;
  return 0;
}

// SCS_B200_CG_BATCH_KERNEL=0 runs every CG iteration as its three kernels (A/B runs); read once
static std::atomic<int> g_cg_batch{-1};
extern "C" void scs_b200_set_cg_batch_kernel(int on) { g_cg_batch = on ? 1 : 0; }
static bool cg_batch_enabled() {
  if (g_cg_batch < 0) {
    const char *e = getenv("SCS_B200_CG_BATCH_KERNEL");
    g_cg_batch = (e && atoi(e) == 0) ? 0 : 1;
  }
  return g_cg_batch == 1;
}
// the views of the reordered pair when the batch kernel can run this workspace's CG loop
static bool cg_batch_ready(const B200Cg *cg, B200FlagView *A, B200FlagView *At) {
  return cg->k34_batch && cg->nranks == 1 && cg->P == nullptr && cg->A_cg != nullptr && cg->At_cg != nullptr &&
         cg->d_ry_cg != nullptr && b200_spmv_flag_view(cg->A_cg, A) == 0 && b200_spmv_flag_view(cg->At_cg, At) == 0;
}
static void k1_operand(const B200Cg *cg, bool re, B200SpmvArgs &a);
static void k2_operand(const B200Cg *cg, bool re, B200SpmvArgs &a);
// `iters` CG iterations as one cooperative launch of k_cg_batch; the caller holds the K34 token
static cudaError_t cg_batch_launch(B200Cg *cg, const B200FlagView &A, const B200FlagView &At, double *d_x, int iters,
                                   unsigned long long *stamps) {
  B200CgBatchArgs a;
  memset(&a, 0, sizeof(a));
  a.x = d_x; a.r = cg->d_r; a.p = cg->d_p; a.Gp = cg->d_Gp; a.tmp = cg->d_tmp; a.M = cg->d_M;
  B200SpmvArgs k;
  memset(&k, 0, sizeof(k));
  k1_operand(cg, true, k);
  a.d1 = k.d_d; a.dmask1 = k.d_dmask; a.dform1 = k.dform;
  k2_operand(cg, true, k);
  a.d2 = k.d_d; a.dform2 = k.dform;
  a.ctl = cg->d_ctl; a.partials = cg->d_partials; a.counter = cg->d_counter; a.bar = cg->d_counter + 8;
  a.seq = (int *)cg->d_counter + 9;
  a.g34 = k34_grid(cg->n);
  a.stamps = stamps;
  int grid = (a.g34 + 1) / 2;
  if (A.grid > grid) grid = A.grid;
  if (At.grid > grid) grid = At.grid;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(SPMV3_THREADS);
  cfg.dynamicSmemBytes = CG_BATCH_SMEM;
  cfg.stream = (cudaStream_t)b200_stream();
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, cg_batch_fn(A.packed != 0, At.packed != 0), cg->n, iters, A, At, a);
}

// fused: K3 and K4 as k_cg_update_p (the caller holds the token when its grid has more than one block)
static int cg_iteration(B200Cg *cg, double *d_x, bool fused) {
  if (shard_x_active(cg)) return cg_iteration_shard_x(cg, d_x);
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int n = cg->n;
  const int g = k34_grid(n);
  if (mat_vec(cg, cg->d_p, cg->d_Gp, 1, &cg->d_ctl->done) != 0) return -1;
  if (fused) {
    CUDA_OK(b200_launch(k_cg_update_p, dim3(g), dim3(VEC_THREADS), 0, st, true, n, d_x, cg->d_r, cg->d_p,
                        (const double *)cg->d_Gp, (const double *)cg->d_M, cg->d_ctl, cg->d_partials, cg->d_counter,
                        (unsigned long long *)nullptr));
    b200_count_launch(1);
    return 0;
  }
  CUDA_OK(b200_launch(k_cg_update, dim3(g), dim3(VEC_THREADS), 0, st, true, n, d_x, cg->d_r, (const double *)cg->d_p,
                      (const double *)cg->d_Gp, (const double *)cg->d_M, cg->d_z, cg->d_ctl, cg->d_partials,
                      cg->d_counter));
  CUDA_OK(b200_launch(k_cg_pupdate, dim3(g), dim3(VEC_THREADS), 0, st, true, n, cg->d_p, (const double *)cg->d_z,
                      (const B200CgCtl *)cg->d_ctl));
  b200_count_launch(2);
  return 0;
}

// timing only (bench.py): runs the path planned at setup without taking the token, so it must not overlap a solve of
// another thread
extern "C" int b200_cg_one_iteration(B200Cg *cg, double *d_x) { return cg_iteration(cg, d_x, cg->k34_fused != 0); }

// The fused kernel's grid barrier under concurrency (k_cg_batch's barriers likewise: it runs only under the token).
// k_cg_update_p needs all of its blocks resident at once; setup
// checks that against the whole GPU. Two such grids on two streams could each get part of the SMs and wait for each
// other until the spin gives up. So a KKT solve whose fused grid has more than one block runs it only while it holds
// this process-wide token, taken with a try-lock (never a wait) at the start of b200_cg_solve and given back once the
// host has seen the solve's stream drain -- also when the solve fails, so no fused launch it enqueued can still be
// waiting to run; without it the solve runs the pair k_cg_update + k_cg_pupdate,
// which computes the same bits (tests/test_cg_fused_gpu.py). A single-block grid has no barrier to wait at.
// The token lives in libscs_b200_token.so, which every library flavour links, so a process that loads several flavours
// (the int, DLONG and spectral builds) still has one token.
// Why this cannot deadlock: with the token, at most one spinning grid of this process is on the device (nranks > 1
// keeps one solve at a time per process; grids of other processes are outside the token). Every other resident block belongs to a kernel that does not wait for another grid, so it
// finishes and frees its slot. A PDL dependent -- in particular the next K1 behind the fused kernel on its own
// stream -- becomes resident only after every block of its predecessor has been scheduled, so it cannot take the slot
// a block of the spinning grid still needs. Hence every block of the fused grid is eventually resident and the
// barrier releases.
namespace {
struct K34Token {
  bool held = false;
  bool take() { return held = b200_k34_token_take() != 0; }
  // after the host has seen the stream drain
  void give_back() {
    if (held) b200_k34_token_give_back();
    held = false;
  }
  // an error return: the fused launches already enqueued must have run (or the stream have failed) first
  ~K34Token() {
    if (held) cudaStreamSynchronize((cudaStream_t)b200_stream());
    give_back();
  }
};
}  // namespace

// Per-kernel device times of the CG loop AS IT RUNS IN A SOLVE (bench.py roofline): `reps` genuine iterations on
// the solver's own p / tmp / r, every kernel bracketed by CUDA events on the library stream. out_ms[0..3] = average
// per launch of K1 (tmp = R_y^-1 A p, spmv POST_MUL), K2 (Gp = R_x p + A' tmp, p'Gp, alpha: spmv POST_FMA_DOT + hook),
// K3 (k_cg_update), K4 (k_cg_pupdate); out_ms[4] = whole iteration (first event to last, launch gaps included).
// With k34_fused, out_ms[2] / [3] are the two phases of k_cg_update_p from its globaltimer stamps: entry to the grid
// barrier's release (K3's work and reductions, the barrier) and release to the end of the last block (K4's stores).
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
  const int g = k34_grid(n);
  std::vector<cudaEvent_t> ev((size_t)reps * 5);
  for (auto &e : ev) e = nullptr;
  int rc = -1;
  bool ok = true;
  for (auto &e : ev)
    if (cudaEventCreate(&e) != cudaSuccess) ok = false;
  // fused K3 + K4: 3 globaltimer stamps per iteration (entry, release, end), see k_cg_update_p
  unsigned long long *d_stamps = nullptr;
  if (ok && cg->k34_fused) {
    d_stamps = (unsigned long long *)b200_malloc((size_t)reps * 3 * sizeof(unsigned long long));
    if (!d_stamps || cudaMemsetAsync(d_stamps, 0, (size_t)reps * 3 * sizeof(unsigned long long), st) != cudaSuccess)
      ok = false;
  }
  if (ok) {
    const int *d_skip = &cg->d_ctl->done;
    for (int r = 0; r < reps && ok; ++r) {
      B200SpmvArgs a;
      memset(&a, 0, sizeof(a));
      cudaEventRecord(ev[(size_t)r * 5 + 0], st);
      const bool re = cg->A_cg != nullptr && cg->At_cg != nullptr && cg->d_ry_cg != nullptr;
      a.d_x = cg->d_p; a.d_y = cg->d_tmp; a.init_sign = 1.0; a.post = B200_POST_MUL;
      k1_operand(cg, re, a);
      a.d_skip = d_skip;
      if (b200_spmv(re ? cg->A_cg : cg->A, &a) != 0) ok = false;
      cudaEventRecord(ev[(size_t)r * 5 + 1], st);
      a.d_x = cg->d_tmp; a.d_y = cg->d_Gp; a.post = B200_POST_FMA_DOT; a.d_v = cg->d_p;
      k2_operand(cg, re, a);
      a.d_dot = &cg->d_ctl->pGp; a.hook = B200_HOOK_CG_ALPHA; a.d_hook_arg = cg->d_ctl;
      if (b200_spmv(re ? cg->At_cg : cg->At, &a) != 0) ok = false;
      cudaEventRecord(ev[(size_t)r * 5 + 2], st);
      if (cg->k34_fused) {
        k_cg_update_p<<<g, VEC_THREADS, 0, st>>>(n, d_x, cg->d_r, cg->d_p, cg->d_Gp, cg->d_M, cg->d_ctl,
                                                 cg->d_partials, cg->d_counter, d_stamps + (size_t)r * 3);
        cudaEventRecord(ev[(size_t)r * 5 + 3], st);
        cudaEventRecord(ev[(size_t)r * 5 + 4], st);
        b200_count_launch(1);
      } else {
        k_cg_update<<<g, VEC_THREADS, 0, st>>>(n, d_x, cg->d_r, cg->d_p, cg->d_Gp, cg->d_M, cg->d_z, cg->d_ctl,
                                               cg->d_partials, cg->d_counter);
        cudaEventRecord(ev[(size_t)r * 5 + 3], st);
        k_cg_pupdate<<<g, VEC_THREADS, 0, st>>>(n, cg->d_p, cg->d_z, cg->d_ctl);
        cudaEventRecord(ev[(size_t)r * 5 + 4], st);
        b200_count_launch(2);
      }
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) ok = false;
  }
  std::vector<unsigned long long> h_stamps(d_stamps ? (size_t)reps * 3 : 0);
  if (ok && d_stamps &&
      cudaMemcpy(h_stamps.data(), d_stamps, h_stamps.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost) !=
          cudaSuccess)
    ok = false;
  if (ok) {
    for (int k = 0; k < 5; ++k) out_ms[k] = 0.0;
    for (int r = 0; r < reps; ++r) {
      for (int k = 0; k < (d_stamps ? 2 : 4); ++k) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[(size_t)r * 5 + k], ev[(size_t)r * 5 + k + 1]);
        out_ms[k] += ms;
      }
      if (d_stamps) {
        // fused: slot 2 = entry to the barrier's release (block 0), slot 3 = release to the last block's end
        const unsigned long long *s = &h_stamps[(size_t)r * 3];
        out_ms[2] += (double)(long long)(s[1] - s[0]) * 1e-6;
        out_ms[3] += (double)(long long)(s[2] - s[1]) * 1e-6;
      }
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[(size_t)r * 5], ev[(size_t)r * 5 + 4]);
      out_ms[4] += ms;
    }
    for (int k = 0; k < 5; ++k) out_ms[k] /= reps;
    rc = 0;
  }
  b200_free(d_stamps);
  for (auto &e : ev)
    if (e) cudaEventDestroy(e);
  return rc;
}

// The batch kernel's phases (scripts/prof_cg_batch.py): one launch of `reps` genuine iterations with the globaltimer
// stamps of block 0. out_ms[0..3] = average per iteration of the K1 phase, the K2 phase, the update up to its beta
// wait and the p update, each with the barrier or wait that ends it; out_ms[4] = the launch (CUDA events) per iteration.
// -1 when the workspace cannot run the batch kernel. Timing only: it must not overlap a solve of another thread.
extern "C" int b200_cg_time_batch(B200Cg *cg, double *d_x, int reps, double *out_ms) {
  B200FlagView A, At;
  if (reps <= 0 || !cg_batch_ready(cg, &A, &At)) return -1;
  cudaStream_t st = (cudaStream_t)b200_stream();
  const size_t bytes = (size_t)reps * 5 * sizeof(unsigned long long);
  unsigned long long *d_stamps = (unsigned long long *)b200_malloc(bytes);
  cudaEvent_t ev[2] = {nullptr, nullptr};
  int rc = -1;
  std::vector<unsigned long long> h((size_t)reps * 5);
  if (d_stamps && cudaEventCreate(&ev[0]) == cudaSuccess && cudaEventCreate(&ev[1]) == cudaSuccess &&
      cudaEventRecord(ev[0], st) == cudaSuccess && cg_batch_launch(cg, A, At, d_x, reps, d_stamps) == cudaSuccess &&
      cudaEventRecord(ev[1], st) == cudaSuccess && cudaStreamSynchronize(st) == cudaSuccess &&
      cudaMemcpy(h.data(), d_stamps, bytes, cudaMemcpyDeviceToHost) == cudaSuccess) {
    b200_count_launch(1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev[0], ev[1]);
    for (int k = 0; k < 4; ++k) out_ms[k] = 0.0;
    for (int r = 0; r < reps; ++r)
      for (int k = 0; k < 4; ++k) out_ms[k] += (double)(long long)(h[(size_t)r * 5 + k + 1] - h[(size_t)r * 5 + k]) * 1e-6;
    for (int k = 0; k < 4; ++k) out_ms[k] /= reps;
    out_ms[4] = ms / reps;
    rc = 0;
  }
  for (auto e : ev)
    if (e) cudaEventDestroy(e);
  b200_free(d_stamps);
  return rc;
}

extern "C" double b200_cg_iter_alg_bytes(const B200Cg *cg, double *per_kernel) {
  const double nnz = (double)b200_spmv_nnz(cg->A), n = cg->n, m = cg->m;
  const bool re = cg->A_cg != nullptr && cg->At_cg != nullptr && cg->d_ry_cg != nullptr;
  // the row operand of K1 (1 / R_y) and of K2 (R_x): a vector, or a table (K1: one mask bit per row)
  const double ry = re && cg->ry_form == B200_D_TWO ? m / 8.0 : 8.0 * m;
  const double rx = re && cg->rx_form == B200_D_ONE ? 0.0 : 8.0 * n;
  // bytes per stored entry: 12, or 11 with a packed index stream
  const double e1 = b200_spmv_entry_bytes(re ? cg->A_cg : cg->A), e2 = b200_spmv_entry_bytes(re ? cg->At_cg : cg->At);
  double k[4];
  k[0] = e1 * nnz + 4.0 * (m + 1.0) + 8.0 * n + 8.0 * m + ry;
  k[1] = e2 * nnz + 4.0 * (n + 1.0) + 8.0 * m + 16.0 * n + rx;
  // K3 reads x, r, p, Gp, M and writes x, r, z; K4 reads z, p and writes p. Fused: z is never stored and p is read
  // once, so phase 1 moves 56 n and phase 2 writes p (8 n).
  k[2] = cg->k34_fused ? 56.0 * n : 64.0 * n;
  k[3] = cg->k34_fused ? 8.0 * n : 24.0 * n;
  if (per_kernel)
    for (int i = 0; i < 4; ++i) per_kernel[i] = k[i];
  return k[0] + k[1] + k[2] + k[3];
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

  // main loop in batches. An iteration enqueued after `done` costs 3 or 4 empty launches (~12 us; nothing in the batch
  // kernel), a host poll costs a ~40 us bubble: the first batch is the hint, the previous count of a solve of the same kind
  // (host/linsys_b200.c), plus a 6 % margin (consecutive ADMM iterations need nearly the same number of CG steps),
  // later batches are small.
  int batch = its_hint + (its_hint / 16 > 2 ? its_hint / 16 : 2);
  if (batch < 4) batch = 4;
  if (batch > 512) batch = 512;  // a sharp drop of the CG count between two solves wastes at most 512 empty iterations
  const int follow = its_hint / 8 > 8 ? (its_hint / 8 < 256 ? its_hint / 8 : 256) : 8;
  long long enq = 0;
  int polls = 0;
  // the batch kernel when this workspace can run it and the token is free; without the token the K3 / K4 pair
  K34Token token;
  B200FlagView vA, vAt;
  const bool want_batch = cg_batch_enabled() && cg_batch_ready(cg, &vA, &vAt);
  const bool held = cg->k34_fused && (want_batch || k34_grid(n) > 1) && token.take();
  bool one_launch = want_batch && held;
  const bool fused = cg->k34_fused && (k34_grid(n) == 1 || held);
  ++cg->k34_solves[fused ? 0 : 1];
  for (;;) {
    if (one_launch) {
      const cudaError_t e = cg_batch_launch(cg, vA, vAt, d_b, batch, nullptr);
      if (e == cudaErrorCooperativeLaunchTooLarge || e == cudaErrorNotSupported) {
        (void)cudaGetLastError();  // refused: this solve runs the three kernels
        one_launch = false;
      } else {
        CUDA_OK(e);
        b200_count_launch(1);
      }
    }
    if (!one_launch)
      for (int i = 0; i < batch; ++i)
        if (cg_iteration(cg, d_b, fused) != 0) return -1;
    enq += batch;
    CUDA_OK(cudaMemcpyAsync(cg->h_ctl, cg->d_ctl, sizeof(B200CgCtl), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (cg->h_ctl->pad[0]) {
      b200_set_error(cg->nranks > 1 ? "peer-memory wait timed out in k_cg_finish_p2p"
                                    : "grid barrier wait timed out in k_cg_update_p or k_cg_batch",
                     cudaErrorUnknown, __FILE__, __LINE__);
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
  token.give_back();  // the last fused launch has finished: the host has seen the stream drain
  if (one_launch) ++cg->k34_batch_solves;
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

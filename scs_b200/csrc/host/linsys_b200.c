/* linsys_b200.c -- the SCS linear-system plugin ("sparse-indirect B200") in C.
 *
 * Implements the five link-time symbols of reference include/linsys.h:25-71 on
 * top of the device CG (kernels/cg.cu) and SpMV (kernels/spmv.cu):
 *
 *   scs_init_lin_sys_work     <- reference cpu/indirect/private.c:225-270
 *   scs_solve_lin_sys         <- :284-324
 *   scs_update_lin_sys_diag_r <- :327-331
 *   scs_free_lin_sys_work     <- :333-349
 *   scs_get_lin_sys_method    <- :221-223
 *
 * plus device-pointer variants (b200_linsys_*_dev) used by the device-resident
 * ADMM driver (host/scs_driver.c) so that the hot loop never crosses PCIe.
 */
#include "linsys_b200.h"
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

const char *scs_get_lin_sys_method(void) { return "sparse-indirect-b200-cuda"; }

/* Host threads for the setup-time passes over nnz of the multi-GPU path (row counts, row-block cut, below):
 * SCS_B200_HOST_THREADS, else min(16, online CPUs); 1 for small inputs. */
static int b200_host_threads(long long work_items) {
  const char *e = getenv("SCS_B200_HOST_THREADS");
  long t = e ? atol(e) : sysconf(_SC_NPROCESSORS_ONLN);
  if (!e && t > 16) t = 16;
  if (!e && work_items < 500000) t = 1;
  if (t < 1) t = 1;
  if (t > 64) t = 64;
  return (int)t;
}

/* expand upper-triangular CSC P into the full symmetric matrix in CSR
 * (reference gpu/indirect/private.c:174-202 does the same for cuSPARSE);
 * also extracts diag(P) for the preconditioner. The input is of scs_int width, the output int: a P whose full
 * symmetric form has more than B200_MAX_STORED entries, or a row index outside [0, n), is refused. */
static int expand_sym_upper(int n, const scs_int *Pp, const scs_int *Pi, const double *Px, int **Fp_out,
                            int **Fi_out, double **Fx_out, double *diag) {
  int *cnt = (int *)calloc((size_t)n + 1, sizeof(int));
  int *Fp = (int *)calloc((size_t)n + 1, sizeof(int));
  int *Fi;
  double *Fx;
  int i, j, tot = 0;
  scs_int k;
  long long full = 0;
  if (!cnt || !Fp) { free(cnt); free(Fp); return -1; }
  for (j = 0; j < n; ++j)
    for (k = Pp[j]; k < Pp[j + 1]; ++k) {
      if (Pi[k] < 0 || Pi[k] >= n) {
        fprintf(stderr, "scs_b200: P row index %lld outside [0, %d)\n", (long long)Pi[k], n);
        free(cnt); free(Fp);
        return -1;
      }
      full += Pi[k] == j ? 1 : 2;
    }
  if (full > B200_MAX_STORED) {
    fprintf(stderr, "scs_b200: the full symmetric P has %lld stored entries, above the limit 2^31 - 129 of one "
            "operator\n", full);
    free(cnt); free(Fp);
    return -1;
  }
  for (j = 0; j < n; ++j) diag[j] = 0.0;
  for (j = 0; j < n; ++j)
    for (k = Pp[j]; k < Pp[j + 1]; ++k) {
      i = (int)Pi[k];
      cnt[i]++;              /* entry (i,j) goes to row i */
      if (i != j) cnt[j]++;  /* mirrored entry (j,i) goes to row j */
      else diag[j] += Px[k];
    }
  for (i = 0; i < n; ++i) { Fp[i + 1] = Fp[i] + cnt[i]; }
  tot = Fp[n];
  Fi = (int *)malloc(((size_t)tot + 1) * sizeof(int));
  Fx = (double *)malloc(((size_t)tot + 1) * sizeof(double));
  if (!Fi || !Fx) { free(cnt); free(Fp); free(Fi); free(Fx); return -1; }
  for (i = 0; i < n; ++i) cnt[i] = Fp[i];
  /* rows get their entries in ascending column order: first the lower part
   * (mirrors, columns < row) then the upper part. Two passes keep it sorted. */
  for (j = 0; j < n; ++j)
    for (k = Pp[j]; k < Pp[j + 1]; ++k) {
      i = (int)Pi[k];
      if (i != j) { /* (i,j) with i<j stored; mirror (j,i): row j, col i < j */
        const int q = cnt[j]++;
        Fi[q] = i; Fx[q] = Px[k];
      }
    }
  for (j = 0; j < n; ++j)
    for (k = Pp[j]; k < Pp[j + 1]; ++k) {
      i = (int)Pi[k];
      { const int q = cnt[i]++; Fi[q] = j; Fx[q] = Px[k]; } /* row i, col j >= i */
    }
  free(cnt);
  *Fp_out = Fp; *Fi_out = Fi; *Fx_out = Fx;
  return 0;
}

/* Row partition for the sharded KKT solve (SURVEY 8e): contiguous blocks with (nearly) equal
 * numbers of nonzeros. */
/* generic fork-join over an array of job records (threads that cannot be created run inline) */
static void run_jobs(void *(*fn)(void *), void *jobs, size_t stride, int T) {
  pthread_t th[64];
  int t, started = 0;
  for (t = 1; t < T; ++t) {
    if (pthread_create(&th[t], NULL, fn, (char *)jobs + (size_t)t * stride) != 0) break;
    started = t;
  }
  fn(jobs);
  for (t = started + 1; t < T; ++t) fn((char *)jobs + (size_t)t * stride);
  for (t = 1; t <= started; ++t) pthread_join(th[t], NULL);
}

typedef struct {
  long long k0, k1;
  const scs_int *Ai;
  int *cnt;
} PcJob;
static void *pc_worker(void *arg) { /* entries per row: integer counts, order-independent */
  PcJob *jb = (PcJob *)arg;
  long long k;
  for (k = jb->k0; k < jb->k1; ++k) __atomic_fetch_add(&jb->cnt[jb->Ai[k]], 1, __ATOMIC_RELAXED);
  return NULL;
}

void b200_row_partition(int m, int n, const scs_int *Ap, const scs_int *Ai, int nranks, int *offsets) {
  const long long nnz = Ap[n];
  int *cnt = (int *)calloc((size_t)m + 1, sizeof(int));
  long long acc = 0;
  int i, r = 1;
  offsets[0] = 0;
  if (!cnt) { /* fall back to equal rows */
    for (r = 1; r <= nranks; ++r) offsets[r] = (int)(((long long)m * r) / nranks);
    return;
  }
  {
    PcJob jobs[64];
    const int T = b200_host_threads(nnz);
    int t;
    for (t = 0; t < T; ++t) {
      jobs[t].k0 = nnz * t / T; jobs[t].k1 = nnz * (t + 1) / T; jobs[t].Ai = Ai; jobs[t].cnt = cnt;
    }
    run_jobs(pc_worker, jobs, sizeof(PcJob), T);
  }
  for (i = 0; i < m && r < nranks; ++i) {
    acc += (long long)cnt[i] + 1; /* +1: empty rows still cost a row */
    while (r < nranks && acc >= ((nnz + m) * (long long)r) / nranks) offsets[r++] = i + 1;
  }
  while (r <= nranks) offsets[r++] = m;
  offsets[nranks] = m;
  free(cnt);
}
scs_int scs_b200_row_partition(scs_int m, scs_int n, const scs_int *Ap, const scs_int *Ai,
                               scs_int nranks, scs_int *offsets) {
  int *offs;
  scs_int r;
  if (m <= 0 || n <= 0 || nranks <= 0 || !Ap || !Ai || !offsets) return -1;
  if (b200_over_dim("m", -1, m) || b200_over_dim("n", -1, n) || b200_over_dim("nranks", -1, nranks) ||
      b200_over_stored("nnz", Ap[n]))
    return -1;
  if (sizeof(scs_int) == sizeof(int)) {
    b200_row_partition((int)m, (int)n, Ap, Ai, (int)nranks, (int *)offsets);
    return 0;
  }
  offs = (int *)malloc(((size_t)nranks + 1) * sizeof(int));
  if (!offs) return -1;
  b200_row_partition((int)m, (int)n, Ap, Ai, (int)nranks, offs);
  for (r = 0; r <= nranks; ++r) offsets[r] = offs[r];
  free(offs);
  return 0;
}

/* CSC restricted to rows [r0, r1), row indices shifted by -r0. Threaded over column ranges of equal nnz: a count pass
 * (kept entries per column), a serial prefix over the n columns, a fill pass -- the output does not depend on the
 * number of threads. */
typedef struct {
  int j0, j1, r0, r1, phase;
  const scs_int *Ap, *Ai;
  const double *Ax;
  int *Lp, *Li;
  double *Lx;
} RrJob;
static void *rr_worker(void *arg) {
  RrJob *jb = (RrJob *)arg;
  const int r0 = jb->r0, r1 = jb->r1;
  int j;
  scs_int k;
  if (jb->phase == 0) {
    for (j = jb->j0; j < jb->j1; ++j) {
      int c = 0;
      for (k = jb->Ap[j]; k < jb->Ap[j + 1]; ++k) c += (jb->Ai[k] >= r0 && jb->Ai[k] < r1);
      jb->Lp[j + 1] = c;
    }
  } else {
    for (j = jb->j0; j < jb->j1; ++j) {
      int q = jb->Lp[j];
      for (k = jb->Ap[j]; k < jb->Ap[j + 1]; ++k)
        if (jb->Ai[k] >= r0 && jb->Ai[k] < r1) { jb->Li[q] = (int)(jb->Ai[k] - r0); jb->Lx[q] = jb->Ax[k]; ++q; }
    }
  }
  return NULL;
}
static int restrict_rows(int n, const scs_int *Ap, const scs_int *Ai, const double *Ax, int r0, int r1,
                         int **Lp_out, int **Li_out, double **Lx_out) {
  RrJob jobs[64];
  const long long nnz = Ap[n];
  int T = b200_host_threads(nnz);
  int j, t, cnt;
  int *Lp = (int *)calloc((size_t)n + 1, sizeof(int));
  int *Li;
  double *Lx;
  if (!Lp) return -1;
  if (T > n) T = n > 0 ? n : 1;
  for (t = 0, j = 0; t < T; ++t) { /* column ranges balanced by their number of entries */
    const long long target = nnz * (t + 1) / T;
    jobs[t].j0 = j;
    if (t == T - 1) {
      j = n;
    } else {
      int lo = j, hi = n;
      while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (Ap[mid] < target) lo = mid + 1; else hi = mid;
      }
      j = lo;
    }
    jobs[t].j1 = j;
    jobs[t].r0 = r0; jobs[t].r1 = r1; jobs[t].phase = 0;
    jobs[t].Ap = Ap; jobs[t].Ai = Ai; jobs[t].Ax = Ax; jobs[t].Lp = Lp; jobs[t].Li = NULL; jobs[t].Lx = NULL;
  }
  run_jobs(rr_worker, jobs, sizeof(RrJob), T);
  for (j = 0; j < n; ++j) Lp[j + 1] += Lp[j];
  cnt = Lp[n];
  Li = (int *)malloc(((size_t)cnt + 1) * sizeof(int));
  Lx = (double *)malloc(((size_t)cnt + 1) * sizeof(double));
  if (!Li || !Lx) { free(Lp); free(Li); free(Lx); return -1; }
  for (t = 0; t < T; ++t) { jobs[t].phase = 1; jobs[t].Li = Li; jobs[t].Lx = Lx; }
  run_jobs(rr_worker, jobs, sizeof(RrJob), T);
  *Lp_out = Lp; *Li_out = Li; *Lx_out = Lx;
  return 0;
}
/* test entry point (tests/test_sharding_cpu.py); the arrays are malloc'ed, the caller frees them */
int scs_b200_restrict_rows_csc(int n, const scs_int *Ap, const scs_int *Ai, const double *Ax, int r0, int r1,
                               int **Lp_out, int **Li_out, double **Lx_out) {
  return restrict_rows(n, Ap, Ai, Ax, r0, r1, Lp_out, Li_out, Lx_out);
}

#include <time.h>
static double wall_ms(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec;
}
/* SCS_B200_SETUP_TIMING=1: wall-clock breakdown of the setup on stderr (syncs the stream at every mark) */
static void setup_mark(const char *what, double *t_last) {
  if (!getenv("SCS_B200_SETUP_TIMING")) return;
  b200_sync();
  {
    const double t = wall_ms();
    fprintf(stderr, "scs_b200 setup: %-44s %8.1f ms\n", what, t - *t_last);
    *t_last = t;
  }
}

/* Both resident orientations of a CSC matrix, built on the device (kernels/setup.cu): *A_out = the m x n operator
 * (rows of A), *At_out = the n x m one (rows of A' = columns of A). */
static int build_both_ops(int m, int n, const int *Ap, const int *Ai, const double *Ax, B200Spmv **A_out,
                          B200Spmv **At_out, double *t_mark) {
  if (b200_setup_ops_from_csc(m, n, Ap, Ai, Ax, A_out, At_out) != 0) return -1;
  setup_mark("linsys: both operators built on the device", t_mark);
  return 0;
}
/* the same from the caller's CSC, of scs_int width: with DLONG its 64-bit indices are narrowed on the device */
static int build_both_ops_user(int m, int n, const scs_int *Ap, const scs_int *Ai, const double *Ax, B200Spmv **A_out,
                               B200Spmv **At_out, double *t_mark) {
#ifdef DLONG
  if (b200_setup_ops_from_csc64(m, n, Ap, Ai, Ax, A_out, At_out) != 0) return -1;
  setup_mark("linsys: both operators built on the device (64-bit indices narrowed there)", t_mark);
  return 0;
#else
  return build_both_ops(m, n, Ap, Ai, Ax, A_out, At_out, t_mark);
#endif
}

/* The reordered pair used inside the CG operator (kernels/spmv.cu "Reordered copies", DESIGN.md section 3.1): the rows
 * of A sorted by their smallest column make one gather per row of K1 and of K2 sequential, and every row is placed
 * where the kernel sums it as in A, so the pair computes what the plain pair computes. Built once on a single GPU whenever both
 * operators are one-pass flagged streams (the only form the permuted copy and the renumbered view are built for);
 * other inputs keep the plain pair. Values and R_y are refreshed whenever the resident operators may have been
 * rescaled (b200_linsys_update_diag_r_dev). */
static int cg_ops_build(ScsLinSysWork *w) {
  long long empty;
  int kept;
  if (w->nranks > 1) return 0;
  if (!b200_spmv_can_route(w->A) || !b200_spmv_can_route(w->At)) return 0; /* one-pass flagged streams only */
  /* empty rows (one stored SKIP entry each) sort last and no column of A references them: A_cg leaves them out, their
   * entries of the permuted tmp are never written and never read */
  empty = b200_spmv_stored(w->A) - b200_spmv_nnz(w->A);
  kept = w->m - (int)empty;
  if (kept <= 0) return 0;
  w->d_perm = (int *)b200_malloc((size_t)w->m * 4);
  w->d_inv = (int *)b200_malloc((size_t)w->m * 4);
  w->d_ry_cg = (double *)b200_malloc((size_t)w->m * 8);
  w->cg.d_diag_tab = (double *)b200_malloc(3 * 8);
  w->cg.d_diag_mixed = (unsigned *)b200_malloc(4);
  w->cg.d_ry_mask = (unsigned *)b200_malloc(((size_t)kept + 31) / 32 * 4);
  if (!w->d_perm || !w->d_inv || !w->d_ry_cg || !w->cg.d_diag_tab || !w->cg.d_diag_mixed || !w->cg.d_ry_mask)
    return -1;
  if (b200_perm_rows_by_min_col(w->A, w->d_perm) != 0) return -1;
  /* the placement reorders the sorted rows slightly: d_perm is final, and d_inv computed from it, only after this */
  w->A_cg = b200_spmv_permuted_rows(w->A, w->d_perm, w->d_inv, kept);
  if (!w->A_cg) return -1;
  w->At_cg = b200_spmv_renumbered_cols(w->At, w->d_inv);
  if (!w->At_cg) return -1;
  /* only the CG loop reads these two: their index streams go to 3 bytes per entry where the columns allow it */
  if (b200_spmv_pack_indices(w->A_cg) != 0 || b200_spmv_pack_indices(w->At_cg) != 0) return -1;
  w->cg.A_cg = w->A_cg; w->cg.At_cg = w->At_cg; w->cg.d_ry_cg = w->d_ry_cg;
  return 0;
}
/* R_y and R_x as tables when SCS's form of diag_r holds (two values of R_y, one of R_x; any other diag_r, e.g. through
 * scs_update_lin_sys_diag_r, takes the vectors): K1 and K2 then stream no row vector for them */
static int cg_ops_refresh(ScsLinSysWork *w) {
  if (!w->A_cg) return 0;
  if (b200_spmv_refresh_permuted(w->A_cg, w->A, w->d_perm) != 0) return -1;
  if (b200_gather_vec(w->m, w->d_perm, w->cg.d_ry_inv, w->d_ry_cg) != 0) return -1; /* 1 / R_y, permuted order */
  return b200_cg_classify_diag(&w->cg, w->d_perm);
}

ScsLinSysWork *scs_init_lin_sys_work(const ScsMatrix *A, const ScsMatrix *P,
                                     const scs_float *diag_r) {
  ScsLinSysWork *w;
  double t_mark = wall_ms();
  int *Lp = NULL, *Li = NULL;
  double *Lx = NULL;
  int n, m;
  if (!A || b200_matrix_over_limits(A, P)) { /* in scs_int width, before anything is narrowed */
    fprintf(stderr, "scs_b200: init_lin_sys_work refused its input\n");
    return SCS_NULL;
  }
  n = (int)A->n;
  m = (int)A->m;
  if (b200_runtime_init() != 0) {
    fprintf(stderr, "scs_b200: no usable sm_90 device: %s\n", b200_last_error());
    return SCS_NULL;
  }
  w = (ScsLinSysWork *)calloc(1, sizeof(ScsLinSysWork));
  if (!w) return SCS_NULL;
  w->n = n; w->m = m;
  w->nnz = A->p[n];
  w->nranks = b200_comm_nranks();
  w->rank = b200_comm_rank();
  w->row0 = 0;
  w->mloc = m;
  if (w->nranks > 1) {
    /* row-sharded: keep only rows [row0, row0+mloc) of A, in both orientations */
    w->offsets = (int *)calloc((size_t)w->nranks + 1, sizeof(int));
    if (!w->offsets) goto fail;
    b200_row_partition(m, n, A->p, A->i, w->nranks, w->offsets);
    w->row0 = w->offsets[w->rank];
    w->mloc = w->offsets[w->rank + 1] - w->row0;
    if (restrict_rows(n, A->p, A->i, A->x, w->row0, w->row0 + w->mloc, &Lp, &Li, &Lx) != 0) goto fail;
    setup_mark("linsys: row block cut out of A (host)", &t_mark);
    {
      const int rc = build_both_ops(w->mloc, n, Lp, Li, Lx, &w->A, &w->At, &t_mark);
      free(Lp); free(Li); free(Lx);
      if (rc != 0) goto fail;
    }
  } else if (build_both_ops_user(m, n, A->p, A->i, A->x, &w->A, &w->At, &t_mark) != 0) {
    goto fail;
  }
  if (!w->A || !w->At) goto fail;
  if (P) {
    int *Fp = NULL, *Fi = NULL;
    double *Fx = NULL;
    double *diag = (double *)malloc((size_t)n * sizeof(double));
    if (!diag || expand_sym_upper(n, P->p, P->i, P->x, &Fp, &Fi, &Fx, diag) != 0) {
      free(diag);
      goto fail;
    }
    w->P = b200_spmv_create(n, n, Fp, Fi, Fx);
    w->d_Pdiag = (double *)b200_malloc((size_t)n * 8);
    if (w->d_Pdiag) b200_h2d(w->d_Pdiag, diag, (size_t)n * 8);
    free(Fp); free(Fi); free(Fx); free(diag);
    if (!w->P || !w->d_Pdiag) goto fail;
    setup_mark("linsys: operator P (host expansion, device build)", &t_mark);
  }
  w->d_diag_r = (double *)b200_malloc(((size_t)n + m + 1) * 8);
  w->d_b = (double *)b200_malloc(((size_t)n + m) * 8);
  w->d_s = (double *)b200_malloc((size_t)n * 8);
  w->cg.d_M = (double *)b200_malloc((size_t)n * 8);
  w->cg.d_p = SCS_NULL; /* allocated below: in the peer-mapped exchange memory when the sharded-x mode is possible */
  w->cg.d_r = (double *)b200_malloc((size_t)n * 8);
  w->cg.d_Gp = (double *)b200_malloc((size_t)n * 8);
  w->cg.d_z = (double *)b200_malloc((size_t)n * 8);
  w->cg.d_tmp = (double *)b200_malloc((size_t)m * 8);
  w->cg.d_ry_inv = (double *)b200_malloc((size_t)m * 8);
  w->cg.d_ctl = (B200CgCtl *)b200_malloc(sizeof(B200CgCtl));
  w->cg.d_partials = (double *)b200_malloc(4 * 2048 * 8);
  w->cg.d_counter = (unsigned int *)b200_malloc(64);
  w->cg.d_red = (double *)b200_malloc((size_t)n * 8);
  w->cg.h_ctl = (B200CgCtl *)b200_host_alloc(sizeof(B200CgCtl));
  if (!w->d_diag_r || !w->d_b || !w->d_s || !w->cg.d_M || !w->cg.d_r ||
      !w->cg.d_Gp || !w->cg.d_z || !w->cg.d_tmp || !w->cg.d_ctl || !w->cg.d_partials ||
      !w->cg.d_counter || !w->cg.h_ctl || !w->cg.d_red || !w->cg.d_ry_inv)
    goto fail;
  b200_memset0(w->cg.d_counter, 64);
  b200_memset0(w->cg.d_ctl, sizeof(B200CgCtl));
  memset(w->cg.h_ctl, 0, sizeof(B200CgCtl));
  w->cg.n = n; w->cg.m = m;
  w->cg.A = w->A; w->cg.At = w->At; w->cg.P = w->P;
  w->cg.d_rx = w->d_diag_r;
  w->cg.d_ry = w->d_diag_r + n;
  w->cg.nranks = w->nranks; w->cg.row0 = w->row0; w->cg.mloc = w->mloc; w->cg.offsets = w->offsets;
  /* fused peer-memory reduction (NVLink, CUDA IPC) when every rank could map every peer */
  w->cg.use_p2p = (w->nranks > 1 && b200_p2p_setup(n) == 0 && b200_p2p_ok(n)) ? 1 : 0;
  if (w->cg.use_p2p) {
    B200P2pSignal sig;
    int r;
    memset(&sig, 0, sizeof(sig));
    sig.nranks = w->nranks; sig.rank = w->rank;
    for (r = 0; r < w->nranks && r < 8; ++r) sig.flags[r] = b200_p2p_flags(r);
    w->cg.d_p2p_sig = (B200P2pSignal *)b200_malloc(sizeof(sig));
    if (!w->cg.d_p2p_sig || b200_h2d(w->cg.d_p2p_sig, &sig, sizeof(sig)) != 0) goto fail;
    /* sharded-x push mode (kernels/cg.cu k_cgx_iteration): p lives in the exchange allocation so that the peers can
     * store their slices into it, and the K2 SpMV pushes its rows to the owners' inboxes. Needs the flagged-stream
     * kernel without virtual rows for A' and the (single) exchange p vector. */
    if (b200_spmv_can_route(w->At) && b200_p2p_claim_pvec() == 0) {
      B200P2pRoute rt;
      const int G = w->nranks, S = (n + G - 1) / G;
      memset(&rt, 0, sizeof(rt));
      rt.nranks = G; rt.rank = w->rank;
      for (r = 0; r <= G; ++r) rt.lo[r] = (int)(((long long)n * r) / G);
      for (r = 0; r < G; ++r) {
        rt.dst[r] = (unsigned long long *)b200_p2p_inbox(r) + 2 * (size_t)w->rank * S; /* my lane of rank r's inbox */
        rt.flags[r] = b200_p2p_flags(r);
      }
      w->p_in_exchange = 1;
      w->cg.d_p = b200_p2p_pvec(w->rank);
      w->cg.d_p2p_route = (B200P2pRoute *)b200_malloc(sizeof(rt));
      if (!w->cg.d_p2p_route || b200_h2d(w->cg.d_p2p_route, &rt, sizeof(rt)) != 0) goto fail;
    }
  }
  if (!w->cg.d_p) {
    w->cg.d_p = (double *)b200_malloc((size_t)n * 8);
    if (!w->cg.d_p) goto fail;
  }
  if (b200_h2d(w->d_diag_r, diag_r, ((size_t)n + m) * 8) != 0) goto fail;
  if (b200_cg_set_preconditioner(&w->cg, w->d_Pdiag) != 0) goto fail;
  if (b200_sync() != 0) goto fail;
  setup_mark("linsys: vectors, preconditioner", &t_mark);
  if (cg_ops_build(w) != 0 || cg_ops_refresh(w) != 0 || b200_sync() != 0) goto fail;
  setup_mark("linsys: reordered pair for the CG operator", &t_mark);
  return w;
fail:
  fprintf(stderr, "scs_b200: init_lin_sys_work failed: %s\n", b200_last_error());
  scs_free_lin_sys_work(w);
  return SCS_NULL;
}

void scs_free_lin_sys_work(ScsLinSysWork *w) {
  if (!w) return;
  b200_sync();
  b200_spmv_destroy(w->At_cg); /* a view of At: before At itself */
  b200_spmv_destroy(w->A_cg);
  b200_free(w->d_ry_cg);
  b200_free(w->cg.d_diag_tab);
  b200_free(w->cg.d_diag_mixed);
  b200_free(w->cg.d_ry_mask);
  b200_free(w->d_perm);
  b200_free(w->d_inv);
  b200_spmv_destroy(w->A);
  b200_spmv_destroy(w->At);
  b200_spmv_destroy(w->P);
  b200_free(w->d_Pdiag);
  b200_free(w->d_diag_r);
  b200_free(w->d_b);
  b200_free(w->d_s);
  b200_free(w->cg.d_M);
  if (w->p_in_exchange) b200_p2p_release_pvec(); else b200_free(w->cg.d_p);
  b200_free(w->cg.d_r);
  b200_free(w->cg.d_Gp);
  b200_free(w->cg.d_z);
  b200_free(w->cg.d_tmp);
  b200_free(w->cg.d_ry_inv);
  b200_free(w->cg.d_ctl);
  b200_free(w->cg.d_partials);
  b200_free(w->cg.d_counter);
  b200_free(w->cg.d_red);
  b200_free(w->cg.d_p2p_sig);
  b200_free(w->cg.d_p2p_route);
  b200_host_free(w->cg.h_ctl);
  free(w->offsets);
  free(w);
}

/* Row-sharded setup: D, E of the FULL matrix are computed on every rank from temporary full
 * copies (both orientations) on its GPU; the resident local blocks are then scaled once. */
int b200_linsys_full_equilibrate(const ScsMatrix *A, const int *bnd, int nbnd, double *d_D, double *d_E) {
  int rc = -1;
  double t_mark = wall_ms();
  B200Spmv *At = NULL, *Ar = NULL;
  if (build_both_ops_user((int)A->m, (int)A->n, A->p, A->i, A->x, &Ar, &At, &t_mark) == 0)
    rc = b200_equilibrate_dev(Ar, At, bnd, nbnd, d_D, d_E);
  setup_mark("linsys: D, E from a temporary full copy", &t_mark);
  b200_spmv_destroy(Ar);
  b200_spmv_destroy(At);
  return rc;
}
int b200_linsys_scale_local(ScsLinSysWork *w, const double *d_D, const double *d_E) {
  if (b200_rescale_dev(w->A, d_D + w->row0, d_E, 1) != 0) return -1;   /* rows of A_g */
  if (b200_rescale_dev(w->At, d_E, d_D + w->row0, 0) != 0) return -1;  /* columns of A_g */
  return 0;
}

/* device-pointer solve used by the ADMM driver; d_tol optional device scalar */
int b200_linsys_solve_dev(ScsLinSysWork *w, double *d_b, const double *d_s, double tol,
                          const double *d_tol) {
  long long max_its = 10LL * w->n; /* reference private.c:307 */
  int its;
  if (max_its > 2000000000LL) max_its = 2000000000LL;
  its = b200_cg_solve(&w->cg, d_b, d_s, tol, (int)max_its, w->last_cg_its, d_tol);
  if (its < 0) return -1;
  w->last_cg_its = its;
  w->tot_cg_its += its;
  w->n_solves += 1;
  return 0;
}

int b200_linsys_update_diag_r_dev(ScsLinSysWork *w, const double *d_diag_r) {
  if (d_diag_r != w->d_diag_r) {
    if (b200_d2d(w->d_diag_r, d_diag_r, ((size_t)w->n + w->m) * 8) != 0) return -1;
  }
  if (b200_cg_set_preconditioner(&w->cg, w->d_Pdiag) != 0) return -1; /* also refreshes 1 / R_y */
  return cg_ops_refresh(w); /* the operators may have been rescaled in place; R_y has changed */
}

scs_int scs_solve_lin_sys(ScsLinSysWork *w, scs_float *b, const scs_float *s, scs_float tol) {
  const size_t nm = (size_t)w->n + w->m;
  if (tol <= 0.) {
    fprintf(stderr, "Warning: tol = %4f <= 0, likely compiled without setting INDIRECT flag.\n",
            tol);
  }
  if (b200_h2d(w->d_b, b, nm * 8) != 0) return -1;
  if (s && b200_h2d(w->d_s, s, (size_t)w->n * 8) != 0) return -1;
  if (b200_linsys_solve_dev(w, w->d_b, s ? w->d_s : NULL, tol, NULL) != 0) return -1;
  if (b200_d2h(b, w->d_b, nm * 8) != 0) return -1;
  if (b200_sync() != 0) return -1;
  return 0;
}

scs_int scs_update_lin_sys_diag_r(ScsLinSysWork *w, const scs_float *new_diag_r) {
  if (b200_h2d(w->d_diag_r, new_diag_r, ((size_t)w->n + w->m) * 8) != 0) return -1;
  if (b200_linsys_update_diag_r_dev(w, w->d_diag_r) != 0) return -1;
  return b200_sync() == 0 ? 0 : -1;
}

scs_int scs_b200_linsys_last_cg_its(const ScsLinSysWork *w) { return w->last_cg_its; }
long long scs_b200_linsys_total_cg_its(const ScsLinSysWork *w) { return w->tot_cg_its; }

static scs_int accum_generic(ScsLinSysWork *w, const B200Spmv *M, int ncols, int nrows,
                             const scs_float *x, scs_float *y, scs_int accumulate) {
  B200SpmvArgs a;
  double *d_x = (double *)b200_malloc((size_t)ncols * 8);
  double *d_y = (double *)b200_malloc((size_t)nrows * 8);
  int rc = -1;
  if (w->nranks > 1) { b200_free(d_x); b200_free(d_y); return -1; } /* operator-level API is single-GPU */
  if (!d_x || !d_y) goto out;
  if (b200_h2d(d_x, x, (size_t)ncols * 8) != 0) goto out;
  if (accumulate && b200_h2d(d_y, y, (size_t)nrows * 8) != 0) goto out;
  memset(&a, 0, sizeof(a));
  a.d_x = d_x; a.d_y = d_y; a.d_init = accumulate ? d_y : NULL; a.init_sign = 1.0;
  a.post = B200_POST_NONE; a.hook = B200_HOOK_NONE;
  if (b200_spmv(M, &a) != 0) goto out;
  if (b200_d2h(y, d_y, (size_t)nrows * 8) != 0) goto out;
  if (b200_sync() != 0) goto out;
  rc = 0;
out:
  b200_free(d_x);
  b200_free(d_y);
  return rc;
}

scs_int scs_b200_accum_by_a(ScsLinSysWork *w, const scs_float *x, scs_float *y,
                            scs_int accumulate) {
  return accum_generic(w, w->A, w->n, w->m, x, y, accumulate);
}
scs_int scs_b200_accum_by_atrans(ScsLinSysWork *w, const scs_float *x, scs_float *y,
                                 scs_int accumulate) {
  return accum_generic(w, w->At, w->m, w->n, x, y, accumulate);
}

/* --- device timing helpers for bench.py (inputs resident in HBM) --------- */
double scs_b200_time_spmv(ScsLinSysWork *w, scs_int op, scs_int reps, double *alg_bytes) {
  double ms[2] = {-1.0, -1.0};
  if (b200_spmv_time_pair(w->A, w->At, reps, ms) != 0) return -1.0;
  if (alg_bytes) *alg_bytes = b200_spmv_alg_bytes(op == 0 ? w->A : w->At, 0);
  return ms[op == 0 ? 0 : 1];
}

/* bench.py roofline: the kernels of the CG loop as they run inside a solve (the solver's own p / tmp / r after
 * a genuine start on the right-hand side b, which the caller provides: length n + m, host). out_ms[0..4] = ms
 * per launch of K1, K2, K3, K4 and of the whole iteration; out_bytes[0..4] = the algorithmic bytes of each
 * (b200_cg_iter_alg_bytes, DESIGN.md section 3). */
scs_int scs_b200_time_cg_kernels(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms,
                                 double *out_bytes) {
  const size_t nm = (size_t)w->n + w->m;
  int k;
  if (w->P) return -1;
  if (b200_h2d(w->d_b, b, nm * 8) != 0) return -1;
  if (b200_cg_solve(&w->cg, w->d_b, NULL, 0.0, 1, 0, NULL) < 0) return -1; /* genuine start: p, r, z, ctl */
  w->cg.h_ctl->done = 0;
  w->cg.h_ctl->max_its = 2000000000;
  if (b200_h2d(w->cg.d_ctl, w->cg.h_ctl, sizeof(B200CgCtl)) != 0) return -1;
  for (k = 0; k < 3; ++k) if (b200_cg_one_iteration(&w->cg, w->d_b) != 0) return -1;
  if (b200_sync() != 0) return -1;
  if (b200_cg_time_kernels(&w->cg, w->d_b, (int)reps, out_ms) != 0) return -1;
  if (out_bytes) out_bytes[4] = b200_cg_iter_alg_bytes(&w->cg, out_bytes);
  return 0;
}

double scs_b200_time_cg_iter(ScsLinSysWork *w, scs_int reps, double *alg_bytes) {
  /* run `reps` genuine CG iterations on a synthetic rhs with the stop test
   * disabled (tol = 0 never satisfies ||r|| < tol) and time them on the stream */
  const size_t nm = (size_t)w->n + w->m;
  double *hb = (double *)malloc(nm * 8);
  double ms = -1.0;
  size_t i;
  int k;
  if (!hb) return -1.0;
  for (i = 0; i < nm; ++i) hb[i] = 0.5 + 1e-3 * (double)(i % 997);
  if (b200_h2d(w->d_b, hb, nm * 8) != 0) goto out;
  /* set up p, r, z, ctl with a 1-iteration solve, then time raw iterations */
  if (b200_cg_solve(&w->cg, w->d_b, NULL, 0.0, 1, 0, NULL) < 0) goto out;
  w->cg.h_ctl->done = 0;
  w->cg.h_ctl->max_its = 2000000000;
  if (b200_h2d(w->cg.d_ctl, w->cg.h_ctl, sizeof(B200CgCtl)) != 0) goto out;
  for (k = 0; k < 3; ++k) if (b200_cg_one_iteration(&w->cg, w->d_b) != 0) goto out;
  if (b200_sync() != 0) goto out;
  if (b200_timer_start() != 0) goto out;
  for (k = 0; k < reps; ++k) if (b200_cg_one_iteration(&w->cg, w->d_b) != 0) goto out;
  ms = b200_timer_stop_ms();
  if (ms >= 0) ms /= (double)reps;
  if (alg_bytes) *alg_bytes = b200_cg_iter_alg_bytes(&w->cg, NULL);
out:
  free(hb);
  return ms;
}

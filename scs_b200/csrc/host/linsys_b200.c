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
 * ADMM driver (host/scs_driver.c) so that the hot loop never crosses PCIe, and
 * the operator level's device twins of the plugin calls and of the SpMV pair
 * (scs_b200_*_device, include/scs_b200.h group (3)) on the caller's buffers.
 */
#include "driver.h" /* ScsWork, for scs_b200_cg_k34_paths */
#include "linsys_b200.h"
#include <pthread.h>
#include <stdint.h>
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

/* One upload of a host CSC into the int32 / fp64 device arrays the builder takes: p and i, of 8 bytes (idx64) or 4,
 * are staged on the device and go through the validating copy (kernels/setup.cu), which narrows them; x is copied as
 * is and not checked. upper: the upper triangle of P, *ndiag (else NULL) then receives its diagonal entries. Refused
 * with a message naming `what` when p[0] != 0, a pointer decreases or leaves [0, nnz], or a row index leaves [0, rows)
 * or, with upper, lies below the diagonal: no kernel reads an index before it has been checked, in its own width (a
 * truncated 2^32 + 3 would look valid). The staging is freed before this returns, so the builder that runs next does
 * not hold it too. On success the caller frees *d_p, *d_i and *d_x. */
int b200_csc_upload(const char *what, int rows, int n, const void *p, const void *i, const double *x, int idx64,
                    int upper, int **d_p, int **d_i, double **d_x, long long *nnz_out, long long *ndiag) {
  const size_t w = idx64 ? 8 : 4;
  const long long nnz = idx64 ? ((const long long *)p)[n] : ((const int *)p)[n];
  void *s_p = NULL, *s_i = NULL;
  unsigned flags = 0;
  unsigned long long first = ~0ULL;
  long long nd = 0;
  int rc = -1;
  *d_p = NULL; *d_i = NULL; *d_x = NULL;
  if (nnz < 0 || nnz > B200_MAX_STORED) {
    fprintf(stderr, "scs_b200: %s refused: nnz = %lld must lie in [0, 2^31 - 129]\n", what, nnz);
    return -1;
  }
  s_p = b200_malloc((size_t)(n + 1) * w);
  s_i = b200_malloc((size_t)nnz * w);
  *d_p = (int *)b200_malloc((size_t)(n + 1) * 4);
  *d_i = (int *)b200_malloc((size_t)nnz * 4);
  *d_x = (double *)b200_malloc((size_t)nnz * 8);
  if (s_p && s_i && *d_p && *d_i && *d_x && b200_h2d(s_p, p, (size_t)(n + 1) * w) == 0 &&
      b200_h2d(s_i, i, (size_t)nnz * w) == 0 && b200_csc_check_ptrs(n, nnz, s_p, idx64, *d_p, &flags) == 0) {
    if (flags == 0 &&
        b200_csc_copy_entries(rows, n, nnz, s_i, NULL, idx64, *d_p, upper, *d_i, NULL, &first, &nd) == 0 &&
        first == ~0ULL)
      rc = 0;
    if (flags != 0 || first != ~0ULL)
      fprintf(stderr, "scs_b200: %s refused: column pointers must start at 0 and not decrease, and row indices must "
              "lie in [0, %s)%s\n", what, upper ? "n" : "m", upper ? " and on or above the diagonal" : "");
  }
  b200_free(s_p); /* stream-ordered: the entry pass has read them */
  b200_free(s_i);
  if (rc == 0 && b200_h2d(*d_x, x, (size_t)nnz * 8) != 0) rc = -1;
  if (rc != 0) {
    b200_free(*d_p); b200_free(*d_i); b200_free(*d_x);
    *d_p = NULL; *d_i = NULL; *d_x = NULL;
    return -1;
  }
  *nnz_out = nnz;
  if (ndiag) *ndiag = nd;
  return 0;
}

void b200_dev_mats_free(B200DevMats *dm) {
  b200_free(dm->Ap); b200_free(dm->Ai); b200_free(dm->Ax);
  b200_free(dm->Pp); b200_free(dm->Pi); b200_free(dm->Px);
  memset(dm, 0, sizeof(*dm));
}

scs_int b200_read_dev_int(const scs_int *d_v) {
  scs_int v = -1;
  if (b200_d2h(&v, d_v, sizeof(scs_int)) != 0 || b200_sync() != 0) return -1;
  return v;
}
/* scs_init's validate_matrix (host/scs_driver.c) on device arrays, shared by scs_b200_init_device,
 * scs_b200_update_matrix_device and scs_b200_init_lin_sys_work_device: the same checks, in the same order, with the same messages. The host reads p[n],
 * then the pointer flags, then the first failing entry: no kernel reads an index before the check that guards it. */
int b200_validate_matrix_dev(const ScsMatrix *A, const ScsMatrix *P, B200DevMats *dm) {
  const int idx64 = sizeof(scs_int) == 8;
  unsigned flags = 0;
  unsigned long long first = 0;
  long long ndiag = 0;
  scs_int Anz;
  if (!A) { printf("A matrix missing\n"); return -1; }
  if (A->m <= 0 || A->n <= 0) { printf("A matrix dimensions must be positive\n"); return -1; }
  if (!A->x || !A->i || !A->p) { printf("data incompletely specified\n"); return -1; }
  Anz = b200_read_dev_int(A->p + A->n);
  dm->Ap = (int *)b200_malloc(((size_t)A->n + 1) * 4);
  if (!dm->Ap || b200_csc_check_ptrs((int)A->n, (long long)Anz, A->p, idx64, dm->Ap, &flags) != 0) return -1;
  if (flags & B200_CSC_BAD_P0) { printf("A->p[0] must equal 0\n"); return -1; }
  if (b200_over_stored("nnz(A) = A->p[n]", Anz)) return -1;
  if (flags & B200_CSC_BAD_PTR) { printf("A->p (column pointers) must be nonnegative and nondecreasing\n"); return -1; }
  if (((double)Anz / A->m > A->n) || Anz < 0) {
    printf("Anz (nonzeros in A) = %li, outside of valid range\n", (long)Anz);
    return -1;
  }
  dm->nnzA = Anz;
  dm->Ai = (int *)b200_malloc((size_t)Anz * 4);
  dm->Ax = (double *)b200_malloc((size_t)Anz * 8);
  if (!dm->Ai || !dm->Ax ||
      b200_csc_copy_entries((int)A->m, (int)A->n, Anz, A->i, A->x, idx64, dm->Ap, 0, dm->Ai, dm->Ax, &first, &ndiag) != 0)
    return -1;
  if (first != ~0ULL) {
    const long long kk = (long long)(first >> 2);
    if ((first & 3) == B200_CSC_BAD_ROW) {
      printf("A row index %li outside valid range [0, %li]\n", (long)b200_read_dev_int(A->i + kk), (long)A->m - 1);
    } else {
      printf("A contains a non-finite entry\n");
    }
    return -1;
  }
  if (P) {
    scs_int Pnz;
    if (!P->x || !P->i || !P->p) { printf("P matrix incompletely specified\n"); return -1; }
    if (P->n != A->n) { printf("P dimension inconsistent with n\n"); return -1; }
    if (P->m != P->n) { printf("P is not square\n"); return -1; }
    Pnz = b200_read_dev_int(P->p + P->n);
    dm->Pp = (int *)b200_malloc(((size_t)P->n + 1) * 4);
    if (!dm->Pp || b200_csc_check_ptrs((int)P->n, (long long)Pnz, P->p, idx64, dm->Pp, &flags) != 0) return -1;
    if (flags & B200_CSC_BAD_P0) { printf("P->p[0] must equal 0\n"); return -1; }
    if (b200_over_stored("nnz(P) = P->p[n]", Pnz)) return -1;
    if (flags & B200_CSC_BAD_PTR) { printf("P->p (column pointers) must be nonnegative and nondecreasing\n"); return -1; }
    if (((double)Pnz / P->m > P->n) || Pnz < 0) { printf("Pnz outside of valid range\n"); return -1; }
    dm->nnzP = Pnz;
    dm->Pi = (int *)b200_malloc((size_t)Pnz * 4);
    dm->Px = (double *)b200_malloc((size_t)Pnz * 8);
    if (!dm->Pi || !dm->Px ||
        b200_csc_copy_entries((int)P->n, (int)P->n, Pnz, P->i, P->x, idx64, dm->Pp, 1, dm->Pi, dm->Px, &first,
                              &ndiag) != 0)
      return -1;
    if (first != ~0ULL) {
      const int code = (int)(first & 3);
      printf(code == B200_CSC_BAD_ROW ? "P row index outside valid range\n"
             : code == B200_CSC_BAD_UPPER ? "P is not upper triangular\n" : "P contains a non-finite entry\n");
      return -1;
    }
    dm->fullP = 2 * (long long)Pnz - ndiag;
    if (b200_over_stored("stored entries of the full symmetric P", dm->fullP)) return -1;
  }
  return 0;
}

/* Both resident orientations of an m x n host CSC (*A_out = the m x n operator, *At_out = the n x m one): one upload,
 * then the device builder */
static int ops_from_host(int m, int n, const void *p, const void *i, const double *x, int idx64, B200Spmv **A_out,
                         B200Spmv **At_out) {
  int *d_p, *d_i;
  double *d_x;
  long long nnz;
  int rc;
  *A_out = *At_out = NULL;
  if (b200_csc_upload("A", m, n, p, i, x, idx64, 0, &d_p, &d_i, &d_x, &nnz, NULL) != 0) return -1;
  rc = b200_setup_ops_from_dev(m, n, nnz, d_p, d_i, d_x, A_out, At_out);
  b200_free(d_p); b200_free(d_i); b200_free(d_x); /* stream-ordered */
  return rc;
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

static int linsys_vectors(ScsLinSysWork *w, const scs_float *diag_r, int diag_on_dev, double *t_mark_p);

/* P's operator and diagonal (w->P, w->d_Pdiag) from its upper CSC in the builder's validated device arrays (nnzP
 * entries; `full` stored entries once expanded to the full symmetric P). The structure's blocks are freed here,
 * stream-ordered. */
static int p_from_dev_csc(ScsLinSysWork *w, long long nnzP, long long full, const int *Pp, const int *Pi,
                          const double *Px) {
  const int n = w->n;
  int *Fp = (int *)b200_malloc(((size_t)n + 1) * 4);
  int *Fi = (int *)b200_malloc((size_t)full * 4);
  int *Fsrc = (int *)b200_malloc((size_t)full * 4);
  int rc = -1;
  w->d_Pdiag = (double *)b200_malloc((size_t)n * 8);
  if (Fp && Fi && Fsrc && w->d_Pdiag && b200_sym_expand_structure(n, nnzP, full, Pp, Pi, Fp, Fi, Fsrc) == 0 &&
      b200_sym_build(n, full, Fp, Fi, Fsrc, Px, w->d_Pdiag, &w->P) == 0)
    rc = 0;
  b200_free(Fp); b200_free(Fi); b200_free(Fsrc);
  return rc;
}

static ScsLinSysWork *init_lin_sys_work(const ScsMatrix *A, const ScsMatrix *P, const scs_float *diag_r) {
  ScsLinSysWork *w;
  double t_mark = wall_ms();
  int *Lp = NULL, *Li = NULL;
  double *Lx = NULL;
  const int idx64 = sizeof(scs_int) == 8;
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
  w->ctx = b200_ctx_bound();
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
      const int rc = ops_from_host(w->mloc, n, Lp, Li, Lx, 0, &w->A, &w->At);
      free(Lp); free(Li); free(Lx);
      if (rc != 0) goto fail;
    }
  } else if (ops_from_host(m, n, A->p, A->i, A->x, idx64, &w->A, &w->At) != 0) {
    goto fail;
  }
  setup_mark("linsys: both operators built on the device", &t_mark);
  if (P) { /* replicated on every rank: the upper CSC uploaded, then expanded to the full symmetric P on the device */
    int *Pp = NULL, *Pi = NULL;
    double *Px = NULL;
    long long nnzP = 0, ndiag = 0, full;
    int rc = -1;
    if (b200_csc_upload("P", n, n, P->p, P->i, P->x, idx64, 1, &Pp, &Pi, &Px, &nnzP, &ndiag) != 0) goto fail;
    full = 2 * nnzP - ndiag;
    if (full > B200_MAX_STORED)
      fprintf(stderr, "scs_b200: the full symmetric P has %lld stored entries, above the limit 2^31 - 129 of one "
              "operator\n", full);
    else
      rc = p_from_dev_csc(w, nnzP, full, Pp, Pi, Px);
    b200_free(Pp); b200_free(Pi); b200_free(Px); /* stream-ordered */
    if (rc != 0) goto fail;
    setup_mark("linsys: operator P (device expansion)", &t_mark);
  }
  if (linsys_vectors(w, diag_r, 0, &t_mark) != 0) goto fail;
  return w;
fail:
  fprintf(stderr, "scs_b200: init_lin_sys_work failed: %s\n", b200_last_error());
  scs_free_lin_sys_work(w);
  return SCS_NULL;
}

/* Inside scs_init the workspace shares the ScsWork's execution context; called as a plugin it gets one of its own, so
 * that linear-system workspaces of different threads solve on different streams. */
ScsLinSysWork *scs_init_lin_sys_work(const ScsMatrix *A, const ScsMatrix *P,
                                     const scs_float *diag_r) {
  B200Ctx *own = SCS_NULL, *prev = SCS_NULL;
  ScsLinSysWork *w;
  if (!b200_ctx_bound()) {
    own = b200_ctx_create();
    prev = b200_ctx_enter(own);
  }
  w = init_lin_sys_work(A, P, diag_r);
  if (w) w->own_ctx = own != SCS_NULL;
  if (own) {
    b200_ctx_leave(prev);
    if (!w) b200_ctx_release(own);
  }
  return w;
}

/* scs_init_lin_sys_work with A, P and diag_r in device memory (single GPU): scs_b200_init_device's validating copy
 * of the caller's CSC arrays, then the builder the host init runs on the blocks it uploads */
static ScsLinSysWork *init_lin_sys_work_device(const ScsMatrix *A, const ScsMatrix *P, const scs_float *d_diag_r,
                                               void *stream) {
  double t_mark = wall_ms();
  B200DevMats dm;
  ScsLinSysWork *w = SCS_NULL;
  memset(&dm, 0, sizeof(dm));
  if (!A) { printf("A matrix missing\n"); return SCS_NULL; }
  if (b200_runtime_init() != 0) {
    fprintf(stderr, "scs_b200: no usable sm_90 device: %s\n", b200_last_error());
    return SCS_NULL;
  }
  if (!b200_single_gpu() || b200_over_dim("A->m", -1, A->m) || b200_over_dim("A->n", -1, A->n)) return SCS_NULL;
  if ((A->p && !b200_dev_ptr_ok(A->p, "A->p")) || (A->i && !b200_dev_ptr_ok(A->i, "A->i")) ||
      (A->x && !b200_dev_ptr_ok(A->x, "A->x")) ||
      (P && ((P->p && !b200_dev_ptr_ok(P->p, "P->p")) || (P->i && !b200_dev_ptr_ok(P->i, "P->i")) ||
             (P->x && !b200_dev_ptr_ok(P->x, "P->x")))) ||
      !b200_dev_ptr_ok(d_diag_r, "diag_r"))
    return SCS_NULL;
  if (b200_wait_for_caller(stream) != 0) return SCS_NULL;
  if (b200_validate_matrix_dev(A, P, &dm) != 0) {
    printf("invalid linear system input data\n");
  } else if ((w = (ScsLinSysWork *)calloc(1, sizeof(ScsLinSysWork))) != SCS_NULL) {
    w->ctx = b200_ctx_bound();
    w->n = (int)A->n; w->m = (int)A->m;
    w->nnz = dm.nnzA;
    w->nranks = 1;
    w->mloc = w->m;
    if (b200_setup_ops_from_dev(w->m, w->n, dm.nnzA, dm.Ap, dm.Ai, dm.Ax, &w->A, &w->At) != 0 ||
        (P && p_from_dev_csc(w, dm.nnzP, dm.fullP, dm.Pp, dm.Pi, dm.Px) != 0) ||
        linsys_vectors(w, d_diag_r, 1, &t_mark) != 0) {
      fprintf(stderr, "scs_b200: init_lin_sys_work failed: %s\n", b200_last_error());
      scs_free_lin_sys_work(w);
      w = SCS_NULL;
    }
  }
  b200_sync(); /* the builder's blocks are free only once its kernels have run */
  b200_dev_mats_free(&dm);
  b200_caller_waits(stream);
  return w;
}
ScsLinSysWork *scs_b200_init_lin_sys_work_device(const ScsMatrix *A, const ScsMatrix *P, const scs_float *d_diag_r,
                                                 void *stream) {
  B200Ctx *own = SCS_NULL, *prev = SCS_NULL;
  ScsLinSysWork *w;
  if (!b200_ctx_bound()) {
    own = b200_ctx_create();
    prev = b200_ctx_enter(own);
  }
  w = init_lin_sys_work_device(A, P, d_diag_r, stream);
  if (w) w->own_ctx = own != SCS_NULL;
  if (own) {
    b200_ctx_leave(prev);
    if (!w) b200_ctx_release(own);
  }
  return w;
}

/* single GPU, from operators built on the device (the device-data entry points, host/scs_driver.c): the workspace takes
 * A, At, P and d_Pdiag over, also when it fails */
ScsLinSysWork *b200_linsys_from_ops(int m, int n, B200Spmv *A, B200Spmv *At, B200Spmv *P, double *d_Pdiag,
                                    const scs_float *diag_r) {
  double t_mark = wall_ms();
  ScsLinSysWork *w = (ScsLinSysWork *)calloc(1, sizeof(ScsLinSysWork));
  if (!w) {
    b200_spmv_destroy(A); b200_spmv_destroy(At); b200_spmv_destroy(P); b200_free(d_Pdiag);
    return SCS_NULL;
  }
  w->ctx = b200_ctx_bound();
  w->n = n; w->m = m;
  w->nnz = b200_spmv_nnz(At);
  w->nranks = 1;
  w->mloc = m;
  w->A = A; w->At = At; w->P = P; w->d_Pdiag = d_Pdiag;
  if (linsys_vectors(w, diag_r, 0, &t_mark) != 0) {
    fprintf(stderr, "scs_b200: init_lin_sys_work failed: %s\n", b200_last_error());
    scs_free_lin_sys_work(w);
    return SCS_NULL;
  }
  return w;
}

/* the work vectors, the preconditioner and the CG loop's reordered pair of a workspace whose operators are built;
 * diag_r (n + m) in host memory, or with diag_on_dev in device memory */
static int linsys_vectors(ScsLinSysWork *w, const scs_float *diag_r, int diag_on_dev, double *t_mark_p) {
  const int n = w->n, m = w->m;
  double t_mark = *t_mark_p;
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
    return -1;
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
    if (!w->cg.d_p2p_sig || b200_h2d(w->cg.d_p2p_sig, &sig, sizeof(sig)) != 0) return -1;
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
      if (!w->cg.d_p2p_route || b200_h2d(w->cg.d_p2p_route, &rt, sizeof(rt)) != 0) return -1;
    }
  }
  if (!w->cg.d_p) {
    w->cg.d_p = (double *)b200_malloc((size_t)n * 8);
    if (!w->cg.d_p) return -1;
  }
  if ((diag_on_dev ? b200_d2d(w->d_diag_r, diag_r, ((size_t)n + m) * 8)
                   : b200_h2d(w->d_diag_r, diag_r, ((size_t)n + m) * 8)) != 0)
    return -1;
  if (b200_cg_set_preconditioner(&w->cg, w->d_Pdiag) != 0) return -1;
  if (b200_cg_plan_k34(&w->cg) != 0) return -1;
  if (b200_sync() != 0) return -1;
  setup_mark("linsys: vectors, preconditioner", &t_mark);
  if (cg_ops_build(w) != 0 || cg_ops_refresh(w) != 0 || b200_sync() != 0) return -1;
  setup_mark("linsys: reordered pair for the CG operator", &t_mark);
  *t_mark_p = t_mark;
  return 0;
}

static void free_lin_sys_work(ScsLinSysWork *w) {
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
void scs_free_lin_sys_work(ScsLinSysWork *w) {
  B200Ctx *prev, *own;
  if (!w) return;
  own = w->own_ctx ? w->ctx : SCS_NULL;
  prev = b200_ctx_enter(w->ctx);
  free_lin_sys_work(w);
  b200_ctx_leave(prev);
  b200_ctx_release(own);
}

/* Row-sharded setup: D, E of the FULL matrix are computed on every rank from temporary full
 * copies (both orientations) on its GPU; the resident local blocks are then scaled once. */
int b200_linsys_full_equilibrate(const ScsMatrix *A, const int *bnd, int nbnd, double *d_D, double *d_E) {
  int rc = -1;
  double t_mark = wall_ms();
  B200Spmv *At = NULL, *Ar = NULL;
  if (ops_from_host((int)A->m, (int)A->n, A->p, A->i, A->x, sizeof(scs_int) == 8, &Ar, &At) == 0)
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
  int *hint = d_s ? &w->last_admm_its : &w->last_g_its; /* batching only: no result depends on it */
  int its;
  if (max_its > 2000000000LL) max_its = 2000000000LL;
  its = b200_cg_solve(&w->cg, d_b, d_s, tol, (int)max_its, *hint, d_tol);
  if (its < 0) return -1;
  *hint = its;
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

static void warn_tol(scs_float tol) {
  if (tol <= 0.) {
    fprintf(stderr, "Warning: tol = %4f <= 0, likely compiled without setting INDIRECT flag.\n",
            tol);
  }
}
static scs_int solve_lin_sys(ScsLinSysWork *w, scs_float *b, const scs_float *s, scs_float tol) {
  const size_t nm = (size_t)w->n + w->m;
  warn_tol(tol);
  if (b200_h2d(w->d_b, b, nm * 8) != 0) return -1;
  if (s && b200_h2d(w->d_s, s, (size_t)w->n * 8) != 0) return -1;
  if (b200_linsys_solve_dev(w, w->d_b, s ? w->d_s : NULL, tol, NULL) != 0) return -1;
  if (b200_d2h(b, w->d_b, nm * 8) != 0) return -1;
  if (b200_sync() != 0) return -1;
  return 0;
}
scs_int scs_solve_lin_sys(ScsLinSysWork *w, scs_float *b, const scs_float *s, scs_float tol) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_int rc = solve_lin_sys(w, b, s, tol);
  b200_ctx_leave(prev);
  return rc;
}

static scs_int update_lin_sys_diag_r(ScsLinSysWork *w, const scs_float *new_diag_r) {
  if (b200_h2d(w->d_diag_r, new_diag_r, ((size_t)w->n + w->m) * 8) != 0) return -1;
  if (b200_linsys_update_diag_r_dev(w, w->d_diag_r) != 0) return -1;
  return b200_sync() == 0 ? 0 : -1;
}
scs_int scs_update_lin_sys_diag_r(ScsLinSysWork *w, const scs_float *new_diag_r) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_int rc = update_lin_sys_diag_r(w, new_diag_r);
  b200_ctx_leave(prev);
  return rc;
}

/* The device twins (include/scs_b200.h group (3)): the host twin's device function on the caller's buffers, after
 * the argument checks, between b200_wait_for_caller and b200_caller_waits. */
static int device_call_ok(const ScsLinSysWork *w) {
  if (!w) { printf("ERROR: missing ScsLinSysWork input\n"); return 0; }
  return b200_single_gpu();
}

static scs_int solve_lin_sys_device(ScsLinSysWork *w, scs_float *d_b, const scs_float *d_s, scs_float tol,
                                    void *stream) {
  int rc;
  if (!b200_dev_ptr_ok(d_b, "b") || (d_s && !b200_dev_ptr_ok(d_s, "s")) ||
      b200_overlap("b", d_b, ((size_t)w->n + w->m) * 8, "s", d_s, (size_t)w->n * 8))
    return -1;
  if ((uintptr_t)d_b % 16 != 0) { /* the CG loop's update kernels read and write x two entries at a time */
    printf("ERROR: b must be 16-byte aligned\n");
    return -1;
  }
  warn_tol(tol);
  if (b200_wait_for_caller(stream) != 0) return -1;
  rc = b200_linsys_solve_dev(w, d_b, d_s, tol, NULL); /* returns once the host has read the CG count */
  b200_caller_waits(stream);
  return rc == 0 ? 0 : -1;
}
scs_int scs_b200_solve_lin_sys_device(ScsLinSysWork *w, scs_float *d_b, const scs_float *d_s, scs_float tol,
                                      void *stream) {
  B200Ctx *prev;
  scs_int rc;
  if (!device_call_ok(w)) return -1;
  prev = b200_ctx_enter(w->ctx);
  rc = solve_lin_sys_device(w, d_b, d_s, tol, stream);
  b200_ctx_leave(prev);
  return rc;
}

static scs_int update_lin_sys_diag_r_device(ScsLinSysWork *w, const scs_float *d_diag_r, void *stream) {
  int rc;
  if (!b200_dev_ptr_ok(d_diag_r, "diag_r")) return -1;
  if (b200_wait_for_caller(stream) != 0) return -1;
  rc = b200_linsys_update_diag_r_dev(w, d_diag_r); /* its classification of R_y reads 4 bytes back */
  b200_caller_waits(stream);
  return rc == 0 ? 0 : -1;
}
scs_int scs_b200_update_lin_sys_diag_r_device(ScsLinSysWork *w, const scs_float *d_diag_r, void *stream) {
  B200Ctx *prev;
  scs_int rc;
  if (!device_call_ok(w)) return -1;
  prev = b200_ctx_enter(w->ctx);
  rc = update_lin_sys_diag_r_device(w, d_diag_r, stream);
  b200_ctx_leave(prev);
  return rc;
}

scs_int scs_b200_linsys_last_cg_its(const ScsLinSysWork *w) { return w->last_cg_its; }
long long scs_b200_linsys_cg_batch_solves(const ScsLinSysWork *w) { return w->cg.k34_batch_solves; }
long long scs_b200_linsys_total_cg_its(const ScsLinSysWork *w) { return w->tot_cg_its; }

/* SCS_B200_G_REUSE=0 makes the ADMM driver's update_work re-solve g at every scs_solve, as the reference does, for A/B
 * runs (DESIGN.md section 3.2). Here rather than in the driver so that every library flavour exports what the header
 * declares, the plugin-only ones included */
scs_int scs_b200_g_reuse(void) {
  const char *e = getenv("SCS_B200_G_REUSE");
  return !(e && strcmp(e, "0") == 0);
}

/* the CG path counts of the last scs_solve (host/scs_driver.c fills them); here rather than in the driver for the same
 * reason as scs_b200_g_reuse */
scs_int scs_b200_cg_k34_paths(const ScsWork *w, long long out[2]) {
  if (!w || !out) return -1;
  out[0] = w->stat_k34[0];
  out[1] = w->stat_k34[1];
  return 0;
}

/* y (+)= M x on device vectors: accumulating, the chain of each row starts at y's own entry */
static int accum_dev(const B200Spmv *M, const double *d_x, double *d_y, scs_int accumulate) {
  B200SpmvArgs a;
  memset(&a, 0, sizeof(a));
  a.d_x = d_x; a.d_y = d_y; a.d_init = accumulate ? d_y : NULL; a.init_sign = 1.0;
  a.post = B200_POST_NONE; a.hook = B200_HOOK_NONE;
  return b200_spmv(M, &a);
}

static scs_int accum_generic(ScsLinSysWork *w, const B200Spmv *M, int ncols, int nrows,
                             const scs_float *x, scs_float *y, scs_int accumulate) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  double *d_x = (double *)b200_malloc((size_t)ncols * 8);
  double *d_y = (double *)b200_malloc((size_t)nrows * 8);
  int rc = -1;
  if (w->nranks > 1) goto out; /* operator-level API is single-GPU */
  if (!d_x || !d_y) goto out;
  if (b200_h2d(d_x, x, (size_t)ncols * 8) != 0) goto out;
  if (accumulate && b200_h2d(d_y, y, (size_t)nrows * 8) != 0) goto out;
  if (accum_dev(M, d_x, d_y, accumulate) != 0) goto out;
  if (b200_d2h(y, d_y, (size_t)nrows * 8) != 0) goto out;
  if (b200_sync() != 0) goto out;
  rc = 0;
out:
  b200_free(d_x);
  b200_free(d_y);
  b200_ctx_leave(prev);
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

/* enqueued only: the SpMV reports nothing, and the caller's stream waits for it */
static scs_int accum_device(ScsLinSysWork *w, int trans, const scs_float *d_x, scs_float *d_y, scs_int accumulate,
                            void *stream) {
  size_t ncols, nrows;
  B200Ctx *prev;
  int rc = -1;
  if (!device_call_ok(w)) return -1;
  ncols = (size_t)(trans ? w->m : w->n);
  nrows = (size_t)(trans ? w->n : w->m);
  prev = b200_ctx_enter(w->ctx);
  if (b200_dev_ptr_ok(d_x, "x") && b200_dev_ptr_ok(d_y, "y") && !b200_overlap("x", d_x, ncols * 8, "y", d_y, nrows * 8) &&
      b200_wait_for_caller(stream) == 0) {
    rc = accum_dev(trans ? w->At : w->A, d_x, d_y, accumulate) == 0 ? 0 : -1;
    b200_caller_waits(stream);
  }
  b200_ctx_leave(prev);
  return rc;
}
scs_int scs_b200_accum_by_a_device(ScsLinSysWork *w, const scs_float *d_x, scs_float *d_y, scs_int accumulate,
                                   void *stream) {
  return accum_device(w, 0, d_x, d_y, accumulate, stream);
}
scs_int scs_b200_accum_by_atrans_device(ScsLinSysWork *w, const scs_float *d_x, scs_float *d_y, scs_int accumulate,
                                        void *stream) {
  return accum_device(w, 1, d_x, d_y, accumulate, stream);
}

/* --- device timing helpers for bench.py (inputs resident in HBM) --------- */
double scs_b200_time_spmv(ScsLinSysWork *w, scs_int op, scs_int reps, double *alg_bytes) {
  double ms[2] = {-1.0, -1.0};
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const int rc = b200_spmv_time_pair(w->A, w->At, reps, ms);
  b200_ctx_leave(prev);
  if (rc != 0) return -1.0;
  if (alg_bytes) *alg_bytes = b200_spmv_alg_bytes(op == 0 ? w->A : w->At, 0);
  return ms[op == 0 ? 0 : 1];
}

/* bench.py roofline: the kernels of the CG loop as they run inside a solve (the solver's own p / tmp / r after
 * a genuine start on the right-hand side b, which the caller provides: length n + m, host). out_ms[0..4] = ms
 * per launch of K1, K2, K3, K4 and of the whole iteration; out_bytes[0..4] = the algorithmic bytes of each
 * (b200_cg_iter_alg_bytes, DESIGN.md section 3). */
static scs_int time_cg_kernels(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms,
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
/* the batch kernel's phases (b200_cg_time_batch) on the solver's own vectors after a genuine start on b (n + m, host) */
static scs_int time_cg_batch(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms) {
  const size_t nm = (size_t)w->n + w->m;
  if (b200_h2d(w->d_b, b, nm * 8) != 0) return -1;
  if (b200_cg_solve(&w->cg, w->d_b, NULL, 0.0, 1, 0, NULL) < 0) return -1;
  w->cg.h_ctl->done = 0;
  w->cg.h_ctl->max_its = 2000000000;
  if (b200_h2d(w->cg.d_ctl, w->cg.h_ctl, sizeof(B200CgCtl)) != 0) return -1;
  if (b200_cg_time_batch(&w->cg, w->d_b, 3, out_ms) != 0) return -1; /* warm-up */
  return b200_cg_time_batch(&w->cg, w->d_b, (int)reps, out_ms) == 0 ? 0 : -1;
}
scs_int scs_b200_time_cg_batch(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_int rc = time_cg_batch(w, b, reps, out_ms);
  b200_ctx_leave(prev);
  return rc;
}
scs_int scs_b200_time_cg_kernels(ScsLinSysWork *w, const scs_float *b, scs_int reps, double *out_ms,
                                 double *out_bytes) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_int rc = time_cg_kernels(w, b, reps, out_ms, out_bytes);
  b200_ctx_leave(prev);
  return rc;
}

static double time_cg_iter(ScsLinSysWork *w, scs_int reps, double *alg_bytes) {
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
double scs_b200_time_cg_iter(ScsLinSysWork *w, scs_int reps, double *alg_bytes) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const double ms = time_cg_iter(w, reps, alg_bytes);
  b200_ctx_leave(prev);
  return ms;
}

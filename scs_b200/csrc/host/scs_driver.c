/* scs_driver.c -- the public SCS ABI (scs_init / scs_update / scs_solve /
 * scs_finish / scs / scs_set_default_settings / scs_version) with a
 * DEVICE-RESIDENT ADMM loop.
 *
 * Host C orchestrates; every O(n+m) or O(nnz) operation of the iteration is a
 * hand-written sm_90a kernel (kernels/ *.cu) reached through the thin C layer
 * of dev_api.h / admm_api.h.  The host sees only scalars (CG flags every
 * iteration, 18 residual scalars every CONVERGED_INTERVAL iterations) and the
 * solution vectors once at the end.
 *
 * Follows, step by step, reference src/scs.c (v3.2.11):
 *   validate :376-451, init_work :982-1116, scs_update :1287-1325,
 *   update_work(_cache) :1118-1157, the iteration loop :1356-1455,
 *   populate_residual_struct :535-607 (+ compute_residuals :463-485,
 *   unnormalize_residuals :487-531), has_converged :611-649, update_scale
 *   :1164-1241, finalize :916-966 (+ set_solved/infeasible/unbounded/unfinished
 *   :847-913), failure :361-371.
 */
#include "driver.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ----------------------------------------------------------------- utils */
static double now_ms(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return 1e3 * (double)ts.tv_sec + 1e-6 * (double)ts.tv_nsec;
}

const char *scs_version(void) { return SCS_VERSION_STR; }

/* reference src/util.c:158-179, include/glbopts.h:35-50 */
void scs_set_default_settings(ScsSettings *stgs) {
  stgs->max_iters = 100000;
  stgs->eps_abs = 1e-4;
  stgs->eps_rel = 1e-4;
  stgs->eps_infeas = 1e-7;
  stgs->alpha = 1.5;
  stgs->rho_x = 1e-6;
  stgs->scale = 0.1;
  stgs->verbose = 1;
  stgs->normalize = 1;
  stgs->warm_start = 0;
  stgs->acceleration_lookback = 10;
  stgs->acceleration_interval = 10;
  stgs->acceleration_type_1 = 1;
  stgs->acceleration_regularization = 1e-8;
  stgs->acceleration_relaxation = 1.0;
  stgs->adaptive_scale = 1;
  stgs->write_data_filename = SCS_NULL;
  stgs->log_csv_filename = SCS_NULL;
  stgs->time_limit_secs = 0.;
}

/* ----------------------------------------------------------------- validation */
/* Every count is read in scs_int width: nnz(A) is checked against the operator limit before i[] or x[] is read, and a
 * 64-bit index that would truncate to a valid int (2^32 + 3 -> 3) fails the range checks. */
static int validate_matrix(const ScsMatrix *A, const ScsMatrix *P) {
  scs_int i, j, Anz;
  if (!A) { printf("A matrix missing\n"); return -1; }
  if (A->m <= 0 || A->n <= 0) { printf("A matrix dimensions must be positive\n"); return -1; }
  if (!A->x || !A->i || !A->p) { printf("data incompletely specified\n"); return -1; }
  if (A->p[0] != 0) { printf("A->p[0] must equal 0\n"); return -1; }
  if (b200_over_stored("nnz(A) = A->p[n]", A->p[A->n])) return -1;
  for (j = 0; j < A->n; ++j)
    if (A->p[j] < 0 || A->p[j] > A->p[j + 1]) {
      printf("A->p (column pointers) must be nonnegative and nondecreasing\n");
      return -1;
    }
  Anz = A->p[A->n];
  if (((double)Anz / A->m > A->n) || Anz < 0) {
    printf("Anz (nonzeros in A) = %li, outside of valid range\n", (long)Anz);
    return -1;
  }
  for (i = 0; i < Anz; ++i) {
    if (A->i[i] < 0 || A->i[i] >= A->m) {
      printf("A row index %li outside valid range [0, %li]\n", (long)A->i[i], (long)A->m - 1);
      return -1;
    }
    if (!isfinite(A->x[i])) { printf("A contains a non-finite entry\n"); return -1; }
  }
  if (P) {
    scs_int Pnz;
    long long full = 0; /* stored entries of the full symmetric P */
    if (!P->x || !P->i || !P->p) { printf("P matrix incompletely specified\n"); return -1; }
    if (P->n != A->n) { printf("P dimension inconsistent with n\n"); return -1; }
    if (P->m != P->n) { printf("P is not square\n"); return -1; }
    if (P->p[0] != 0) { printf("P->p[0] must equal 0\n"); return -1; }
    if (b200_over_stored("nnz(P) = P->p[n]", P->p[P->n])) return -1;
    for (j = 0; j < P->n; ++j)
      if (P->p[j] < 0 || P->p[j] > P->p[j + 1]) {
        printf("P->p (column pointers) must be nonnegative and nondecreasing\n");
        return -1;
      }
    Pnz = P->p[P->n];
    if (((double)Pnz / P->m > P->n) || Pnz < 0) { printf("Pnz outside of valid range\n"); return -1; }
    for (j = 0; j < P->n; j++)
      for (i = P->p[j]; i < P->p[j + 1]; i++) {
        if (P->i[i] < 0 || P->i[i] >= P->n) { printf("P row index outside valid range\n"); return -1; }
        if (P->i[i] > j) { printf("P is not upper triangular\n"); return -1; }
        if (!isfinite(P->x[i])) { printf("P contains a non-finite entry\n"); return -1; }
        full += P->i[i] == j ? 1 : 2;
      }
    if (b200_over_stored("stored entries of the full symmetric P", full)) return -1;
  }
  return 0;
}

/* the same blocks from a host A and P that validate_matrix has accepted (scs_init on one GPU) */
static int dev_mats_from_host(const ScsMatrix *A, const ScsMatrix *P, B200DevMats *dm) {
  const int idx64 = sizeof(scs_int) == 8;
  long long ndiag = 0;
  if (b200_csc_upload("A", (int)A->m, (int)A->n, A->p, A->i, A->x, idx64, 0, &dm->Ap, &dm->Ai, &dm->Ax, &dm->nnzA,
                      SCS_NULL) != 0)
    return -1;
  if (P) {
    if (b200_csc_upload("P", (int)P->n, (int)P->n, P->p, P->i, P->x, idx64, 1, &dm->Pp, &dm->Pi, &dm->Px, &dm->nnzP,
                        &ndiag) != 0)
      return -1;
    dm->fullP = 2 * dm->nnzP - ndiag;
  }
  return 0;
}
static int validate(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, B200DevMats *dm) {
  if (d->m <= 0 || d->n <= 0) {
    printf("m and n must both be greater than 0; m = %li, n = %li\n", (long)d->m, (long)d->n);
    return -1;
  }
  if (b200_over_dim("m", -1, d->m) || b200_over_dim("n", -1, d->n)) return -1;
  if (d->A && (d->A->m != d->m || d->A->n != d->n)) {
    printf("A dimensions inconsistent with m, n\n");
    return -1;
  }
  if (!d->b || !d->c) { printf("b or c missing\n"); return -1; }
  if ((dm ? b200_validate_matrix_dev(d->A, d->P, dm) : validate_matrix(d->A, d->P)) < 0) {
    printf("invalid linear system input data\n");
    return -1;
  }
  if (b200_validate_cones(k, d->m) < 0) { printf("cone validation error\n"); return -1; }
  if (stgs->max_iters <= 0) { printf("max_iters must be positive\n"); return -1; }
  if (!isfinite(stgs->eps_abs) || stgs->eps_abs < 0) { printf("eps_abs tolerance must be a nonnegative finite number\n"); return -1; }
  if (!isfinite(stgs->eps_rel) || stgs->eps_rel < 0) { printf("eps_rel tolerance must be a nonnegative finite number\n"); return -1; }
  if (!isfinite(stgs->eps_infeas) || stgs->eps_infeas < 0) { printf("eps_infeas tolerance must be a nonnegative finite number\n"); return -1; }
  if (!isfinite(stgs->alpha) || stgs->alpha <= 0 || stgs->alpha >= 2) { printf("alpha must be in (0,2)\n"); return -1; }
  if (!isfinite(stgs->rho_x) || stgs->rho_x <= 0) { printf("rho_x must be a positive finite number (1e-3 works well).\n"); return -1; }
  if (!isfinite(stgs->scale) || stgs->scale <= 0) { printf("scale must be a positive finite number (1 works well).\n"); return -1; }
  if (!isfinite(stgs->time_limit_secs) || stgs->time_limit_secs < 0) { printf("time_limit_secs must be a nonnegative finite number.\n"); return -1; }
  if (stgs->acceleration_interval <= 0) { printf("acceleration_interval must be positive (10 works well).\n"); return -1; }
  if (stgs->acceleration_lookback < 0) { printf("acceleration_lookback must be nonnegative\n"); return -1; }
  if (b200_over_dim("acceleration_lookback", -1, stgs->acceleration_lookback)) return -1;
  if (!isfinite(stgs->acceleration_regularization) || stgs->acceleration_regularization < 0) {
    printf("acceleration_regularization must be a nonnegative finite number.\n");
    return -1;
  }
  if (!isfinite(stgs->acceleration_relaxation) || stgs->acceleration_relaxation < 0 ||
      stgs->acceleration_relaxation > 2) {
    printf("acceleration_relaxation must be in [0, 2].\n");
    return -1;
  }
  return 0;
}

/* ----------------------------------------------------------------- deep copies */
static ScsMatrix *copy_matrix(const ScsMatrix *src) {
  ScsMatrix *A;
  scs_int nz;
  if (!src) return SCS_NULL;
  nz = src->p[src->n];
  A = (ScsMatrix *)calloc(1, sizeof(ScsMatrix));
  if (!A) return SCS_NULL;
  A->n = src->n; A->m = src->m;
  A->x = (double *)malloc(((size_t)nz + 1) * sizeof(double));
  A->i = (scs_int *)malloc(((size_t)nz + 1) * sizeof(scs_int));
  A->p = (scs_int *)malloc(((size_t)src->n + 1) * sizeof(scs_int));
  if (!A->x || !A->i || !A->p) { free(A->x); free(A->i); free(A->p); free(A); return SCS_NULL; }
  memcpy(A->x, src->x, (size_t)nz * sizeof(double));
  memcpy(A->i, src->i, (size_t)nz * sizeof(scs_int));
  memcpy(A->p, src->p, ((size_t)src->n + 1) * sizeof(scs_int));
  return A;
}
static void free_matrix(ScsMatrix *A) {
  if (A) { free(A->x); free(A->i); free(A->p); free(A); }
}
static void *dup_mem(const void *src, size_t bytes) {
  void *p;
  if (!src || bytes == 0) return SCS_NULL;
  p = malloc(bytes);
  if (p) memcpy(p, src, bytes);
  return p;
}

/* ----------------------------------------------------------------- workspace */
/* SCS_B200_SETUP_TIMING=1: wall-clock breakdown of scs_init / scs_finish on stderr (syncs the stream at every mark) */
static void init_mark(const char *what, double *t_last) {
  if (!getenv("SCS_B200_SETUP_TIMING")) return;
  b200_sync();
  {
    const double t = now_ms();
    fprintf(stderr, "scs_b200 setup: %-44s %8.1f ms\n", what, t - *t_last);
    *t_last = t;
  }
}

static void finish_work(ScsWork *w) {
  double t_mark = now_ms();
  b200_sync();
  init_mark("finish: stream drained", &t_mark);
  if (w->log_csv_fout) fclose(w->log_csv_fout);
  free(w->log_csv_name);
  free(w->log_host);
  if (w->cones) b200_cones_destroy(w->cones);
  init_mark("finish: cones", &t_mark);
  if (w->p) scs_free_lin_sys_work(w->p);
  init_mark("finish: linear-system workspace", &t_mark);
  if (w->accel) b200_aa_destroy(w->accel);
  init_mark("finish: acceleration workspace", &t_mark);
  b200_free(w->adm.d_u); b200_free(w->adm.d_u_t); b200_free(w->adm.d_v); b200_free(w->adm.d_v_prev);
  b200_free(w->adm.d_rsk); b200_free(w->adm.d_g); b200_free(w->adm.d_R); b200_free(w->adm.d_ws);
  b200_free(w->adm.d_sc); b200_free(w->adm.d_part); b200_free(w->adm.d_cnt);
  b200_free(w->d_b); b200_free(w->d_c); b200_free(w->d_D); b200_free(w->d_E);
  b200_free(w->d_ax); b200_free(w->d_aty); b200_free(w->d_px);
  b200_free(w->d_sol_x); b200_free(w->d_sol_y); b200_free(w->d_sol_s);
  b200_free(w->d_b_orig); b200_free(w->d_c_orig);
  init_mark("finish: device vectors", &t_mark);
  b200_host_free(w->h_sc);
  init_mark("finish: pinned scalars", &t_mark);
  free(w->D); free(w->E); free(w->h_diag_r);
  free(w->cone_boundaries);
  free(w->bl_orig); free(w->bu_orig);
  if (w->d) {
    free_matrix(w->d->A); free_matrix(w->d->P); free(w->d);
  }
  if (w->k) {
    free(w->k->bu); free(w->k->bl); free(w->k->q); free(w->k->s); free(w->k->p); free(w->k->cs);
#ifdef USE_SPECTRAL_CONES
    free(w->k->d); free(w->k->nuc_m); free(w->k->nuc_n); free(w->k->ell1); free(w->k->sl_n); free(w->k->sl_k);
#endif
    free(w->k);
  }
  free(w->stgs);
  free(w);
  init_mark("finish: host copies", &t_mark);
}
void scs_finish(ScsWork *w) {
  B200Ctx *ctx, *prev;
  if (!w) return;
  ctx = w->ctx;
  prev = b200_ctx_enter(ctx);
  finish_work(w);
  b200_ctx_leave(prev);
  b200_ctx_release(ctx); /* its stream has drained: the blocks freed under it join the shared pool */
}

static void set_diag_r_host(ScsWork *w) {
  int i, n = w->n, m = w->m;
  for (i = 0; i < n; ++i) w->h_diag_r[i] = w->stgs->rho_x;
  for (i = 0; i < w->k->z; ++i) w->h_diag_r[n + i] = 1.0 / (1000. * w->stgs->scale);
  for (i = w->k->z; i < m; ++i) w->h_diag_r[n + i] = 1.0 / w->stgs->scale;
  w->h_diag_r[n + m] = TAU_FACTOR;
}

static int set_cone_boundaries(ScsWork *w) {
  const ScsCone *k = w->k;
  int i, count = 0;
  int total = k->qsize + k->ssize + k->cssize + k->ep + k->ed + k->psize;
  int *b;
#ifdef USE_SPECTRAL_CONES
  total += k->dsize + k->nucsize + k->ell1_size + k->sl_size;
#endif
  b = (int *)calloc((size_t)total + 1, sizeof(int));
  if (!b) return -1;
  b[count++] = k->z + k->l + k->bsize;
  for (i = 0; i < k->qsize; ++i) b[count++] = k->q[i];
  for (i = 0; i < k->ssize; ++i) b[count++] = k->s[i] * (k->s[i] + 1) / 2;
  for (i = 0; i < k->cssize; ++i) b[count++] = k->cs[i] * k->cs[i];
  for (i = 0; i < k->ep + k->ed + k->psize; ++i) b[count++] = 3; /* every triple shares one D (cones.c:405-408) */
#ifdef USE_SPECTRAL_CONES /* one D value per spectral cone (cones.c:411-419) */
  for (i = 0; i < k->dsize; ++i) b[count++] = k->d[i] * (k->d[i] + 1) / 2 + 2;
  for (i = 0; i < k->nucsize; ++i) b[count++] = k->nuc_m[i] * k->nuc_n[i] + 1;
  for (i = 0; i < k->ell1_size; ++i) b[count++] = k->ell1[i] + 1;
  for (i = 0; i < k->sl_size; ++i) b[count++] = k->sl_n[i] * (k->sl_n[i] + 1) / 2 + 1;
#endif
  w->cone_boundaries = b;
  w->cone_boundaries_len = total + 1;
  return 0;
}

static int update_bc_dev(ScsWork *w);
/* the originals given (NULL: the resident one is kept) uploaded, then normalised on the device like every door's */
scs_int scs_update(ScsWork *w, scs_float *b, scs_float *c) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  scs_int rc = -1;
  if ((!b || b200_h2d(w->d_b_orig, b, (size_t)w->m * 8) == 0) &&
      (!c || b200_h2d(w->d_c_orig, c, (size_t)w->n * 8) == 0))
    rc = update_bc_dev(w);
  b200_ctx_leave(prev);
  return rc;
}

static void print_header(const ScsWork *w) {
  const ScsCone *k = w->k;
  int i;
  for (i = 0; i < 78; ++i) printf("-");
  printf("\n\t       SCS hot path on H100 (scs_b200 %s, API of SCS 3.2.11)\n", SCS_VERSION_STR);
  for (i = 0; i < 78; ++i) printf("-");
  printf("\nproblem:  variables n: %i, constraints m: %i\n", w->n, w->m);
  printf("cones: \t  z: %i, l: %i, b: %i, q: %i cones, s: %i cones, exp: %i + %i dual, pow: %i\n", (int)k->z,
         (int)k->l, (int)k->bsize, (int)k->qsize, (int)k->ssize, (int)k->ep, (int)k->ed, (int)k->psize);
  printf("settings: eps_abs: %.1e, eps_rel: %.1e, eps_infeas: %.1e\n\t  alpha: %.2f, scale: %.2e, "
         "adaptive_scale: %lli\n\t  max_iters: %lli, normalize: %lli, rho_x: %.2e\n",
         w->stgs->eps_abs, w->stgs->eps_rel, w->stgs->eps_infeas, w->stgs->alpha, w->stgs->scale,
         (long long)w->stgs->adaptive_scale, (long long)w->stgs->max_iters, (long long)w->stgs->normalize,
         w->stgs->rho_x);
  if (w->stgs->acceleration_lookback)
    printf("\t  acceleration_lookback: %lli, acceleration_interval: %lli\n",
           (long long)w->stgs->acceleration_lookback, (long long)w->stgs->acceleration_interval);
  printf("lin-sys:  %s\n\t  nnz(A): %li, nnz(P): %li\n", scs_get_lin_sys_method(),
         (long)w->nnzA, (long)w->nnzP);
}

static int build_ops_dev(ScsWork *w, B200DevMats *dm);
static void write_data_dev(const char *filename, const ScsData *d, const ScsCone *k, const ScsSettings *stgs);

/* dev_data: the device-data entry point, d's arrays are device pointers, validated into dm's blocks; else scs_init,
 * the data in host memory, validated there. On one GPU (dm != NULL) the operators are built on the device from dm's
 * blocks (build_ops_dev), which scs_init fills from the host A and P. Several GPUs (dm == NULL, scs_init only) cut A
 * into row blocks on the host (scs_init_lin_sys_work). */
static ScsWork *init_work(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, B200DevMats *dm, int dev_data,
                          B200Ctx *ctx) {
  ScsWork *w;
  const double t0 = now_ms();
  double t_mark = t0;
  int n, m, i, host_copy;
  size_t l;
  if (!d || !k || !stgs) {
    printf("ERROR: Missing ScsData, ScsCone, or ScsSettings input\n");
    return SCS_NULL;
  }
  if (validate(d, k, stgs, dev_data ? dm : SCS_NULL) < 0) {
    printf("ERROR: Validation returned failure\n");
    return SCS_NULL;
  }
  if (b200_runtime_init() != 0) {
    printf("ERROR: scs_b200 needs an sm_90 (H100) CUDA device: %s\n", b200_last_error());
    return SCS_NULL;
  }
  if (!ctx) {
    printf("ERROR: could not create the workspace's stream: %s\n", b200_last_error());
    return SCS_NULL;
  }
  if (stgs->write_data_filename) { /* reference scs.c:1270-1273 */
    printf("Writing raw problem data to %s\n", stgs->write_data_filename);
    if (dev_data) write_data_dev(stgs->write_data_filename, d, k, stgs);
    else scs_b200_write_data(stgs->write_data_filename, d, k, stgs);
  }
  w = (ScsWork *)calloc(1, sizeof(ScsWork));
  if (!w) return SCS_NULL;
  w->ctx = ctx;
  n = w->n = d->n;
  m = w->m = d->m;
  l = (size_t)n + m + 1;
  /* deep copies */
  w->d = (ScsData *)calloc(1, sizeof(ScsData));
  w->k = (ScsCone *)calloc(1, sizeof(ScsCone));
  w->stgs = (ScsSettings *)calloc(1, sizeof(ScsSettings));
  if (!w->d || !w->k || !w->stgs) goto fail;
  w->d->n = n; w->d->m = m;
  w->nnzA = dev_data ? dm->nnzA : d->A->p[n];
  w->nnzP = dev_data ? dm->nnzP : d->P ? d->P->p[n] : 0;
  /* the equilibration, for init and for scs_b200_update_matrix_device. One GPU: on the device, the pair of A alone
   * (P = 0) or with P (b200_equilibrate_qp_dev), so no host copy of A or P is made. Several GPUs: with P = 0 on the
   * device from temporary full copies of A; otherwise (P != 0, or no equilibration) from a host copy of A and P,
   * equilibrated there (host/equilibrate.c) */
  w->equil = !stgs->normalize ? B200_EQUIL_NONE : d->P ? B200_EQUIL_QP : B200_EQUIL_PAIR;
  host_copy = !dm && w->equil != B200_EQUIL_PAIR;
  w->scale0 = stgs->scale;
  if (host_copy) {
    w->d->A = copy_matrix(d->A);
    w->d->P = d->P ? copy_matrix(d->P) : SCS_NULL;
    if (!w->d->A || (d->P && !w->d->P)) goto fail;
  }
  *w->k = *k;
  w->k->bu = w->k->bl = SCS_NULL; w->k->q = SCS_NULL; w->k->s = SCS_NULL;
  w->k->cs = SCS_NULL; w->k->p = SCS_NULL;
#ifdef USE_SPECTRAL_CONES
  w->k->d = SCS_NULL; w->k->nuc_m = w->k->nuc_n = SCS_NULL; w->k->ell1 = SCS_NULL; w->k->sl_n = w->k->sl_k = SCS_NULL;
#endif
  if (k->bsize > 1) {
    w->k->bu = (double *)dup_mem(k->bu, (size_t)(k->bsize - 1) * 8);
    w->k->bl = (double *)dup_mem(k->bl, (size_t)(k->bsize - 1) * 8);
    w->bu_orig = (double *)dup_mem(k->bu, (size_t)(k->bsize - 1) * 8);
    w->bl_orig = (double *)dup_mem(k->bl, (size_t)(k->bsize - 1) * 8);
    if (!w->k->bu || !w->k->bl || !w->bu_orig || !w->bl_orig) goto fail;
  }
  if (k->qsize > 0) { w->k->q = (scs_int *)dup_mem(k->q, (size_t)k->qsize * sizeof(scs_int)); if (!w->k->q) goto fail; }
  if (k->psize > 0) { w->k->p = (double *)dup_mem(k->p, (size_t)k->psize * 8); if (!w->k->p) goto fail; }
  if (k->cssize > 0) { w->k->cs = (scs_int *)dup_mem(k->cs, (size_t)k->cssize * sizeof(scs_int)); if (!w->k->cs) goto fail; }
  if (k->ssize > 0) { w->k->s = (scs_int *)dup_mem(k->s, (size_t)k->ssize * sizeof(scs_int)); if (!w->k->s) goto fail; }
#ifdef USE_SPECTRAL_CONES
  if (k->dsize > 0) { w->k->d = (scs_int *)dup_mem(k->d, (size_t)k->dsize * sizeof(scs_int)); if (!w->k->d) goto fail; }
  if (k->nucsize > 0) {
    w->k->nuc_m = (scs_int *)dup_mem(k->nuc_m, (size_t)k->nucsize * sizeof(scs_int));
    w->k->nuc_n = (scs_int *)dup_mem(k->nuc_n, (size_t)k->nucsize * sizeof(scs_int));
    if (!w->k->nuc_m || !w->k->nuc_n) goto fail;
  }
  if (k->ell1_size > 0) { w->k->ell1 = (scs_int *)dup_mem(k->ell1, (size_t)k->ell1_size * sizeof(scs_int)); if (!w->k->ell1) goto fail; }
  if (k->sl_size > 0) {
    w->k->sl_n = (scs_int *)dup_mem(k->sl_n, (size_t)k->sl_size * sizeof(scs_int));
    w->k->sl_k = (scs_int *)dup_mem(k->sl_k, (size_t)k->sl_size * sizeof(scs_int));
    if (!w->k->sl_n || !w->k->sl_k) goto fail;
  }
#endif
  *w->stgs = *stgs;
  w->stgs->write_data_filename = SCS_NULL;
  w->stgs->log_csv_filename = SCS_NULL;
  if (stgs->log_csv_filename) { /* reference scs.c:1275-1278; the file is opened by every scs_solve */
    printf("Logging run data to %s\n", stgs->log_csv_filename);
    w->log_csv_name = (char *)dup_mem(stgs->log_csv_filename, strlen(stgs->log_csv_filename) + 1);
    if (!w->log_csv_name) goto fail;
  }
  if (w->stgs->verbose) print_header(w);

  w->h_diag_r = (double *)malloc(l * 8);
  if (!w->h_diag_r) goto fail;
  if (set_cone_boundaries(w) != 0) goto fail;
  set_diag_r_host(w);

  /* equilibrate A, P on the host copy (setup) */
  w->primal_scale = w->dual_scale = 1.0;
  if (w->stgs->normalize) {
    w->D = (double *)malloc((size_t)m * 8);
    w->E = (double *)malloc((size_t)n * 8);
    if (!w->D || !w->E) goto fail;
    if (host_copy) {
      if (b200_equilibrate(w->d->P, w->d->A, w->cone_boundaries, w->cone_boundaries_len, w->D, w->E) != 0)
        goto fail;
      b200_normalize_box(w->k, w->D, w->k->bl, w->k->bu);
    }
  }

  /* device state */
  w->adm.n = n; w->adm.m = m;
  w->adm.d_u = (double *)b200_malloc(l * 8);
  w->adm.d_u_t = (double *)b200_malloc(l * 8);
  w->adm.d_v = (double *)b200_malloc(l * 8);
  w->adm.d_v_prev = (double *)b200_malloc(l * 8);
  w->adm.d_rsk = (double *)b200_malloc(l * 8);
  w->adm.d_g = (double *)b200_malloc(l * 8);
  w->adm.d_R = (double *)b200_malloc(l * 8);
  w->adm.d_ws = (double *)b200_malloc((size_t)n * 8);
  w->adm.d_sc = (double *)b200_malloc(SC_COUNT * 8);
  w->adm.d_part = (double *)b200_malloc(8 * 2048 * 8);
  w->adm.d_cnt = (unsigned int *)b200_malloc(64);
  w->d_b = (double *)b200_malloc((size_t)m * 8);
  w->d_c = (double *)b200_malloc((size_t)n * 8);
  w->d_ax = (double *)b200_malloc((size_t)m * 8);
  w->d_aty = (double *)b200_malloc((size_t)n * 8);
  w->d_px = d->P ? (double *)b200_malloc((size_t)n * 8) : SCS_NULL;
  w->d_sol_x = (double *)b200_malloc((size_t)n * 8);
  w->d_sol_y = (double *)b200_malloc((size_t)m * 8);
  w->d_sol_s = (double *)b200_malloc((size_t)m * 8);
  w->h_sc = (double *)b200_host_alloc(SC_COUNT * 8);
  if (!w->adm.d_u || !w->adm.d_u_t || !w->adm.d_v || !w->adm.d_v_prev || !w->adm.d_rsk ||
      !w->adm.d_g || !w->adm.d_R || !w->adm.d_ws || !w->adm.d_sc || !w->adm.d_part ||
      !w->adm.d_cnt || !w->d_b || !w->d_c || !w->d_ax || !w->d_aty || (d->P && !w->d_px) ||
      !w->d_sol_x || !w->d_sol_y || !w->d_sol_s || !w->h_sc) {
    printf("ERROR: device memory allocation failure: %s\n", b200_last_error());
    goto fail;
  }
  i = 0;
  i |= b200_memset0(w->adm.d_cnt, 64);
  i |= b200_memset0(w->adm.d_sc, SC_COUNT * 8);
  i |= b200_memset0(w->adm.d_u, l * 8);
  i |= b200_memset0(w->adm.d_u_t, l * 8);
  i |= b200_memset0(w->adm.d_v, l * 8);
  i |= b200_memset0(w->adm.d_v_prev, l * 8);
  i |= b200_memset0(w->adm.d_rsk, l * 8);
  i |= b200_memset0(w->adm.d_g, l * 8);
  i |= b200_h2d(w->adm.d_R, w->h_diag_r, l * 8);
  if (w->D) {
    w->d_D = (double *)b200_malloc((size_t)m * 8);
    w->d_E = (double *)b200_malloc((size_t)n * 8);
    if (!w->d_D || !w->d_E) goto fail;
    if (host_copy) {
      i |= b200_h2d(w->d_D, w->D, (size_t)m * 8);
      i |= b200_h2d(w->d_E, w->E, (size_t)n * 8);
    }
  }
  if (i != 0) goto fail;
  init_mark("init: validate, copies, device vectors", &t_mark);
  if (dm) {
    if (!dev_data && dev_mats_from_host(d->A, d->P, dm) != 0) goto fail;
    if (build_ops_dev(w, dm) != 0) goto fail;
    init_mark("init: operators, equilibration and preconditioner on the device", &t_mark);
  } else if (!host_copy) {
    /* row-sharded, P = 0: D, E from temporary full copies on the device, then the resident row block scaled once */
    if (b200_linsys_full_equilibrate(d->A, w->cone_boundaries, w->cone_boundaries_len, w->d_D, w->d_E) != 0)
      goto fail;
    w->p = scs_init_lin_sys_work(d->A, SCS_NULL, w->h_diag_r);
    if (!w->p) { printf("ERROR: init_lin_sys_work failure\n"); goto fail; }
    t_mark = now_ms();
    if (b200_linsys_scale_local(w->p, w->d_D, w->d_E) != 0) goto fail;
    if (b200_linsys_update_diag_r_dev(w->p, w->p->d_diag_r) != 0) goto fail; /* preconditioner of D A E */
    if (b200_d2h(w->D, w->d_D, (size_t)m * 8) != 0 || b200_d2h(w->E, w->d_E, (size_t)n * 8) != 0 ||
        b200_sync() != 0)
      goto fail;
    b200_normalize_box(w->k, w->D, w->k->bl, w->k->bu);
    init_mark("init: device equilibration + preconditioner", &t_mark);
  }
  w->cones = b200_cones_build(w->k, m, w->k->bl, w->k->bu);
  if (!w->cones) {
    printf("ERROR: init_cone failure\n");
    goto fail;
  }
  if (!w->p) w->p = scs_init_lin_sys_work(w->d->A, w->d->P, w->h_diag_r);
  if (!w->p) { printf("ERROR: init_lin_sys_work failure\n"); goto fail; }
  if (w->stgs->acceleration_lookback) {
    w->accel = b200_aa_create((int)l, (int)w->stgs->acceleration_lookback, (int)w->stgs->acceleration_lookback,
                              w->stgs->acceleration_type_1 != 0, w->stgs->acceleration_regularization,
                              w->stgs->acceleration_relaxation, AA_SAFEGUARD_FACTOR,
                              AA_MAX_WEIGHT_NORM, AA_IR_MAX_STEPS, 0);
    if (!w->accel && w->stgs->verbose) printf("WARN: aa_init returned NULL, no acceleration applied.\n");
  }
  /* b, c: the originals onto the device, normalised there. Allocated last: placed before the blocks the ADMM loop
   * streams, their 32 MB at C2 moved those and bench.py ran 0.7 % fewer iterations/s (H100 80GB HBM3, 700 W). */
  w->d_b_orig = (double *)b200_malloc((size_t)m * 8);
  w->d_c_orig = (double *)b200_malloc((size_t)n * 8);
  if (!w->d_b_orig || !w->d_c_orig) goto fail;
  if (dev_data)
    i = b200_d2d(w->d_b_orig, d->b, (size_t)m * 8) | b200_d2d(w->d_c_orig, d->c, (size_t)n * 8);
  else
    i = b200_h2d(w->d_b_orig, d->b, (size_t)m * 8) | b200_h2d(w->d_c_orig, d->c, (size_t)n * 8);
  if (i != 0 || update_bc_dev(w) != 0) goto fail;
  if (b200_sync() != 0) goto fail;
  init_mark("init: cones, AA workspace, b, c", &t_mark);
  w->r_orig.last_iter = w->r_norm.last_iter = -1;
  w->setup_time = now_ms() - t0;
  return w;
fail:
  printf("ERROR: scs_init failed (%s)\n", b200_last_error());
  finish_work(w); /* the caller releases ctx */
  return SCS_NULL;
}

/* Every workspace gets an execution context of its own (a parked one when a finished workspace left one): its stream,
 * events, timers and free lists, so that workspaces of different threads solve concurrently. */
ScsWork *scs_init(const ScsData *d, const ScsCone *k, const ScsSettings *stgs) {
  B200DevMats dm;
  ScsWork *w;
  B200Ctx *ctx = d && k && stgs ? b200_ctx_create() : SCS_NULL, *prev = b200_ctx_enter(ctx);
  memset(&dm, 0, sizeof(dm));
  w = init_work(d, k, stgs, b200_comm_nranks() > 1 ? SCS_NULL : &dm, 0, ctx);
  if (dm.Ap) { /* uploaded (a refused input never reaches the GPU): free only once the builder's kernels have run */
    b200_sync();
    b200_dev_mats_free(&dm);
  }
  b200_ctx_leave(prev);
  if (!w) b200_ctx_release(ctx);
  return w;
}

/* ----------------------------------------------------------------- residuals */
static void compute_residuals(B200Residuals *r, double pd) {
  const double tol = INFEAS_NEGATIVITY_TOL / pd;
  r->res_pri = SAFEDIV_POS(r->nm_ax_s_btau, r->tau);
  r->res_dual = SAFEDIV_POS(r->nm_px_aty_ctau, r->tau);
  r->res_unbdd_a = NAN;
  r->res_unbdd_p = NAN;
  r->res_infeas = NAN;
  if (r->ctx_tau < -tol) {
    r->res_unbdd_a = SAFEDIV_POS(r->nm_ax_s, -r->ctx_tau);
    r->res_unbdd_p = SAFEDIV_POS(r->nm_px, -r->ctx_tau);
  }
  if (r->bty_tau < -tol) r->res_infeas = SAFEDIV_POS(r->nm_aty, -r->bty_tau);
}

static int populate_residual_struct(ScsWork *w, int iter) {
  B200Residuals *r = &w->r_norm, *ro = &w->r_orig;
  B200SpmvArgs a;
  const int n = w->n;
  const double *h;
  double pd;
  if (r->last_iter == iter) return 0;
  r->last_iter = iter;
  memset(&a, 0, sizeof(a));
  a.init_sign = 1.0; a.post = B200_POST_NONE; a.hook = B200_HOOK_NONE;
  /* ax = A x (row-sharded: local rows, then all-gather) */
  a.d_x = w->adm.d_u; a.d_y = w->d_ax + w->p->row0;
  if (b200_spmv(w->p->A, &a) != 0) return -1;
  if (w->p->nranks > 1 && b200_allgatherv(w->d_ax, w->p->offsets) != 0) return -1;
  /* aty = A' y (row-sharded: local partial, then all-reduce) */
  a.d_x = w->adm.d_u + n + w->p->row0; a.d_y = w->d_aty;
  if (b200_spmv(w->p->At, &a) != 0) return -1;
  if (w->p->nranks > 1 && b200_allreduce_sum(w->d_aty, (size_t)n) != 0) return -1;
  if (w->p->P) {
    a.d_x = w->adm.d_u; a.d_y = w->d_px;
    if (b200_spmv(w->p->P, &a) != 0) return -1;
  }
  if (b200_admm_resid_rows(&w->adm, w->d_ax, w->d_b, w->d_D, 1.0 / w->dual_scale, w->dual_scale) != 0) return -1;
  if (b200_admm_resid_cols(&w->adm, w->d_aty, w->d_px, w->d_c, w->d_E, 1.0 / w->primal_scale) != 0) return -1;
  if (b200_d2h(w->h_sc, w->adm.d_sc, SC_COUNT * 8) != 0) return -1;
  if (b200_sync() != 0) return -1;
  h = w->h_sc;
  /* normalised quantities (scs.c:553-598) */
  r->tau = h[SC_TAU];
  r->kap = h[SC_KAP];
  r->xt_p_x_tau = w->p->P ? h[SC_XPX_TAU] : 0.;
  r->bty_tau = h[SC_BTY_TAU];
  r->ctx_tau = h[SC_CTX_TAU];
  r->bty = SAFEDIV_POS(r->bty_tau, r->tau);
  r->ctx = SAFEDIV_POS(r->ctx_tau, r->tau);
  r->xt_p_x = SAFEDIV_POS(r->xt_p_x_tau, r->tau * r->tau);
  r->gap = fabs(r->xt_p_x + r->ctx + r->bty);
  r->pobj = r->xt_p_x / 2. + r->ctx;
  r->dobj = -r->xt_p_x / 2. - r->bty;
  r->nm_ax_s_btau = h[SC_NM_AXSB];
  r->nm_px_aty_ctau = h[SC_NM_PXATYC];
  /* un-normalised (scs.c:487-531); with normalize == 0 the factors are all 1 */
  pd = w->primal_scale * w->dual_scale;
  ro->last_iter = iter;
  ro->tau = r->tau;
  ro->kap = r->kap / pd;
  ro->bty_tau = r->bty_tau / pd;
  ro->ctx_tau = r->ctx_tau / pd;
  ro->xt_p_x_tau = r->xt_p_x_tau / pd;
  ro->xt_p_x = r->xt_p_x / pd;
  ro->ctx = r->ctx / pd;
  ro->bty = r->bty / pd;
  ro->pobj = r->pobj / pd;
  ro->dobj = r->dobj / pd;
  ro->gap = r->gap / pd;
  ro->nm_ax_s_btau = h[SC_O_AXSB];
  ro->nm_ax = h[SC_O_AX];
  ro->nm_ax_s = h[SC_O_AXS];
  ro->nm_s = h[SC_O_S];
  ro->nm_px_aty_ctau = h[SC_O_PXATYC];
  ro->nm_px = h[SC_O_PX];
  ro->nm_aty = h[SC_O_ATY];
  compute_residuals(ro, pd);
  return 0;
}

static int has_converged(const ScsWork *w) {
  const B200Residuals *r = &w->r_orig;
  const double eps_abs = w->stgs->eps_abs, eps_rel = w->stgs->eps_rel, eps_infeas = w->stgs->eps_infeas;
  if (r->tau > 0.) {
    const double grl = MAX(MAX(fabs(r->xt_p_x), fabs(r->ctx)), fabs(r->bty));
    const double prl = MAX(MAX(w->nm_b_orig * r->tau, r->nm_s), r->nm_ax) / r->tau;
    const double drl = MAX(MAX(w->nm_c_orig * r->tau, r->nm_px), r->nm_aty) / r->tau;
    if (isless(r->res_pri, eps_abs + eps_rel * prl) && isless(r->res_dual, eps_abs + eps_rel * drl) &&
        isless(r->gap, eps_abs + eps_rel * grl))
      return SCS_SOLVED;
  }
  if (isless(r->res_unbdd_a, eps_infeas) && isless(r->res_unbdd_p, eps_infeas)) return SCS_UNBOUNDED;
  if (isless(r->res_infeas, eps_infeas)) return SCS_INFEASIBLE;
  return 0;
}

/* ----------------------------------------------------------------- per-solve setup */
/* g = (I + M)^{-1} [c; -b]  (scs.c:1118-1128). h lives only in d_g and the CG overwrites it in place, so g is valid only
 * once the solve has returned */
static int update_work_cache(ScsWork *w) {
  w->g_valid = 0;
  if (b200_admm_build_h(&w->adm, w->d_c, w->d_b) != 0) return -1;
  if (b200_linsys_solve_dev(w->p, w->adm.d_g, SCS_NULL, CG_BEST_TOL, SCS_NULL) != 0) return -1;
  w->g_valid = 1;
  return 0;
}

static int update_work(ScsWork *w, ScsSolution *sol) {
  const int n = w->n, m = w->m;
  w->last_scale_update_iter = 0;
  w->sum_log_scale_factor = 0.;
  w->n_log_scale_factor = 0;
  w->scale_updates = 0;
  w->time_limit_reached = 0;
  w->rejected_accel_steps = 0;
  w->accepted_accel_steps = 0;
  w->aa_norm = 0.;
  w->r_norm.last_iter = -1;
  w->r_orig.last_iter = -1;
  if (w->stgs->warm_start && sol && sol->x && sol->y && sol->s) {
    int (*in)(void *, const void *, size_t) = w->sol_on_dev ? b200_d2d : b200_h2d;
    if (in(w->d_sol_x, sol->x, (size_t)n * 8) != 0) return -1;
    if (in(w->d_sol_y, sol->y, (size_t)m * 8) != 0) return -1;
    if (in(w->d_sol_s, sol->s, (size_t)m * 8) != 0) return -1;
    if (w->D && b200_admm_normalize_sol(n, m, w->d_D, w->d_E, w->primal_scale, w->dual_scale,
                                        w->d_sol_x, w->d_sol_y, w->d_sol_s) != 0)
      return -1;
    if (b200_admm_warm_start(&w->adm, w->d_sol_x, w->d_sol_y, w->d_sol_s) != 0) return -1;
  } else {
    if (b200_admm_cold_start(&w->adm) != 0) return -1;
  }
  /* g does not depend on the starting point: a solve on unchanged data reuses it (the CG would return the same bits) */
  if (w->g_valid && scs_b200_g_reuse()) return 0;
  return update_work_cache(w);
}

/* scs.c:1164-1241 */
static int update_scale(ScsWork *w, int iter) {
  const B200Residuals *r = &w->r_orig;
  double factor, new_scale, relative_res_pri, relative_res_dual, denom_pri, denom_dual;
  const int iters_since_last_update = iter - w->last_scale_update_iter;
  denom_pri = MAX(r->nm_ax, r->nm_s);
  denom_pri = MAX(denom_pri, w->nm_b_orig * r->tau);
  relative_res_pri = SAFEDIV_POS(r->nm_ax_s_btau, denom_pri);
  denom_dual = MAX(r->nm_px, r->nm_aty);
  denom_dual = MAX(denom_dual, w->nm_c_orig * r->tau);
  relative_res_dual = SAFEDIV_POS(r->nm_px_aty_ctau, denom_dual);
  relative_res_pri = MAX(relative_res_pri, DIV_EPS_TOL);
  relative_res_dual = MAX(relative_res_dual, DIV_EPS_TOL);
  w->sum_log_scale_factor += log(relative_res_pri) - log(relative_res_dual);
  w->n_log_scale_factor++;
  factor = sqrt(exp(w->sum_log_scale_factor / (double)(w->n_log_scale_factor)));
  if (iters_since_last_update < RESCALING_MIN_ITERS) return 0;
  new_scale = MIN(MAX(w->stgs->scale * factor, MIN_SCALE_VALUE), MAX_SCALE_VALUE);
  if (new_scale == w->stgs->scale) return 0;
  if (factor > sqrt(10.) || factor < 1. / sqrt(10.)) {
    w->scale_updates++;
    w->sum_log_scale_factor = 0;
    w->n_log_scale_factor = 0;
    w->last_scale_update_iter = iter;
    w->stgs->scale = new_scale;
    w->g_valid = 0; /* new diag_r; g is re-solved just below */
    set_diag_r_host(w);
    if (b200_admm_set_diag_r(&w->adm, w->k->z, w->stgs->rho_x, w->stgs->scale) != 0) return -1;
    if (b200_linsys_update_diag_r_dev(w->p, w->adm.d_R) != 0) return -1;
    if (update_work_cache(w) != 0) return -1;
    if (w->accel) b200_aa_reset_dev(w->accel);
    if (b200_admm_remap_v(&w->adm) != 0) return -1;
  }
  return 0;
}

/* ----------------------------------------------------------------- finalize */
static void fill_nan(double *v, int len) {
  int i;
  for (i = 0; i < len; ++i) v[i] = NAN;
}

/* Ctrl-C handling, same contract as the reference (src/ctrlc.c:84-126, src/scs.c:1344,1400-1403,1482): a SIGINT
 * handler is installed for the duration of scs_solve (reference counted, the previous handler is restored) and the
 * iteration polls the flag -- here once per ADMM iteration on the host, between two enqueues -- returning SCS_SIGINT. */
#include <pthread.h>
#include <signal.h>
static volatile sig_atomic_t int_detected;
static struct sigaction int_oact;
static pthread_mutex_t int_mutex = PTHREAD_MUTEX_INITIALIZER;
static int int_listeners = 0;
static void handle_ctrlc(int sig) { int_detected = sig ? sig : -1; }
static void start_interrupt_listener(void) {
  pthread_mutex_lock(&int_mutex);
  if (int_listeners == 0) {
    struct sigaction act;
    int_detected = 0;
    act.sa_flags = 0;
    sigemptyset(&act.sa_mask);
    act.sa_handler = handle_ctrlc;
    sigaction(SIGINT, &act, &int_oact);
  }
  int_listeners++;
  pthread_mutex_unlock(&int_mutex);
}
static void end_interrupt_listener(void) {
  pthread_mutex_lock(&int_mutex);
  if (int_listeners > 0 && --int_listeners == 0) {
    struct sigaction act;
    sigaction(SIGINT, &int_oact, &act);
  }
  pthread_mutex_unlock(&int_mutex);
}

static int failure(ScsWork *w, int m, int n, ScsSolution *sol, ScsInfo *info, int status,
                   const char *msg, const char *ststr) {
  if (info) {
    info->gap = info->res_pri = info->res_dual = info->pobj = info->dobj = NAN;
    info->iter = -1;
    info->status_val = status;
    info->solve_time = NAN;
    strcpy(info->status, ststr);
    memset(&info->aa_stats, 0, sizeof(info->aa_stats));
    info->aa_stats.last_aa_norm = NAN;
  }
  if (sol && w && w->sol_on_dev) { /* device buffers, checked at entry */
    b200_vec_fill(n, sol->x, NAN);
    b200_vec_fill(m, sol->y, NAN);
    b200_vec_fill(m, sol->s, NAN);
  } else if (sol) {
    if (n > 0) {
      if (!sol->x) sol->x = (double *)calloc((size_t)n, sizeof(double));
      if (sol->x) fill_nan(sol->x, n);
    }
    if (m > 0) {
      if (!sol->y) sol->y = (double *)calloc((size_t)m, sizeof(double));
      if (sol->y) fill_nan(sol->y, m);
      if (!sol->s) sol->s = (double *)calloc((size_t)m, sizeof(double));
      if (sol->s) fill_nan(sol->s, m);
    }
  }
  printf("Failure:%s\n", msg);
  end_interrupt_listener(); /* every failure() inside scs_solve leaves the solve; outside it the count is 0: no-op */
  return status;
}

static void set_info_aa_stats(ScsInfo *info, const B200Aa *accel) {
  memset(&info->aa_stats, 0, sizeof(info->aa_stats));
  info->aa_stats.last_aa_norm = NAN;
  if (accel) {
    int o[8];
    double dd[2];
    b200_aa_stats(accel, o, dd);
    info->aa_stats.iter = o[0]; info->aa_stats.n_accept = o[1];
    info->aa_stats.n_reject_lapack = o[2]; info->aa_stats.n_reject_rank0 = o[3];
    info->aa_stats.n_reject_nonfinite = o[4]; info->aa_stats.n_reject_weight_cap = o[5];
    info->aa_stats.n_safeguard_reject = o[6]; info->aa_stats.last_rank = o[7];
    info->aa_stats.last_aa_norm = dd[0]; info->aa_stats.last_regularization = dd[1];
  }
}

/* scaling factors decided on the host, applied on the device, then one D2H */
static int finalize(ScsWork *w, ScsSolution *sol, ScsInfo *info, int iter) {
  const int n = w->n, m = w->m;
  const B200Residuals *r = &w->r_orig;
  double fx = 1.0, fy = 1.0, fs = 1.0; /* NaN means "fill with NaN" */
  double nm_s, nm_y, sty;
  int (*out)(void *, const void *, size_t) = w->sol_on_dev ? b200_d2d : b200_d2h;
  if (!w->sol_on_dev) {
    if (!sol->x) sol->x = (double *)calloc((size_t)n, sizeof(double));
    if (!sol->y) sol->y = (double *)calloc((size_t)m, sizeof(double));
    if (!sol->s) sol->s = (double *)calloc((size_t)m, sizeof(double));
  }
  if (!sol->x || !sol->y || !sol->s) return -1;
  if (b200_admm_unnormalize_sol(&w->adm, w->d_D, w->d_E, w->primal_scale, w->dual_scale, w->d_sol_x,
                                w->d_sol_y, w->d_sol_s) != 0)
    return -1;
  if (populate_residual_struct(w, iter) != 0) return -1;
  if (b200_vec_norms_dot(m, w->d_sol_s, w->d_sol_y, w->adm.d_sc + SC_TMP0, w->adm.d_part,
                         w->adm.d_cnt) != 0)
    return -1;
  if (b200_d2h(w->h_sc, w->adm.d_sc, SC_COUNT * 8) != 0 || b200_sync() != 0) return -1;
  nm_s = w->h_sc[SC_TMP0];
  nm_y = w->h_sc[SC_TMP0 + 1];
  sty = w->h_sc[SC_TMP0 + 2];

  info->setup_time = w->setup_time;
  info->iter = iter;
  info->res_infeas = r->res_infeas;
  info->res_unbdd_a = r->res_unbdd_a;
  info->res_unbdd_p = r->res_unbdd_p;
  info->scale = w->stgs->scale;
  info->scale_updates = w->scale_updates;
  info->rejected_accel_steps = w->rejected_accel_steps;
  info->accepted_accel_steps = w->accepted_accel_steps;
  set_info_aa_stats(info, w->accel);
  info->comp_slack = fabs(sty);
  if (info->comp_slack > 1e-5 * MAX(nm_s, nm_y))
    printf("WARNING - large complementary slackness residual: %f\n", info->comp_slack);

  {
    int st = info->status_val, inaccurate = 0;
    if (st == SCS_UNFINISHED) { /* set_unfinished, scs.c:887-913 */
      inaccurate = 1;
      if (r->kap > r->tau && (r->bty_tau < 0 || r->ctx_tau < 0)) {
        st = (r->bty_tau < 0 && r->bty_tau < r->ctx_tau) ? SCS_INFEASIBLE : SCS_UNBOUNDED;
      } else if (r->tau > 0) {
        st = SCS_SOLVED;
      } else {
        printf("ERROR: could not determine problem status.\n");
        st = SCS_FAILED;
      }
    }
    if (st == SCS_SOLVED) {
      fx = fy = fs = SAFEDIV_POS(1.0, r->tau);
      info->gap = r->gap;
      info->res_pri = r->res_pri;
      info->res_dual = r->res_dual;
      info->pobj = r->xt_p_x / 2. + r->ctx;
      info->dobj = -r->xt_p_x / 2. - r->bty;
      strcpy(info->status, "solved");
      info->status_val = inaccurate ? SCS_SOLVED_INACCURATE : SCS_SOLVED;
    } else if (st == SCS_INFEASIBLE) {
      fy = -1 / r->bty_tau;
      fx = fs = NAN;
      info->gap = info->res_pri = info->res_dual = NAN;
      info->pobj = info->dobj = INFINITY;
      strcpy(info->status, "infeasible");
      info->status_val = inaccurate ? SCS_INFEASIBLE_INACCURATE : SCS_INFEASIBLE;
    } else if (st == SCS_UNBOUNDED) {
      fx = fs = -1 / r->ctx_tau;
      fy = NAN;
      info->gap = info->res_pri = info->res_dual = NAN;
      info->pobj = info->dobj = -INFINITY;
      strcpy(info->status, "unbounded");
      info->status_val = inaccurate ? SCS_UNBOUNDED_INACCURATE : SCS_UNBOUNDED;
    } else {
      info->status_val = SCS_FAILED;
      strcpy(info->status, "failure");
    }
    if (inaccurate && info->status_val != SCS_FAILED) {
      if (w->time_limit_reached) strcat(info->status, " (inaccurate - reached time_limit_secs)");
      else if (info->iter >= w->stgs->max_iters) strcat(info->status, " (inaccurate - reached max_iters)");
      else printf("ERROR: should not be in this state (1).\n");
    }
  }
  if (isnan(fx)) { if (b200_vec_fill(n, w->d_sol_x, NAN) != 0) return -1; }
  else if (b200_vec_scale(n, w->d_sol_x, fx) != 0) return -1;
  if (isnan(fy)) { if (b200_vec_fill(m, w->d_sol_y, NAN) != 0) return -1; }
  else if (b200_vec_scale(m, w->d_sol_y, fy) != 0) return -1;
  if (isnan(fs)) { if (b200_vec_fill(m, w->d_sol_s, NAN) != 0) return -1; }
  else if (b200_vec_scale(m, w->d_sol_s, fs) != 0) return -1;
  if (out(sol->x, w->d_sol_x, (size_t)n * 8) != 0) return -1;
  if (out(sol->y, w->d_sol_y, (size_t)m * 8) != 0) return -1;
  if (out(sol->s, w->d_sol_s, (size_t)m * 8) != 0) return -1;
  return b200_sync();
}

static void print_summary(ScsWork *w, int i, double t0) {
  const B200Residuals *r = &w->r_orig;
  printf("%*i|", 6, i);
  printf("%*.2e ", 9, r->res_pri);
  printf("%*.2e ", 9, r->res_dual);
  printf("%*.2e ", 9, r->gap);
  printf("%*.2e ", 10, SAFEDIV_POS(r->pobj + r->dobj, 2.));
  printf("%*.2e ", 9, w->stgs->scale);
  printf("%*.2e ", 9, (now_ms() - t0 + w->setup_time) / 1e3);
  printf("\n");
  fflush(stdout);
}

/* ----------------------------------------------------------------- CSV trace
 * One row per ADMM iteration, the columns of the reference's log_data_to_csv (src/rw.c:707-861) in the same order and
 * format (%.16e), so that two traces can be diffed column by column. A debugging mode: the iterates and the residual
 * vectors are copied to the host every iteration and every norm is recomputed there with the reference's formulas
 * (populate_residual_struct / unnormalize_residuals, src/scs.c:487-607). As in the reference, logging refreshes the
 * residual struct EVERY iteration, which feeds the CG tolerance of the next one (scs.c:1448-1453). */
static double h_ninf(const double *v, long long len) {
  double mx = 0.;
  long long i;
  for (i = 0; i < len; ++i) { const double a = fabs(v[i]); if (a > mx) mx = a; }
  return mx;
}
static double h_n2(const double *v, long long len) {
  double s = 0.;
  long long i;
  for (i = 0; i < len; ++i) s += v[i] * v[i];
  return sqrt(s);
}
static int log_data_to_csv(ScsWork *w, int iter, double t_solve) {
  const int n = w->n, m = w->m;
  const long long l = (long long)n + m + 1;
  const B200Residuals *r = &w->r_orig;
  B200Residuals rn_local, *rn = &rn_local;
  FILE *f = w->log_csv_fout;
  double *u, *ut, *v, *vp, *rsk, *ax, *aty, *px, *bv, *cv;
  double acc[16];
  double tau, inv_ds, inv_ps;
  long long i;
  if (!f) return 0;
  if (populate_residual_struct(w, iter) != 0) return -1;
  if (!w->log_host) {
    w->log_host = (double *)malloc((size_t)(5 * l + 2 * (long long)m + 3 * (long long)n) * sizeof(double));
    if (!w->log_host) return -1;
  }
  u = w->log_host; ut = u + l; v = ut + l; vp = v + l; rsk = vp + l; ax = rsk + l; aty = ax + m; px = aty + n;
  bv = px + n; cv = bv + m;
  if (b200_d2h(u, w->adm.d_u, (size_t)l * 8) != 0 || b200_d2h(ut, w->adm.d_u_t, (size_t)l * 8) != 0 ||
      b200_d2h(v, w->adm.d_v, (size_t)l * 8) != 0 || b200_d2h(vp, w->adm.d_v_prev, (size_t)l * 8) != 0 ||
      b200_d2h(rsk, w->adm.d_rsk, (size_t)l * 8) != 0 || b200_d2h(ax, w->d_ax, (size_t)m * 8) != 0 ||
      b200_d2h(aty, w->d_aty, (size_t)n * 8) != 0 || b200_d2h(bv, w->d_b, (size_t)m * 8) != 0 ||
      b200_d2h(cv, w->d_c, (size_t)n * 8) != 0 || b200_sync() != 0)
    return -1;
  if (w->p->P) {
    if (b200_d2h(px, w->d_px, (size_t)n * 8) != 0 || b200_sync() != 0) return -1;
  } else {
    memset(px, 0, (size_t)n * 8);
  }
  if (iter == 0) {
    fprintf(f, "iter,res_pri,res_dual,gap,x_nrm_inf,y_nrm_inf,s_nrm_inf,x_nrm_2,y_nrm_2,s_nrm_2,"
               "x_nrm_inf_normalized,y_nrm_inf_normalized,s_nrm_inf_normalized,x_nrm_2_normalized,y_nrm_2_normalized,"
               "s_nrm_2_normalized,ax_s_btau_nrm_inf,px_aty_ctau_nrm_inf,ax_s_btau_nrm_2,px_aty_ctau_nrm_2,res_infeas,"
               "res_unbdd_a,res_unbdd_p,pobj,dobj,tau,kap,res_pri_normalized,res_dual_normalized,gap_normalized,"
               "ax_s_btau_nrm_inf_normalized,px_aty_ctau_nrm_inf_normalized,ax_s_btau_nrm_2_normalized,"
               "px_aty_ctau_nrm_2_normalized,res_infeas_normalized,res_unbdd_a_normalized,res_unbdd_p_normalized,"
               "pobj_normalized,dobj_normalized,tau_normalized,kap_normalized,ax_nrm_inf,ax_s_nrm_inf,px_nrm_inf,"
               "aty_nrm_inf,xt_p_x,xt_p_x_tau,ctx,ctx_tau,bty,bty_tau,b_nrm_inf,c_nrm_inf,scale,diff_u_ut_nrm_2,"
               "diff_v_v_prev_nrm_2,diff_u_ut_nrm_inf,diff_v_v_prev_nrm_inf,aa_norm,accepted_accel_steps,"
               "rejected_accel_steps,time,spectral_Newton_iter,plain_Newton_success,res_dual_spectral,res_pri_spectral,"
               "comp_spectral,\n");
  }
  tau = fabs(u[l - 1]);
  inv_ds = 1.0 / w->dual_scale;
  inv_ps = 1.0 / w->primal_scale;
  /* the normalised residual struct with its infeasibility ratios (scs.c:598 compute_residuals(r, m, n, 1.0)): the
   * device path keeps only what the iteration needs, the remaining normalised norms are taken from the host copies */
  rn_local = w->r_norm;
  rn_local.nm_aty = h_ninf(aty, n);
  rn_local.nm_px = h_ninf(px, n);
  {
    double mx = 0.;
    for (i = 0; i < m; ++i) { const double a = fabs(ax[i] + rsk[n + i]); if (a > mx) mx = a; }
    rn_local.nm_ax_s = mx;
  }
  compute_residuals(&rn_local, 1.0);
  /* acc: 0..5 inf/2-norms of x, y, s (original), 6..7 2-norms of ax_s_btau / px_aty_ctau (original),
   * 8..9 the same normalised */
  memset(acc, 0, sizeof(acc));
  {
    double xi = 0, x2 = 0, yi = 0, y2 = 0, si = 0, s2 = 0, p2 = 0, p2n = 0, d2 = 0, d2n = 0;
    for (i = 0; i < n; ++i) {
      const double e = w->E ? w->E[i] : 1.0;
      const double xo = w->E ? u[i] * (e / w->dual_scale) : u[i];
      const double rr = px[i] + aty[i] + tau * cv[i];
      const double ro = rr * (inv_ps / e);
      if (fabs(xo) > xi) xi = fabs(xo);
      x2 += xo * xo;
      d2n += rr * rr;
      d2 += ro * ro;
    }
    for (i = 0; i < m; ++i) {
      const double d = w->D ? w->D[i] : 1.0;
      const double yo = w->D ? u[n + i] * (d / w->primal_scale) : u[n + i];
      const double so = w->D ? rsk[n + i] / (d * w->dual_scale) : rsk[n + i];
      const double rr = ax[i] + rsk[n + i] - tau * bv[i];
      const double ro = rr * (inv_ds / d);
      if (fabs(yo) > yi) yi = fabs(yo);
      if (fabs(so) > si) si = fabs(so);
      y2 += yo * yo;
      s2 += so * so;
      p2n += rr * rr;
      p2 += ro * ro;
    }
    acc[0] = xi; acc[1] = yi; acc[2] = si; acc[3] = sqrt(x2); acc[4] = sqrt(y2); acc[5] = sqrt(s2);
    acc[6] = sqrt(p2); acc[7] = sqrt(d2); acc[8] = sqrt(p2n); acc[9] = sqrt(d2n);
  }
  fprintf(f, "%li,", (long)iter);
  fprintf(f, "%.16e,%.16e,%.16e,", r->res_pri, r->res_dual, r->gap);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,%.16e,%.16e,", acc[0], acc[1], acc[2], acc[3], acc[4], acc[5]);
  fprintf(f, "%.16e,%.16e,%.16e,", h_ninf(u, n), h_ninf(u + n, m), h_ninf(rsk + n, m));
  fprintf(f, "%.16e,%.16e,%.16e,", h_n2(u, n), h_n2(u + n, m), h_n2(rsk + n, m));
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,", r->nm_ax_s_btau, r->nm_px_aty_ctau, acc[6], acc[7]);
  fprintf(f, "%.16e,%.16e,%.16e,", r->res_infeas, r->res_unbdd_a, r->res_unbdd_p);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,", r->pobj, r->dobj, r->tau, r->kap);
  fprintf(f, "%.16e,%.16e,%.16e,", rn->res_pri, rn->res_dual, rn->gap);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,", rn->nm_ax_s_btau, rn->nm_px_aty_ctau, acc[8], acc[9]);
  fprintf(f, "%.16e,%.16e,%.16e,", rn->res_infeas, rn->res_unbdd_a, rn->res_unbdd_p);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,", rn->pobj, rn->dobj, rn->tau, rn->kap);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,", r->nm_ax, r->nm_ax_s, r->nm_px, r->nm_aty);
  fprintf(f, "%.16e,%.16e,%.16e,%.16e,%.16e,%.16e,", r->xt_p_x, r->xt_p_x_tau, r->ctx, r->ctx_tau, r->bty, r->bty_tau);
  fprintf(f, "%.16e,%.16e,%.16e,", w->nm_b_orig, w->nm_c_orig, w->stgs->scale);
  {
    double du2 = 0, dv2 = 0, dui = 0, dvi = 0;
    for (i = 0; i < l; ++i) {
      const double a = u[i] - ut[i], b = v[i] - vp[i];
      du2 += a * a;
      dv2 += b * b;
      if (fabs(a) > dui) dui = fabs(a);
      if (fabs(b) > dvi) dvi = fabs(b);
    }
    fprintf(f, "%.16e,%.16e,%.16e,%.16e,", sqrt(du2), sqrt(dv2), dui, dvi);
  }
  fprintf(f, "%.16e,%li,%li,", w->aa_norm, (long)w->accepted_accel_steps, (long)w->rejected_accel_steps);
  fprintf(f, "%.16e,", (now_ms() - t_solve) / 1e3);
  {
    /* the Newton_stats record of the last log-det cone projected (rw.c:854-858); zeros without log-det cones */
    int st_iter = 0, st_success = 0;
    double st_res[3] = {0.0, 0.0, 0.0};
#ifdef USE_SPECTRAL_CONES
    if (w->k->dsize > 0 && b200_cones_logdet_stats(w->cones, &st_iter, &st_success, st_res) != 0) return -1;
#endif
    fprintf(f, "%i,%i,%.16e,%.16e,%.16e,", st_iter, st_success, st_res[0], st_res[1], st_res[2]);
  }
  fprintf(f, "\n");
  return 0;
}

/* ----------------------------------------------------------------- the solve */
static scs_int solve(ScsWork *w, ScsSolution *sol, ScsInfo *info, scs_int warm_start) {
  int i, l;
  double t_solve, total_accel = 0.0, total_cone = 0.0, total_lin = 0.0;
  const long long launches0 = b200_ctx_launches();
  long long cg0, solves0, k34_0[2];
  ScsSettings *stgs;
  if (!sol || !w || !info) {
    printf("ERROR: missing ScsWork, ScsSolution or ScsInfo input\n");
    return SCS_FAILED;
  }
  l = w->m + w->n + 1;
  stgs = w->stgs;
  stgs->warm_start = warm_start;
  t_solve = now_ms();
  if (w->log_csv_name) { /* reference rw.c:686-698, scs.c:1349 */
    if (w->log_csv_fout) fclose(w->log_csv_fout);
    w->log_csv_fout = fopen(w->log_csv_name, "w");
    if (!w->log_csv_fout) printf("Error: Could not open %s for writing\n", w->log_csv_name);
  }
  start_interrupt_listener();
  strcpy(info->lin_sys_solver, scs_get_lin_sys_method());
  info->status_val = SCS_UNFINISHED;
  cg0 = w->p->tot_cg_its;
  solves0 = w->p->n_solves;
  k34_0[0] = w->p->cg.k34_solves[0];
  k34_0[1] = w->p->cg.k34_solves[1];
  if (update_work(w, sol) != 0)
    return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in update_work", "failure");
  if (stgs->verbose) {
    int k;
    for (k = 0; k < 78; ++k) printf("-");
    printf("\n iter | pri res | dua res |   gap   |   obj   |  scale  | time (s)\n");
    for (k = 0; k < 78; ++k) printf("-");
    printf("\n");
  }

  b200_section_begin();
  for (i = 0; i < stgs->max_iters; ++i) {
    const int check = (i % CONVERGED_INTERVAL == 0);
    int dual_done = 0;
    if (int_detected) /* reference scs.c:1400-1403 */
      return failure(w, w->m, w->n, sol, info, SCS_SIGINT, "interrupted", "interrupted");
    /* ---- Anderson acceleration (scs.c:1359-1366) */
    if (w->accel) {
      if (i > 0 && i % stgs->acceleration_interval == 0) {
        b200_section_mark(B200_SEC_OTHER);
        w->aa_norm = b200_aa_apply_dev(w->accel, w->adm.d_v, w->adm.d_v_prev);
        b200_section_mark(B200_SEC_ACCEL);
      }
    }
    /* ---- normalize v, v_prev = v, u_t = R v, warm start, CG tolerance */
    b200_section_mark(B200_SEC_OTHER);
    if (b200_admm_prep_linsys(&w->adm, i, w->accel != SCS_NULL, pow((double)i + 1, CG_RATE)) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_lin_sys", "failure");
    /* ---- KKT solve (device PCG), tau from root_plus */
    if (b200_linsys_solve_dev(w->p, w->adm.d_u_t, w->adm.d_ws, 0.0, w->adm.d_sc + SC_TOL) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_lin_sys", "failure");
    if (b200_admm_root_plus(&w->adm, i) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_lin_sys", "failure");
    b200_section_mark(B200_SEC_LINSYS);
    /* ---- cone projection */
    if (b200_admm_cone_pre(&w->adm, i, w->k->z, w->k->l, b200_cones_scratch(w->cones)) != 0 ||
        b200_cones_project_rest(w->cones, w->adm.d_u + w->n, b200_cones_scratch(w->cones),
                                w->adm.d_R + w->n) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_cones", "failure");
    b200_section_mark(B200_SEC_CONE);
    /* ---- rsk (and, when nothing intervenes, the dual update in the same pass) */
    {
      const int fuse_dual = !check;
      if (b200_admm_rsk_dual(&w->adm, fuse_dual, stgs->alpha) != 0)
        return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in compute_rsk", "failure");
      dual_done = fuse_dual;
    }

    if (check) {
      b200_section_mark(B200_SEC_OTHER);
      if (b200_section_flush() != 0 || b200_cones_check(w->cones) != 0)
        return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_cones", "failure");
      if (populate_residual_struct(w, i) != 0)
        return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in residuals", "failure");
      if ((info->status_val = has_converged(w)) != 0) break;
      if (stgs->time_limit_secs) {
        if (now_ms() - t_solve > 1000. * stgs->time_limit_secs) {
          w->time_limit_reached = 1;
          break;
        }
      }
    }
    if (stgs->verbose && i % PRINT_INTERVAL == 0) {
      populate_residual_struct(w, i);
      print_summary(w, i, t_solve);
    }
    if (stgs->adaptive_scale && i == w->r_orig.last_iter) {
      if (update_scale(w, i) < 0)
        return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in update_scale", "failure");
    }
    /* ---- dual variable step */
    if (!dual_done && b200_admm_dual_update(&w->adm, stgs->alpha) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in update_dual_vars", "failure");
    /* ---- AA safeguard (scs.c:1439-1447) */
    if (w->accel && i % stgs->acceleration_interval == 0 && w->aa_norm > 0) {
      b200_section_mark(B200_SEC_OTHER);
      if (b200_aa_safeguard_dev(w->accel, w->adm.d_v, w->adm.d_v_prev) < 0) w->rejected_accel_steps++;
      else w->accepted_accel_steps++;
      b200_section_mark(B200_SEC_ACCEL);
    }
    /* log AFTER the scale update so that the residual recalculation does not affect the algorithm (scs.c:1448-1453) */
    if (w->log_csv_fout && log_data_to_csv(w, i, t_solve) != 0)
      return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in log_data_to_csv", "failure");
  }
  if (w->log_csv_fout && log_data_to_csv(w, i, t_solve) != 0) /* final row after the full run (scs.c:1457-1461) */
    return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in log_data_to_csv", "failure");
  b200_section_mark(B200_SEC_OTHER);
  if (b200_section_flush() != 0 || b200_cones_check(w->cones) != 0)
    return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in project_cones", "failure");
  total_lin = b200_section_ms(B200_SEC_LINSYS);
  total_cone = b200_section_ms(B200_SEC_CONE);
  total_accel = b200_section_ms(B200_SEC_ACCEL);
  (void)l;
  if (stgs->verbose) {
    populate_residual_struct(w, i);
    print_summary(w, i, t_solve);
  }
  if (finalize(w, sol, info, i) != 0)
    return failure(w, w->m, w->n, sol, info, SCS_FAILED, "error in finalize", "failure");
  info->solve_time = now_ms() - t_solve;
  info->lin_sys_time = total_lin;
  info->cone_time = total_cone;
  info->accel_time = total_accel;
  w->stat_cg_iters = w->p->tot_cg_its - cg0;
  w->stat_solves = w->p->n_solves - solves0;
  w->stat_launches = b200_ctx_launches() - launches0;
  w->stat_k34[0] = w->p->cg.k34_solves[0] - k34_0[0];
  w->stat_k34[1] = w->p->cg.k34_solves[1] - k34_0[1];
  if (w->log_csv_fout) { /* scs.c:1481 */
    fclose(w->log_csv_fout);
    w->log_csv_fout = SCS_NULL;
  }
  end_interrupt_listener();
  if (stgs->verbose) {
    int k;
    for (k = 0; k < 78; ++k) printf("-");
    printf("\nstatus:  %s\ntimings: total: %1.2es = setup: %1.2es + solve: %1.2es\n", info->status,
           (info->setup_time + info->solve_time) / 1e3, info->setup_time / 1e3, info->solve_time / 1e3);
    printf("\t lin-sys: %1.2es, cones: %1.2es, accel: %1.2es\n", info->lin_sys_time / 1e3,
           info->cone_time / 1e3, info->accel_time / 1e3);
    printf("\t cg iterations: %lld over %lld solves, kernel launches: %lld\n", w->stat_cg_iters,
           w->stat_solves, w->stat_launches);
    for (k = 0; k < 78; ++k) printf("-");
    printf("\nobjective = %.6f\n", info->pobj);
    for (k = 0; k < 78; ++k) printf("-");
    printf("\n");
  }
  return info->status_val;
}
scs_int scs_solve(ScsWork *w, ScsSolution *sol, ScsInfo *info, scs_int warm_start) {
  B200Ctx *prev = b200_ctx_enter(w ? w->ctx : SCS_NULL);
  const scs_int status = solve(w, sol, info, warm_start);
  b200_ctx_leave(prev);
  return status;
}

scs_int scs(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, ScsSolution *sol,
            ScsInfo *info) {
  scs_int status;
  ScsWork *w = scs_init(d, k, stgs);
  if (w) {
    scs_solve(w, sol, info, stgs->warm_start);
    status = info->status_val;
  } else {
    status = failure(SCS_NULL, d ? d->m : -1, d ? d->n : -1, sol, info, SCS_FAILED,
                     "could not initialize work", "failure");
  }
  scs_finish(w);
  return status;
}

scs_int scs_b200_get_stats(const ScsWork *w, ScsB200Stats *out) {
  if (!w || !out) return -1;
  out->cg_iters = w->stat_cg_iters;
  out->lin_sys_solves = w->stat_solves;
  out->kernel_launches = w->stat_launches;
  out->spmv_ms = 0.0;
  out->n_gpus = b200_comm_nranks();
  return 0;
}
scs_int scs_b200_set_max_iters(ScsWork *w, scs_int max_iters) {
  if (!w || max_iters <= 0) return -1;
  w->stgs->max_iters = max_iters;
  return 0;
}
long long scs_b200_launch_count(void) { return b200_launches(); }
scs_int scs_b200_device_ok(void) { return b200_device_ok(); }

/* ----------------------------------------------------------------- device-data entry points */
/* b and c normalised from the device originals, for every door (reference scs_update and normalize_b_c, scs.c:1287-1325
 * and normalize.c:33-61; the maxima skip NaN like its norm_inf): the four maxima are the only values that reach the
 * host */
static int update_bc_dev(ScsWork *w) {
  const double t0 = now_ms();
  double mx[4], sigma;
  w->g_valid = 0; /* new normalised b and c */
  if (b200_normalize_b_c_dev(w->m, w->n, w->d_b_orig, w->d_c_orig, w->D ? w->d_D : SCS_NULL, w->D ? w->d_E : SCS_NULL,
                             w->d_b, w->d_c, mx) != 0)
    return -1;
  w->nm_b_orig = mx[0];
  w->nm_c_orig = mx[2];
  if (w->D) {
    sigma = mx[3] > mx[1] ? mx[3] : mx[1];
    sigma = sigma < 1e-4 ? 1.0 : sigma;
    sigma = sigma > 1e4 ? 1e4 : sigma;
    sigma = SAFEDIV_POS(1.0, sigma);
    if (b200_scale_b_c(w->m, w->n, w->d_b, w->d_c, sigma) != 0) return -1;
    w->primal_scale = sigma;
    w->dual_scale = sigma;
  }
  if (b200_sync() != 0) return -1;
  w->setup_time = now_ms() - t0;
  return 0;
}

/* the linear-system workspace from dm's blocks: both operators of A; with P, the structure of the full P, the
 * P-aware equilibration on the device and then P's operator and diagonal; with P = 0, b200_equilibrate_dev on the
 * built pair */
static int build_ops_dev(ScsWork *w, B200DevMats *dm) {
  const int n = w->n, m = w->m;
  B200Spmv *A = SCS_NULL, *At = SCS_NULL, *P = SCS_NULL;
  int *Fp = SCS_NULL, *Fi = SCS_NULL, *Fsrc = SCS_NULL;
  double *d_Pdiag = SCS_NULL;
  int rc = -1;
  do {
    if (b200_setup_ops_from_dev(m, n, dm->nnzA, dm->Ap, dm->Ai, dm->Ax, &A, &At) != 0) break;
    if (dm->Pp) {
      Fp = (int *)b200_malloc(((size_t)n + 1) * 4);
      Fi = (int *)b200_malloc((size_t)dm->fullP * 4);
      Fsrc = (int *)b200_malloc((size_t)dm->fullP * 4);
      d_Pdiag = (double *)b200_malloc((size_t)n * 8);
      if (!Fp || !Fi || !Fsrc || !d_Pdiag ||
          b200_sym_expand_structure(n, dm->nnzP, dm->fullP, dm->Pp, dm->Pi, Fp, Fi, Fsrc) != 0)
        break;
      if (w->D && b200_equilibrate_qp_dev(A, At, dm->Pp, dm->Pi, dm->Px, Fp, Fi, Fsrc, w->cone_boundaries,
                                          w->cone_boundaries_len, w->d_D, w->d_E) != 0)
        break;
      if (b200_sym_build(n, dm->fullP, Fp, Fi, Fsrc, dm->Px, d_Pdiag, &P) != 0) break;
    }
    w->p = b200_linsys_from_ops(m, n, A, At, P, d_Pdiag, w->h_diag_r); /* takes them over */
    A = At = P = SCS_NULL;
    d_Pdiag = SCS_NULL;
    if (!w->p) break;
    if (w->D && !dm->Pp) {
      if (b200_equilibrate_dev(w->p->A, w->p->At, w->cone_boundaries, w->cone_boundaries_len, w->d_D, w->d_E) != 0 ||
          b200_linsys_update_diag_r_dev(w->p, w->p->d_diag_r) != 0)
        break;
    }
    if (w->D) {
      if (b200_d2h(w->D, w->d_D, (size_t)m * 8) != 0 || b200_d2h(w->E, w->d_E, (size_t)n * 8) != 0 ||
          b200_sync() != 0)
        break;
      b200_normalize_box(w->k, w->D, w->k->bl, w->k->bu);
    }
    rc = 0;
  } while (0);
  b200_sync();
  b200_spmv_destroy(A); b200_spmv_destroy(At); b200_spmv_destroy(P);
  b200_free(Fp); b200_free(Fi); b200_free(Fsrc); b200_free(d_Pdiag);
  return rc;
}

/* ScsSettings.write_data_filename with device data: a debugging mode, the arrays are copied to the host to be written */
static int dev_to_host(void **dst, const void *d_src, size_t bytes) {
  *dst = malloc(bytes ? bytes : 1);
  return *dst && b200_d2h(*dst, d_src, bytes) == 0 ? 0 : -1;
}
static void write_data_dev(const char *filename, const ScsData *d, const ScsCone *k, const ScsSettings *stgs) {
  ScsData hd = *d;
  ScsMatrix hA = *d->A, hP;
  const long long nnzA = b200_read_dev_int(d->A->p + d->A->n), nnzP = d->P ? b200_read_dev_int(d->P->p + d->P->n) : 0;
  int ok = dev_to_host((void **)&hA.p, d->A->p, ((size_t)d->n + 1) * sizeof(scs_int)) == 0 &&
           dev_to_host((void **)&hA.i, d->A->i, (size_t)nnzA * sizeof(scs_int)) == 0 &&
           dev_to_host((void **)&hA.x, d->A->x, (size_t)nnzA * 8) == 0 &&
           dev_to_host((void **)&hd.b, d->b, (size_t)d->m * 8) == 0 &&
           dev_to_host((void **)&hd.c, d->c, (size_t)d->n * 8) == 0;
  hd.A = &hA;
  hd.P = SCS_NULL;
  memset(&hP, 0, sizeof(hP));
  if (d->P) {
    hP = *d->P;
    hP.p = SCS_NULL; hP.i = SCS_NULL; hP.x = SCS_NULL;
    ok = ok && dev_to_host((void **)&hP.p, d->P->p, ((size_t)d->n + 1) * sizeof(scs_int)) == 0 &&
         dev_to_host((void **)&hP.i, d->P->i, (size_t)nnzP * sizeof(scs_int)) == 0 &&
         dev_to_host((void **)&hP.x, d->P->x, (size_t)nnzP * 8) == 0;
    hd.P = &hP;
  }
  if (ok && b200_sync() == 0) scs_b200_write_data(filename, &hd, k, stgs);
  else printf("Error: could not copy the problem data to the host for %s\n", filename);
  free(hA.p); free(hA.i); free(hA.x); free(hP.p); free(hP.i); free(hP.x); free(hd.b); free(hd.c);
}

static ScsWork *init_device(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, void *stream, B200Ctx *ctx) {
  B200DevMats dm;
  ScsWork *w;
  memset(&dm, 0, sizeof(dm));
  if (!d || !k || !stgs) {
    printf("ERROR: Missing ScsData, ScsCone, or ScsSettings input\n");
    return SCS_NULL;
  }
  if (b200_runtime_init() != 0) {
    printf("ERROR: scs_b200 needs an sm_90 (H100) CUDA device: %s\n", b200_last_error());
    return SCS_NULL;
  }
  if (!b200_single_gpu()) return SCS_NULL;
  if ((d->A && ((d->A->p && !b200_dev_ptr_ok(d->A->p, "A->p")) || (d->A->i && !b200_dev_ptr_ok(d->A->i, "A->i")) ||
                (d->A->x && !b200_dev_ptr_ok(d->A->x, "A->x")))) ||
      (d->P && ((d->P->p && !b200_dev_ptr_ok(d->P->p, "P->p")) || (d->P->i && !b200_dev_ptr_ok(d->P->i, "P->i")) ||
                (d->P->x && !b200_dev_ptr_ok(d->P->x, "P->x")))) ||
      (d->b && !b200_dev_ptr_ok(d->b, "b")) || (d->c && !b200_dev_ptr_ok(d->c, "c"))) {
    printf("ERROR: Validation returned failure\n");
    return SCS_NULL;
  }
  if (!ctx || b200_wait_for_caller(stream) != 0) return SCS_NULL;
  w = init_work(d, k, stgs, &dm, 1, ctx);
  b200_sync(); /* the builder's blocks are free only once its kernels have run */
  b200_dev_mats_free(&dm);
  b200_caller_waits(stream);
  return w;
}
ScsWork *scs_b200_init_device(const ScsData *d, const ScsCone *k, const ScsSettings *stgs, void *stream) {
  B200Ctx *ctx = d && k && stgs ? b200_ctx_create() : SCS_NULL, *prev = b200_ctx_enter(ctx);
  ScsWork *w = init_device(d, k, stgs, stream, ctx);
  b200_ctx_leave(prev);
  if (!w) b200_ctx_release(ctx);
  return w;
}

static scs_int update_device(ScsWork *w, const scs_float *d_b, const scs_float *d_c, void *stream) {
  int rc = -1;
  if (!w || !b200_single_gpu() || (d_b && !b200_dev_ptr_ok(d_b, "b")) || (d_c && !b200_dev_ptr_ok(d_c, "c"))) return -1;
  if (b200_wait_for_caller(stream) != 0) return -1;
  if ((!d_b || b200_d2d(w->d_b_orig, d_b, (size_t)w->m * 8) == 0) &&
      (!d_c || b200_d2d(w->d_c_orig, d_c, (size_t)w->n * 8) == 0))
    rc = update_bc_dev(w);
  b200_caller_waits(stream);
  return rc;
}
scs_int scs_b200_update_device(ScsWork *w, const scs_float *d_b, const scs_float *d_c, void *stream) {
  B200Ctx *prev = b200_ctx_enter(w ? w->ctx : SCS_NULL);
  const scs_int rc = update_device(w, d_b, d_c, stream);
  b200_ctx_leave(prev);
  return rc;
}

/* New values of A (and P) on the pattern the workspace was built with (DESIGN.md section 1, "Matrix update"): the
 * validating copy of init, the builder's transpose, a pattern check of every entry against the resident streams (one
 * 4-byte read-back), and only then the values scattered into A, A' and P, the equilibration init chose, the
 * preconditioner and the CG copy refreshed, and the state of a fresh init restored. */
static void pattern_differs(const char *which) {
  printf("ERROR: the pattern of %s differs from the one the workspace was built with\n", which);
}
static scs_int update_matrix_device(ScsWork *w, const ScsMatrix *A, const ScsMatrix *P, void *stream) {
  const double t0 = now_ms();
  double t_mark = t0;
  const int n = w ? w->n : 0, m = w ? w->m : 0;
  B200DevMats dm;
  int *Tp = SCS_NULL, *Ti = SCS_NULL, *Fp = SCS_NULL, *Fi = SCS_NULL, *Fsrc = SCS_NULL;
  double *Tx = SCS_NULL, *Fx = SCS_NULL;
  unsigned *d_bad = SCS_NULL, bad = ~0u;
  int rc = -1;
  memset(&dm, 0, sizeof(dm));
  if (!w) { printf("ERROR: missing ScsWork input\n"); return -1; }
  if (!b200_single_gpu()) return -1;
  if (!A) { printf("ERROR: A matrix missing\n"); return -1; }
  if (P && !w->p->P) { printf("ERROR: P is given, but the workspace was built without P\n"); return -1; }
  if (!P && w->p->P) { printf("ERROR: the workspace was built with P, and no P is given\n"); return -1; }
  if (A->m != m || A->n != n) {
    printf("ERROR: A is %li x %li; the workspace was built for %i x %i\n", (long)A->m, (long)A->n, m, n);
    return -1;
  }
  if (P && (P->m != n || P->n != n)) {
    printf("ERROR: P is %li x %li; the workspace was built for %i x %i\n", (long)P->m, (long)P->n, n, n);
    return -1;
  }
  if ((A->p && !b200_dev_ptr_ok(A->p, "A->p")) || (A->i && !b200_dev_ptr_ok(A->i, "A->i")) ||
      (A->x && !b200_dev_ptr_ok(A->x, "A->x")) ||
      (P && ((P->p && !b200_dev_ptr_ok(P->p, "P->p")) || (P->i && !b200_dev_ptr_ok(P->i, "P->i")) ||
             (P->x && !b200_dev_ptr_ok(P->x, "P->x")))))
    return -1;
  if (b200_wait_for_caller(stream) != 0) return -1;
  do {
    /* 1. everything is checked before the first write to a resident array */
    if (b200_validate_matrix_dev(A, P, &dm) != 0) { printf("invalid linear system input data\n"); break; }
    if (dm.nnzA != w->nnzA) { pattern_differs("A"); break; }
    if (P && (dm.nnzP != w->nnzP || dm.fullP != b200_spmv_nnz(w->p->P))) { pattern_differs("P"); break; }
    init_mark("update: validating copy", &t_mark);
    Tp = (int *)b200_malloc(((size_t)m + 1) * 4);
    Ti = (int *)b200_malloc((size_t)dm.nnzA * 4);
    Tx = (double *)b200_malloc((size_t)dm.nnzA * 8);
    d_bad = (unsigned *)b200_malloc(4);
    if (!Tp || !Ti || !Tx || !d_bad || b200_memset0(d_bad, 4) != 0 ||
        b200_csc_transpose(m, n, dm.nnzA, dm.Ap, dm.Ai, dm.Ax, Tp, Ti, Tx) != 0)
      goto dev_fail;
    init_mark("update: transpose", &t_mark);
    if (P) {
      Fp = (int *)b200_malloc(((size_t)n + 1) * 4);
      Fi = (int *)b200_malloc((size_t)dm.fullP * 4);
      Fsrc = (int *)b200_malloc((size_t)dm.fullP * 4);
      if (!Fp || !Fi || !Fsrc || b200_sym_expand_structure(n, dm.nnzP, dm.fullP, dm.Pp, dm.Pi, Fp, Fi, Fsrc) != 0)
        goto dev_fail;
    }
    if (b200_spmv_check_pattern(w->p->At, dm.Ap, dm.Ai, dm.nnzA, 1u, d_bad) != 0 ||
        b200_spmv_check_pattern(w->p->A, Tp, Ti, dm.nnzA, 1u, d_bad) != 0 ||
        (P && b200_spmv_check_pattern(w->p->P, Fp, Fi, dm.fullP, 2u, d_bad) != 0) ||
        b200_d2h(&bad, d_bad, 4) != 0 || b200_sync() != 0)
      goto dev_fail;
    init_mark("update: pattern check", &t_mark);
    if (bad) { pattern_differs(bad & 1u ? "A" : "P"); break; }
    w->g_valid = 0; /* from here on the operators, diag_r, b and c change (d_g is zeroed in step 6) */
    /* 2. the raw values into both orientations of A, equilibrated in place as init did */
    if (b200_spmv_scatter_values(w->p->At, dm.Ap, dm.Ax) != 0 || b200_spmv_scatter_values(w->p->A, Tp, Tx) != 0)
      goto dev_fail;
    if (w->equil == B200_EQUIL_PAIR) {
      if (b200_equilibrate_dev(w->p->A, w->p->At, w->cone_boundaries, w->cone_boundaries_len, w->d_D, w->d_E) != 0)
        goto dev_fail;
    } else if (w->equil == B200_EQUIL_QP) {
      if (b200_equilibrate_qp_dev(w->p->A, w->p->At, dm.Pp, dm.Pi, dm.Px, Fp, Fi, Fsrc, w->cone_boundaries,
                                  w->cone_boundaries_len, w->d_D, w->d_E) != 0)
        goto dev_fail;
    }
    /* 3. P's values and diagonal from the (equilibrated) upper CSC */
    if (P) {
      Fx = (double *)b200_malloc((size_t)(dm.fullP > 0 ? dm.fullP : 1) * 8);
      if (!Fx || b200_sym_values(n, Fp, Fi, Fsrc, dm.Px, Fx, w->p->d_Pdiag) != 0 ||
          b200_spmv_scatter_values(w->p->P, Fp, Fx) != 0)
        goto dev_fail;
    }
    init_mark("update: values, equilibration", &t_mark);
    /* 4. the initial scale and diag_r; the preconditioner, A_cg's values and the R_y tables follow them */
    w->stgs->scale = w->scale0;
    set_diag_r_host(w);
    if (b200_admm_set_diag_r(&w->adm, w->k->z, w->stgs->rho_x, w->stgs->scale) != 0 ||
        b200_linsys_update_diag_r_dev(w->p, w->adm.d_R) != 0)
      goto dev_fail;
    w->p->last_cg_its = w->p->last_admm_its = w->p->last_g_its = 0;
    init_mark("update: preconditioner, CG copy", &t_mark);
    /* 5. D and E on the host (box bounds, CSV log); the box bounds renormalised from the originals */
    if (w->D && (b200_d2h(w->D, w->d_D, (size_t)m * 8) != 0 || b200_d2h(w->E, w->d_E, (size_t)n * 8) != 0 ||
                 b200_sync() != 0))
      goto dev_fail;
    if (w->k->bsize > 1) {
      memcpy(w->k->bl, w->bl_orig, (size_t)(w->k->bsize - 1) * 8);
      memcpy(w->k->bu, w->bu_orig, (size_t)(w->k->bsize - 1) * 8);
      b200_normalize_box(w->k, w->D, w->k->bl, w->k->bu);
    }
    if (b200_cones_set_box(w->cones, w->k->bl, w->k->bu) != 0) goto dev_fail;
    /* the log-det cones' warm starts and saved projections, as init leaves them */
    if (b200_cones_reset_spectral(w->cones) != 0) goto dev_fail;
    /* 6. the iterates, the scalar board, AA and the residual caches as init leaves them */
    if (b200_memset0(w->adm.d_cnt, 64) != 0 || b200_memset0(w->adm.d_sc, SC_COUNT * 8) != 0 ||
        b200_memset0(w->adm.d_u, ((size_t)n + m + 1) * 8) != 0 ||
        b200_memset0(w->adm.d_u_t, ((size_t)n + m + 1) * 8) != 0 ||
        b200_memset0(w->adm.d_v, ((size_t)n + m + 1) * 8) != 0 ||
        b200_memset0(w->adm.d_v_prev, ((size_t)n + m + 1) * 8) != 0 ||
        b200_memset0(w->adm.d_rsk, ((size_t)n + m + 1) * 8) != 0 ||
        b200_memset0(w->adm.d_g, ((size_t)n + m + 1) * 8) != 0)
      goto dev_fail;
    if (w->accel) b200_aa_restart_dev(w->accel);
    w->r_orig.last_iter = w->r_norm.last_iter = -1;
    /* 7. b and c renormalised from the originals with the new D, E */
    if (update_bc_dev(w) != 0) goto dev_fail;
    init_mark("update: box bounds, resets, b and c", &t_mark);
    rc = 0;
    break;
  dev_fail:
    printf("ERROR: scs_b200_update_matrix_device failed (%s)\n", b200_last_error());
  } while (0);
  b200_sync();
  b200_free(Tp); b200_free(Ti); b200_free(Tx); b200_free(d_bad);
  b200_free(Fp); b200_free(Fi); b200_free(Fsrc); b200_free(Fx);
  b200_dev_mats_free(&dm);
  if (rc == 0) w->setup_time = now_ms() - t0;
  b200_caller_waits(stream);
  return rc;
}
scs_int scs_b200_update_matrix_device(ScsWork *w, const ScsMatrix *A, const ScsMatrix *P, void *stream) {
  B200Ctx *prev = b200_ctx_enter(w ? w->ctx : SCS_NULL);
  const scs_int rc = update_matrix_device(w, A, P, stream);
  b200_ctx_leave(prev);
  return rc;
}

static scs_int solve_device(ScsWork *w, ScsSolution *d_sol, ScsInfo *info, scs_int warm_start, void *stream) {
  scs_int status;
  if (!w || !d_sol || !info) {
    printf("ERROR: missing ScsWork, ScsSolution or ScsInfo input\n");
    return -1;
  }
  if (!b200_single_gpu() || !b200_dev_ptr_ok(d_sol->x, "sol->x") || !b200_dev_ptr_ok(d_sol->y, "sol->y") ||
      !b200_dev_ptr_ok(d_sol->s, "sol->s"))
    return -1;
  if (b200_wait_for_caller(stream) != 0) return -1;
  w->sol_on_dev = 1;
  status = solve(w, d_sol, info, warm_start);
  w->sol_on_dev = 0;
  b200_caller_waits(stream);
  return status;
}
scs_int scs_b200_solve_device(ScsWork *w, ScsSolution *d_sol, ScsInfo *info, scs_int warm_start, void *stream) {
  B200Ctx *prev = b200_ctx_enter(w ? w->ctx : SCS_NULL);
  const scs_int status = solve_device(w, d_sol, info, warm_start, stream);
  b200_ctx_leave(prev);
  return status;
}

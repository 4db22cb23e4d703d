/* operators.c -- operator-level C-ABI entry points: the cone projection (reference src/cones.c:1498-1596) and
 * Anderson acceleration (reference src/aa.c:657-979), each through two doors. The host door stages host arrays
 * through the workspace's device buffers (the parity tests and bench.py compare one operator at a time against the
 * reference with it); the device door (scs_b200_*_device) runs on the caller's device buffers, ordered with the
 * caller's stream. Both run the same kernels the ADMM driver uses. Each workspace has an execution context of its own
 * (dev_api.h), bound by every call. */
#include "driver.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

struct SCS_B200_CONE_WORK {
  int m;
  B200Cones *cones;
  double *d_x, *d_ry;
  B200Ctx *ctx;
};

static void cone_free(ScsB200ConeWork *c) {
  b200_cones_destroy(c->cones);
  b200_free(c->d_x);
  b200_free(c->d_ry);
  free(c);
}

static ScsB200ConeWork *init_cone(const ScsCone *k, scs_int m, const scs_float *D) {
  ScsB200ConeWork *c;
  double *bl = SCS_NULL, *bu = SCS_NULL;
  if (!k || m <= 0) return SCS_NULL;
  if (b200_over_dim("m", -1, m) || b200_validate_cones(k, m) != 0) return SCS_NULL; /* before any device work */
  c = (ScsB200ConeWork *)calloc(1, sizeof(*c));
  if (!c) return SCS_NULL;
  c->ctx = b200_ctx_bound();
  c->m = (int)m;
  if (k->bsize > 1) { /* the caller's bounds stay as given */
    bl = (double *)malloc((size_t)(k->bsize - 1) * 8);
    bu = (double *)malloc((size_t)(k->bsize - 1) * 8);
    if (!bl || !bu) goto fail;
    memcpy(bl, k->bl, (size_t)(k->bsize - 1) * 8);
    memcpy(bu, k->bu, (size_t)(k->bsize - 1) * 8);
    b200_normalize_box(k, D, bl, bu);
  }
  c->cones = b200_cones_build(k, m, bl, bu);
  if (!c->cones) goto fail;
  c->d_x = (double *)b200_malloc((size_t)m * 8);
  c->d_ry = (double *)b200_malloc((size_t)m * 8);
  if (!c->d_x || !c->d_ry) goto fail;
  free(bl);
  free(bu);
  return c;
fail:
  free(bl);
  free(bu);
  cone_free(c);
  return SCS_NULL;
}

ScsB200ConeWork *scs_b200_init_cone(const ScsCone *k, scs_int m, const scs_float *D) {
  B200Ctx *ctx = b200_ctx_create(), *prev = b200_ctx_enter(ctx);
  ScsB200ConeWork *c = init_cone(k, m, D); /* a failed init has freed its blocks under ctx */
  b200_ctx_leave(prev);
  if (!c) b200_ctx_release(ctx);
  return c;
}

static scs_int proj_dual_cone(ScsB200ConeWork *c, scs_float *x, const scs_float *r_y) {
  const size_t bytes = (size_t)c->m * 8;
  if (b200_h2d(c->d_x, x, bytes) != 0) return -1;
  if (r_y && b200_h2d(c->d_ry, r_y, bytes) != 0) return -1;
  if (b200_cones_proj_dual(c->cones, c->d_x, r_y ? c->d_ry : SCS_NULL) != 0) return -1;
  if (b200_d2h(x, c->d_x, bytes) != 0) return -1;
  if (b200_sync() != 0) return -1;
  return b200_cones_check(c->cones); /* a failed eigen-decomposition is an error, like cones.c:1048-1052 */
}
scs_int scs_b200_proj_dual_cone(ScsB200ConeWork *c, scs_float *x, const scs_float *r_y) {
  B200Ctx *prev = b200_ctx_enter(c->ctx);
  const scs_int rc = proj_dual_cone(c, x, r_y);
  b200_ctx_leave(prev);
  return rc;
}

/* The device twins (include/scs_b200.h group (3)): the host twin's device function on the caller's buffers, after
 * the argument checks, between b200_wait_for_caller and b200_caller_waits. */
static scs_int proj_dual_cone_device(ScsB200ConeWork *c, scs_float *d_x, const scs_float *d_r_y, void *stream) {
  const size_t bytes = (size_t)c->m * 8;
  int rc;
  if (!b200_dev_ptr_ok(d_x, "x") || (d_r_y && !b200_dev_ptr_ok(d_r_y, "r_y")) ||
      b200_overlap("x", d_x, bytes, "r_y", d_r_y, bytes))
    return -1;
  if (b200_wait_for_caller(stream) != 0) return -1;
  rc = b200_cones_proj_dual(c->cones, d_x, d_r_y);
  b200_caller_waits(stream);
  if (rc != 0) return -1;
  return b200_cones_check(c->cones); /* reads the sticky flag back when there are eigen-decomposition cones */
}
scs_int scs_b200_proj_dual_cone_device(ScsB200ConeWork *c, scs_float *d_x, const scs_float *d_r_y, void *stream) {
  B200Ctx *prev;
  scs_int rc;
  if (!c) { printf("ERROR: missing ScsB200ConeWork input\n"); return -1; }
  if (!b200_single_gpu()) return -1;
  prev = b200_ctx_enter(c->ctx);
  rc = proj_dual_cone_device(c, d_x, d_r_y, stream);
  b200_ctx_leave(prev);
  return rc;
}

scs_int scs_b200_cone_logdet_stats(ScsB200ConeWork *c, scs_int *iter, scs_int *newton_success,
                                   scs_float *residuals) {
  int it = 0, success = 0, rc;
  B200Ctx *prev;
  if (!c) return -1;
  prev = b200_ctx_enter(c->ctx);
  rc = b200_cones_logdet_stats(c->cones, &it, &success, residuals);
  b200_ctx_leave(prev);
  if (rc != 0) return -1;
  *iter = it;
  *newton_success = success;
  return 0;
}

void scs_b200_finish_cone(ScsB200ConeWork *c) {
  B200Ctx *ctx, *prev;
  if (!c) return;
  ctx = c->ctx;
  prev = b200_ctx_enter(ctx);
  cone_free(c);
  b200_ctx_leave(prev);
  b200_ctx_release(ctx);
}

/* ------------------------------------------------------------------ AA */
struct SCS_B200_AA_WORK {
  int dim;
  B200Aa *a;
  double *d_f, *d_x;
  B200Ctx *ctx;
};

static int over_int(long long v) { return v > 2147483647LL; }

static void aa_free(ScsB200AaWork *w) {
  b200_aa_destroy(w->a);
  b200_free(w->d_f);
  b200_free(w->d_x);
  free(w);
}

ScsB200AaWork *scs_b200_aa_init(scs_int dim, scs_int mem, scs_int min_len, scs_int type1,
                                scs_float regularization, scs_float relaxation,
                                scs_float safeguard_factor, scs_float max_weight_norm,
                                scs_int ir_max_steps, scs_int verbosity) {
  ScsB200AaWork *w;
  B200Ctx *prev;
  /* the vector length and the memory are int inside; larger 64-bit values are refused, not truncated */
  if (over_int(dim) || b200_over_dim("mem", -1, mem) || b200_over_dim("min_len", -1, min_len) ||
      b200_over_dim("ir_max_steps", -1, ir_max_steps))
    return SCS_NULL;
  w = (ScsB200AaWork *)calloc(1, sizeof(*w));
  if (!w) return SCS_NULL;
  w->dim = (int)dim;
  w->ctx = b200_ctx_create();
  prev = b200_ctx_enter(w->ctx);
  w->a = b200_aa_create((int)dim, (int)mem, (int)min_len, type1 != 0, regularization, relaxation, safeguard_factor,
                        max_weight_norm, (int)ir_max_steps,
                        verbosity > 2 ? 2 : verbosity < 0 ? 0 : (int)verbosity); /* levels 0, 1, 2 */
  if (w->a) {
    w->d_f = (double *)b200_malloc((size_t)dim * 8);
    w->d_x = (double *)b200_malloc((size_t)dim * 8);
  }
  if (!w->a || !w->d_f || !w->d_x) {
    B200Ctx *ctx = w->ctx;
    aa_free(w);
    b200_ctx_leave(prev);
    b200_ctx_release(ctx);
    return SCS_NULL;
  }
  b200_ctx_leave(prev);
  return w;
}

static scs_float aa_apply(ScsB200AaWork *w, scs_float *f, const scs_float *x) {
  const size_t bytes = (size_t)w->dim * 8;
  double nrm;
  if (b200_h2d(w->d_f, f, bytes) != 0 || b200_h2d(w->d_x, x, bytes) != 0) return NAN;
  nrm = b200_aa_apply_dev(w->a, w->d_f, w->d_x);
  if (b200_d2h(f, w->d_f, bytes) != 0 || b200_sync() != 0) return NAN;
  return nrm;
}
scs_float scs_b200_aa_apply(ScsB200AaWork *w, scs_float *f, const scs_float *x) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_float nrm = aa_apply(w, f, x);
  b200_ctx_leave(prev);
  return nrm;
}

static scs_int aa_safeguard(ScsB200AaWork *w, scs_float *f_new, scs_float *x_new) {
  const size_t bytes = (size_t)w->dim * 8;
  int rc;
  if (b200_h2d(w->d_f, f_new, bytes) != 0 || b200_h2d(w->d_x, x_new, bytes) != 0) return 0;
  rc = b200_aa_safeguard_dev(w->a, w->d_f, w->d_x);
  if (rc < 0) {
    b200_d2h(f_new, w->d_f, bytes);
    b200_d2h(x_new, w->d_x, bytes);
    b200_sync();
  }
  return rc;
}
scs_int scs_b200_aa_safeguard(ScsB200AaWork *w, scs_float *f_new, scs_float *x_new) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  const scs_int rc = aa_safeguard(w, f_new, x_new);
  b200_ctx_leave(prev);
  return rc;
}

/* the AA twins: refused with NaN (apply) or -1 (safeguard), the workspace and both vectors untouched */
static int aa_device_ok(const ScsB200AaWork *w, const char *f_name, const scs_float *d_f, const char *x_name,
                        const scs_float *d_x) {
  const size_t bytes = w ? (size_t)w->dim * 8 : 0;
  if (!w) { printf("ERROR: missing ScsB200AaWork input\n"); return 0; }
  return b200_single_gpu() && b200_dev_ptr_ok(d_f, f_name) && b200_dev_ptr_ok(d_x, x_name) &&
         !b200_overlap(f_name, d_f, bytes, x_name, d_x, bytes);
}
scs_float scs_b200_aa_apply_device(ScsB200AaWork *w, scs_float *d_f, const scs_float *d_x, void *stream) {
  B200Ctx *prev;
  scs_float nrm = NAN;
  if (!aa_device_ok(w, "f", d_f, "x", d_x)) return NAN;
  prev = b200_ctx_enter(w->ctx);
  if (b200_wait_for_caller(stream) == 0) {
    nrm = b200_aa_apply_dev(w->a, d_f, d_x); /* the scalars it needs are read back before it returns */
    b200_caller_waits(stream);
  }
  b200_ctx_leave(prev);
  return nrm;
}
scs_int scs_b200_aa_safeguard_device(ScsB200AaWork *w, scs_float *d_f_new, scs_float *d_x_new, void *stream) {
  B200Ctx *prev;
  scs_int rc = -1;
  if (!aa_device_ok(w, "f_new", d_f_new, "x_new", d_x_new)) return -1;
  prev = b200_ctx_enter(w->ctx);
  if (b200_wait_for_caller(stream) == 0) {
    rc = b200_aa_safeguard_dev(w->a, d_f_new, d_x_new);
    b200_caller_waits(stream);
  }
  b200_ctx_leave(prev);
  return rc;
}

void scs_b200_aa_reset(ScsB200AaWork *w) {
  B200Ctx *prev = b200_ctx_enter(w->ctx);
  b200_aa_reset_dev(w->a);
  b200_ctx_leave(prev);
}

void scs_b200_aa_finish(ScsB200AaWork *w) {
  B200Ctx *ctx, *prev;
  if (!w) return;
  ctx = w->ctx;
  prev = b200_ctx_enter(ctx);
  aa_free(w);
  b200_ctx_leave(prev);
  b200_ctx_release(ctx);
}

AaStats scs_b200_aa_get_stats(const ScsB200AaWork *w) {
  AaStats s;
  int o[8];
  double d[2];
  b200_aa_stats(w->a, o, d);
  s.iter = o[0]; s.n_accept = o[1]; s.n_reject_lapack = o[2]; s.n_reject_rank0 = o[3];
  s.n_reject_nonfinite = o[4]; s.n_reject_weight_cap = o[5]; s.n_safeguard_reject = o[6];
  s.last_rank = o[7]; s.last_aa_norm = d[0]; s.last_regularization = d[1];
  return s;
}

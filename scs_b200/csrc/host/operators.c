/* operators.c -- operator-level C-ABI entry points with HOST buffers, used by
 * the parity tests and bench.py to compare one operator at a time against the
 * reference: the cone projection (reference src/cones.c:1498-1596) and Anderson
 * acceleration (reference src/aa.c:657-979). Each call stages the host arrays
 * through device memory and runs the same kernels the ADMM driver uses. */
#include "driver.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

struct SCS_B200_CONE_WORK {
  int m;
  B200Cones *cones;
  double *d_x, *d_ry;
};

ScsB200ConeWork *scs_b200_init_cone(const ScsCone *k, scs_int m, const scs_float *D) {
  ScsB200ConeWork *c;
  double *bl = SCS_NULL, *bu = SCS_NULL;
  scs_int j;
  long long dims;
  B200ConeInts ci;
  if (!k || m <= 0) return SCS_NULL;
  if (b200_over_dim("m", -1, m) || b200_cone_over_limits(k)) return SCS_NULL; /* in scs_int width, before narrowing */
  if (k->cssize < 0 || (k->cssize > 0 && !k->cs)) return SCS_NULL;
  if (k->ep < 0 || k->ed < 0 || k->psize < 0 || (k->psize > 0 && !k->p)) return SCS_NULL;
  dims = (long long)k->z + k->l + k->bsize;
  for (j = 0; j < k->qsize; ++j) dims += k->q[j];
  for (j = 0; j < k->ssize; ++j) dims += ((long long)k->s[j] * (k->s[j] + 1)) / 2;
  for (j = 0; j < k->cssize; ++j) dims += (long long)k->cs[j] * k->cs[j];
  dims += 3LL * ((long long)k->ep + k->ed + k->psize);
#ifdef USE_SPECTRAL_CONES
  if (k->dsize != 0 || k->nucsize < 0 || k->ell1_size < 0 || k->sl_size < 0) return SCS_NULL; /* no log-det cones */
  if ((k->nucsize > 0 && (!k->nuc_m || !k->nuc_n)) || (k->ell1_size > 0 && !k->ell1) ||
      (k->sl_size > 0 && (!k->sl_n || !k->sl_k)))
    return SCS_NULL;
  for (j = 0; j < k->nucsize; ++j)
    if (k->nuc_m[j] < 1 || k->nuc_n[j] < 1 || k->nuc_n[j] > k->nuc_m[j]) return SCS_NULL;
  for (j = 0; j < k->ell1_size; ++j)
    if (k->ell1[j] < 1) return SCS_NULL;
  for (j = 0; j < k->sl_size; ++j)
    if (k->sl_k[j] <= 0 || k->sl_k[j] >= k->sl_n[j]) return SCS_NULL;
  dims += b200_spectral_rows(k);
#endif
  if (dims != m) {
    fprintf(stderr, "scs_b200: cone dims %lld != m %lld\n", dims, (long long)m);
    return SCS_NULL;
  }
  c = (ScsB200ConeWork *)calloc(1, sizeof(*c));
  if (!c) return SCS_NULL;
  c->m = (int)m;
  if (k->bsize > 1) {
    /* box bounds follow the row scaling (reference normalize_box_cone, cones.c:1160-1177);
     * as in the reference, the +-1e15 -> inf mapping only happens when a scaling is given */
    const double *Db = D ? D + k->z + k->l : SCS_NULL;
    bl = (double *)malloc((size_t)(k->bsize - 1) * 8);
    bu = (double *)malloc((size_t)(k->bsize - 1) * 8);
    if (!bl || !bu) goto fail;
    for (j = 0; j < k->bsize - 1; ++j) {
      bl[j] = k->bl[j];
      bu[j] = k->bu[j];
      if (Db) {
        const double factor = Db[j + 1] / Db[0];
        if (bu[j] >= MAX_BOX_VAL) bu[j] = INFINITY; else bu[j] *= factor;
        if (bl[j] <= -MAX_BOX_VAL) bl[j] = -INFINITY; else bl[j] *= factor;
      }
    }
  }
  if (b200_cone_ints(k, &ci) != 0) goto fail; /* int copies for the kernel layer */
  c->cones = b200_cones_create(c->m, (int)k->z, (int)k->l, (int)k->bsize, bl, bu, (int)k->qsize, ci.q, (int)k->ssize,
                               ci.s);
  free(bl);
  free(bu);
  bl = bu = SCS_NULL;
  if (!c->cones) goto fail_ints;
#ifdef USE_SPECTRAL_CONES
  if (b200_cones_set_spectral(c->cones, (int)k->nucsize, ci.nuc_m, ci.nuc_n, (int)k->ell1_size, ci.ell1,
                              (int)k->sl_size, ci.sl_n, ci.sl_k) != 0)
    goto fail_ints;
#endif
  if (b200_cones_set_triples(c->cones, (int)k->ep, (int)k->ed, (int)k->psize, k->p) != 0) goto fail_ints;
  if (b200_cones_set_complex_psd(c->cones, (int)k->cssize, ci.cs, (int)(k->ep + k->ed + k->psize)) != 0)
    goto fail_ints;
  b200_cone_ints_free(&ci);
  c->d_x = (double *)b200_malloc((size_t)m * 8);
  c->d_ry = (double *)b200_malloc((size_t)m * 8);
  if (!c->d_x || !c->d_ry) goto fail;
  return c;
fail_ints:
  b200_cone_ints_free(&ci);
fail:
  free(bl);
  free(bu);
  scs_b200_finish_cone(c);
  return SCS_NULL;
}

scs_int scs_b200_proj_dual_cone(ScsB200ConeWork *c, scs_float *x, const scs_float *r_y) {
  const size_t bytes = (size_t)c->m * 8;
  if (b200_h2d(c->d_x, x, bytes) != 0) return -1;
  if (r_y && b200_h2d(c->d_ry, r_y, bytes) != 0) return -1;
  if (b200_cones_proj_dual(c->cones, c->d_x, r_y ? c->d_ry : SCS_NULL) != 0) return -1;
  if (b200_d2h(x, c->d_x, bytes) != 0) return -1;
  if (b200_sync() != 0) return -1;
  return b200_cones_check(c->cones); /* a failed eigen-decomposition is an error, like cones.c:1048-1052 */
}

void scs_b200_finish_cone(ScsB200ConeWork *c) {
  if (!c) return;
  b200_cones_destroy(c->cones);
  b200_free(c->d_x);
  b200_free(c->d_ry);
  free(c);
}

/* ------------------------------------------------------------------ AA */
struct SCS_B200_AA_WORK {
  int dim;
  B200Aa *a;
  double *d_f, *d_x;
};

static int over_int(long long v) { return v > 2147483647LL; }

ScsB200AaWork *scs_b200_aa_init(scs_int dim, scs_int mem, scs_int min_len, scs_int type1,
                                scs_float regularization, scs_float relaxation,
                                scs_float safeguard_factor, scs_float max_weight_norm,
                                scs_int ir_max_steps, scs_int verbosity) {
  ScsB200AaWork *w;
  /* the vector length and the memory are int inside; larger 64-bit values are refused, not truncated */
  if (over_int(dim) || b200_over_dim("mem", -1, mem) || b200_over_dim("min_len", -1, min_len) ||
      b200_over_dim("ir_max_steps", -1, ir_max_steps))
    return SCS_NULL;
  w = (ScsB200AaWork *)calloc(1, sizeof(*w));
  if (!w) return SCS_NULL;
  w->dim = (int)dim;
  w->a = b200_aa_create((int)dim, (int)mem, (int)min_len, type1 != 0, regularization, relaxation, safeguard_factor,
                        max_weight_norm, (int)ir_max_steps,
                        verbosity > 2 ? 2 : verbosity < 0 ? 0 : (int)verbosity); /* levels 0, 1, 2 */
  if (!w->a) { free(w); return SCS_NULL; }
  w->d_f = (double *)b200_malloc((size_t)dim * 8);
  w->d_x = (double *)b200_malloc((size_t)dim * 8);
  if (!w->d_f || !w->d_x) { scs_b200_aa_finish(w); return SCS_NULL; }
  return w;
}

scs_float scs_b200_aa_apply(ScsB200AaWork *w, scs_float *f, const scs_float *x) {
  const size_t bytes = (size_t)w->dim * 8;
  double nrm;
  if (b200_h2d(w->d_f, f, bytes) != 0 || b200_h2d(w->d_x, x, bytes) != 0) return NAN;
  nrm = b200_aa_apply_dev(w->a, w->d_f, w->d_x);
  if (b200_d2h(f, w->d_f, bytes) != 0 || b200_sync() != 0) return NAN;
  return nrm;
}

scs_int scs_b200_aa_safeguard(ScsB200AaWork *w, scs_float *f_new, scs_float *x_new) {
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

void scs_b200_aa_reset(ScsB200AaWork *w) { b200_aa_reset_dev(w->a); }

void scs_b200_aa_finish(ScsB200AaWork *w) {
  if (!w) return;
  b200_aa_destroy(w->a);
  b200_free(w->d_f);
  b200_free(w->d_x);
  free(w);
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

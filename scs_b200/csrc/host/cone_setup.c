/* cone_setup.c -- the cone setup shared by scs_init (host/scs_driver.c) and scs_b200_init_cone (host/operators.c):
 * the validation of an ScsCone against the rows it covers, the scaling of the box bounds by D and the build of the
 * device cone workspace. Here because every library flavour links this file; the plugin-only ones leave out the
 * driver. */
#include "driver.h"
#include <math.h>
#include <stdio.h>

/* reference src/cones.c:583-765 (validate_cones) for a cone of m rows; every count and size is checked below 2^30
 * before any sum of them */
int b200_validate_cones(const ScsCone *k, scs_int m) {
  scs_int i;
  long long dims;
#ifdef USE_SPECTRAL_CONES
  static const char *names[4] = {"log-det", "nuclear-norm", "l1-norm", "sum-of-largest-eigenvalues"};
  const scs_int counts[4] = {k->dsize, k->nucsize, k->ell1_size, k->sl_size};
  long long rows[4] = {0, 0, 0, 0};
  int f, first = 1;
#endif
  if (b200_cone_over_limits(k)) return -1;
  if (k->z < 0) { printf("free cone dimension error\n"); return -1; }
  if (k->l < 0) { printf("lp cone dimension error\n"); return -1; }
  if (k->bsize < 0) { printf("box cone dimension error\n"); return -1; }
  if (k->bsize > 1) {
    if (!k->bl || !k->bu) { printf("box cone bounds missing\n"); return -1; }
    for (i = 0; i < k->bsize - 1; ++i) {
      if (isnan(k->bl[i]) || isnan(k->bu[i])) { printf("box cone bounds cannot be NaN\n"); return -1; }
      if (k->bl[i] == INFINITY || k->bu[i] == -INFINITY) {
        printf("box cone bounds use invalid infinity direction\n");
        return -1;
      }
      if (k->bl[i] > k->bu[i]) {
        printf("infeasible: box lower bound larger than upper bound\n");
        return -1;
      }
    }
  }
  if (k->qsize < 0 || (k->qsize > 0 && !k->q)) { printf("soc cone dimension error\n"); return -1; }
  for (i = 0; i < k->qsize; ++i)
    if (k->q[i] < 0) { printf("soc cone dimension error\n"); return -1; }
  if (k->ssize < 0 || (k->ssize > 0 && !k->s)) { printf("sd cone dimension error\n"); return -1; }
  for (i = 0; i < k->ssize; ++i)
    if (k->s[i] < 0) { printf("sd cone dimension error\n"); return -1; }
  if (k->cssize < 0 || k->ed < 0 || k->ep < 0 || k->psize < 0) {
    printf("cone dimension error\n");
    return -1;
  }
  if (k->cssize > 0) {
    if (!k->cs) { printf("complex sd cone array missing\n"); return -1; }
    for (i = 0; i < k->cssize; ++i)
      if (k->cs[i] < 0) { printf("complex sd cone dimension error\n"); return -1; }
  }
  if (k->psize > 0) { /* reference cones.c:678-690 */
    if (!k->p) { printf("power cone array missing\n"); return -1; }
    for (i = 0; i < k->psize; ++i)
      if (!isfinite(k->p[i]) || k->p[i] < -1 || k->p[i] > 1) { printf("power cone error, values must be in [-1,1]\n"); return -1; }
  }
#ifdef USE_SPECTRAL_CONES /* reference cones.c:690-754 */
  if (k->dsize < 0 || (k->dsize > 0 && !k->d)) { printf("logdet cone dimension error\n"); return -1; }
  for (i = 0; i < k->dsize; ++i)
    if (k->d[i] < 1) { printf("logdet cone dimension error\n"); return -1; }
  if (k->nucsize < 0) { printf("nuclear cone dimension error\n"); return -1; }
  if (k->nucsize > 0 && (!k->nuc_m || !k->nuc_n)) { printf("nuclear cone arrays missing\n"); return -1; }
  for (i = 0; i < k->nucsize; ++i)
    if (k->nuc_m[i] < 1 || k->nuc_n[i] < 1 || k->nuc_n[i] > k->nuc_m[i]) {
      printf("nuclear norm cone dimension error\n");
      return -1;
    }
  if (k->ell1_size < 0) { printf("ell1 cone dimension error\n"); return -1; }
  if (k->ell1_size > 0 && !k->ell1) { printf("ell1 cone array missing\n"); return -1; }
  for (i = 0; i < k->ell1_size; ++i)
    if (k->ell1[i] < 1) { printf("ell1 cone dimension error\n"); return -1; }
  if (k->sl_size < 0) { printf("sum-of-largest-eigenvalues cone dimension error\n"); return -1; }
  if (k->sl_size > 0 && (!k->sl_n || !k->sl_k)) { printf("sum-of-largest-eigenvalues cone arrays missing\n"); return -1; }
  for (i = 0; i < k->sl_size; ++i)
    if (k->sl_k[i] >= k->sl_n[i] || k->sl_k[i] <= 0) {
      printf("sum-of-largest-eigenvalues cone dimension error\n");
      return -1;
    }
#endif
  dims = (long long)k->z + k->l + k->bsize;
  for (i = 0; i < k->qsize; ++i) dims += k->q[i];
  for (i = 0; i < k->ssize; ++i) dims += (long long)k->s[i] * (k->s[i] + 1) / 2;
  for (i = 0; i < k->cssize; ++i) dims += (long long)k->cs[i] * k->cs[i];
  dims += 3LL * ((long long)k->ep + k->ed + k->psize);
#ifdef USE_SPECTRAL_CONES /* rows of the spectral cones (reference cones.c:435-443) */
  for (i = 0; i < k->dsize; ++i) rows[0] += (long long)k->d[i] * (k->d[i] + 1) / 2 + 2;
  for (i = 0; i < k->nucsize; ++i) rows[1] += (long long)k->nuc_m[i] * k->nuc_n[i] + 1;
  for (i = 0; i < k->ell1_size; ++i) rows[2] += (long long)k->ell1[i] + 1;
  for (i = 0; i < k->sl_size; ++i) rows[3] += (long long)k->sl_n[i] * (k->sl_n[i] + 1) / 2 + 1;
  dims += rows[0] + rows[1] + rows[2] + rows[3];
#endif
  if (dims != m) {
    printf("Error: Cone dims %li != rows in A %li", (long)dims, (long)m);
#ifdef USE_SPECTRAL_CONES /* name the spectral families: a wrong cone array usually comes from one of them */
    for (f = 0; f < 4; ++f) {
      if (counts[f] == 0) continue;
      printf("%s%lli rows in %lli %s cone%s", first ? " (spectral: " : ", ", rows[f], (long long)counts[f], names[f],
             counts[f] == 1 ? "" : "s");
      first = 0;
    }
    if (!first) printf(")");
#endif
    printf("\n");
    return -1;
  }
  return 0;
}

/* box bounds follow the row scaling (reference normalize_box_cone, cones.c:1160-1177); as in the reference, the
 * +-1e15 -> inf mapping only happens when a scaling is given, so D == NULL leaves them as they are */
void b200_normalize_box(const ScsCone *k, const double *D, double *bl, double *bu) {
  scs_int j;
  if (!D) return;
  D += k->z + k->l; /* the rows of the box cone */
  for (j = 0; j < k->bsize - 1; ++j) {
    const double factor = D[j + 1] / D[0];
    if (bu[j] >= MAX_BOX_VAL) bu[j] = INFINITY; else bu[j] *= factor;
    if (bl[j] <= -MAX_BOX_VAL) bl[j] = -INFINITY; else bl[j] *= factor;
  }
}

B200Cones *b200_cones_build(const ScsCone *k, scs_int m, const double *bl, const double *bu) {
  B200ConeInts ci;
  B200Cones *c;
  int bad;
  if (b200_cone_ints(k, &ci) != 0) return SCS_NULL; /* int copies for the kernel layer */
  c = b200_cones_create((int)m, (int)k->z, (int)k->l, (int)k->bsize, bl, bu, (int)k->qsize, ci.q, (int)k->ssize,
                        ci.s);
  bad = !c;
#ifdef USE_SPECTRAL_CONES
  bad = bad || b200_cones_set_spectral(c, (int)k->dsize, ci.d, (int)k->nucsize, ci.nuc_m, ci.nuc_n,
                                       (int)k->ell1_size, ci.ell1, (int)k->sl_size, ci.sl_n, ci.sl_k) != 0;
#endif
  bad = bad || b200_cones_set_triples(c, (int)k->ep, (int)k->ed, (int)k->psize, k->p) != 0 ||
        b200_cones_set_complex_psd(c, (int)k->cssize, ci.cs, (int)(k->ep + k->ed + k->psize)) != 0;
  b200_cone_ints_free(&ci);
  if (bad && c) {
    b200_cones_destroy(c);
    c = SCS_NULL;
  }
  return c;
}

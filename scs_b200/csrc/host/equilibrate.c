/* equilibrate.c -- Ruiz + L2 equilibration of A and P on the host at setup.
 * Setup path (runs once per scs_init), not part of the per-iteration hot
 * loop. It serves the multi-GPU path with P != 0 only; one GPU runs its
 * device form, b200_equilibrate_qp_dev (kernels/equil.cu), with the same bits.
 *
 * Same algorithm and constants as reference linsys/scs_matrix.c:229-496
 * (compute_ruiz_mats / compute_l2_mats / rescale / normalize_a_p: 25 Ruiz
 * passes + 1 L2 pass, limits 1e-4 / 1e4, D constant inside every cone of
 * size > 1).
 */
#include "driver.h"
#include <math.h>
#include <stdlib.h>

#define MIN_NORMALIZATION_FACTOR (1e-4)
#define MAX_NORMALIZATION_FACTOR (1e4)
#define NUM_RUIZ_PASSES (25)
#define NUM_L2_PASSES (1)

static double apply_limit(double x) {
  x = x < MIN_NORMALIZATION_FACTOR ? 1.0 : x;
  x = x > MAX_NORMALIZATION_FACTOR ? MAX_NORMALIZATION_FACTOR : x;
  return x;
}

/* aggregate vec over every cone block after the first z+l+bsize rows;
 * mode 0: max |.|, mode 1: mean  (reference enforce_cone_boundaries, cones.c:366-379) */
static void enforce_boundaries(const int *bnd, int nbnd, double *vec, int mode) {
  int i, j, count = bnd[0];
  for (i = 1; i < nbnd; ++i) {
    const int delta = bnd[i];
    double wrk = 0.0;
    if (mode == 0) {
      for (j = count; j < count + delta; ++j) {
        const double t = fabs(vec[j]);
        if (t > wrk) wrk = t;
      }
    } else {
      for (j = count; j < count + delta; ++j) wrk += vec[j];
      wrk = delta > 0 ? wrk / delta : 0.0;
    }
    for (j = count; j < count + delta; ++j) vec[j] = wrk;
    count += delta;
  }
}

static void ruiz_mats(const ScsMatrix *P, const ScsMatrix *A, double *Dt, double *Et, const int *bnd,
                      int nbnd) {
  scs_int i, j, kk;
  for (i = 0; i < A->m; ++i) Dt[i] = 0.;
  for (i = 0; i < A->n; ++i)
    for (j = A->p[i]; j < A->p[i + 1]; ++j) {
      const double t = fabs(A->x[j]);
      if (t > Dt[A->i[j]]) Dt[A->i[j]] = t;
    }
  enforce_boundaries(bnd, nbnd, Dt, 0);
  for (i = 0; i < A->m; ++i) {
    Dt[i] = sqrt(apply_limit(Dt[i]));
    Dt[i] = SAFEDIV_POS(1.0, Dt[i]);
  }
  for (i = 0; i < A->n; ++i) Et[i] = 0.;
  if (P) {
    for (j = 0; j < P->n; j++)
      for (kk = P->p[j]; kk < P->p[j + 1]; kk++) {
        const double wrk = fabs(P->x[kk]);
        i = P->i[kk];
        if (wrk > Et[j]) Et[j] = wrk;
        if (i != j && wrk > Et[i]) Et[i] = wrk;
      }
  }
  for (i = 0; i < A->n; ++i) {
    double nm = 0.0;
    for (j = A->p[i]; j < A->p[i + 1]; ++j) {
      const double t = fabs(A->x[j]);
      if (t > nm) nm = t;
    }
    if (nm > Et[i]) Et[i] = nm;
    Et[i] = sqrt(apply_limit(Et[i]));
    Et[i] = SAFEDIV_POS(1.0, Et[i]);
  }
}

static void l2_mats(const ScsMatrix *P, const ScsMatrix *A, double *Dt, double *Et, const int *bnd,
                    int nbnd) {
  scs_int i, j, kk;
  for (i = 0; i < A->m; ++i) Dt[i] = 0.;
  for (i = 0; i < A->n; ++i)
    for (j = A->p[i]; j < A->p[i + 1]; ++j) Dt[A->i[j]] += A->x[j] * A->x[j];
  for (i = 0; i < A->m; ++i) Dt[i] = sqrt(Dt[i]);
  enforce_boundaries(bnd, nbnd, Dt, 1);
  for (i = 0; i < A->m; ++i) {
    Dt[i] = sqrt(apply_limit(Dt[i]));
    Dt[i] = SAFEDIV_POS(1.0, Dt[i]);
  }
  for (i = 0; i < A->n; ++i) Et[i] = 0.;
  if (P) {
    for (j = 0; j < P->n; j++)
      for (kk = P->p[j]; kk < P->p[j + 1]; kk++) {
        const double wrk = P->x[kk] * P->x[kk];
        i = P->i[kk];
        Et[j] += wrk;
        if (i != j) Et[i] += wrk;
      }
  }
  for (i = 0; i < A->n; ++i) {
    double s = 0.0;
    for (j = A->p[i]; j < A->p[i + 1]; ++j) s += A->x[j] * A->x[j];
    Et[i] += s;
    Et[i] = sqrt(apply_limit(sqrt(Et[i])));
    Et[i] = SAFEDIV_POS(1.0, Et[i]);
  }
}

static void rescale(ScsMatrix *P, ScsMatrix *A, const double *Dt, const double *Et, double *D,
                    double *E) {
  scs_int i, j;
  for (i = 0; i < A->n; ++i) {
    const double ei = Et[i];
    for (j = A->p[i]; j < A->p[i + 1]; ++j) A->x[j] *= Dt[A->i[j]] * ei;
  }
  if (P) {
    for (i = 0; i < P->n; ++i) {
      const double ei = Et[i];
      for (j = P->p[i]; j < P->p[i + 1]; ++j) P->x[j] *= Et[P->i[j]] * ei;
    }
  }
  for (i = 0; i < A->m; ++i) D[i] *= Dt[i];
  for (i = 0; i < A->n; ++i) E[i] *= Et[i];
}

/* A -> D A E, P -> E P E in place; D (m), E (n) are outputs. bnd[0] = z+l+bsize,
 * bnd[1..] = sizes of the cones that must share one D value. */
int b200_equilibrate(ScsMatrix *P, ScsMatrix *A, const int *bnd, int nbnd, double *D, double *E) {
  int i;
  double *Dt = (double *)calloc((size_t)A->m, sizeof(double));
  double *Et = (double *)calloc((size_t)A->n, sizeof(double));
  if (!Dt || !Et) {
    free(Dt);
    free(Et);
    return -1;
  }
  for (i = 0; i < A->m; ++i) D[i] = 1.;
  for (i = 0; i < A->n; ++i) E[i] = 1.;
  for (i = 0; i < NUM_RUIZ_PASSES; ++i) {
    ruiz_mats(P, A, Dt, Et, bnd, nbnd);
    rescale(P, A, Dt, Et, D, E);
  }
  for (i = 0; i < NUM_L2_PASSES; ++i) {
    l2_mats(P, A, Dt, Et, bnd, nbnd);
    rescale(P, A, Dt, Et, D, E);
  }
  free(Dt);
  free(Et);
  return 0;
}

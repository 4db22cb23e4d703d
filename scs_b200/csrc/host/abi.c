/* abi.c -- the integer width of the C ABI (include/scs_b200.h) and its boundary with the kernel layer.
 *
 * scs_int is int in the default build and long long in the DLONG build (the reference's include/scs_types.h:14-24 on
 * LP64). The kernel layer (dev_api.h, admm_api.h) takes int everywhere. Every count, size or index a caller passes is
 * checked here in scs_int width against the limits of the operators (dev_api.h B200_MAX_DIM, B200_MAX_STORED) and only
 * then narrowed; a value that does not fit is refused with a message that names the limit, never truncated. The
 * matrix indices of A and P are checked and narrowed on the device, by the validating copy (kernels/setup.cu) that
 * b200_csc_upload (host/linsys_b200.c) runs them through. The argument checks of the device-pointer entry points
 * (device pointers, a single GPU, disjoint vectors) are here too. */
#include "driver.h"
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* The struct layouts of the reference's headers, compiled with gcc on x86-64 in the matching configuration: a caller
 * built against them passes exactly these bytes. */
#ifdef DLONG
_Static_assert(sizeof(scs_int) == 8, "DLONG: scs_int is 64 bits");
_Static_assert(sizeof(ScsMatrix) == 40, "ScsMatrix layout (DLONG)");
_Static_assert(sizeof(ScsData) == 48, "ScsData layout (DLONG)");
_Static_assert(sizeof(ScsSettings) == 152 && offsetof(ScsSettings, write_data_filename) == 136 &&
                   offsetof(ScsSettings, log_csv_filename) == 144,
               "ScsSettings layout (DLONG)");
#ifdef USE_SPECTRAL_CONES
_Static_assert(sizeof(ScsCone) == 200 && offsetof(ScsCone, d) == 120 && offsetof(ScsCone, nuc_m) == 136 &&
                   offsetof(ScsCone, ell1) == 160 && offsetof(ScsCone, sl_n) == 176 && offsetof(ScsCone, sl_size) == 192,
               "ScsCone layout (DLONG, spectral cones)");
#else
_Static_assert(sizeof(ScsCone) == 120 && offsetof(ScsCone, p) == 104 && offsetof(ScsCone, psize) == 112,
               "ScsCone layout (DLONG)");
#endif
_Static_assert(sizeof(AaStats) == 80, "AaStats layout (DLONG)");
_Static_assert(sizeof(ScsInfo) == 496 && offsetof(ScsInfo, status) == 8 && offsetof(ScsInfo, lin_sys_solver) == 136 &&
                   offsetof(ScsInfo, pobj) == 280 && offsetof(ScsInfo, aa_stats) == 392 &&
                   offsetof(ScsInfo, lin_sys_time) == 472,
               "ScsInfo layout (DLONG)");
#else
_Static_assert(sizeof(scs_int) == 4, "scs_int is int");
_Static_assert(sizeof(ScsMatrix) == 32, "ScsMatrix layout");
_Static_assert(sizeof(ScsData) == 40, "ScsData layout");
_Static_assert(sizeof(ScsSettings) == 136 && offsetof(ScsSettings, write_data_filename) == 120 &&
                   offsetof(ScsSettings, log_csv_filename) == 128,
               "ScsSettings layout");
#ifdef USE_SPECTRAL_CONES
_Static_assert(sizeof(ScsCone) == 184 && offsetof(ScsCone, d) == 104 && offsetof(ScsCone, nuc_m) == 120 &&
                   offsetof(ScsCone, ell1) == 144 && offsetof(ScsCone, sl_n) == 160 && offsetof(ScsCone, sl_size) == 176,
               "ScsCone layout (spectral cones)");
#else
_Static_assert(sizeof(ScsCone) == 104 && offsetof(ScsCone, p) == 88 && offsetof(ScsCone, psize) == 96,
               "ScsCone layout");
#endif
_Static_assert(sizeof(AaStats) == 48, "AaStats layout");
_Static_assert(sizeof(ScsInfo) == 448 && offsetof(ScsInfo, status) == 4 && offsetof(ScsInfo, lin_sys_solver) == 132 &&
                   offsetof(ScsInfo, pobj) == 272 && offsetof(ScsInfo, aa_stats) == 376 &&
                   offsetof(ScsInfo, lin_sys_time) == 424,
               "ScsInfo layout");
#endif
_Static_assert(sizeof(ScsSolution) == 24, "ScsSolution layout");

int b200_over_dim(const char *what, long long index, scs_int v) {
  if (v <= B200_MAX_DIM) return 0;
  if (index >= 0)
    printf("%s[%lld] = %lld exceeds the limit 2^30 - 1 on dimensions and cone sizes\n", what, index, (long long)v);
  else
    printf("%s = %lld exceeds the limit 2^30 - 1 on dimensions and cone sizes\n", what, (long long)v);
  return 1;
}

int b200_over_stored(const char *what, scs_int v) {
  if (v <= B200_MAX_STORED) return 0;
  printf("%s = %lld exceeds the limit 2^31 - 129 on the stored entries of one operator\n", what, (long long)v);
  return 1;
}

static int over_dims(const char *what, const scs_int *v, scs_int n) {
  scs_int i;
  if (!v) return 0;
  for (i = 0; i < n; ++i)
    if (b200_over_dim(what, (long long)i, v[i])) return 1;
  return 0;
}

int b200_cone_over_limits(const ScsCone *k) {
  if (b200_over_dim("z", -1, k->z) || b200_over_dim("l", -1, k->l) || b200_over_dim("bsize", -1, k->bsize) ||
      b200_over_dim("qsize", -1, k->qsize) || b200_over_dim("ssize", -1, k->ssize) ||
      b200_over_dim("cssize", -1, k->cssize) || b200_over_dim("ep", -1, k->ep) || b200_over_dim("ed", -1, k->ed) ||
      b200_over_dim("psize", -1, k->psize))
    return 1;
  if (over_dims("q", k->q, k->qsize) || over_dims("s", k->s, k->ssize) || over_dims("cs", k->cs, k->cssize)) return 1;
#ifdef USE_SPECTRAL_CONES
  if (b200_over_dim("dsize", -1, k->dsize) || b200_over_dim("nucsize", -1, k->nucsize) ||
      b200_over_dim("ell1_size", -1, k->ell1_size) || b200_over_dim("sl_size", -1, k->sl_size))
    return 1;
  if (over_dims("d", k->d, k->dsize) || over_dims("nuc_m", k->nuc_m, k->nucsize) ||
      over_dims("nuc_n", k->nuc_n, k->nucsize) || over_dims("ell1", k->ell1, k->ell1_size) ||
      over_dims("sl_n", k->sl_n, k->sl_size) || over_dims("sl_k", k->sl_k, k->sl_size))
    return 1;
#endif
  return 0;
}

int b200_matrix_over_limits(const ScsMatrix *A, const ScsMatrix *P) {
  if (b200_over_dim("A->m", -1, A->m) || b200_over_dim("A->n", -1, A->n)) return 1;
  if (A->m < 0 || A->n < 0 || !A->p) { printf("A matrix dimensions must be nonnegative, A->p given\n"); return 1; }
  if (b200_over_stored("nnz(A)", A->p[A->n])) return 1;
  if (P) {
    if (b200_over_dim("P->n", -1, P->n)) return 1;
    if (P->n < 0 || !P->p) { printf("P matrix dimensions must be nonnegative, P->p given\n"); return 1; }
    if (b200_over_stored("nnz(P)", P->p[P->n])) return 1;
  }
  return 0;
}

/* The argument checks of the device-pointer entry points (scs_b200_*_device: host/scs_driver.c, host/operators.c,
 * host/linsys_b200.c), here because every library flavour links this file. */
int b200_dev_ptr_ok(const void *p, const char *what) {
  if (b200_is_device_ptr(p)) return 1;
  printf("ERROR: %s must point to device memory of the library's CUDA device\n", what);
  return 0;
}
int b200_single_gpu(void) {
  if (b200_comm_nranks() <= 1) return 1;
  printf("ERROR: the device-data entry points drive a single GPU; this process is one of %d ranks\n",
         b200_comm_nranks());
  return 0;
}
int b200_overlap(const char *a_name, const void *a, size_t a_bytes, const char *b_name, const void *b,
                 size_t b_bytes) {
  const uintptr_t pa = (uintptr_t)a, pb = (uintptr_t)b;
  if (!a || !b || pa >= pb + b_bytes || pb >= pa + a_bytes) return 0;
  printf("ERROR: %s and %s must not overlap\n", a_name, b_name);
  return 1;
}

/* an int copy of v[0..n) (values already checked); NULL when n <= 0. 0, or -1 when out of memory */
static int narrow(const scs_int *v, scs_int n, int **out) {
  scs_int i;
  *out = SCS_NULL;
  if (!v || n <= 0) return 0;
  *out = (int *)malloc((size_t)n * sizeof(int));
  if (!*out) return -1;
  for (i = 0; i < n; ++i) (*out)[i] = (int)v[i];
  return 0;
}

int b200_cone_ints(const ScsCone *k, B200ConeInts *c) {
  int rc = 0;
  memset(c, 0, sizeof(*c));
  rc |= narrow(k->q, k->qsize, &c->q);
  rc |= narrow(k->s, k->ssize, &c->s);
  rc |= narrow(k->cs, k->cssize, &c->cs);
#ifdef USE_SPECTRAL_CONES
  rc |= narrow(k->d, k->dsize, &c->d);
  rc |= narrow(k->nuc_m, k->nucsize, &c->nuc_m);
  rc |= narrow(k->nuc_n, k->nucsize, &c->nuc_n);
  rc |= narrow(k->ell1, k->ell1_size, &c->ell1);
  rc |= narrow(k->sl_n, k->sl_size, &c->sl_n);
  rc |= narrow(k->sl_k, k->sl_size, &c->sl_k);
#endif
  if (rc != 0) b200_cone_ints_free(c);
  return rc;
}

void b200_cone_ints_free(B200ConeInts *c) {
  free(c->q); free(c->s); free(c->cs); free(c->d);
  free(c->nuc_m); free(c->nuc_n); free(c->ell1); free(c->sl_n); free(c->sl_k);
  c->q = c->s = c->cs = c->d = c->nuc_m = c->nuc_n = c->ell1 = c->sl_n = c->sl_k = SCS_NULL;
}

/* rw_b200.c -- the SCS problem-file format (reference src/rw.c:574-684), reader and writer.
 *
 * SURVEY.md 8(f)-4: parity tooling. A problem dumped by the reference (`write_data_filename`) can be
 * fed to this library byte for byte and vice versa, so CPU and GPU runs read identical inputs; the
 * reference's own binary fixtures (test/problems/{random_prob, max_ent, mpc_bug1..3}) become inputs of
 * the device-resident solver. Host code only -- nothing here touches the GPU.
 *
 * File layout (all native endianness; I = integer of the width stored in the header, F = fp64):
 *   u32 sizeof(I), u32 sizeof(F), u32 len, char version[len]
 *   cone     I z, l, bsize; F bl[bsize-1], bu[bsize-1]; I qsize, q[]; I ssize, s[]; I ep, ed; I psize; F p[]
 *   data     I m, n; F b[m], c[n]; matrix A; I has_P; [matrix P]
 *            matrix = I m, n; I colptr[n+1]; F x[nnz]; I rowidx[nnz]
 *   settings I normalize; F scale, rho_x; I max_iters; F eps_abs, eps_rel, eps_infeas, alpha;
 *            I verbose, warm_start, acceleration_lookback, acceleration_interval;
 *            then, when version == "3.2.11":  I acceleration_type_1; F acceleration_regularization,
 *            acceleration_relaxation; I adaptive_scale       (older files: I adaptive_scale only)
 *   optional extension block: u32 magic "SCSE", u32 1; I cssize, cs[]; I dsize, d[]; I nucsize, nuc_m[],
 *            nuc_n[]; I ell1_size, ell1[]; I sl_size, sl_n[], sl_k[]; F time_limit_secs
 * The default build skips the spectral arrays on reading and writes them empty; the spectral build
 * (USE_SPECTRAL_CONES) reads them into ScsCone and writes them as the reference's spectral build does.
 * The writer emits I = sizeof(scs_int) -- 4 bytes, or 8 in the DLONG build, as the reference's writer of the same
 * width does -- and the version string of the API it implements ("3.2.11"). The reader accepts I = 4 or 8 and both
 * settings layouts: the DLONG build widens 4-byte files, the int build narrows 8-byte ones (values must fit an int). */
#include "driver.h"
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define FILE_API_VERSION "3.2.11"
#define EXT_MAGIC 0x53435345u

/* ------------------------------------------------------------------ byte streams with a sticky error */
typedef struct {
  FILE *f;
  int bad;        /* set on the first short read / write or invalid value; later calls are no-ops */
  int int_bytes;  /* width of I in the file (reader) */
} Stream;

static void put_raw(Stream *s, const void *p, size_t bytes) {
  if (s->bad || bytes == 0) return;
  if (!p || fwrite(p, 1, bytes, s->f) != bytes) s->bad = 1;
}
static void put_i(Stream *s, scs_int v) { put_raw(s, &v, sizeof(scs_int)); }
static void put_f(Stream *s, double v) { put_raw(s, &v, sizeof(double)); }
static void put_is(Stream *s, const scs_int *v, scs_int n) { if (n > 0) put_raw(s, v, (size_t)n * sizeof(scs_int)); }
static void put_fs(Stream *s, const double *v, scs_int n) { if (n > 0) put_raw(s, v, (size_t)n * sizeof(double)); }

static void get_raw(Stream *s, void *p, size_t bytes) {
  if (s->bad || bytes == 0) return;
  if (fread(p, 1, bytes, s->f) != bytes) s->bad = 1;
}
static void get_is(Stream *s, scs_int *dst, size_t n) {
  size_t i;
  if (s->bad || n == 0) return;
  if (s->int_bytes == (int)sizeof(scs_int)) {
    get_raw(s, dst, n * sizeof(scs_int));
    return;
  }
  if (s->int_bytes == 4) { /* 4-byte integers on file, 8-byte scs_int (DLONG): widen */
    for (i = 0; i < n && !s->bad; ++i) {
      int32_t narrow = 0;
      get_raw(s, &narrow, sizeof(narrow));
      dst[i] = narrow;
    }
    return;
  }
  for (i = 0; i < n && !s->bad; ++i) { /* 8-byte integers on file, int scs_int: narrow, refusing overflow */
    int64_t wide = 0;
    get_raw(s, &wide, sizeof(wide));
    if (wide > 2147483647LL || wide < -2147483647LL - 1) s->bad = 1;
    dst[i] = (scs_int)wide;
  }
}
static scs_int get_i(Stream *s) {
  scs_int v = 0;
  get_is(s, &v, 1);
  return v;
}
static double get_f(Stream *s) {
  double v = 0.0;
  get_raw(s, &v, sizeof(double));
  return v;
}
/* allocate-and-read; a negative count is a format error, count 0 gives NULL */
static scs_int *get_i_array(Stream *s, scs_int n) {
  scs_int *v;
  if (n < 0) s->bad = 1;
  if (s->bad || n == 0) return SCS_NULL;
  v = (scs_int *)calloc((size_t)n, sizeof(scs_int));
  if (!v) { s->bad = 1; return SCS_NULL; }
  get_is(s, v, (size_t)n);
  return v;
}
static double *get_f_array(Stream *s, scs_int n) {
  double *v;
  if (n < 0) s->bad = 1;
  if (s->bad || n == 0) return SCS_NULL;
  v = (double *)calloc((size_t)n, sizeof(double));
  if (!v) { s->bad = 1; return SCS_NULL; }
  get_raw(s, v, (size_t)n * sizeof(double));
  return v;
}
#ifndef USE_SPECTRAL_CONES
static void skip_i_array(Stream *s, scs_int n) {
  char buf[4096];
  uint64_t left;
  if (n < 0) s->bad = 1;
  if (s->bad) return;
  left = (uint64_t)n * (uint64_t)s->int_bytes;
  while (left > 0 && !s->bad) {
    const size_t chunk = left < sizeof(buf) ? (size_t)left : sizeof(buf);
    get_raw(s, buf, chunk);
    left -= chunk;
  }
}
#endif

/* ------------------------------------------------------------------ writer */
static void put_matrix(Stream *s, const ScsMatrix *M) {
  const scs_int nnz = M->p[M->n];
  if (nnz < 0) { s->bad = 1; return; }
  put_i(s, M->m);
  put_i(s, M->n);
  put_is(s, M->p, M->n + 1);
  put_fs(s, M->x, nnz);
  put_is(s, M->i, nnz);
}

scs_int scs_b200_write_data(const char *filename, const ScsData *d, const ScsCone *k,
                            const ScsSettings *stgs) {
  Stream s;
  const uint32_t head[3] = {(uint32_t)sizeof(scs_int), (uint32_t)sizeof(double), (uint32_t)strlen(FILE_API_VERSION)};
  const uint32_t ext[2] = {EXT_MAGIC, 1u};
  scs_int nbox;
  if (!filename || !d || !k || !stgs || !d->A) return -1;
  nbox = k->bsize > 1 ? k->bsize - 1 : 0;
  s.f = fopen(filename, "wb");
  s.bad = 0;
  s.int_bytes = (int)sizeof(scs_int);
  if (!s.f) {
    printf("Error: could not open %s for writing\n", filename);
    return -1;
  }
  put_raw(&s, head, sizeof(head));
  put_raw(&s, FILE_API_VERSION, head[2]);
  /* cone */
  put_i(&s, k->z); put_i(&s, k->l); put_i(&s, k->bsize);
  put_fs(&s, k->bl, nbox); put_fs(&s, k->bu, nbox);
  put_i(&s, k->qsize); put_is(&s, k->q, k->qsize);
  put_i(&s, k->ssize); put_is(&s, k->s, k->ssize);
  put_i(&s, k->ep); put_i(&s, k->ed);
  put_i(&s, k->psize); put_fs(&s, k->p, k->psize);
  /* data */
  put_i(&s, d->m); put_i(&s, d->n);
  put_fs(&s, d->b, d->m); put_fs(&s, d->c, d->n);
  put_matrix(&s, d->A);
  put_i(&s, d->P ? 1 : 0);
  if (d->P) put_matrix(&s, d->P);
  /* settings (3.2.11 layout; warm_start is stored as 0 like the reference does) */
  put_i(&s, stgs->normalize); put_f(&s, stgs->scale); put_f(&s, stgs->rho_x);
  put_i(&s, stgs->max_iters);
  put_f(&s, stgs->eps_abs); put_f(&s, stgs->eps_rel); put_f(&s, stgs->eps_infeas); put_f(&s, stgs->alpha);
  put_i(&s, stgs->verbose); put_i(&s, 0);
  put_i(&s, stgs->acceleration_lookback); put_i(&s, stgs->acceleration_interval);
  put_i(&s, stgs->acceleration_type_1);
  put_f(&s, stgs->acceleration_regularization); put_f(&s, stgs->acceleration_relaxation);
  put_i(&s, stgs->adaptive_scale);
  /* extension block: complex PSD orders, four empty spectral-cone groups, the time limit */
  put_raw(&s, ext, sizeof(ext));
  put_i(&s, k->cssize); put_is(&s, k->cs, k->cssize);
#ifdef USE_SPECTRAL_CONES
  put_i(&s, k->dsize); put_is(&s, k->d, k->dsize);
  put_i(&s, k->nucsize); put_is(&s, k->nuc_m, k->nucsize); put_is(&s, k->nuc_n, k->nucsize);
  put_i(&s, k->ell1_size); put_is(&s, k->ell1, k->ell1_size);
  put_i(&s, k->sl_size); put_is(&s, k->sl_n, k->sl_size); put_is(&s, k->sl_k, k->sl_size);
#else
  put_i(&s, 0); put_i(&s, 0); put_i(&s, 0); put_i(&s, 0);
#endif
  put_f(&s, stgs->time_limit_secs);
  if (fclose(s.f) != 0) s.bad = 1;
  if (s.bad) printf("Error: failed writing SCS data to %s\n", filename);
  return s.bad ? -1 : 0;
}

/* ------------------------------------------------------------------ reader */
static ScsMatrix *get_matrix(Stream *s) {
  ScsMatrix *M = (ScsMatrix *)calloc(1, sizeof(ScsMatrix));
  scs_int nnz;
  if (!M) { s->bad = 1; return SCS_NULL; }
  M->m = get_i(s);
  M->n = get_i(s);
  if (M->m < 0 || M->n < 0) s->bad = 1;
  M->p = get_i_array(s, s->bad ? 0 : M->n + 1);
  nnz = (M->p && !s->bad) ? M->p[M->n] : 0;
  if (nnz < 0) { s->bad = 1; nnz = 0; }
  M->x = get_f_array(s, nnz);
  M->i = get_i_array(s, nnz);
  return M;
}
static void drop_matrix(ScsMatrix *M) {
  if (!M) return;
  free(M->x); free(M->i); free(M->p); free(M);
}

void scs_b200_free_data(ScsData *d, ScsCone *k, ScsSettings *stgs) {
  if (d) {
    drop_matrix(d->A); drop_matrix(d->P);
    free(d->b); free(d->c); free(d);
  }
  if (k) {
    free(k->bu); free(k->bl); free(k->q); free(k->s); free(k->cs); free(k->p);
#ifdef USE_SPECTRAL_CONES
    free(k->d); free(k->nuc_m); free(k->nuc_n); free(k->ell1); free(k->sl_n); free(k->sl_k);
#endif
    free(k);
  }
  free(stgs);
}

scs_int scs_b200_read_data(const char *filename, ScsData **d_out, ScsCone **k_out, ScsSettings **stgs_out) {
  Stream s;
  uint32_t head[3] = {0, 0, 0};
  char ver[16];
  int current_layout;
  scs_int nbox;
  ScsData *d = SCS_NULL;
  ScsCone *k = SCS_NULL;
  ScsSettings *st = SCS_NULL;
  if (!filename || !d_out || !k_out || !stgs_out) return -1;
  *d_out = SCS_NULL; *k_out = SCS_NULL; *stgs_out = SCS_NULL;
  s.f = fopen(filename, "rb");
  s.bad = 0;
  s.int_bytes = (int)sizeof(scs_int);
  if (!s.f) {
    printf("Error reading file %s\n", filename);
    return -1;
  }
  get_raw(&s, head, sizeof(head));
  if (!s.bad && head[0] != 4 && head[0] != 8) { printf("Error: unsupported file integer size %u\n", head[0]); s.bad = 1; }
  if (!s.bad && head[1] != sizeof(double)) { printf("Error: file float size %u, this build uses 8\n", head[1]); s.bad = 1; }
  if (!s.bad && head[2] >= sizeof(ver)) { printf("Error: file version string too long\n"); s.bad = 1; }
  if (s.bad) goto fail;
  s.int_bytes = (int)head[0];
  memset(ver, 0, sizeof(ver));
  get_raw(&s, ver, head[2]);
  current_layout = strcmp(ver, FILE_API_VERSION) == 0;
  if (!s.bad && !current_layout)
    printf("Warning: SCS file version %s, this library implements the API of %s (older settings layout assumed)\n",
           ver, FILE_API_VERSION);

  k = (ScsCone *)calloc(1, sizeof(ScsCone));
  d = (ScsData *)calloc(1, sizeof(ScsData));
  st = (ScsSettings *)calloc(1, sizeof(ScsSettings));
  if (!k || !d || !st) { s.bad = 1; goto fail; }
  /* cone */
  k->z = get_i(&s); k->l = get_i(&s); k->bsize = get_i(&s);
  if (k->bsize < 0) s.bad = 1;
  nbox = k->bsize > 1 ? k->bsize - 1 : 0;
  k->bl = get_f_array(&s, nbox); k->bu = get_f_array(&s, nbox);
  k->qsize = get_i(&s); k->q = get_i_array(&s, k->qsize);
  k->ssize = get_i(&s); k->s = get_i_array(&s, k->ssize);
  k->ep = get_i(&s); k->ed = get_i(&s);
  k->psize = get_i(&s); k->p = get_f_array(&s, k->psize);
  /* data */
  d->m = get_i(&s); d->n = get_i(&s);
  if (d->m < 0 || d->n < 0) s.bad = 1;
  d->b = get_f_array(&s, s.bad ? 0 : d->m);
  d->c = get_f_array(&s, s.bad ? 0 : d->n);
  d->A = get_matrix(&s);
  if (get_i(&s)) d->P = get_matrix(&s);
  /* settings */
  scs_set_default_settings(st);
  st->normalize = get_i(&s); st->scale = get_f(&s); st->rho_x = get_f(&s);
  st->max_iters = get_i(&s);
  st->eps_abs = get_f(&s); st->eps_rel = get_f(&s); st->eps_infeas = get_f(&s); st->alpha = get_f(&s);
  st->verbose = get_i(&s); st->warm_start = get_i(&s);
  st->acceleration_lookback = get_i(&s); st->acceleration_interval = get_i(&s);
  if (current_layout) {
    st->acceleration_type_1 = get_i(&s);
    st->acceleration_regularization = get_f(&s); st->acceleration_relaxation = get_f(&s);
  }
  st->adaptive_scale = get_i(&s);
  if (s.bad) goto fail;
  /* optional extension block (older files end here) */
  {
    uint32_t magic = 0;
    const size_t got = fread(&magic, 1, sizeof(magic), s.f);
    if (got == sizeof(magic) && magic == EXT_MAGIC) {
      uint32_t ev = 0;
      scs_int cnt;
      get_raw(&s, &ev, sizeof(ev));
      if (ev != 1u) { printf("Error: unsupported SCS file extension version %u\n", ev); s.bad = 1; }
      k->cssize = get_i(&s); k->cs = get_i_array(&s, k->cssize);
#ifdef USE_SPECTRAL_CONES /* the spectral arrays (reference rw.c:540-557) */
      (void)cnt;
      k->dsize = get_i(&s); k->d = get_i_array(&s, k->dsize);
      k->nucsize = get_i(&s); k->nuc_m = get_i_array(&s, k->nucsize); k->nuc_n = get_i_array(&s, k->nucsize);
      k->ell1_size = get_i(&s); k->ell1 = get_i_array(&s, k->ell1_size);
      k->sl_size = get_i(&s); k->sl_n = get_i_array(&s, k->sl_size); k->sl_k = get_i_array(&s, k->sl_size);
#else
      cnt = get_i(&s); skip_i_array(&s, cnt);                              /* log-det cones */
      cnt = get_i(&s); skip_i_array(&s, cnt); skip_i_array(&s, cnt);       /* nuclear-norm cones */
      cnt = get_i(&s); skip_i_array(&s, cnt);                              /* ell-1 cones */
      cnt = get_i(&s); skip_i_array(&s, cnt); skip_i_array(&s, cnt);       /* sum-of-largest cones */
#endif
      st->time_limit_secs = get_f(&s);
    } else if (got != 0 && got != sizeof(magic)) {
      printf("Error: incomplete extension header in %s\n", filename);
      s.bad = 1;
    } else if (got == sizeof(magic)) {
      printf("Warning: ignoring unrecognized trailing data in SCS file\n");
    }
  }
  if (s.bad) goto fail;
  fclose(s.f);
  *d_out = d; *k_out = k; *stgs_out = st;
  return 0;
fail:
  printf("Error: could not read SCS data from %s\n", filename);
  fclose(s.f);
  scs_b200_free_data(d, k, st);
  return -1;
}

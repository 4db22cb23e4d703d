/* driver.h -- private workspace of the device-resident ADMM driver
 * (counterpart of reference include/scs_work.h:55-86, with the iterate vectors
 * living in HBM instead of host memory). */
#include <stdio.h>
#ifndef B200_DRIVER_H
#define B200_DRIVER_H
#include "../../../include/scs_b200.h"
#include "../admm_api.h"
#include "../dev_api.h"
#include "linsys_b200.h"

/* constants that are part of parity: reference include/glbopts.h:184-257 */
#define SCS_VERSION_STR "3.2.11-b200"
#define FEASIBLE_ITERS (1)
#define RESCALING_MIN_ITERS (100)
#define CONVERGED_INTERVAL (25)
#define PRINT_INTERVAL (250)
#define TAU_FACTOR (10.)
#define INFEAS_NEGATIVITY_TOL (1e-9)
#define AA_SAFEGUARD_FACTOR (1.)
#define AA_MAX_WEIGHT_NORM (1e10)
#define AA_IR_MAX_STEPS (5)
#define MAX_SCALE_VALUE (1e6)
#define MIN_SCALE_VALUE (1e-6)
#define CG_BEST_TOL (1e-12)
#define CG_RATE (1.5)
#define MAX_BOX_VAL (1e15)
#define DIV_EPS_TOL (1E-18)
#define SAFEDIV_POS(X, Y) ((Y) < DIV_EPS_TOL ? ((X) / DIV_EPS_TOL) : (X) / (Y))

#ifdef USE_SPECTRAL_CONES
/* rows of the spectral cones (reference cones.c:435-443); a log-det cone of order d has d(d+1)/2 + 2 */
static inline long long b200_spectral_rows(const ScsCone *k) {
  long long rows = 0;
  scs_int i;
  for (i = 0; i < k->dsize; ++i) rows += (long long)k->d[i] * (k->d[i] + 1) / 2 + 2;
  for (i = 0; i < k->nucsize; ++i) rows += (long long)k->nuc_m[i] * k->nuc_n[i] + 1;
  for (i = 0; i < k->ell1_size; ++i) rows += (long long)k->ell1[i] + 1;
  for (i = 0; i < k->sl_size; ++i) rows += (long long)k->sl_n[i] * (k->sl_n[i] + 1) / 2 + 1;
  return rows;
}
#endif
#ifndef MAX
#define MAX(a, b) (((a) > (b)) ? (a) : (b))
#endif
#ifndef MIN
#define MIN(a, b) (((a) < (b)) ? (a) : (b))
#endif

typedef struct {
  int last_iter;
  double xt_p_x, xt_p_x_tau, ctx, ctx_tau, bty, bty_tau, pobj, dobj, gap, tau, kap;
  double res_pri, res_dual, res_infeas, res_unbdd_p, res_unbdd_a;
  /* inf-norms of the vectors the reference keeps on the host */
  double nm_ax_s_btau, nm_px_aty_ctau, nm_ax, nm_ax_s, nm_px, nm_aty, nm_s;
} B200Residuals;

struct SCS_WORK {
  int n, m;
  long long nnzA, nnzP;
  double setup_time;
  int time_limit_reached;
  /* host copies */
  ScsData *d;       /* deep copy, A/P/b/c NORMALISED */
  ScsCone *k;       /* deep copy, box bounds normalised */
  ScsSettings *stgs;
  double *D, *E;    /* equilibration (NULL when normalize == 0) */
  double primal_scale, dual_scale;
  double *b_orig, *c_orig;
  double nm_b_orig, nm_c_orig;
  double *h_diag_r; /* l */
  int *cone_boundaries;
  int cone_boundaries_len;
  /* device state */
  B200Admm adm;
  double *d_b, *d_c, *d_D, *d_E;
  double *d_ax, *d_aty, *d_px;
  double *d_sol_x, *d_sol_y, *d_sol_s; /* n, m, m staging (finalize / warm start) */
  double *h_sc;                        /* pinned mirror of the scalar board */
  ScsLinSysWork *p;
  B200Cones *cones;
  B200Aa *accel;
  B200Residuals r_orig, r_norm;
  /* scale updating */
  double sum_log_scale_factor;
  int last_scale_update_iter, n_log_scale_factor, scale_updates;
  /* AA */
  double aa_norm;
  int rejected_accel_steps, accepted_accel_steps;
  /* stats of the last solve */
  long long stat_cg_iters, stat_solves, stat_launches;
  /* per-iteration CSV trace (ScsSettings.log_csv_filename, reference src/rw.c:707-861): debugging mode, the
   * iterates are copied to the host every iteration and every column is recomputed there */
  char *log_csv_name; /* deep copy of ScsSettings.log_csv_filename */
  FILE *log_csv_fout; /* opened ("w") at the start of every scs_solve, closed at its end (rw.c:686-705) */
  double *log_host; /* scratch: u, u_t, v, v_prev, rsk (l each), ax (m), aty (n), px (n) */
};

/* the integer-width boundary (host/abi.c): checks in scs_int width that print a message naming the limit and return
 * nonzero, and int copies of the cone arrays for the kernel layer */
int b200_cone_over_limits(const ScsCone *k);
typedef struct {
  int *q, *s, *cs, *nuc_m, *nuc_n, *ell1, *sl_n, *sl_k; /* NULL where the cone has none */
} B200ConeInts;
int b200_cone_ints(const ScsCone *k, B200ConeInts *c); /* 0, or -1 (out of memory, nothing held) */
void b200_cone_ints_free(B200ConeInts *c);

int b200_equilibrate(ScsMatrix *P, ScsMatrix *A, const int *bnd, int nbnd, double *D, double *E);
double b200_normalize_b_c(int m, int n, const double *D, const double *E, double *b, double *c);

#endif

// cones_spectral.cu -- projection onto the log-det, nuclear-norm, l1-norm and sum-of-largest-eigenvalues cones of
// SCS's spectral build, on the device. Only libscs_b200_spectral.so creates these cones; the kernels do not depend on
// the ScsCone layout and are linked into both libraries.
//
// Replaces reference src/spectral_cones/logdeterminant/*.c, src/spectral_cones/nuclear/{ell1_cone.c,
// nuclear_cone.c} and src/spectral_cones/sum-largest/{sum_largest_eval_cone.c, sum_largest_cone.c}. Each block of
// rows holds -R x on entry and Pi_K(.) / R + s on exit (the Moreau wrapper, as every cone of kernels/cones.cu).
//
//  * log-det cone (t, v, X), 2 + d(d+1)/2 rows: groups by order d; sqrt2-scaled unpack -> cusolverDnXsyevBatched ->
//    the reference's log_cone_proj_wrapper on (sqrt2 t, sqrt2 v, eigenvalues) (k_logdet_vector, one warp per cone:
//    analytic exits, Newton, the acceptance test, the interior-point method with and without Mehrotra's correction)
//    -> V diag(lambda') V' on the DMMA path (lambda' >= 0) -> repack, t' / sqrt2, v' / sqrt2. Each cone's warm-start
//    flag and previous projection persist across projections and solves, as in the reference.
//
//  * l1 cone (t, x), 1 + n rows: Pi = (t + mu, sign(x) max(|x| - mu, 0)) with the threshold mu >= 0 of
//    ell1_threshold (sort-free: Michelot's active-set iteration, one CTA per cone, fixed-order block sums). Cones of
//    up to ELL1_INLINE entries are finished by that CTA; the soft thresholding of bigger ones runs on 4096-row chunks.
//  * sum-of-largest cone (t, X), 1 + n(n+1)/2 rows, X packed like the PSD cone: groups by order n; sqrt2-scaled
//    unpack -> cusolverDnXsyevBatched -> the reference's sorted vector projection of (sqrt2 t, eigenvalues
//    descending), one thread per cone -> V diag(e') V' on the DMMA path with every eigenvalue (either sign) ->
//    repack with the diagonal / sqrt2, t' / sqrt2.
//  * nuclear-norm cone (t, X), 1 + m n rows, X m x n column-major with m >= n: groups by (m, n). The SVD comes from
//    the same batched symmetric eigensolver through the embedding E = [[0, X], [X', 0]] of order m + n: its
//    eigenvalues are +-sigma_i and m - n zeros, and an eigenvector of sigma_i > 0 is (u_i; v_i) / sqrt2 with
//    X v_i = sigma_i u_i. The n largest eigenvalues are the singular values; the l1 step of (t, sigma) is the same
//    ell1_threshold as the l1 cone; X' = sum_i sigma'_i u_i v_i' = sum_i 2 sigma'_i top(w_i) bot(w_i)' is the
//    rectangular DMMA contraction. Zero or near-zero sigma need no care: an eigenvector of an eigenvalue near 0 may
//    mix with the null space of E and is not of the form (u; v) / sqrt2, but its weight is sigma'_i, which is 0 when
//    sigma_i <= mu and sigma_i itself when mu = 0 (then Pi is the identity and the term is as small as sigma_i).
//    So such columns contribute nothing or at most their own tiny singular value, exactly as in X.
// Eigensolver status words, and a log-det cone on which all three methods fail, join the sticky error flag of
// kernels/cones.cu (b200_cones_check).
#include "../common.cuh"
#include "../admm_api.h"
#include <cusolverDn.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <utility>
#include <vector>

#define ELL1_INLINE 8192   // l1 cones up to this many entries are soft-thresholded by their own CTA
#define ELL1_CHUNK 4096
#define ELL1_SMALL_T 256   // threads of the per-cone CTA (small cones / big cones)
#define ELL1_BIG_T 1024
#define NUC_T 128
#define TOL_LARGEST_CONE 1e-9  // reference sum_largest_cone.c:9

namespace {

__device__ __forceinline__ double finish(double xnew, const double *ry, const double *sv, long long row) {
  if (sv == nullptr) return xnew;
  return (ry != nullptr) ? xnew / ry[row] + sv[row] : xnew + sv[row];
}

// Threshold of the l1-norm cone projection of (t0, v), returned in every thread of the CTA:
//   Pi(t0, v) = (t0 + mu, sign(v) max(|v| - mu, 0)),   mu >= 0 the root of  sum_i max(|v_i| - mu, 0) = t0 + mu.
// mu = 0 when (t0, v) is in the cone (Pi is the identity); mu = +inf when -t0 >= max |v_i| ((t0, v) is in the polar
// cone and Pi = 0), as the reference's early exit (ell1_cone.c:107).
// Michelot's active-set iteration: A = all; mu = (sum_A |v| - t0) / (|A| + 1); A = {|v_i| > mu}; repeat until A stops
// shrinking. mu never decreases and A only shrinks, so it ends after at most n + 1 passes with the active set of the
// reference's sorted scan: the k largest magnitudes with |v|_(k) > mu >= |v|_(k+1). Sums are block sums in a fixed
// order (deterministic, no atomics). absv(i) returns |v_i|. All threads must call.
template <class F>
__device__ double ell1_threshold(int n, double t0, F absv, double *s_red /* 64 doubles */) {
  __shared__ double s_bc[2];
  double a[1] = {0.0}, mx[1] = {0.0};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = absv(i);
    a[0] += v;
    mx[0] = fmax(mx[0], v);
  }
  block_sum<1>(a, s_red);
  block_max<1>(mx, s_red + 32);
  if (threadIdx.x == 0) { s_bc[0] = a[0]; s_bc[1] = mx[0]; }
  __syncthreads();
  const double sum_all = s_bc[0], vmax = s_bc[1];
  __syncthreads();
  if (-t0 >= vmax) return INFINITY;
  double cnt = (double)n;
  double mu = (sum_all - t0) / (cnt + 1.0);
  if (!(mu > 0.0)) return 0.0;
  for (;;) {
    double r[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double v = absv(i);
      if (v > mu) { r[0] += v; r[1] += 1.0; }
    }
    block_sum<2>(r, s_red);
    if (threadIdx.x == 0) { s_bc[0] = r[0]; s_bc[1] = r[1]; }
    __syncthreads();
    const double s = s_bc[0], c = s_bc[1];
    __syncthreads();
    if (c >= cnt) break;  // the active set no longer shrinks: mu is exact for it
    cnt = c;
    mu = (s - t0) / (c + 1.0);
  }
  return mu;
}

// soft thresholding of one entry (reference ell1_cone.c:139-144, 218-220)
__device__ __forceinline__ double ell1_apply(double xv, double mu, double diff) {
  const double a = fabs(xv);
  if (!(a > mu)) return 0.0;
  return xv >= 0 ? a - diff : -(a - diff);
}

// one CTA per l1 cone: off[b] = row of t, len[b] = n. Cones with n <= ELL1_INLINE are finished here; for the others
// (mu, t' - t) go to par[2 b] for k_ell1_chunks.
__global__ void k_ell1_cones(const int *__restrict__ off, const int *__restrict__ len, double *__restrict__ x,
                             const double *sv, const double *ry, double *__restrict__ par) {
  __shared__ double s_red[64];
  const int b = blockIdx.x;
  const long long base = off[b];
  const int n = len[b];
  const double t0 = x[base];
  const double *v = x + base + 1;
  const double mu = ell1_threshold(n, t0, [v](int i) { return fabs(v[i]); }, s_red);
  const double tn = (mu == INFINITY) ? 0.0 : t0 + mu;
  const double diff = tn - t0;
  if (n <= ELL1_INLINE) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const long long row = base + 1 + i;
      x[row] = finish(ell1_apply(x[row], mu, diff), ry, sv, row);
    }
  } else if (threadIdx.x == 0) {
    par[2 * b] = mu;
    par[2 * b + 1] = diff;
  }
  if (threadIdx.x == 0) x[base] = finish(tn, ry, sv, base);
}

// chunks of the big l1 cones: (index into par, first row, rows, -)
__global__ void k_ell1_chunks(const int4 *__restrict__ chunks, const double *__restrict__ par, double *__restrict__ x,
                              const double *sv, const double *ry) {
  const int4 ch = chunks[blockIdx.x];
  const double mu = par[2 * ch.x], diff = par[2 * ch.x + 1];
  for (int i = threadIdx.x; i < ch.z; i += blockDim.x) {
    const long long row = (long long)ch.y + i;
    x[row] = finish(ell1_apply(x[row], mu, diff), ry, sv, row);
  }
}

// nuclear cone: the embedding E = [[0, X], [X', 0]] of order N = m + n, column-major; off[b] = first row of X
__global__ void k_nuc_embed(int m, int n, int count, const int *__restrict__ off, const double *__restrict__ x,
                            double *__restrict__ mats) {
  const int b = blockIdx.y;
  if (b >= count) return;
  const int N = m + n;
  const double *X = x + off[b];
  double *M = mats + (size_t)b * N * N;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < N * N; e += gridDim.x * blockDim.x) {
    const int I = e % N, J = e / N;
    double v = 0.0;
    if (I < m && J >= m) v = X[I + (size_t)(J - m) * m];
    else if (I >= m && J < m) v = X[J + (size_t)(I - m) * m];
    M[e] = v;
  }
}

// nuclear cone, vector step: one CTA per cone. sigma_i = max(lambda_{N-1-i}, 0), i < n (syevd sorts ascending);
// writes t' and overwrites the eigenvalues with the contraction weights: 2 sigma'_i on column N-1-i, 0 elsewhere.
__global__ void k_nuc_vector(int m, int n, int count, const int *__restrict__ off, double *__restrict__ evals,
                             double *__restrict__ x, const double *sv, const double *ry) {
  __shared__ double s_red[64];
  const int b = blockIdx.x;
  const int N = m + n;
  double *lam = evals + (size_t)b * N;
  const long long trow = (long long)off[b] - 1;
  const double t0 = x[trow];
  const double mu = ell1_threshold(n, t0, [lam, N](int i) { return fmax(lam[N - 1 - i], 0.0); }, s_red);
  const double tn = (mu == INFINITY) ? 0.0 : t0 + mu;
  const double diff = tn - t0;
  // every thread has read lam[] inside ell1_threshold (it ends with a barrier); rewrite it in place
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    double wgt = 0.0;
    if (c >= N - n) {
      const double sigma = fmax(lam[c], 0.0);
      wgt = 2.0 * ell1_apply(sigma, mu, diff);
    }
    lam[c] = wgt;
  }
  if (threadIdx.x == 0) x[trow] = finish(tn, ry, sv, trow);
}

// sum-of-largest cone, vector step: one thread per cone, the reference's sorted algorithm
// (proj_sum_largest_cone_sorted, sum_largest_cone.c:42-147) on x = eigenvalues in DESCENDING order, read through
// the ascending array e (x[i] = e[n-1-i]), and t scaled by sqrt2 as the eigenvalues are (sum_largest_eval_cone.c:111).
__global__ void k_sl_vector(int n, int count, const int *__restrict__ off, const int *__restrict__ kk,
                            double *__restrict__ evals, double *__restrict__ x, const double *sv, const double *ry) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= count) return;
  double *e = evals + (size_t)b * n;
  auto X = [e, n](int i) -> double & { return e[n - 1 - i]; };
  const int k = kk[b];
  const long long trow = (long long)off[b] - 1;
  const double sqrt2 = sqrt(2.0);
  double t = x[trow] * sqrt2;
  int nu = k, nt = 0;
  double eta = 0.0;
  const double t0 = t;
  double S = X(0);
  for (int i = 1; i < k; ++i) S += X(i);
  double a_u = X(nu - 1), a_t = X(nu);
  while (S > t + TOL_LARGEST_CONE) {
    const double ratio = (nu == k) ? 1.0 : (double)nt / (k - nu);
    const double s1 = (nu == k) ? a_u - a_t : (a_u - a_t) / (ratio - 1);
    const double s3 = (S - t) / (ratio * (nu + 1) + (k - nu));
    double s = (nu == 0) ? s3 : fmin(s3, s1);
    if (!(nu + nt == n || nt == 0)) s = fmin(s, a_t - X(nu + nt));
    eta += s * ratio;
    S -= s * (ratio * nu + k - nu);
    t = t0 + eta;
    if (nt > 0) a_t -= s;
    if (nu != 0 && s == s1) nu -= 1;
    if (nu > 0) a_u = X(nu - 1) - eta;
    nt = (nt == 0) ? 2 : nt + 1;
  }
  nt -= 1;
  for (int i = 0; i < nu; ++i) X(i) -= eta;
  for (int i = nu; i < nu + nt; ++i) X(i) = a_t;
  x[trow] = finish(t * (1.0 / sqrt2), ry, sv, trow);
}

// ---------------------------------------------------------------------------------------------- log-det cone
// The vector step of the log-det cone (reference logdeterminant/log_cone_{wrapper,Newton,IPM}.c): the projection of
// (t0, v0, x0) onto the log cone {(t, v, x) : v > 0, x > 0, t <= -v sum log(x_i / v)}. One warp per cone; lane l
// owns the entries i = l (mod 32) of every length-n vector, so a lane reads only what it wrote and no barrier is
// needed. Scalars are computed redundantly in every lane from warp sums (warp_sum's xor butterfly gives every lane
// the same bits), so every lane takes the same branches. A launch is bit-reproducible: no atomics.
#define LD_T 32
#define LD_VECS 16           // length-n vectors of scratch per cone (the IPM's; Newton uses the first 4) ...
#define LD_KEEP 32           // ... and the IPM's saved line-search state
// Newton (log_cone_Newton.c)
#define LD_MIN_INIT 1.0
#define LD_MIN_DENOMINATOR 1e-14
#define LD_MIN_X 1e-17
#define LD_MIN_V 1e-14
#define LD_MAX_ITER_NEWTON 100
#define LD_ALPHA_NEWTON 0.01
#define LD_BETA_NEWTON 0.8
#define LD_TOL_NEWTON 1e-12
#define LD_MAX_GRAD_STEPS 5
#define LD_LS_REL_TOL 1e-14
// IPM (log_cone_IPM.c)
#define LD_FEASTOL_IPM 1e-7
#define LD_ABSTOL_IPM 1e-7
#define LD_RELTOL_IPM 1e-6
#define LD_MAX_ITER_IPM 100
#define LD_BETA_IPM 0.5
#define LD_STEP_IPM 0.99
#define LD_ALPHA_IPM 0.01
#define LD_MAX_RELAXED_ITERS 8
// acceptance (log_cone_wrapper.c)
#define LD_DUAL_FEAS_TOL 1e-2
#define LD_PRI_FEAS_TOL 1e-2
#define LD_COMP_TOL 1e-2
#define LD_DUAL_T_THRESHOLD 1e-8
#define LD_DUAL_X_THRESHOLD 1e-8
// Newton_stats.iter codes (util_spectral_cones.h, log_cone_Newton.c)
#define LD_IN_CONE (-1)
#define LD_IN_NEGATIVE_DUAL_CONE (-2)
#define LD_ANALYTICAL_SOL (-3)
#define LD_TERMINATE_DUE_TO_ZEROS (-5)
#define LD_MAX_GRAD_STEPS_REACHED (-6)
#define LD_ERR_BIT 2         // OR-ed into the sticky error flag when all three methods fail on a cone

template <int K>
__device__ __forceinline__ void warp_sums(double (&v)[K]) {
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ bool warp_all(bool p) { return __all_sync(0xffffffffu, p) != 0; }

struct LdStats {  // Newton_stats of the reference
  int iter, newton_success;
  double res[3];
};

// check_opt_cond_log_cone (log_cone_wrapper.c:132-204) on tvx = (t, v, x)
__device__ __noinline__ void ld_check_opt(int n, double t, double v, const double *x, double t0, double v0, const double *x0,
                             double res[3]) {
  const int lane = threadIdx.x;
  double dualt = t - t0;
  if (fabs(dualt) < LD_DUAL_T_THRESHOLD) dualt = LD_DUAL_T_THRESHOLD;
  const double dualv = v - v0;
  // 0 dot(dualx, x), 1 sum log x, 2 sum_{x<0} x^2, 3 sum log dualx, 4 sum_{dualx<0} dualx^2, 5 |dualx|^2, 6 |x|^2
  double a[7] = {0, 0, 0, 0, 0, 0, 0};
  bool xpos = true, dpos = true;
  for (int i = lane; i < n; i += LD_T) {
    const double xi = x[i];
    double di = xi - x0[i];
    if (fabs(di) < LD_DUAL_X_THRESHOLD) di = LD_DUAL_X_THRESHOLD;
    a[0] += di * xi;
    a[1] += log(xi);
    if (xi < 0) a[2] += xi * xi;
    a[3] += log(di);
    if (di < 0) a[4] += di * di;
    a[5] += di * di;
    a[6] += xi * xi;
    xpos = xpos && xi > 0.0;
    dpos = dpos && di > 0.0;
  }
  warp_sums<7>(a);
  xpos = warp_all(xpos);
  dpos = warp_all(dpos);
  const double comp = t * dualt + v * dualv + a[0];
  double pri;
  if (v > 0 && xpos) {
    pri = -v * (a[1] - n * log(v)) - t;
  } else {
    pri = v * v;
    if (t < 0) pri += t * t;
    pri += a[2];
  }
  double dual;
  if (dualt > 0 && dpos) {
    dual = dualt * (n * log(dualt) - n - a[3]) - dualv;
  } else {
    dual = dualt * dualt;
    if (dualv < 0) dual += dualv * dualv;
    dual += a[4];
  }
  const double dual_norm = sqrt(dualt * dualt + dualv * dualv + a[5]);
  const double pri_norm = sqrt(t * t + v * v + a[6]);
  res[0] = dual / fmax(dual_norm, 1.0);
  res[1] = pri / fmax(pri_norm, 1.0);
  res[2] = comp / fmax(fmax(pri_norm, 1.0), dual_norm);
}

// obj_val (log_cone_Newton.c:40-56) at (v, x)
__device__ double ld_newton_obj(int n, double v, const double *x, double t0, double v0, const double *x0) {
  double a[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < n; i += LD_T) {
    a[0] += log(x[i]);
    const double d = x[i] - x0[i];
    a[1] += 0.5 * d * d;
  }
  warp_sums<2>(a);
  const double sx = -(v * a[0] - n * v * log(v));
  return 0.5 * (sx - t0) * (sx - t0) + 0.5 * (v - v0) * (v - v0) + a[1];
}

// log_cone_Newton (log_cone_Newton.c:58-302). u = (t, v, x) with x = u + 2 (the cone's saved projection).
// ws: 4 n doubles (grad, du, temp1, u_new). Returns 0 or -1; sets *iter and *warm as the reference does.
__device__ __noinline__ int ld_newton(int n, double t0, double v0, const double *x0, double *u, double *ws, int *iter_out,
                         int *warm) {
  const int lane = threadIdx.x;
  double *x = u + 2;
  double *grad = ws, *du = ws + n, *temp1 = ws + 2 * n, *unew = ws + 3 * n;
  bool nonneg = true, pos = true, neg = true;
  double slx = 0.0, sld = 0.0;
  for (int i = lane; i < n; i += LD_T) {
    nonneg = nonneg && x0[i] >= 0;
    pos = pos && x0[i] > 0;
    neg = neg && x0[i] < 0;
  }
  nonneg = warp_all(nonneg);
  pos = warp_all(pos);
  neg = warp_all(neg);
  if (v0 > 0 && pos) {
    for (int i = lane; i < n; i += LD_T) slx += log(x0[i]);
    slx = warp_sum(slx);
  }
  // in the cone
  if ((v0 > 0 && pos && -v0 * (slx - n * log(v0)) <= t0) || (v0 == 0 && nonneg && t0 >= 0)) {
    if (lane == 0) { u[0] = t0; u[1] = v0; }
    for (int i = lane; i < n; i += LD_T) x[i] = x0[i];
    *iter_out = LD_IN_CONE;
    *warm = 1;
    return 0;
  }
  // in the negative dual cone: the projection is 0, and not a warm start for the next call
  if (t0 < 0 && neg) {
    for (int i = lane; i < n; i += LD_T) sld += log(x0[i] / t0);
    const double sum = (-(double)n - warp_sum(sld)) * t0;
    if (v0 <= sum) {
      if (lane == 0) { u[0] = 0.0; u[1] = 0.0; }
      for (int i = lane; i < n; i += LD_T) x[i] = 0.0;
      *iter_out = LD_IN_NEGATIVE_DUAL_CONE;
      *warm = 0;
      return 0;
    }
  }
  // analytic: (t0, 0, max(x0, 0))
  if (v0 <= 0 && t0 >= 0) {
    if (lane == 0) { u[0] = t0; u[1] = 0.0; }
    for (int i = lane; i < n; i += LD_T) x[i] = x0[i] > 0.0 ? x0[i] : 0.0;
    *iter_out = LD_ANALYTICAL_SOL;
    *warm = 1;
    return 0;
  }
  __syncwarp();
  double v;
  if (!*warm) {
    v = (v0 > LD_MIN_INIT) ? v0 : LD_MIN_INIT;
    for (int i = lane; i < n; i += LD_T) x[i] = (x0[i] > LD_MIN_INIT) ? x0[i] : LD_MIN_INIT;
  } else {
    v = u[1];
  }
  double obj_old = ld_newton_obj(n, v, x, t0, v0, x0);
  int num_grad_steps = 0, iter;
  for (iter = 1; iter <= LD_MAX_ITER_NEWTON; ++iter) {
    if (v < LD_MIN_V) {
      if (lane == 0) u[1] = v;
      *iter_out = LD_TERMINATE_DUE_TO_ZEROS;
      return -1;
    }
    double s = 0.0;
    for (int i = lane; i < n; i += LD_T) {
      x[i] = fmax(x[i], LD_MIN_X);
      s += log(x[i]);
    }
    const double temp0 = -warp_sum(s) + n * log(v);
    const double a = v * temp0 - t0;
    const double c = temp0 + n;
    const double grad0 = a * c + v - v0;
    const double v_inv = 1 / v;
    const double d0 = 1 + a * (-a * (v_inv * v_inv) + n * v_inv - 2 * c * v_inv);
    const double w0 = -(a + v * c) * v_inv;
    const double av = a * v;
    double du0 = -grad0 / d0;
    const double tp0 = w0 / d0;
    double nd[2] = {0.0, 0.0};  // nominator, denominator (x parts)
    for (int i = lane; i < n; i += LD_T) {
      const double x_inv = 1 / x[i];
      const double g = -av * x_inv + x[i] - x0[i];
      const double d = 1 + av * (x_inv * x_inv);
      const double w = v * x_inv;
      grad[i] = g;
      du[i] = -g / d;
      temp1[i] = w / d;
      nd[0] += w * du[i];
      nd[1] += w * temp1[i];
    }
    warp_sums<2>(nd);
    const double nominator = w0 * du0 + nd[0];
    const double denominator = (1 + w0 * tp0) + nd[1];
    if (fabs(denominator) < LD_MIN_DENOMINATOR) {
      if (lane == 0) u[1] = v;
      *iter_out = LD_TERMINATE_DUE_TO_ZEROS;
      return -1;
    }
    const double ratio = -nominator / denominator;
    du0 += ratio * tp0;
    double dd = 0.0;
    for (int i = lane; i < n; i += LD_T) {
      du[i] += ratio * temp1[i];
      dd += grad[i] * du[i];
    }
    double dirDer = grad0 * du0 + warp_sum(dd);
    if (dirDer > 0) {
      if (num_grad_steps >= LD_MAX_GRAD_STEPS) {
        if (lane == 0) u[1] = v;
        *iter_out = LD_MAX_GRAD_STEPS_REACHED;
        return -1;
      }
      num_grad_steps += 1;
      du0 = -grad0;
      double gg = 0.0;
      for (int i = lane; i < n; i += LD_T) {
        du[i] = -grad[i];
        gg += grad[i] * grad[i];
      }
      dirDer = -(grad0 * grad0) - warp_sum(gg);
    }
    const double newton_decrement = -dirDer;
    if (newton_decrement <= 2 * LD_TOL_NEWTON) break;
    // the largest step that stays in the domain
    double step = 1.0;
    if (du0 < 0) step = fmin(step, -0.99 * v / du0);
    double ms = 1.0;
    for (int i = lane; i < n; i += LD_T)
      if (du[i] < 0) ms = fmin(ms, -0.99 * x[i] / du[i]);
    step = fmin(step, warp_min(ms));
    // backtracking line search
    double vnew, new_obj;
    for (;;) {
      vnew = v + step * du0;
      for (int i = lane; i < n; i += LD_T) unew[i] = x[i] + step * du[i];
      new_obj = ld_newton_obj(n, vnew, unew, t0, v0, x0);
      if (!((1 - LD_LS_REL_TOL) * new_obj > obj_old + LD_ALPHA_NEWTON * step * dirDer)) break;
      step *= LD_BETA_NEWTON;
    }
    obj_old = new_obj;
    v = vnew;
    for (int i = lane; i < n; i += LD_T) x[i] = unew[i];
  }
  double s = 0.0;
  for (int i = lane; i < n; i += LD_T) s += log(x[i]);
  const double t = -v * (warp_sum(s) - n * log(v));
  if (lane == 0) { u[0] = t; u[1] = v; }
  *warm = 1;
  *iter_out = iter;
  return 0;
}

// A length-(n + 3) vector of the IPM, (t, v, x, r), split into its scalar entries and the x part in scratch.
struct LdVec {
  double t, v, r;
  double *x;
};

// The oracle of log_cone_IPM.c:55-87 and the residuals of its main loop at (t, v, x, r), z, s. With store set, the
// x parts of 1/x, grad_f0, grad_f1 and r_x go to the scratch vectors (the main loop); otherwise only the norms are
// formed (the line search). Returns f_u in f, ||r_x|| in *nrx, and grad_f0, grad_f1, r_x's scalar entries.
__device__ __noinline__ void ld_ipm_oracle(int n, double t, double v, const double *x, double r, double t0, double v0,
                              const double *x0, const double z[3], double *x_inv, LdVec *g0, LdVec *g1, LdVec *rx,
                              bool store, double f[3], double *nrx) {
  // 0 sum log x, 1 ||x - x0||^2, 2 ||r_x (x part)||^2
  double a[3] = {0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < n; i += LD_T) {
    const double xi = x[i];
    const double xinv = 1 / xi;
    const double g0x = xi - x0[i];
    const double g1x = xinv * -v;
    const double rxx = g0x * z[0] + z[1] * g1x;
    a[0] += log(xi);
    a[1] += g0x * g0x;
    a[2] += rxx * rxx;
    if (store) {
      x_inv[i] = xinv;
      g0->x[i] = g0x;
      g1->x[i] = g1x;
      rx->x[i] = rxx;
    }
  }
  warp_sums<3>(a);
  g0->t = t - t0;
  g0->v = v - v0;
  g0->r = -1.0;
  const double sum_log_xv = a[0] - n * log(v);
  const double norm_2 = sqrt(a[1]);
  f[0] = 0.5 * (g0->t * g0->t + g0->v * g0->v + norm_2 * norm_2) - r;
  f[1] = -v * sum_log_xv - t;
  f[2] = -v;
  g1->t = -1.0;
  g1->v = n - sum_log_xv;
  g1->r = 0.0;
  rx->t = g0->t * z[0] + z[1] * g1->t;
  rx->v = g0->v * z[0] + z[1] * g1->v - z[2];
  rx->r = g0->r * z[0] + z[1] * g1->r + 1;
  *nrx = sqrt(((rx->t * rx->t + rx->v * rx->v) + a[2]) + rx->r * rx->r);
}

// sum over the u_dim entries of a .* b, with the x parts' sum given
__device__ __forceinline__ double ld_dot(double at_b_t, double at_b_v, double sx, double ar_br) {
  return ((at_b_t + at_b_v) + sx) + ar_br;
}

struct LdKkt {
  double coeff;
  double R[9];
  LdVec c0, c1;  // G \ g0, G \ g1; G \ e_r = -e_r is implicit
  double *temp1, *temp2, *gres, *res, *bnew;
};

// KKT_precompute (log_cone_IPM.c:149-200)
__device__ __noinline__ void ld_kkt_precompute(int n, double v, const double *x_inv, const double z[3], const double w[3],
                                  const LdVec &g0, const LdVec &g1, LdKkt &K) {
  const double a = z[0] + 1 / (w[2] * w[2]) + z[1] * n / v;
  double s[3] = {0.0, 0.0, 0.0};  // coeff sum, dot(g0x, temp2), dot(g1x, temp2)
  for (int i = threadIdx.x; i < n; i += LD_T) {
    const double xi = x_inv[i];
    const double t1 = z[0] + (z[1] * v) * (xi * xi);
    const double t2 = xi / t1;
    K.temp1[i] = t1;
    K.temp2[i] = t2;
    s[0] += (xi * xi) / t1;
    s[1] += g0.x[i] * t2;
    s[2] += g1.x[i] * t2;
  }
  warp_sums<3>(s);
  K.coeff = a - z[1] * z[1] * s[0];
  K.c0.t = g0.t / z[0];
  K.c0.v = (g0.v + z[1] * s[1]) / K.coeff;
  K.c0.r = -g0.r;
  K.c1.t = g1.t / z[0];
  K.c1.v = (g1.v + z[1] * s[2]) / K.coeff;
  K.c1.r = -g1.r;
  double d[4] = {0.0, 0.0, 0.0, 0.0};  // g0.c0, g0.c1, g1.c0, g1.c1 (x parts)
  for (int i = threadIdx.x; i < n; i += LD_T) {
    const double c0 = (g0.x[i] + (z[1] * K.c0.v) * x_inv[i]) / K.temp1[i];
    const double c1 = (g1.x[i] + (z[1] * K.c1.v) * x_inv[i]) / K.temp1[i];
    K.c0.x[i] = c0;
    K.c1.x[i] = c1;
    d[0] += g0.x[i] * c0;
    d[1] += g0.x[i] * c1;
    d[2] += g1.x[i] * c0;
    d[3] += g1.x[i] * c1;
  }
  warp_sums<4>(d);
  K.R[0] = 1 + ld_dot(g0.t * K.c0.t, g0.v * K.c0.v, d[0], g0.r * K.c0.r);
  K.R[3] = ld_dot(g0.t * K.c1.t, g0.v * K.c1.v, d[1], g0.r * K.c1.r);
  K.R[6] = -g0.r;  // g0 . (G \ e_r) = g0_r * (-1)
  K.R[1] = ld_dot(g1.t * K.c0.t, g1.v * K.c0.v, d[2], g1.r * K.c0.r);
  K.R[4] = 1 + ld_dot(g1.t * K.c1.t, g1.v * K.c1.v, d[3], g1.r * K.c1.r);
  K.R[2] = K.c0.r;
}

// KKT_solve (log_cone_IPM.c:202-331): rhs1 = (r_x, r_znl) of length u_dim + 3, rhs2 of length 3. Writes du (its x
// part to du->x), dr, dz, ds.
__device__ __noinline__ void ld_kkt_solve(int n, const double z[3], const double w[3], const double *x_inv, double v,
                             const double lm[3], const LdVec &rhs1, const double rz_in[3], const double rhs2[3],
                             const LdVec &g0, const LdVec &g1, LdKkt &K, LdVec *du, double *dr, double dz[3],
                             double ds[3]) {
  const int lane = threadIdx.x;
  double rz[3];
  for (int k = 0; k < 3; ++k) rz[k] = rz_in[k] - w[k] * (rhs2[k] / lm[k]);
  const double sc0 = rz[0] / w[0], sc1 = rz[1] / w[1];
  LdVec b;
  b.t = rhs1.t; b.t += sc0 * g0.t; b.t += sc1 * g1.t;
  b.v = rhs1.v; b.v += sc0 * g0.v; b.v += sc1 * g1.v;
  b.r = rhs1.r; b.r += sc0 * g0.r; b.r += sc1 * g1.r;
  b.v -= rz[2] / (w[2] * w[2]);
  for (int i = lane; i < n; i += LD_T) {
    double bx = rhs1.x[i];
    bx += sc0 * g0.x[i];
    bx += sc1 * g1.x[i];
    K.bnew[i] = bx;
    K.res[i] = bx;
    du->x[i] = 0.0;
  }
  LdVec res = b;
  du->t = du->v = 0.0;
  *dr = 0.0;
  for (int it = 0; it < 3; ++it) {
    double s = 0.0;
    for (int i = lane; i < n; i += LD_T) s += K.res[i] * K.temp2[i];
    s = warp_sum(s);
    LdVec G;
    G.t = res.t / z[0];
    G.v = (res.v + z[1] * s) / K.coeff;
    G.r = -res.r;
    double d[2] = {0.0, 0.0};
    for (int i = lane; i < n; i += LD_T) {
      const double gx = (K.res[i] + (z[1] * G.v) * x_inv[i]) / K.temp1[i];
      K.gres[i] = gx;
      d[0] += g0.x[i] * gx;
      d[1] += g1.x[i] * gx;
    }
    warp_sums<2>(d);
    const double ctg0 = ld_dot(g0.t * G.t, g0.v * G.v, d[0], g0.r * G.r);
    const double ctg1 = ld_dot(g1.t * G.t, g1.v * G.v, d[1], g1.r * G.r);
    const double ctg2 = G.r;
    const double ri0 = ctg2 / K.R[2];
    const double ri1 = (ctg1 - K.R[1] * ri0) / K.R[4];
    const double ri2 = (ctg0 - K.R[0] * ri0 - K.R[3] * ri1) / K.R[6];
    // G -= [c0 c1 -e_r] ri, column by column
    G.t += -ri0 * K.c0.t; G.t += -ri1 * K.c1.t;
    G.v += -ri0 * K.c0.v; G.v += -ri1 * K.c1.v;
    G.r += -ri0 * K.c0.r; G.r += -ri1 * K.c1.r; G.r += -ri2 * -1.0;
    du->t += G.t;
    du->v += G.v;
    *dr += G.r;
    const bool more = it != 2;
    double e[3] = {0.0, 0.0, 0.0};  // dot(x_inv, du_x), dot(g0x, du_x), dot(g1x, du_x)
    for (int i = lane; i < n; i += LD_T) {
      double gx = K.gres[i];
      gx += -ri0 * K.c0.x[i];
      gx += -ri1 * K.c1.x[i];
      const double dx = du->x[i] + gx;
      du->x[i] = dx;
      if (more) {
        e[0] += x_inv[i] * dx;
        e[1] += g0.x[i] * dx;
        e[2] += g1.x[i] * dx;
      }
    }
    if (!more) break;
    warp_sums<3>(e);
    const double gdu_t = z[0] * du->t;
    const double gdu_v = (z[0] + 1 / (w[2] * w[2])) * du->v + z[1] * (n / v * du->v - e[0]);
    const double gdu_r = -*dr;
    const double coeff0 = ((g0.t * du->t + g0.v * du->v) + e[1]) + g0.r * *dr;
    const double coeff1 = ((g1.t * du->t + g1.v * du->v) + e[2]) + g1.r * *dr;
    double cct_t = g0.t * coeff0; cct_t += coeff1 * g1.t;
    double cct_v = g0.v * coeff0; cct_v += coeff1 * g1.v;
    double cct_r = g0.r * coeff0; cct_r += coeff1 * g1.r; cct_r += *dr;
    res.t = b.t + -1.0 * (gdu_t + cct_t);
    res.v = b.v + -1.0 * (gdu_v + cct_v);
    res.r = b.r + -1.0 * (gdu_r + cct_r);
    for (int i = lane; i < n; i += LD_T) {
      const double xi = x_inv[i], dx = du->x[i];
      const double gdu = z[0] * dx + z[1] * (-du->v * xi + v * dx * xi * xi);
      double cct = g0.x[i] * coeff0;
      cct += coeff1 * g1.x[i];
      K.res[i] = K.bnew[i] + -1.0 * (gdu + cct);
    }
  }
  double e[2] = {0.0, 0.0};
  for (int i = lane; i < n; i += LD_T) {
    e[0] += g0.x[i] * du->x[i];
    e[1] += g1.x[i] * du->x[i];
  }
  warp_sums<2>(e);
  dz[0] = rz[0] - w[0] * (((g0.t * du->t + g0.v * du->v) + e[0]) + g0.r * *dr);
  dz[1] = rz[1] - w[1] * (((g1.t * du->t + g1.v * du->v) + e[1]) + g1.r * *dr);
  dz[2] = rz[2] + du->v;
  for (int k = 0; k < 3; ++k) {
    dz[k] = -dz[k] / (w[k] * w[k]);
    ds[k] = w[k] * (rhs2[k] / lm[k] - w[k] * dz[k]);
  }
}

// log_cone_IPM (log_cone_IPM.c:338-713) for one variant. u = (t, v, x) (the cone's saved projection); x0 is scaled
// in place and unscaled at the end, as the reference does. ws: LD_VECS n + LD_KEEP doubles. Returns the iteration count.
__device__ __noinline__ int ld_ipm(int n, double t0, double v0, double *x0, double *u, double *ws, int variant) {
  const int lane = threadIdx.x;
  double *x = u + 2;
  double *x_inv = ws;
  LdVec g0, g1, rx, du, du_0;  // du_0: only its x part is used
  g0.x = ws + n; g1.x = ws + 2 * n; rx.x = ws + 3 * n; du.x = ws + 4 * n;
  double *xnew = ws + 5 * n, *x_0 = ws + 6 * n;
  du_0.x = ws + 7 * n;
  LdKkt K;
  K.temp1 = ws + 8 * n; K.temp2 = ws + 9 * n; K.c0.x = ws + 10 * n; K.c1.x = ws + 11 * n;
  K.gres = ws + 12 * n; K.res = ws + 13 * n; K.bnew = ws + 14 * n;
  double *xinv_new = ws + 15 * n;
  // scale (t0, v0, x0)
  double sc = 0.0;
  for (int i = lane; i < n; i += LD_T) sc = fmax(sc, fabs(x0[i]));
  double scale1 = warp_max(sc);
  scale1 = t0 > scale1 ? t0 : scale1;
  scale1 = v0 > scale1 ? v0 : scale1;
  scale1 = 1 / scale1;
  t0 = t0 * scale1;
  v0 = v0 * scale1;
  for (int i = lane; i < n; i += LD_T) {
    x0[i] *= scale1;
    x[i] = 1.0;
  }
  double t = 1.0, v = 1.0, r = 0.0, dr = 0.0, rnew = 0.0;
  double z[3] = {1.0, 1.0, 1.0}, s[3] = {1.0, 1.0, 1.0};
  double dz[3] = {0, 0, 0}, ds[3] = {0, 0, 0};
  // the state the relaxed line search may return to (rarely used: kept in the cone's scratch, not in registers).
  // Every lane writes and reads the same values. 0 t, 1 v, 2 r, 3 dr, 4 z, 7 s, 10 dz, 13 ds, 16 du_t, 17 du_v,
  // 18 phi, 19 dphi, 20 step
  double *keep = ws + 16 * n;
  double tnew = 0, vnew = 0, z_new[3] = {0, 0, 0}, s_new[3] = {0, 0, 0};
  double pres0 = 1, dres0 = 1, theta1 = 0, theta2 = 0, theta3 = 0;
  int relaxed_iters = 0, iter;
  for (iter = 0; iter < LD_MAX_ITER_IPM; ++iter) {
    const double gap = z[0] * s[0] + z[1] * s[1] + z[2] * s[2];
    const double mu = gap / 3;
    double f[3], norm_rx;
    ld_ipm_oracle(n, t, v, x, r, t0, v0, x0, z, x_inv, &g0, &g1, &rx, true, f, &norm_rx);
    double rznl[3] = {f[0] + s[0], f[1] + s[1], f[2] + s[2]};
    double dres = norm_rx;
    double pres = sqrt(rznl[0] * rznl[0] + rznl[1] * rznl[1] + rznl[2] * rznl[2]);
    const double norm_rznl = pres;
    if (iter == 0) {
      pres0 = fmax(pres, 1.0);
      dres0 = fmax(dres, 1.0);
      theta1 = 1.0 / gap;
      theta2 = 1.0 / dres0;
      theta3 = 1.0 / pres0;
    }
    pres = pres / pres0;
    dres = dres / dres0;
    const double relgap = gap / fmax(r, 1.0);
    if (dres < LD_FEASTOL_IPM && pres < LD_FEASTOL_IPM && (gap < LD_ABSTOL_IPM || relgap <= LD_RELTOL_IPM)) break;
    double w[3], lm[3];
    for (int k = 0; k < 3; ++k) {
      w[k] = sqrt(s[k] / z[k]);
      lm[k] = sqrt(s[k] * z[k]);
    }
    const double is0 = 1 / w[0], is1 = 1 / w[1];
    g0.t *= is0; g0.v *= is0; g0.r *= is0;
    g1.t *= is1; g1.v *= is1; g1.r *= is1;
    for (int i = lane; i < n; i += LD_T) {
      g0.x[i] *= is0;
      g1.x[i] *= is1;
      rx.x[i] = -rx.x[i];
    }
    ld_kkt_precompute(n, v, x_inv, z, w, g0, g1, K);
    double rhs2[3] = {-lm[0] * lm[0], -lm[1] * lm[1], -lm[2] * lm[2]};
    rx.t = -rx.t; rx.v = -rx.v; rx.r = -rx.r;
    for (int k = 0; k < 3; ++k) rznl[k] = -rznl[k];
    double sigma = 0.0;
    double phi = theta1 * gap + theta2 * norm_rx + theta3 * norm_rznl;
    double dphi = -theta1 * (1 - sigma) * gap - theta2 * norm_rx - theta3 * norm_rznl;
    double step = 0.0;
    for (int j = 0; j < 2; ++j) {
      if (j == 1 && variant == 0) {
        const double f1s = 1 - sigma;
        rx.t *= f1s; rx.v *= f1s; rx.r *= f1s;
        for (int k = 0; k < 3; ++k) rznl[k] *= f1s;
        for (int i = lane; i < n; i += LD_T) rx.x[i] *= f1s;
        for (int k = 0; k < 3; ++k) rhs2[k] += (sigma * mu - ds[k] * dz[k]);
      }
      ld_kkt_solve(n, z, w, x_inv, v, lm, rx, rznl, rhs2, g0, g1, K, &du, &dr, dz, ds);
      // find_max_step_size (log_cone_IPM.c:90-126)
      {
        double step_max = 10.0;
        for (int k = 0; k < 3; ++k) {
          if (dz[k] < 0) step_max = fmin(step_max, -z[k] / dz[k]);
          if (ds[k] < 0) step_max = fmin(step_max, -s[k] / ds[k]);
        }
        double dom = 10.0;
        if (du.v < 0) dom = fmin(dom, -v / du.v);
        double md = 10.0;
        for (int i = lane; i < n; i += LD_T)
          if (du.x[i] < 0) md = fmin(md, -x[i] / du.x[i]);
        dom = fmin(dom, warp_min(md));
        step = fmin(1.0, LD_STEP_IPM * step_max);
        while (step > dom) step *= LD_BETA_IPM;
      }
      bool backtrack = true;
      while (backtrack) {
        tnew = t + step * du.t;
        vnew = v + step * du.v;
        for (int i = lane; i < n; i += LD_T) xnew[i] = x[i] + step * du.x[i];
        rnew = r + step * dr;
        for (int k = 0; k < 3; ++k) {
          z_new[k] = z[k] + step * dz[k];
          s_new[k] = s[k] + step * ds[k];
        }
        LdVec g0n, g1n, rxn;
        g0n.x = g1n.x = rxn.x = nullptr;
        double fn[3], nrxn;
        ld_ipm_oracle(n, tnew, vnew, xnew, rnew, t0, v0, x0, z_new, xinv_new, &g0n, &g1n, &rxn, false, fn, &nrxn);
        const double rz0 = fn[0] + s_new[0], rz1 = fn[1] + s_new[1], rz2 = fn[2] + s_new[2];
        const double gap_new = z_new[0] * s_new[0] + z_new[1] * s_new[1] + z_new[2] * s_new[2];
        const double phi_new = theta1 * gap_new + theta2 * nrxn + theta3 * sqrt(rz0 * rz0 + rz1 * rz1 + rz2 * rz2);
        if (j == 0) {
          if (phi_new <= (1 - LD_ALPHA_IPM * step) * phi) {
            backtrack = false;
            sigma = gap_new / gap;
            if (sigma < 1) sigma *= (sigma * sigma);
          } else {
            step *= LD_BETA_IPM;
          }
        } else if (relaxed_iters == -1) {
          if (phi_new <= phi + LD_ALPHA_IPM * step * dphi) backtrack = false;
          else step *= LD_BETA_IPM;
        } else if (relaxed_iters == 0) {
          if (!(phi_new <= phi + LD_ALPHA_IPM * step * dphi)) {
            relaxed_iters = 1;
            keep[0] = t; keep[1] = v; keep[2] = r; keep[3] = dr;
            for (int k = 0; k < 3; ++k) { keep[4 + k] = z[k]; keep[7 + k] = s[k]; keep[10 + k] = dz[k]; keep[13 + k] = ds[k]; }
            keep[16] = du.t; keep[17] = du.v;
            for (int i = lane; i < n; i += LD_T) { x_0[i] = x[i]; du_0.x[i] = du.x[i]; }
            keep[18] = phi; keep[19] = dphi; keep[20] = step;
          }
          backtrack = false;
        } else if (relaxed_iters == LD_MAX_RELAXED_ITERS) {
          if (phi_new <= keep[18] + LD_ALPHA_IPM * keep[20] * keep[19]) {
            backtrack = false;
          } else {
            relaxed_iters = -1;
            t = keep[0]; v = keep[1]; r = keep[2]; dr = keep[3];
            for (int k = 0; k < 3; ++k) { z[k] = keep[4 + k]; s[k] = keep[7 + k]; dz[k] = keep[10 + k]; ds[k] = keep[13 + k]; }
            du.t = keep[16]; du.v = keep[17];
            for (int i = lane; i < n; i += LD_T) { x[i] = x_0[i]; du.x[i] = du_0.x[i]; }
            phi = keep[18]; dphi = keep[19]; step = keep[20];
          }
        } else {  // 0 < relaxed_iters < LD_MAX_RELAXED_ITERS
          if (phi_new <= keep[18] + LD_ALPHA_IPM * keep[20] * keep[19]) relaxed_iters = 0;
          else relaxed_iters += 1;
          backtrack = false;
        }
      }
    }
    t = tnew; v = vnew; r = rnew;
    for (int i = lane; i < n; i += LD_T) x[i] = xnew[i];
    for (int k = 0; k < 3; ++k) { z[k] = z_new[k]; s[k] = s_new[k]; }
  }
  scale1 = 1 / scale1;
  for (int i = lane; i < n; i += LD_T) {
    x0[i] *= scale1;
    x[i] *= scale1;
  }
  if (lane == 0) { u[0] = t * scale1; u[1] = v * scale1; }
  __syncwarp();
  return iter;
}

__device__ __forceinline__ bool ld_accept(const double res[3]) {
  return res[0] < LD_DUAL_FEAS_TOL && res[1] < LD_PRI_FEAS_TOL && fabs(res[2]) < LD_COMP_TOL;
}

// log_cone_proj_wrapper (log_cone_wrapper.c:47-129) on (t0, v0, x0). u = the cone's saved projection (t, v, x),
// warm its warm-start flag, st the running stats. Returns 0, or -1 when all three methods fail.
__device__ int ld_wrapper(int n, double t0, double v0, double *x0, double *u, double *ws, int *warm, LdStats &st) {
  int iter = 0;
  int status = ld_newton(n, t0, v0, x0, u, ws, &iter, warm);
  st.iter = iter;
  __syncwarp();
  if (u[0] >= t0 - 0.1 * fabs(t0)) ld_check_opt(n, u[0], u[1], u + 2, t0, v0, x0, st.res);
  else status = -1;
  if (status == 0 && ld_accept(st.res)) {
    st.newton_success = 1;
    return 0;
  }
  for (int variant = 0; variant < 2; ++variant) {
    st.iter = ld_ipm(n, t0, v0, x0, u, ws, variant);
    ld_check_opt(n, u[0], u[1], u + 2, t0, v0, x0, st.res);
    if (variant == 0) *warm = 1;
    if (ld_accept(st.res)) {
      st.newton_success = 2 + variant;
      return 0;
    }
  }
  return -1;
}

// log-det cone, vector step: one warp per cone of the group. off[b] = first row of X (t, v sit just before); idx[b] = the cone's index among the
// log-det cones; poff[b] = offset of its saved projection (2 + n doubles) in proj. Overwrites the eigenvalues with
// lambda' >= 0 and writes t', v'. The cone with index last writes the stats record.
__global__ void __launch_bounds__(LD_T) k_logdet_vector(int n, const int *__restrict__ off, const int *__restrict__ idx,
                                                        const long long *__restrict__ poff, double *__restrict__ evals,
                                                        double *__restrict__ x, const double *sv, const double *ry,
                                                        double *__restrict__ proj, int *__restrict__ warm,
                                                        double *__restrict__ scratch, int last, LdStats *stats,
                                                        int *err) {
  const int b = blockIdx.x, lane = threadIdx.x;
  double *e = evals + (size_t)b * n;
  double *u = proj + poff[b];
  double *ws = scratch + (size_t)b * (LD_VECS * n + LD_KEEP);
  const long long trow = (long long)off[b] - 2;
  const double sqrt2 = sqrt(2.0);
  const double t0 = sqrt2 * x[trow], v0 = sqrt2 * x[trow + 1];
  const int cone = idx[b];
  int wflag = warm[cone];
  LdStats st;
  st.newton_success = 0;
  st.iter = 0;
  st.res[0] = st.res[1] = st.res[2] = 0.0;
  const int status = ld_wrapper(n, t0, v0, e, u, ws, &wflag, st);
  __syncwarp();
  for (int i = lane; i < n; i += LD_T) e[i] = u[2 + i];
  if (lane == 0) {
    warm[cone] = wflag;
    const double inv = 1.0 / sqrt2;
    x[trow] = finish(inv * u[0], ry, sv, trow);
    x[trow + 1] = finish(inv * u[1], ry, sv, trow + 1);
    if (status != 0) atomicOr(err, LD_ERR_BIT);
    if (cone == last) {
      stats->iter = st.iter;
      stats->res[0] = st.res[0];
      stats->res[1] = st.res[1];
      stats->res[2] = st.res[2];
      if (status == 0) stats->newton_success = st.newton_success;
    }
  }
}

// order-1 log-det cones: the unpacked 1 x 1 matrix is its own eigenvalue, with eigenvector 1
__global__ void k_logdet_order1(int count, double *__restrict__ mats, double *__restrict__ evals) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= count) return;
  evals[b] = mats[b];
  mats[b] = 1.0;
}

// one batch of equally shaped matrices for cusolverDnXsyevBatched
struct EigGroup {
  int m, n;    // nuclear: X is m x n (order m + n); sum-of-largest: order n (m = 0)
  int N;       // order of the decomposed matrices
  int count;
  int *d_off;  // first row of each block's matrix (the row after t)
  int *d_k;    // sum-of-largest: k of each cone; log-det: the cone's index among the log-det cones
  long long *d_poff;  // log-det: offset of each cone's saved projection in B200SpecCones::d_ld_proj
  double *d_scratch;  // log-det: LD_VECS n doubles per cone
  double *d_mats, *d_evals;
  int *d_info;
  void *d_work, *h_work;
  size_t work_bytes, h_work_bytes;
};

}  // namespace

struct B200SpecCones {
  std::vector<EigGroup> ld, nuc, sl;
  // log-det state, kept across projections and solves like the reference's ScsConeWork: the warm-start flag of each
  // cone, its previous projection (2 + d doubles, at offsets 2 i + sum_{j<i} d_j) and the stats of the last cone
  int ld_count;
  long long ld_proj_len;
  int *d_ld_warm;
  double *d_ld_proj;
  LdStats *d_ld_stats;
  int n_ell1_small, n_ell1_big, n_chunks;
  int *d_ell1_off, *d_ell1_len;  // small cones first, then big ones
  double *d_par;                 // 2 per big cone
  int4 *d_chunks;
  cusolverDnHandle_t solver;
  cusolverDnParams_t params;
  int *d_err;  // owned by B200Cones
};

static void free_group(EigGroup &g) {
  b200_free(g.d_off); b200_free(g.d_k); b200_free(g.d_poff); b200_free(g.d_scratch); b200_free(g.d_mats); b200_free(g.d_evals); b200_free(g.d_info);
  b200_free(g.d_work); free(g.h_work);
}

extern "C" void b200_spec_destroy(B200SpecCones *c) {
  if (!c) return;
  b200_sync();
  for (auto &g : c->ld) free_group(g);
  for (auto &g : c->nuc) free_group(g);
  for (auto &g : c->sl) free_group(g);
  b200_free(c->d_ld_warm); b200_free(c->d_ld_proj); b200_free(c->d_ld_stats);
  b200_free(c->d_ell1_off); b200_free(c->d_ell1_len); b200_free(c->d_par); b200_free(c->d_chunks);
  if (c->params) cusolverDnDestroyParams(c->params);
  b200_solver_release((void *)c->solver);
  delete c;
}

// offsets / ks: host arrays of the group; allocates the eigensolver batch of order g.N
static bool init_group(B200SpecCones *c, EigGroup &g, const std::vector<int> &offs, const std::vector<int> *ks) {
  g.count = (int)offs.size();
  g.d_off = (int *)b200_malloc((size_t)g.count * 4);
  g.d_mats = (double *)b200_malloc((size_t)g.count * g.N * g.N * 8);
  g.d_evals = (double *)b200_malloc((size_t)g.count * g.N * 8);
  g.d_info = (int *)b200_malloc((size_t)g.count * 4);
  bool ok = g.d_off && g.d_mats && g.d_evals && g.d_info && b200_h2d(g.d_off, offs.data(), offs.size() * 4) == 0;
  if (ok && ks) {
    g.d_k = (int *)b200_malloc((size_t)g.count * 4);
    ok = g.d_k && b200_h2d(g.d_k, ks->data(), ks->size() * 4) == 0;
  }
  ok = ok && b200_sync() == 0;
  if (g.N == 1) return ok;  // order-1 log-det cones need no eigensolver (k_logdet_order1)
  size_t wd = 0, wh = 0;
  ok = ok && cusolverDnXsyevBatched_bufferSize(c->solver, c->params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_LOWER,
                                               g.N, CUDA_R_64F, g.d_mats, g.N, CUDA_R_64F, g.d_evals, CUDA_R_64F,
                                               &wd, &wh, std::min(g.count, B200_EIG_BATCH)) == CUSOLVER_STATUS_SUCCESS;
  if (ok) {
    g.work_bytes = wd;
    g.h_work_bytes = wh;
    g.d_work = b200_malloc(wd ? wd : 16);
    g.h_work = wh ? malloc(wh) : nullptr;
    ok = g.d_work != nullptr && (wh == 0 || g.h_work != nullptr);
  }
  return ok;
}

// zeroes the log-det warm starts, saved projections and stats: the state of a fresh b200_spec_create
extern "C" int b200_spec_reset(B200SpecCones *c) {
  if (!c || c->ld_count == 0) return 0;
  const int rc = b200_memset0(c->d_ld_warm, (size_t)c->ld_count * 4) |
                 b200_memset0(c->d_ld_proj, (size_t)c->ld_proj_len * 8) | b200_memset0(c->d_ld_stats, sizeof(LdStats));
  return rc != 0 || b200_sync() != 0 ? -1 : 0;
}

// the Newton_stats record of the last log-det cone projected: 0, or -1 when there are no log-det cones
extern "C" int b200_spec_logdet_stats(B200SpecCones *c, int *iter, int *newton_success, double res[3]) {
  if (!c || c->ld_count == 0) return -1;
  LdStats h;
  if (b200_d2h(&h, c->d_ld_stats, sizeof(h)) != 0 || b200_sync() != 0) return -1;
  *iter = h.iter;
  *newton_success = h.newton_success;
  res[0] = h.res[0]; res[1] = h.res[1]; res[2] = h.res[2];
  return 0;
}

extern "C" B200SpecCones *b200_spec_create(int dsize, const int *h_d, int nucsize, const int *h_nuc_m,
                                           const int *h_nuc_n, int ell1_size, const int *h_ell1, int sl_size,
                                           const int *h_sl_n, const int *h_sl_k, long long first_row, int *d_err) {
  if (b200_runtime_init() != 0) return nullptr;
  B200SpecCones *c = new B200SpecCones();  // value-initialised: counts and pointers start at 0
  c->d_err = d_err;
  long long row = first_row;
  // log-det cones come first (reference cones.c:1449): (t, v, X), 2 + d(d+1)/2 rows; grouped by order
  struct LdCones { std::vector<int> off, idx; std::vector<long long> poff; };
  std::map<int, LdCones> ld_by;
  long long poff = 0;
  for (int i = 0; i < dsize; ++i) {
    auto &e = ld_by[h_d[i]];
    e.off.push_back((int)(row + 2));
    e.idx.push_back(i);
    e.poff.push_back(poff);
    poff += 2 + (long long)h_d[i];
    row += 2 + (long long)h_d[i] * (h_d[i] + 1) / 2;
  }
  c->ld_count = dsize;
  c->ld_proj_len = poff;
  std::map<std::pair<int, int>, std::vector<int>> nuc_by;
  for (int i = 0; i < nucsize; ++i) {
    nuc_by[{h_nuc_m[i], h_nuc_n[i]}].push_back((int)(row + 1));
    row += 1 + (long long)h_nuc_m[i] * h_nuc_n[i];
  }
  std::vector<int> small_off, small_len, big_off, big_len;
  std::vector<int4> chunks;
  for (int i = 0; i < ell1_size; ++i) {
    const int n = h_ell1[i];
    if (n <= ELL1_INLINE) {
      small_off.push_back((int)row);
      small_len.push_back(n);
    } else {
      for (int done = 0; done < n; done += ELL1_CHUNK)
        chunks.push_back(make_int4((int)big_off.size(), (int)(row + 1 + done), n - done < ELL1_CHUNK ? n - done : ELL1_CHUNK, 0));
      big_off.push_back((int)row);
      big_len.push_back(n);
    }
    row += 1 + (long long)n;
  }
  std::map<int, std::pair<std::vector<int>, std::vector<int>>> sl_by;
  for (int i = 0; i < sl_size; ++i) {
    auto &e = sl_by[h_sl_n[i]];
    e.first.push_back((int)(row + 1));
    e.second.push_back(h_sl_k[i]);
    row += 1 + (long long)h_sl_n[i] * (h_sl_n[i] + 1) / 2;
  }
  // ---- l1 cones: small cones first, then big ones (one CTA per cone each)
  c->n_ell1_small = (int)small_off.size();
  c->n_ell1_big = (int)big_off.size();
  c->n_chunks = (int)chunks.size();
  const int ncones = c->n_ell1_small + c->n_ell1_big;
  if (ncones > 0) {
    std::vector<int> offs(small_off), lens(small_len);
    offs.insert(offs.end(), big_off.begin(), big_off.end());
    lens.insert(lens.end(), big_len.begin(), big_len.end());
    c->d_ell1_off = (int *)b200_malloc((size_t)ncones * 4);
    c->d_ell1_len = (int *)b200_malloc((size_t)ncones * 4);
    c->d_par = (double *)b200_malloc((size_t)(2 * ncones) * 8);
    c->d_chunks = (int4 *)b200_malloc((chunks.size() + 1) * sizeof(int4));
    if (!c->d_ell1_off || !c->d_ell1_len || !c->d_par || !c->d_chunks ||
        b200_h2d(c->d_ell1_off, offs.data(), offs.size() * 4) != 0 ||
        b200_h2d(c->d_ell1_len, lens.data(), lens.size() * 4) != 0 ||
        (!chunks.empty() && b200_h2d(c->d_chunks, chunks.data(), chunks.size() * sizeof(int4)) != 0) ||
        b200_sync() != 0) {
      b200_spec_destroy(c);
      return nullptr;
    }
  }
  if (dsize > 0) {
    c->d_ld_warm = (int *)b200_malloc((size_t)dsize * 4);
    c->d_ld_proj = (double *)b200_malloc((size_t)poff * 8);
    c->d_ld_stats = (LdStats *)b200_malloc(sizeof(LdStats));
    if (!c->d_ld_warm || !c->d_ld_proj || !c->d_ld_stats || b200_spec_reset(c) != 0) {
      b200_spec_destroy(c);
      return nullptr;
    }
  }
  // ---- eigensolver batches
  if (!ld_by.empty() || !nuc_by.empty() || !sl_by.empty()) {
    c->solver = (cusolverDnHandle_t)b200_solver_acquire();
    if (!c->solver || cusolverDnCreateParams(&c->params) != CUSOLVER_STATUS_SUCCESS) {
      b200_spec_destroy(c);
      return nullptr;
    }
  }
  for (auto &kv : ld_by) {
    EigGroup g;
    memset(&g, 0, sizeof(g));
    g.n = g.N = kv.first;
    bool ok = init_group(c, g, kv.second.off, &kv.second.idx);
    if (ok) {
      g.d_poff = (long long *)b200_malloc((size_t)g.count * 8);
      g.d_scratch = (double *)b200_malloc((size_t)g.count * (LD_VECS * g.n + LD_KEEP) * 8);
      ok = g.d_poff && g.d_scratch && b200_h2d(g.d_poff, kv.second.poff.data(), (size_t)g.count * 8) == 0 &&
           b200_sync() == 0;
    }
    c->ld.push_back(g);
    if (!ok) { b200_spec_destroy(c); return nullptr; }
  }
  for (auto &kv : nuc_by) {
    EigGroup g;
    memset(&g, 0, sizeof(g));
    g.m = kv.first.first;
    g.n = kv.first.second;
    g.N = g.m + g.n;
    const bool ok = init_group(c, g, kv.second, nullptr);
    c->nuc.push_back(g);  // pushed before the check so that destroy releases what was allocated
    if (!ok) { b200_spec_destroy(c); return nullptr; }
  }
  for (auto &kv : sl_by) {
    EigGroup g;
    memset(&g, 0, sizeof(g));
    g.n = g.N = kv.first;
    const bool ok = init_group(c, g, kv.second.first, &kv.second.second);
    c->sl.push_back(g);
    if (!ok) { b200_spec_destroy(c); return nullptr; }
  }
  return c;
}

static int syevd(B200SpecCones *c, EigGroup &g, const char *what) {
  return b200_syevd_batched(c->solver, c->params, g.N, g.d_mats, g.d_evals, g.d_work, g.work_bytes, g.h_work,
                            g.h_work_bytes, g.d_info, g.count, c->d_err, what);
}

extern "C" int b200_spec_project(B200SpecCones *c, double *d_x, const double *d_s, const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  // ---- log-det cones. A cone on which all three methods fail sets LD_ERR_BIT in the sticky flag; the solve then
  // fails at the next b200_cones_check (the next convergence check), where the reference fails at once.
  for (auto &g : c->ld) {
    b200_psd_unpack_launch(g.n, g.count, g.d_off, d_x, g.d_mats);
    if (g.N == 1) {
      k_logdet_order1<<<(g.count + 127) / 128, 128, 0, st>>>(g.count, g.d_mats, g.d_evals);
      b200_count_launch(1);
    } else if (syevd(c, g, "cusolverDnXsyevBatched (log-det cone)") != 0) {
      return -1;
    }
    k_logdet_vector<<<g.count, LD_T, 0, st>>>(g.n, g.d_off, g.d_k, g.d_poff, g.d_evals, d_x, d_s, d_ry,
                                              c->d_ld_proj, c->d_ld_warm, g.d_scratch, c->ld_count - 1,
                                              c->d_ld_stats, c->d_err);
    b200_count_launch(1);
    b200_reconstruct_launch(0, g.n, g.n, g.n, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
  }
  // ---- nuclear-norm cones
  for (auto &g : c->nuc) {
    for (int b0 = 0; b0 < g.count; b0 += B200_EIG_BATCH) {
      const int nb = std::min(B200_EIG_BATCH, g.count - b0);
      dim3 eg((g.N * g.N + 255) / 256, nb);
      k_nuc_embed<<<eg, 256, 0, st>>>(g.m, g.n, nb, g.d_off + b0, d_x, g.d_mats + (size_t)b0 * g.N * g.N);
      b200_count_launch(1);
    }
    if (syevd(c, g, "cusolverDnXsyevBatched (nuclear-norm cone embedding)") != 0) return -1;
    k_nuc_vector<<<g.count, NUC_T, 0, st>>>(g.m, g.n, g.count, g.d_off, g.d_evals, d_x, d_s, d_ry);
    b200_count_launch(1);
    b200_reconstruct_launch(2, g.N, g.m, g.n, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
  }
  // ---- l1-norm cones
  if (c->n_ell1_small > 0) {
    k_ell1_cones<<<c->n_ell1_small, ELL1_SMALL_T, 0, st>>>(c->d_ell1_off, c->d_ell1_len, d_x, d_s, d_ry, c->d_par);
    b200_count_launch(1);
  }
  if (c->n_ell1_big > 0) {
    k_ell1_cones<<<c->n_ell1_big, ELL1_BIG_T, 0, st>>>(c->d_ell1_off + c->n_ell1_small,
                                                       c->d_ell1_len + c->n_ell1_small, d_x, d_s, d_ry, c->d_par);
    k_ell1_chunks<<<c->n_chunks, 256, 0, st>>>(c->d_chunks, c->d_par, d_x, d_s, d_ry);
    b200_count_launch(2);
  }
  // ---- sum-of-largest-eigenvalues cones
  for (auto &g : c->sl) {
    b200_psd_unpack_launch(g.n, g.count, g.d_off, d_x, g.d_mats);
    if (syevd(c, g, "cusolverDnXsyevBatched (sum-of-largest-eigenvalues cone)") != 0) return -1;
    k_sl_vector<<<(g.count + 127) / 128, 128, 0, st>>>(g.n, g.count, g.d_off, g.d_k, g.d_evals, d_x, d_s, d_ry);
    b200_count_launch(1);
    b200_reconstruct_launch(1, g.n, g.n, g.n, g.count, g.d_off, g.d_mats, g.d_evals, d_x, d_s, d_ry);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

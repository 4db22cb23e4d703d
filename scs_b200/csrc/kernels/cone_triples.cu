// cone_triples.cu -- the three-dimensional cones of SCS on the device: exponential (primal and
// dual) and power (primal and dual). One thread per triple; no shared state, no reductions.
//
// Replaces reference src/exp_cone.c:365-441 (proj_pd_exp_cone and everything it calls) and
// src/cones.c:1282-1332 (proj_power_cone) + the dispatch of src/cones.c:1406-1443. Widening row
// 8(f)-3 of SURVEY.md: these cones are not in BASELINE.json's configs, they complete the cone
// product so that a reference user's exp/power models run on the device loop.
//
// Exponential cone K_exp = cl{(r,s,t): s > 0, s exp(r/s) <= t}. The projection follows
// H. Friberg, "Projection onto the exponential cone: a univariate root-finding problem" (2021),
// the algorithm the reference implements: (1) two closed-form candidates for the primal and the
// polar projection; accept them when Moreau's optimality conditions hold to 1e-8; otherwise
// (2) bracket the root rho of the univariate function h, (3) damped Newton (<= 20 steps, falling
// back to <= 40 bisections), (4) map rho back and keep it if it beats the closed-form candidate.
// Constants, stop rules and the order of the decisions are the reference's, because they decide
// WHICH branch a triple takes; exp/log come from the CUDA math library (<= 1-2 ulp from glibc),
// so results agree with the CPU to ~1e-15 relative except when a stop test flips (tests: 1e-11).
//
// Power cone K_a = {(x,y,r): x^a y^(1-a) >= |r|, x,y >= 0}: Newton on r (<= 20 steps, stop
// |f| < 1e-9 -- the reference's POW_CONE_TOL, so a borderline stop can differ by ~1e-9).
#include "../common.cuh"
#include "../admm_api.h"
#include <math.h>

#define EXP_BIG 1e15  // the reference's "infinity" for this cone
// the scalar math is host+device so that tests/test_cone_triples_cpu.py can check THIS restatement against
// the reference on the CPU before any GPU time is spent (oracle/Makefile builds it with -DB200_TRIPLES_HOST_TEST
// into a test-only library; the product library contains the device path only)
#define HD __host__ __device__

namespace {

struct V3 {
  double r, s, t;
};
HD inline double dist2(const V3 &a, const V3 &b) {
  const double d0 = a.r - b.r, d1 = a.s - b.s, d2 = a.t - b.t;
  return d0 * d0 + d1 * d1 + d2 * d2;
}
HD inline bool finite_big(double x) { return fabs(x) < EXP_BIG; }
HD inline double clampd(double x, double lo, double hi) { return fmax(lo, fmin(hi, x)); }

// h(rho) (Friberg eq. for the root, multiplied by a positive polynomial) and its derivative
HD inline double h_val(const V3 &v, double rho) {
  const double ep = exp(rho), em = 1.0 / ep;
  return ((rho - 1) * v.r + v.s) * ep - (v.r - rho * v.s) * em - (rho * (rho - 1) + 1) * v.t;
}
HD inline void h_val_der(const V3 &v, double rho, double &f, double &df) {
  const double ep = exp(rho), em = 1.0 / ep;
  f = ((rho - 1) * v.r + v.s) * ep - (v.r - rho * v.s) * em - (rho * (rho - 1) + 1) * v.t;
  df = (rho * v.r + v.s) * ep + (v.r - (rho - 1) * v.s) * em - (2 * rho - 1) * v.t;
}

// closed-form candidates: a point of the cone (resp. polar cone) and its squared distance
HD double primal_candidate(const V3 &v, V3 &p) {
  p.t = fmax(v.t, 0.0);
  p.s = 0.0;
  p.r = fmin(v.r, 0.0);
  double d = dist2(v, p);
  if (v.s > 0.0) {
    const double tp = fmax(v.t, v.s * exp(v.r / v.s));
    const double nd = (tp - v.t) * (tp - v.t);
    if (nd < d) {
      p.t = tp; p.s = v.s; p.r = v.r;
      d = nd;
    }
  }
  return d;
}
HD double polar_candidate(const V3 &v, V3 &q) {
  q.t = fmin(v.t, 0.0);
  q.s = fmin(v.s, 0.0);
  q.r = 0.0;
  double d = dist2(v, q);
  if (v.r > 0.0) {
    const double td = fmin(v.t, -v.r * exp(v.s / v.r - 1.0));
    const double nd = (v.t - td) * (v.t - td);
    if (nd < d) {
      q.t = td; q.s = v.s; q.r = v.r;
      d = nd;
    }
  }
  return d;
}

// bracket of the root (Friberg section 4: psi / omega bounds), made consistent at the end
HD double psi_p(const V3 &v) {
  const double w = sqrt(v.r * v.r + v.s * v.s - v.r * v.s);
  const double psi = (v.r > v.s) ? (v.r - v.s + w) / v.r : -v.s / (v.r - v.s - w);
  return ((psi - 1.0) * v.r + v.s) / (psi * (psi - 1.0) + 1.0);
}
HD double psi_d(const V3 &v) {
  const double w = sqrt(v.r * v.r + v.s * v.s - v.r * v.s);
  const double psi = (v.s > v.r) ? (v.r - w) / v.s : (v.r - v.s) / (v.r + w);
  return (v.r - psi * v.s) / (psi * (psi - 1.0) + 1.0);
}
HD double omega_p(double rho) {
  double val = exp(rho) / (rho * (rho - 1.0) + 1.0);
  if (rho < 2.0) val = fmin(val, exp(2.0) / 3.0);
  return val;
}
HD double omega_d(double rho) {
  double val = -exp(-rho) / (rho * (rho - 1.0) + 1.0);
  if (rho > -1.0) val = fmax(val, -exp(1.0) / 3.0);
  return val;
}
HD inline double safediv_pos(double x, double y) { return x / fmax(y, 1e-18); }

HD void root_bracket(const V3 &v, double pd2, double dd2, double &lo_out, double &hi_out) {
  double base_lo = -EXP_BIG, base_hi = EXP_BIG, lo = -EXP_BIG, hi = EXP_BIG;
  const double sm = fmin(v.s, 0.0), rm = fmin(v.r, 0.0);
  const double Dp = sqrt(fmax(pd2 - sm * sm, 0.0));
  const double Dd = sqrt(fmax(dd2 - rm * rm, 0.0));
  if (v.t > 0.0) {
    lo = fmax(lo, log(v.t / psi_p(v)));
  } else if (v.t < 0.0) {
    hi = fmin(hi, -log(-v.t / psi_d(v)));
  }
  if (v.r > 0.0) {
    base_lo = 1.0 - v.s / v.r;
    lo = fmax(lo, base_lo);
    const double tpu = fmax(1e-12, fmin(Dd, Dp + v.t));
    const double val = v.r * omega_p(lo);
    const double sgn = val < 0 ? -1.0 : 1.0;
    hi = fmin(hi, fmax(lo, base_lo + safediv_pos(tpu, fabs(val)) * sgn));
  }
  if (v.s > 0.0) {
    base_hi = v.r / v.s;
    hi = fmin(hi, base_hi);
    const double tdl = -fmax(1e-12, fmin(Dp, Dd - v.t));
    const double val = v.s * omega_d(hi);
    const double sgn = val < 0 ? -1.0 : 1.0;
    lo = fmax(lo, fmin(hi, base_hi - safediv_pos(tdl, fabs(val)) * sgn));
  }
  // rounding can push the bounds outside the base interval or flip them
  lo = clampd(fmin(lo, hi), base_lo, base_hi);
  hi = clampd(fmax(lo, hi), base_lo, base_hi);
  if (lo != hi) {
    const double fl = h_val(v, lo), fu = h_val(v, hi);
    if (fl * fu > 0.0) {
      if (fabs(fl) < fabs(fu)) hi = lo; else lo = hi;
    }
  }
  lo_out = lo;
  hi_out = hi;
}

HD double root_bisect(const V3 &v, double lo, double hi, double x) {
  double xn = x;
  for (int it = 0; it < 40; ++it) {
    const double f = h_val(v, x);
    if (f < 0.0) lo = x; else hi = x;
    xn = 0.5 * (lo + hi);
    if (fabs(xn - x) <= 1e-12 * fmax(1.0, fabs(xn)) || xn == lo || xn == hi) break;
    x = xn;
  }
  return xn;
}
HD double root_newton(const V3 &v, double lo, double hi, double x) {
  const double EPS = 1e-15, DFTOL = 1e-13, LOD = 0.05, HID = 0.95;
  int it = 0;
  for (; it < 20; ++it) {
    double f, df;
    h_val_der(v, x, f, df);
    if (fabs(f) <= EPS) break;
    if (f < 0.0) lo = x; else hi = x;
    if (hi <= lo) {  // bracket collapsed
      hi = 0.5 * (hi + lo);
      lo = hi;
      break;
    }
    if (!finite_big(f) || df < DFTOL) break;  // flat or overflowing
    const double xn = x - f / df;
    if (fabs(xn - x) <= EPS * fmax(1.0, fabs(xn))) break;
    if (xn >= hi) x = fmin(LOD * x + HID * hi, hi);
    else if (xn <= lo) x = fmax(LOD * x + HID * lo, lo);
    else x = xn;
  }
  if (it < 20) return clampd(x, lo, hi);
  return root_bisect(v, lo, hi, x);
}

HD double primal_from_root(const V3 &v, double rho, V3 &p) {
  const double lin = (rho - 1.0) * v.r + v.s, e = exp(rho);
  if (lin > 0.0 && finite_big(e)) {
    const double q = rho * (rho - 1.0) + 1.0;
    p.t = e * lin / q;
    p.s = lin / q;
    p.r = rho * lin / q;
    return dist2(p, v);
  }
  p.t = EXP_BIG; p.s = 0.0; p.r = 0.0;
  return EXP_BIG;
}
HD double polar_from_root(const V3 &v, double rho, V3 &q) {
  const double lin = v.r - rho * v.s, e = exp(-rho);
  if (lin > 0.0 && finite_big(e)) {
    const double d = rho * (rho - 1.0) + 1.0;
    q.t = -e * lin / d;
    q.s = (1.0 - rho) * lin / d;
    q.r = lin / d;
    return dist2(v, q);
  }
  q.t = -EXP_BIG; q.s = 0.0; q.r = 0.0;
  return EXP_BIG;
}

// in place: v <- Pi_{K_exp}(v) (primal != 0) or Pi_{K_exp^*}(v) = -Pi_{polar}(-v)
HD void project_exp(V3 &v, int primal) {
  const double TOL = 1e-8;
  if (!primal) { v.r = -v.r; v.s = -v.s; v.t = -v.t; }
  V3 p, q;
  double pd2 = primal_candidate(v, p);
  double dd2 = polar_candidate(v, q);
  double err = fabs(p.r + q.r - v.r);
  err = fmax(err, fabs(p.s + q.s - v.s));
  err = fmax(err, fabs(p.t + q.t - v.t));
  const double pq = p.r * q.r + p.s * q.s + p.t * q.t;
  bool done = (v.s <= 0.0 && v.r <= 0.0);
  done = done || (fmin(pd2, dd2) <= TOL * TOL);
  done = done || (err <= TOL && pq <= TOL);
  if (!done) {
    double lo, hi;
    root_bracket(v, pd2, dd2, lo, hi);
    const double rho = root_newton(v, lo, hi, 0.5 * (lo + hi));
    V3 hat;
    if (primal) {
      if (primal_from_root(v, rho, hat) <= pd2) p = hat;
    } else {
      if (polar_from_root(v, rho, hat) <= dd2) q = hat;
    }
  }
  if (primal) v = p;
  else { v.r = -q.r; v.s = -q.s; v.t = -q.t; }
}

// ------------------------------------------------------------------ power cone
HD inline double pow_coord(double r, double xh, double rh, double a) {
  const double x = 0.5 * (xh + sqrt(xh * xh + 4 * a * (rh - r) * r));
  return fmax(x, 1e-12);
}
HD void project_pow(double &v0, double &v1, double &v2, double a) {
  const double PTOL = 1e-9;
  const double xh = v0, yh = v1, rh = fabs(v2);
  if (xh >= 0 && yh >= 0 && PTOL + pow(xh, a) * pow(yh, 1 - a) >= rh) return;  // already inside
  if (xh <= 0 && yh <= 0 &&
      PTOL + pow(-xh, a) * pow(-yh, 1 - a) >= rh * pow(a, a) * pow(1 - a, 1 - a)) {
    v0 = v1 = v2 = 0.0;  // -v is in the polar cone
    return;
  }
  double x = 0.0, y = 0.0, r = rh / 2;
  for (int it = 0; it < 20; ++it) {
    x = pow_coord(r, xh, rh, a);
    y = pow_coord(r, yh, rh, 1 - a);
    const double xa = pow(x, a), yb = pow(y, 1 - a);
    const double f = xa * yb - r;
    if (fabs(f) < PTOL) break;
    const double dxdr = a * (rh - 2 * r) / (2 * x - xh);
    const double dydr = (1 - a) * (rh - 2 * r) / (2 * y - yh);
    const double fp = xa * yb * (a * dxdr / x + (1 - a) * dydr / y) - 1;
    r = fmax(r - f / fp, 0.0);
    r = fmin(r, rh);
  }
  v0 = x;
  v1 = y;
  v2 = (v2 < 0) ? -r : r;
}

__global__ void k_exp_triples(int n_primal, int n_total, long long off, double *__restrict__ x,
                              const double *sv, const double *ry) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += gridDim.x * blockDim.x) {
    const long long b = off + 3LL * i;
    V3 v;
    v.r = x[b]; v.s = x[b + 1]; v.t = x[b + 2];
    project_exp(v, i < n_primal);
    x[b] = moreau_post(v.r, ry, sv, b);
    x[b + 1] = moreau_post(v.s, ry, sv, b + 1);
    x[b + 2] = moreau_post(v.t, ry, sv, b + 2);
  }
}
__global__ void k_pow_triples(int n, long long off, const double *__restrict__ pw, double *__restrict__ x,
                              const double *sv, const double *ry) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long b = off + 3LL * i;
    const double a = pw[i];
    double v0 = x[b], v1 = x[b + 1], v2 = x[b + 2];
    if (a >= 0) {
      project_pow(v0, v1, v2, a);
    } else {
      // dual power cone through Moreau: Pi_{K*}(v) = v + Pi_K(-v)   (cones.c:1432-1440)
      double w0 = -v0, w1 = -v1, w2 = -v2;
      project_pow(w0, w1, w2, -a);
      v0 += w0; v1 += w1; v2 += w2;
    }
    x[b] = moreau_post(v0, ry, sv, b);
    x[b + 1] = moreau_post(v1, ry, sv, b + 1);
    x[b + 2] = moreau_post(v2, ry, sv, b + 2);
  }
}

}  // namespace

#ifdef B200_TRIPLES_HOST_TEST
// test-only host entry points (NOT compiled into libscs_b200.so)
extern "C" void b200_triples_host_exp(double *v, int primal) {
  V3 t;
  t.r = v[0]; t.s = v[1]; t.t = v[2];
  project_exp(t, primal);
  v[0] = t.r; v[1] = t.s; v[2] = t.t;
}
extern "C" void b200_triples_host_pow(double *v, double a) {
  if (a >= 0) {
    project_pow(v[0], v[1], v[2], a);
  } else {
    double w0 = -v[0], w1 = -v[1], w2 = -v[2];
    project_pow(w0, w1, w2, -a);
    v[0] += w0; v[1] += w1; v[2] += w2;
  }
}
#endif

#ifndef B200_TRIPLES_HOST_TEST
// d_x: the m-vector being projected (rows off.. hold -R x on entry, Pi(.)/R + s on exit)
extern "C" int b200_cone_triples_project(int n_exp_primal, int n_exp_dual, int n_pow, long long exp_off,
                                         const double *d_pow, double *d_x, const double *d_s,
                                         const double *d_ry) {
  cudaStream_t st = (cudaStream_t)b200_stream();
  const int ne = n_exp_primal + n_exp_dual;
  const int cap = 8 * b200_num_sms();
  if (ne > 0) {
    int g = (ne + 127) / 128;
    if (g > cap) g = cap;
    k_exp_triples<<<g, 128, 0, st>>>(n_exp_primal, ne, exp_off, d_x, d_s, d_ry);
    b200_count_launch(1);
  }
  if (n_pow > 0) {
    int g = (n_pow + 127) / 128;
    if (g > cap) g = cap;
    k_pow_triples<<<g, 128, 0, st>>>(n_pow, exp_off + 3LL * ne, d_pow, d_x, d_s, d_ry);
    b200_count_launch(1);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}
#endif

// spmv_flag.cuh -- the flagged-stream SpMV's per-stage work (kernels/spmv.cu, see the block comment above
// spmv_flag_kernel): the producer's bulk copies of one ring stage and one consumer warp's warp-tile. Shared by
// spmv_flag_kernel and by the CG loop's batch kernel (kernels/cg.cu k_cg_batch), which runs the CG pair's two
// products as phases of one launch: the same lanes, the same sums, the same bits.
#pragma once
#include "common.cuh"
#include "dev_api.h"

// defaults: ONE CTA of 768 threads per SM (1 producer + 23 consumer warps), 3 stages = 130 kB of shared
// memory (within the H100's 227 kB per block), which leaves ~125 kB of the 256 kB L1/shared array to the gathers
#ifndef SPMV3_THREADS
#define SPMV3_THREADS 768
#endif
#ifndef SPMV3_STAGES
#define SPMV3_STAGES 3
#endif
#ifndef SPMV3_CTAS_PER_SM
#define SPMV3_CTAS_PER_SM 1
#endif
#define SPMV3_NCW (SPMV3_THREADS / 32 - 1)
#define SPMV3_WT 128
#define SPMV3_CAP (SPMV3_NCW * SPMV3_WT + 8)
#define SPMV3_MAXROW 124
// the kernel forms stream positions up to stored + 128 in 32-bit int (kb = (k0 & ~3) + 4 * lane, ka + cnt)
#define SPMV3_MAX_STORED B200_MAX_STORED

// Packed index stream of the CG loop's operators (an operator with at most 2^22 columns): 3 bytes per entry, the
// column in bits 0..21, END in bit 22, SKIP in bit 23. The one encode / decode of that format; decode gives back the
// int32 entry (flags in bits 31 / 30) bit for bit.
#define SPMV3_IDX24_MAXCOLS (1 << 22)
__host__ __device__ __forceinline__ unsigned spmv3_idx24_encode(int v) {
  const unsigned u = (unsigned)v;
  return (u & 0x3fffffu) | ((u >> 31) & 1u) << 22 | ((u >> 30) & 1u) << 23;
}
__host__ __device__ __forceinline__ int spmv3_idx24_decode(unsigned e) {
  return (int)((e & 0x3fffffu) | ((e >> 22) & 1u) << 31 | ((e >> 23) & 1u) << 30);
}
// The packed slice of a stage's entries [ka, ka + cnt) (ka a multiple of 4): a 1-D bulk copy needs a 16-byte aligned
// address and a length that is a multiple of 16, so it starts at entry ka & ~15 (byte 3 * (ka & ~15)) and its length
// is rounded up. At most 12 + 5 entries more than the int32 slice, which is still less than 4 * cnt bytes.
__host__ __device__ __forceinline__ unsigned spmv3_idx24_slice_bytes(int ka, int cnt) {
  return (unsigned)((3 * (ka + cnt - (ka & ~15)) + 15) & ~15);
}

// random 8-byte gather of the dense vector. NC: the read-only path, optionally without L1 allocation; it requires x
// to stay unwritten for the whole launch. !NC: a weak load, for a launch that rewrites x between its phases (the
// acquire of the grid barrier in between invalidates stale L1 lines)
template <bool NC>
__device__ __forceinline__ double gather_ld(const double *p) {
  if (!NC) return *p;
#ifdef SPMV_GATHER_NOALLOC
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  return r;
#else
  return __ldg(p);
#endif
}
// epilogue; the caller fetches the operands d[row] (dv) and v[row] (vv), the flag kernel EARLY (before the gathers
// are consumed) so that their latency overlaps the row's chain instead of adding to it
template <int POST>
__device__ __forceinline__ void spmv_epilogue(double s, int row, double *__restrict__ y, double dv, double vv,
                                              double &dot_acc) {
  double out = s;
  if (POST == B200_POST_DIV) {
    out = s / dv;
  } else if (POST == B200_POST_MUL) {
    out = s * dv;
  } else if (POST == B200_POST_FMA_DOT) {
    out = fma(dv, vv, s);
    dot_acc = fma(vv, out, dot_acc);
  } else if (POST == B200_POST_FMA) {
    out = fma(dv, vv, s);
  }
  y[row] = out;
}

// The shared-memory ring of one CTA: SPMV3_STAGES stages of value slice, index slice and SPMV3_NCW descriptors
struct Spmv3Ring {
  double *vals;     // [SPMV3_STAGES][SPMV3_CAP]
  int *idx;         // [SPMV3_STAGES][SPMV3_CAP] (IDX24: the packed bytes)
  int4 *desc;       // [SPMV3_STAGES][SPMV3_NCW]
  uint64_t *full, *empty;
  double *out;      // [SPMV3_NCW][SPMV3_WT]: per consumer warp, the row sums of its warp-tile by row number
};

// producer: the bulk copies of group i of a CTA's warp-tiles (g = its first descriptor) into stage st, extent [ka,
// ka + cnt) of the stream
template <bool IDX24>
__device__ __forceinline__ void spmv3_issue_stage(const Spmv3Ring &R, int st, const int4 *g, int i, int ka, int cnt,
                                                  const void *colidx, const double *vals, uint64_t pol) {
  const unsigned ib = IDX24 ? spmv3_idx24_slice_bytes(ka, cnt) : (unsigned)cnt * 4u;
  mbar_expect_tx(&R.full[st], (unsigned)cnt * 8u + ib + (unsigned)(SPMV3_NCW * 16));
  tma_load_1d(R.desc + (size_t)st * SPMV3_NCW, g + (size_t)i * SPMV3_NCW, SPMV3_NCW * 16, &R.full[st], pol);
  if (IDX24)
    tma_load_1d(R.idx + (size_t)st * SPMV3_CAP, static_cast<const unsigned char *>(colidx) + 3 * (size_t)(ka & ~15),
                ib, &R.full[st], pol);
  else
    tma_load_1d(R.idx + (size_t)st * SPMV3_CAP, static_cast<const int *>(colidx) + ka, ib, &R.full[st], pol);
  tma_load_1d(R.vals + (size_t)st * SPMV3_CAP, vals + ka, (unsigned)cnt * 8u, &R.full[st], pol);
}

// Row operands and outputs of one product, as the consumer warps read them
struct Spmv3Epi {
  const double *x;    // gathered vector
  double *y;
  const double *init;
  double init_sign;
  const double *d;
  const unsigned *dmask;
  int dform;
  double dt0, dt1;    // the table forms of d: its values
  const double *v;
  // multi-GPU push mode (B200_HOOK_P2P_ROUTE): the routing table in shared memory, else unused
  bool routed;
  const int *rt_lo;
  unsigned long long *const *rt_dst;
  unsigned long long hook_val;
};

template <bool NC>
struct Spmv3Ro {
  typedef const double *__restrict__ D;
  typedef const unsigned *__restrict__ U;
};
template <>
struct Spmv3Ro<false> {
  typedef const double *D;
  typedef const unsigned *U;
};
// consumer warp cw: waits for stage st (phase parity par), takes its warp-tile, hands the stage back and sums and
// stores the warp-tile's rows. NC: the flavour of the gathers (gather_ld) and of the epilogue's reads; without it no
// pointer is restrict-qualified, so the compiler cannot turn a read into a non-coherent one either
template <int POST, bool IDX24, bool NC>
__device__ __forceinline__ void spmv3_consume_stage(const Spmv3Ring &R, int st, unsigned par, int cw, int lane,
                                                    const Spmv3Epi &E, double &dot_acc) {
  constexpr bool TAB = POST == B200_POST_MUL || POST == B200_POST_FMA_DOT || POST == B200_POST_FMA;
  typename Spmv3Ro<NC>::D x = E.x;
  typename Spmv3Ro<NC>::D d = E.d;
  typename Spmv3Ro<NC>::U dmask = E.dmask;
  typename Spmv3Ro<NC>::D v = E.v;
  const double *init = E.init;
  const int dform = E.dform;
  double *ws = R.out + cw * SPMV3_WT;
  const unsigned FULL = 0xffffffffu;
  const unsigned lt = (1u << lane) - 1u;
  const unsigned le = lt | (1u << lane);
  const int sw = (lane >> 2) & 1;
  mbar_wait(&R.full[st], par);
  const int4 dsc = R.desc[st * SPMV3_NCW + cw];
  const int ka = R.desc[st * SPMV3_NCW].y & ~3;
  const int row0 = dsc.x, k0 = dsc.y, cnt = dsc.z;
  const int kend = k0 + cnt;
  const int kb = (k0 & ~3) + 4 * lane;  // global index of this lane's first entry
  int4 iv = make_int4(0, 0, 0, 0);
  double2 t0 = make_double2(0.0, 0.0), t1 = make_double2(0.0, 0.0);
  const bool any = (kb < kend) && (kb + 4 > k0);
  if (any) {
    const int e = kb - ka;
    if (IDX24) {  // 12 bytes from byte 3 * (kb - (ka & ~15)), a multiple of 12: three conflict-free 32-bit LDS
      const unsigned *wp = reinterpret_cast<const unsigned *>(
          reinterpret_cast<const unsigned char *>(R.idx + (size_t)st * SPMV3_CAP) + 3 * (kb - (ka & ~15)));
      const unsigned w0 = wp[0], w1 = wp[1], w2 = wp[2];
      iv = make_int4(spmv3_idx24_decode(w0 & 0xffffffu), spmv3_idx24_decode(w0 >> 24 | (w1 & 0xffffu) << 8),
                     spmv3_idx24_decode(w1 >> 16 | (w2 & 0xffu) << 16), spmv3_idx24_decode(w2 >> 8));
    } else {
      iv = *reinterpret_cast<const int4 *>(R.idx + (size_t)st * SPMV3_CAP + e);
    }
    t0 = *reinterpret_cast<const double2 *>(R.vals + (size_t)st * SPMV3_CAP + e + 2 * sw);
    t1 = *reinterpret_cast<const double2 *>(R.vals + (size_t)st * SPMV3_CAP + e + 2 - 2 * sw);
  }
  const bool v0 = any && (kb >= k0), v1 = any && (kb + 1 >= k0) && (kb + 1 < kend),
             v2 = any && (kb + 2 >= k0) && (kb + 2 < kend), v3 = any && (kb + 3 < kend);
  const bool g0 = v0 && !(iv.x & B200_FLAG_SKIP), g1 = v1 && !(iv.y & B200_FLAG_SKIP),
             g2 = v2 && !(iv.z & B200_FLAG_SKIP), g3 = v3 && !(iv.w & B200_FLAG_SKIP);
  // 4 independent gathers in flight per lane
  const double x0 = g0 ? gather_ld<NC>(&x[iv.x & B200_COLMASK]) : 0.0;
  const double x1 = g1 ? gather_ld<NC>(&x[iv.y & B200_COLMASK]) : 0.0;
  const double x2 = g2 ? gather_ld<NC>(&x[iv.z & B200_COLMASK]) : 0.0;
  const double x3 = g3 ? gather_ld<NC>(&x[iv.w & B200_COLMASK]) : 0.0;
  // the stage's bytes are in registers (the gather addresses depend on them): hand it back
  __syncwarp();
  if (lane == 0) mbar_arrive(&R.empty[st]);
  if (cnt == 0) return;  // padding descriptor (warp-uniform)
  const int nrows_w = dsc.w;
  // epilogue operands of the first two rounds (rows row0 + lane, row0 + lane + 32): in flight
  // together with the gathers
  // (B200_D_TWO: the mask words, at most two per round; the table value is selected at the use)
  double pd0 = 0.0, pd1 = 0.0, pv0 = 0.0, pv1 = 0.0, pi0 = 0.0, pi1 = 0.0;
  unsigned pw0 = 0u, pw1 = 0u;
  {
    const bool r0ok = lane < nrows_w, r1ok = lane + 32 < nrows_w;
    if (POST != B200_POST_NONE) {
      if (!TAB || dform == B200_D_VEC) {
        if (r0ok) pd0 = d[row0 + lane];
        if (r1ok) pd1 = d[row0 + lane + 32];
      } else if (TAB && dform == B200_D_TWO) {
        if (r0ok) pw0 = dmask[(row0 + lane) >> 5];
        if (r1ok) pw1 = dmask[(row0 + lane + 32) >> 5];
      }
    }
    if (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) {
      if (r0ok) pv0 = v[row0 + lane];
      if (r1ok) pv1 = v[row0 + lane + 32];
    }
    if (init != nullptr) {
      if (r0ok) pi0 = init[row0 + lane];
      if (r1ok) pi1 = init[row0 + lane + 32];
    }
  }

  const double a0 = sw ? t1.x : t0.x, a1 = sw ? t1.y : t0.y;
  const double a2 = sw ? t0.x : t1.x, a3 = sw ? t0.y : t1.y;
  const bool e0 = v0 && (iv.x < 0), e1 = v1 && (iv.y < 0), e2 = v2 && (iv.z < 0), e3 = v3 && (iv.w < 0);
  const unsigned b0 = __ballot_sync(FULL, e0), b1 = __ballot_sync(FULL, e1);
  const unsigned b2 = __ballot_sync(FULL, e2), b3 = __ballot_sync(FULL, e3);
  const unsigned ends = b0 | b1 | b2 | b3;  // lanes in which at least one row ends
  // row number (within the warp-tile) of the first END of this lane = number of ENDs in the lanes before it
  int r = __popc(b0 & lt) + __popc(b1 & lt) + __popc(b2 & lt) + __popc(b3 & lt);
  // open-row segments: the tail of lane h (the last lane <= me in which a row ends) starts the
  // row that is open when my entries begin
  const unsigned mle = ends & le;
  const int h = mle ? 31 - __clz(mle) : 0;
  const int maxdist = __reduce_max_sync(FULL, lane - h);

  const double p0 = g0 ? __dmul_rn(a0, x0) : 0.0, p1 = g1 ? __dmul_rn(a1, x1) : 0.0;
  const double p2 = g2 ? __dmul_rn(a2, x2) : 0.0, p3 = g3 ? __dmul_rn(a3, x3) : 0.0;
  // in-lane sequential sums, restarted after every END (0 + p is exact)
  double acc = p0;
  double o0 = acc;
  if (e0) acc = 0.0;
  acc = __dadd_rn(acc, p1);
  double o1 = acc;
  if (e1) acc = 0.0;
  acc = __dadd_rn(acc, p2);
  double o2 = acc;
  if (e2) acc = 0.0;
  acc = __dadd_rn(acc, p3);
  double o3 = acc;
  if (e3) acc = 0.0;
  // segmented inclusive scan of the tails (Hillis-Steele, fixed order)
  double I = acc;
  for (int dd = 1; dd <= maxdist; dd <<= 1) {
    const double up = __shfl_up_sync(FULL, I, dd);
    if (lane - dd >= h) I = __dadd_rn(up, I);
  }
  double carry = __shfl_up_sync(FULL, I, 1);
  if (lane == 0) carry = 0.0;  // warp-tiles hold whole rows: nothing is open at entry 0
  // the first END of the lane closes the row that was open on entry
  if (e0) o0 = __dadd_rn(carry, o0);
  else if (e1) o1 = __dadd_rn(carry, o1);
  else if (e2) o2 = __dadd_rn(carry, o2);
  else if (e3) o3 = __dadd_rn(carry, o3);
  // transpose through the warp's scratch: row sums by row number, then a COALESCED epilogue
  // (one row per lane and round: full-sector stores of y, one division per row, operands of the
  // first two rounds were fetched before the gathers were consumed)
  if (e0) { ws[r] = o0; ++r; }
  if (e1) { ws[r] = o1; ++r; }
  if (e2) { ws[r] = o2; ++r; }
  if (e3) { ws[r] = o3; }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < SPMV3_WT / 32; ++j) {
    const int rr = lane + 32 * j;
    if (j * 32 >= nrows_w) break;  // warp-uniform
    if (rr < nrows_w) {
      const int row = row0 + rr;
      double sres = ws[rr];
      double dv, vv, iv0;
      unsigned dw;
      if (j == 0) { dv = pd0; dw = pw0; vv = pv0; iv0 = pi0; }
      else if (j == 1) { dv = pd1; dw = pw1; vv = pv1; iv0 = pi1; }
      else {
        dv = (POST != B200_POST_NONE && (!TAB || dform == B200_D_VEC)) ? d[row] : 0.0;
        dw = (TAB && dform == B200_D_TWO) ? dmask[row >> 5] : 0u;
        vv = (POST == B200_POST_FMA_DOT || POST == B200_POST_FMA) ? v[row] : 0.0;
        iv0 = (init != nullptr) ? init[row] : 0.0;
      }
      if (TAB && dform != B200_D_VEC) dv = (dw >> (row & 31)) & 1u ? E.dt1 : E.dt0;
      if (init != nullptr) sres = __dadd_rn(sres, E.init_sign * iv0);
      if (E.routed) {  // push the row to the rank that owns it, as a self-validating 16-byte element
        int o = 0;
        while (row >= E.rt_lo[o + 1]) ++o;
        ll_store(E.rt_dst[o] + 2 * (size_t)(row - E.rt_lo[o]), sres, (unsigned)E.hook_val);
      } else {
        spmv_epilogue<POST>(sres, row, E.y, dv, vv, dot_acc);
      }
    }
  }
  __syncwarp();  // the scratch is rewritten by the next warp-tile
}

// A flagged-stream operator as a kernel that runs it as one phase among others reads it (b200_spmv_flag_view)
struct B200FlagView {
  const void *idx;          // int32 or packed index stream
  const double *vals;
  const int4 *wt;
  const int *cta_begin;
  int grid;                 // CTAs of its partition
  int packed;               // 1: idx is the packed stream
  double *partials;         // its reduction slots and ticket counter (the dot product's finish)
  unsigned int *counter;
};
// 0 and *out filled for a one-pass operator (no virtual rows) with rows, else -1
extern "C" int b200_spmv_flag_view(const B200Spmv *M, B200FlagView *out);

// Register-resident path for small channel groups (GS = 1, 2, 4): domain batch norm
// (GS = 1) and the whitening layers of the shipped ResNet-50-DWT / LeNet (GS = 4).
//
// Each thread owns VEC consecutive pixels of all GS channels of one group, so a warp
// reads GS fully coalesced row segments; every kernel is one HBM pass:
//   stats       read x                    -> shifted moments -> mean, cov, W, running-stat EMA
//   apply       read x, write y           y = W (x - mean) [* gamma + beta] [relu]
//   bwd_reduce  read x, dout              -> R = sum dz xc^T, sum dz -> A1, Bm, cvec, dgamma, dbeta
//   bwd_apply   read x, dout, write dx    dx = A1 dz + Bm x + cvec
// i.e. 12 B/element forward + 20 B/element backward, the algorithmic minimum of SURVEY.md §8d.
//
// Activation storage T: float, or __nv_bfloat16 (DWT_DTYPE_BF16; half the bytes).  A thread's VEC = 4 pixels of one
// channel row are one float4 or 8 bytes of bf16 (ld4 / st4, dwt_common.cuh); the pilot shift's scalar loads and the
// residual widen the same way.  Everything between load and store is the fp32 code on the fp32 plan of the shape, so a
// bf16 call's sums, statistics, W, coefficients, dgamma / dbeta, running buffers and status bits are those of the fp32
// kernels on x.float(), and y / dx are their outputs rounded to nearest-even.
//
// Work decomposition.  A "problem" is one (domain, group).  A CTA of 8 warps serves `ppc`
// consecutive groups of one domain, 8/ppc warps ("team") per problem, so that sites with
// thousands of tiny problems (domain BN at 7x7: 6144 problems of 12.5 KB) still run a few
// hundred long-lived CTAs instead of thousands of short ones whose prologue/epilogue
// round trips dominate; sites with few large problems instead split each problem over
// `nchunks` CTAs (then ppc = 1) that meet through per-CTA partials and an arrival counter.
// The small dense algebra (4x4 Cholesky, triangular inverse, backward coefficients, EMA)
// is done by ONE thread per problem, entirely in registers.
//
// Reference: utils/whitening.py:37-61, utils/batch_norm.py:54-69 (/root/reference).
#include "dwt_common.cuh"
#include "norm_launch.h"
#include "small_algebra.cuh"

namespace dwt {
namespace {

// Team geometry of the calling thread.
struct Team {
  int wpp;       // warps per problem
  int team;      // team index inside the CTA
  int ttid;      // thread index inside the team
  int tthreads;  // threads per team
  int g;         // group served (may be >= G in the last CTA of a row: then !valid)
  bool valid;
  __device__ __forceinline__ Team(const Geom& gm) {
    wpp = kWarps / gm.ppc;
    tthreads = wpp * 32;
    team = threadIdx.x / tthreads;
    ttid = threadIdx.x - team * tthreads;
    g = blockIdx.y * gm.ppc + team;
    valid = g < gm.G;
  }
};

// item -> (image n, pixel-vector pv) of the flattened per-group work list
struct ItemMap {
  unsigned PV;          // pixel vectors per row
  unsigned img_stride;  // C*HW   (N*C*HW < 2^31 is checked on the host: 32-bit element offsets)
  __device__ __forceinline__ unsigned offset(unsigned item, int VEC) const {
    unsigned n = item / PV, pv = item - n * PV;
    return n * img_stride + pv * VEC;
  }
};

template <int GS, int VEC> struct Unroll {
  static constexpr int raw = 16 / (GS * VEC);                                   // ~16 floats per tensor per batch
  static constexpr int one = raw < 1 ? 1 : (raw > 8 ? 8 : raw);
  static constexpr int stats = 2 * one;                                        // ~32 floats in flight per thread
};

// Team-level reduction of NACC per-thread accumulators into sAcc[team][NACC] (or, when the
// problem is split over several CTAs, through the global partials + arrival counter).
// Returns true in the threads that should finalize (team thread 0 of a valid problem, and only
// in the last-arriving CTA when nchunks > 1).
template <int NACC>
__device__ __forceinline__ bool team_reduce(const Geom& gm, const Team& tm, int d, const float (&acc)[NACC],
                                            float (*sRed)[NACC], float (*sAcc)[NACC], float* partial,
                                            int* counters, int* sFlag) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < NACC; ++i) {
    const float v = warp_sum(acc[i]);
    if (lane == 0) sRed[warp][i] = v;
  }
  __syncthreads();
  if (tm.ttid < NACC) {
    float t = 0.f;
    for (int w = 0; w < tm.wpp; ++w) t += sRed[tm.team * tm.wpp + w][tm.ttid];
    sAcc[tm.team][tm.ttid] = t;
  }
  if (gm.nchunks > 1) {      // ppc == 1: one problem per CTA, split over gridDim.x CTAs
    float* prob = partial + ((size_t)d * gm.G + tm.g) * gm.nchunks * NACC;
    if (threadIdx.x < NACC) prob[(size_t)blockIdx.x * NACC + threadIdx.x] = sAcc[0][threadIdx.x];
    if (!arrive_is_last(counters + d * gm.G + tm.g, gm.nchunks, sFlag)) return false;
    if (threadIdx.x < NACC) {
      double s = 0.0;
      for (int c = 0; c < gm.nchunks; ++c) s += (double)__ldcg(prob + (size_t)c * NACC + threadIdx.x);
      sAcc[0][threadIdx.x] = (float)s;
    }
  }
  __syncthreads();
  return tm.valid && tm.ttid == 0;
}

// ------------------------------------------------------------------------------------------
// stats
// ------------------------------------------------------------------------------------------
template <class T, int GS, int VEC>
__global__ void __launch_bounds__(kThreads, (GS * VEC >= 16) ? 3 : 4) small_stats_kernel(const T* __restrict__ x, const Geom gm,
                                                                const FwdFin fin, float* __restrict__ partial,
                                                                int* counters) {
  constexpr int NM = GS * (GS + 1) / 2, NACC = GS + NM, UNROLL = Unroll<GS, VEC>::stats;
  __shared__ float sK[kWarps][GS];
  __shared__ float sRed[kWarps][NACC];
  __shared__ float sAcc[kWarps][NACC];
  __shared__ int sFlag;
  const Team tm(gm);
  const int d = blockIdx.z;
  const int g = tm.valid ? tm.g : gm.G - 1;          // out-of-range teams shadow the last group, results dropped
  const T* xg = x + ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const ItemMap map{(unsigned)(gm.HW / VEC), (unsigned)(gm.C * gm.HW)};
  const unsigned items = (unsigned)gm.N * map.PV, stride = gridDim.x * tm.tthreads;
  unsigned i0 = blockIdx.x * tm.tthreads + tm.ttid;

  // Pilot shift (mean of <=32 mid-image pixels of image 0, per channel, checked against 32 samples spread over the
  // domain: pilot_shift in dwt_common.cuh) overlapped with the first batch of loads: the loads do not depend on K,
  // only the arithmetic does.
  const bool spread = (long long)gm.N * gm.HW > kPilotSpread;
  const bool spread_lane = spread && tm.ttid < kPilotSpread;
  float pv[GS], ps[GS];
  {
    const int np = gm.HW < 32 ? gm.HW : 32, p0 = ((gm.HW - np) / 2) & ~3, lane = threadIdx.x & 31;
    const size_t so = spread_lane ? pilot_spread_offset(tm.ttid, gm.N, gm.HW, (size_t)gm.C * gm.HW) : 0;
#pragma unroll
    for (int c = 0; c < GS; ++c) {
      pv[c] = (tm.ttid < 32 && lane < np) ? ld1(xg + (size_t)c * gm.HW + p0 + lane) : 0.f;
      ps[c] = spread_lane ? ld1(xg + (size_t)c * gm.HW + so) : 0.f;
    }
  }
  HeldVec<T, VEC> v[UNROLL][GS];        // the next batch stays in flight across the accumulation of this one
  bool have[UNROLL];
  auto load_batch = [&](unsigned base) {
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = base + u * stride;
      have[u] = it < items;
      if (have[u]) {
        const T* p = xg + map.offset(it, VEC);
#pragma unroll
        for (int c = 0; c < GS; ++c) v[u][c].load(p + (size_t)c * gm.HW);
      }
    }
  };
  if (i0 < items) load_batch(i0);
  if (tm.ttid < 32) {
    const int np = gm.HW < 32 ? gm.HW : 32;
#pragma unroll
    for (int c = 0; c < GS; ++c) {
      const float K0 = warp_sum(pv[c]) / (float)np;
      const float e = spread_lane ? ps[c] - K0 : 0.f;
      const float s1 = warp_sum(e), s2 = warp_sum(e * e);
      if (tm.ttid == 0) sK[tm.team][c] = spread ? pilot_refine(K0, s1, s2) : K0;
    }
  }
  __syncthreads();
  float K[GS], acc[NACC];
#pragma unroll
  for (int c = 0; c < GS; ++c) K[c] = sK[tm.team][c];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  while (i0 < items) {
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (have[u]) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
          float xs[GS];
#pragma unroll
          for (int c = 0; c < GS; ++c) { xs[c] = v[u][c][e] - K[c]; acc[c] += xs[c]; }
#pragma unroll
          for (int c = 0; c < GS; ++c)
#pragma unroll
            for (int j = 0; j <= c; ++j) acc[GS + c * (c + 1) / 2 + j] = fmaf(xs[c], xs[j], acc[GS + c * (c + 1) / 2 + j]);
        }
      }
    }
    i0 += stride * UNROLL;
    if (i0 < items) load_batch(i0);
  }
  if (!team_reduce<NACC>(gm, tm, d, acc, sRed, sAcc, partial, counters, &sFlag)) return;

  const float invM = 1.f / gm.M;
  const float* a = sAcc[tm.team];
  float mean[GS], cov[GS][GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) mean[i] = K[i] + a[i] * invM;
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      const float cij = a[GS + i * (i + 1) / 2 + j] * invM - (a[i] * invM) * (a[j] * invM);
      cov[i][j] = cij; cov[j][i] = cij;
    }
  const bool bad = factor_thread<GS>(gm, fin, d, tm.g, mean, cov, true);
  ema_thread<GS>(gm, fin, d, tm.g, mean, cov, bad);
}

// Eval mode: W and mean straight from the running buffers (whitening.py:42-43,50-53).
template <int GS>
__global__ void __launch_bounds__(kThreads) small_eval_prep_kernel(const Geom gm, const FwdFin fin) {
  const int g = blockIdx.x * kThreads + threadIdx.x, d = blockIdx.z;
  if (g >= gm.G) return;
  float mean[GS], cov[GS][GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    mean[i] = fin.rmean[d][g * GS + i];
#pragma unroll
    for (int j = 0; j < GS; ++j) cov[i][j] = fin.rcov[d][(size_t)g * GS * GS + i * GS + j];
  }
  factor_thread<GS>(gm, fin, d, g, mean, cov, false);
}

// ------------------------------------------------------------------------------------------
// apply
// ------------------------------------------------------------------------------------------
template <class T, int GS, int VEC, int EPI>
__global__ void __launch_bounds__(kThreads, (GS * VEC >= 16) ? 3 : 4) small_apply_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                                const Geom gm, const float* __restrict__ save_mean,
                                                                const float* __restrict__ save_w,
                                                                const float* __restrict__ gamma,
                                                                const float* __restrict__ beta,
                                                                const T* __restrict__ res) {
  constexpr bool RES = (EPI & DWT_EPI_RESIDUAL) != 0;
  constexpr int NM = GS * (GS + 1) / 2, UNROLL = RES ? Unroll<GS, VEC>::one : Unroll<GS, VEC>::stats;
  const Team tm(gm);
  if (!tm.valid) return;
  const int g = tm.g, d = blockIdx.z;
  float Wp[NM], bp[GS];
  load_forward_map<GS, EPI>(save_w + ((size_t)d * gm.G + g) * GS * GS, save_mean + (size_t)d * gm.C + g * GS,
                            gamma + g * GS, beta + g * GS, Wp, bp);
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const T* xg = x + base;
  T* yg = y + base;
  const ItemMap map{(unsigned)(gm.HW / VEC), (unsigned)(gm.C * gm.HW)};
  const unsigned items = (unsigned)gm.N * map.PV, stride = gridDim.x * tm.tthreads;
  const T* rg = res + base;
  for (unsigned i0 = blockIdx.x * tm.tthreads + tm.ttid; i0 < items; i0 += stride * UNROLL) {
    float v[UNROLL][GS][VEC], rs[RES ? UNROLL : 1][GS][VEC];
    unsigned off[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = i0 + u * stride;
      if (it < items) {
        off[u] = map.offset(it, VEC);
#pragma unroll
        for (int c = 0; c < GS; ++c) {
          load_vec<VEC>(xg + off[u] + (size_t)c * gm.HW, v[u][c]);
          if constexpr (RES) load_vec<VEC>(rg + off[u] + (size_t)c * gm.HW, rs[u][c]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = i0 + u * stride;
      if (it < items) {
        float o[GS][VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
          float xi[GS], oi[GS];
#pragma unroll
          for (int c = 0; c < GS; ++c) xi[c] = v[u][c][e];
          apply_group<GS>(Wp, bp, xi, oi);
#pragma unroll
          for (int c = 0; c < GS; ++c) {
            float z = oi[c];
            if constexpr (RES) z += rs[u][c][e];
            o[c][e] = (EPI & DWT_EPI_RELU) ? fmaxf(z, 0.f) : z;
          }
        }
#pragma unroll
        for (int c = 0; c < GS; ++c) store_vec<VEC>(yg + off[u] + (size_t)c * gm.HW, o[c]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// backward reduce
// ------------------------------------------------------------------------------------------
template <class T, int GS, int VEC, int EPI>
__global__ void __launch_bounds__(kThreads, 3) small_bwd_reduce_kernel(const T* __restrict__ x,
                                                                     const T* __restrict__ dout, const Geom gm,
                                                                     const BwdFin fin, const float* __restrict__ beta,
                                                                     float* __restrict__ partial, int* counters) {
  constexpr int NM = GS * (GS + 1) / 2, NACC = GS * GS + GS, UNROLL = Unroll<GS, VEC>::one;
  constexpr bool RELU = (EPI & DWT_EPI_RELU) != 0;
  __shared__ float sRed[kWarps][NACC];
  __shared__ float sAcc[kWarps][NACC];
  __shared__ int sFlag;
  const Team tm(gm);
  const int d = blockIdx.z;
  const int g = tm.valid ? tm.g : gm.G - 1;
  float Wp[NM], bp[GS], mu[GS];
  const float* mean_g = fin.save_mean + (size_t)d * gm.C + g * GS;
  if constexpr (RELU)
    load_forward_map<GS, EPI>(fin.save_w + ((size_t)d * gm.G + g) * GS * GS, mean_g, fin.gamma + g * GS,
                              beta + g * GS, Wp, bp);
#pragma unroll
  for (int c = 0; c < GS; ++c) mu[c] = __ldg(mean_g + c);
  float acc[NACC];          // R[i][j] at i*GS+j, then sdz
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const T* xg = x + base;
  const T* gg = dout + base;
  const ItemMap map{(unsigned)(gm.HW / VEC), (unsigned)(gm.C * gm.HW)};
  const unsigned items = (unsigned)gm.N * map.PV, stride = gridDim.x * tm.tthreads;
  for (unsigned i0 = blockIdx.x * tm.tthreads + tm.ttid; i0 < items; i0 += stride * UNROLL) {
    float v[UNROLL][GS][VEC], q[UNROLL][GS][VEC];
    bool have[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = i0 + u * stride;
      have[u] = it < items;
      if (have[u]) {
        const unsigned off = map.offset(it, VEC);
#pragma unroll
        for (int c = 0; c < GS; ++c) {
          load_vec<VEC>(xg + off + (size_t)c * gm.HW, v[u][c]);
          load_vec<VEC>(gg + off + (size_t)c * gm.HW, q[u][c]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (have[u]) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
          float xi[GS], dz[GS];
#pragma unroll
          for (int c = 0; c < GS; ++c) { xi[c] = v[u][c][e]; dz[c] = q[u][c][e]; }
          if constexpr (RELU) {
            float oi[GS];
            apply_group<GS>(Wp, bp, xi, oi);
#pragma unroll
            for (int c = 0; c < GS; ++c) dz[c] = oi[c] > 0.f ? dz[c] : 0.f;
          }
#pragma unroll
          for (int i = 0; i < GS; ++i) {
            acc[GS * GS + i] += dz[i];
#pragma unroll
            for (int j = 0; j < GS; ++j) acc[i * GS + j] = fmaf(dz[i], xi[j] - mu[j], acc[i * GS + j]);
          }
        }
      }
    }
  }
  if (!team_reduce<NACC>(gm, tm, d, acc, sRed, sAcc, partial, counters, &sFlag)) return;
  const float* a = sAcc[tm.team];
  float R[GS][GS], sdz[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    sdz[i] = a[GS * GS + i];
#pragma unroll
    for (int j = 0; j < GS; ++j) R[i][j] = a[i * GS + j];
  }
  bwd_finalize_thread<GS>(gm, fin, d, tm.g, R, sdz);
}

// Backward coefficients when no reduction is needed (eval mode, no affine gradient): A1 = W^T diag(gamma).
template <int GS>
__global__ void __launch_bounds__(kThreads) small_bwd_prep_kernel(const Geom gm, const BwdFin fin) {
  const int g = blockIdx.x * kThreads + threadIdx.x, d = blockIdx.z;
  if (g >= gm.G) return;
  float R[GS][GS], sdz[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    sdz[i] = 0.f;
#pragma unroll
    for (int j = 0; j < GS; ++j) R[i][j] = 0.f;
  }
  bwd_finalize_thread<GS>(gm, fin, d, g, R, sdz);
}

// ------------------------------------------------------------------------------------------
// backward apply
// ------------------------------------------------------------------------------------------
template <class T, int GS, int VEC, int EPI>
__global__ void __launch_bounds__(kThreads, 3) small_bwd_apply_kernel(const T* __restrict__ x,
                                                                    const T* __restrict__ dout,
                                                                    T* __restrict__ dx, const Geom gm,
                                                                    const float* __restrict__ coef,
                                                                    const float* __restrict__ save_mean,
                                                                    const float* __restrict__ save_w,
                                                                    const float* __restrict__ gamma,
                                                                    const float* __restrict__ beta) {
  constexpr int NM = GS * (GS + 1) / 2, UNROLL = Unroll<GS, VEC>::one;
  constexpr bool RELU = (EPI & DWT_EPI_RELU) != 0;
  const Team tm(gm);
  if (!tm.valid) return;
  const int g = tm.g, d = blockIdx.z;
  float Wp[NM], bp[GS];
  if constexpr (RELU)
    load_forward_map<GS, EPI>(save_w + ((size_t)d * gm.G + g) * GS * GS, save_mean + (size_t)d * gm.C + g * GS,
                              gamma + g * GS, beta + g * GS, Wp, bp);
  // A1 upper-triangular (packed by rows), Bm symmetric (packed lower), cvec
  float A1[NM], Bm[NM], cv[GS];
  const float* cf = coef + ((size_t)d * gm.G + g) * coef_stride(GS);
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    cv[i] = __ldg(cf + 2 * GS * GS + i);
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      A1[i * (i + 1) / 2 + j] = __ldg(cf + j * GS + i);             // A1[j][i], j <= i
      Bm[i * (i + 1) / 2 + j] = __ldg(cf + GS * GS + i * GS + j);   // Bm[i][j] = Bm[j][i]
    }
  }
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const T* xg = x + base;
  const T* gg = dout + base;
  T* dg = dx + base;
  const ItemMap map{(unsigned)(gm.HW / VEC), (unsigned)(gm.C * gm.HW)};
  const unsigned items = (unsigned)gm.N * map.PV, stride = gridDim.x * tm.tthreads;
  for (unsigned i0 = blockIdx.x * tm.tthreads + tm.ttid; i0 < items; i0 += stride * UNROLL) {
    float v[UNROLL][GS][VEC], q[UNROLL][GS][VEC];
    unsigned off[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = i0 + u * stride;
      if (it < items) {
        off[u] = map.offset(it, VEC);
#pragma unroll
        for (int c = 0; c < GS; ++c) {
          load_vec<VEC>(xg + off[u] + (size_t)c * gm.HW, v[u][c]);
          load_vec<VEC>(gg + off[u] + (size_t)c * gm.HW, q[u][c]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const unsigned it = i0 + u * stride;
      if (it < items) {
        float o[GS][VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) {
          float xi[GS], dz[GS];
#pragma unroll
          for (int c = 0; c < GS; ++c) { xi[c] = v[u][c][e]; dz[c] = q[u][c][e]; }
          if constexpr (RELU) {
            float oi[GS];
            apply_group<GS>(Wp, bp, xi, oi);
#pragma unroll
            for (int c = 0; c < GS; ++c) dz[c] = oi[c] > 0.f ? dz[c] : 0.f;
          }
#pragma unroll
          for (int i = 0; i < GS; ++i) {
            float acc = cv[i];
#pragma unroll
            for (int j = i; j < GS; ++j) acc = fmaf(A1[j * (j + 1) / 2 + i], dz[j], acc);   // A1[i][j], j >= i
#pragma unroll
            for (int j = 0; j < GS; ++j) {
              const int hi = i > j ? i : j, lo = i > j ? j : i;
              acc = fmaf(Bm[hi * (hi + 1) / 2 + lo], xi[j], acc);
            }
            o[i][e] = acc;
          }
        }
#pragma unroll
        for (int c = 0; c < GS; ++c) store_vec<VEC>(dg + off[u] + (size_t)c * gm.HW, o[c]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// launch tables
// ------------------------------------------------------------------------------------------
inline dim3 grid_of(const Geom& gm, int chunks) { return dim3(chunks, (gm.G + gm.ppc - 1) / gm.ppc, gm.D); }
inline dim3 grid_prep(const Geom& gm) { return dim3((gm.G + kThreads - 1) / kThreads, 1, gm.D); }

#define DWT_DISPATCH_GS(GS_, ...)                      \
  switch (GS_) {                                       \
    case 1: { constexpr int kGS = 1; __VA_ARGS__; break; } \
    case 2: { constexpr int kGS = 2; __VA_ARGS__; break; } \
    case 4: { constexpr int kGS = 4; __VA_ARGS__; break; } \
    default: break;                                    \
  }
#define DWT_DISPATCH_VEC(V_, ...)                      \
  if ((V_) == 4) { constexpr int kVEC = 4; __VA_ARGS__; } else { constexpr int kVEC = 1; __VA_ARGS__; }
#define DWT_DISPATCH_EPI(E_, ...)                                         \
  if ((E_) == 3) { constexpr int kEPI = 3; __VA_ARGS__; }                 \
  else if ((E_) == 1) { constexpr int kEPI = 1; __VA_ARGS__; }            \
  else { constexpr int kEPI = 0; __VA_ARGS__; }
// Activation storage and row vector of a launch: TT = float with VEC 4 or 1, or __nv_bfloat16 with VEC 4 (the C ABI
// takes bf16 only where the float32 call of the shape has vec == 4, and runs that call's plan)
#define DWT_DISPATCH_T_VEC(BF16_, V_, ...)                                                \
  if (BF16_) { using TT = __nv_bfloat16; constexpr int kVEC = 4; __VA_ARGS__; }           \
  else { using TT = float; DWT_DISPATCH_VEC(V_, __VA_ARGS__); }
#define DWT_IN(P_) static_cast<const TT*>(P_)
#define DWT_OUT(P_) static_cast<TT*>(P_)

}  // namespace

bool small_supports(int GS) { return GS == 1 || GS == 2 || GS == 4; }

void small_stats(const void* x, bool bf16, const Geom& gm, int vec, const FwdFin& fin, float* partial, int* counters,
                 cudaStream_t st) {
  DWT_DISPATCH_GS(gm.GS, DWT_DISPATCH_T_VEC(bf16, vec, (small_stats_kernel<TT, kGS, kVEC><<<grid_of(gm, gm.nchunks), kThreads, 0, st>>>(
                                                            DWT_IN(x), gm, fin, partial, counters))));
}

void small_eval_prep(const Geom& gm, const FwdFin& fin, cudaStream_t st) {
  DWT_DISPATCH_GS(gm.GS, (small_eval_prep_kernel<kGS><<<grid_prep(gm), kThreads, 0, st>>>(gm, fin)));
}

void small_apply(const void* x, void* y, bool bf16, const Geom& gm, int vec, int chunks, int epi, const float* mean,
                 const float* w, const float* gamma, const float* beta, const void* residual, cudaStream_t st) {
  if (epi == 7) {
    DWT_DISPATCH_GS(gm.GS, DWT_DISPATCH_T_VEC(bf16, vec, (small_apply_kernel<TT, kGS, kVEC, 7><<<grid_of(gm, chunks), kThreads, 0, st>>>(
                                                              DWT_IN(x), DWT_OUT(y), gm, mean, w, gamma, beta, DWT_IN(residual)))));
    return;
  }
  DWT_DISPATCH_GS(gm.GS, DWT_DISPATCH_T_VEC(bf16, vec, DWT_DISPATCH_EPI(epi, (small_apply_kernel<TT, kGS, kVEC, kEPI><<<grid_of(gm, chunks), kThreads, 0, st>>>(
                                                                                  DWT_IN(x), DWT_OUT(y), gm, mean, w, gamma, beta, nullptr)))));
}

void small_bwd_reduce(const void* x, const void* dout, bool bf16, const Geom& gm, int vec, const BwdFin& fin,
                      const float* beta, float* partial, int* counters, cudaStream_t st) {
  DWT_DISPATCH_GS(gm.GS, DWT_DISPATCH_T_VEC(bf16, vec, DWT_DISPATCH_EPI(fin.epi, (small_bwd_reduce_kernel<TT, kGS, kVEC, kEPI><<<grid_of(gm, gm.nchunks), kThreads, 0, st>>>(
                                                                                      DWT_IN(x), DWT_IN(dout), gm, fin, beta, partial, counters)))));
}

void small_bwd_prep(const Geom& gm, const BwdFin& fin, cudaStream_t st) {
  DWT_DISPATCH_GS(gm.GS, (small_bwd_prep_kernel<kGS><<<grid_prep(gm), kThreads, 0, st>>>(gm, fin)));
}

void small_bwd_apply(const void* x, const void* dout, void* dx, bool bf16, const Geom& gm, int vec, int chunks, int epi,
                     const float* coef, const float* mean, const float* w, const float* gamma, const float* beta,
                     cudaStream_t st) {
  DWT_DISPATCH_GS(gm.GS, DWT_DISPATCH_T_VEC(bf16, vec, DWT_DISPATCH_EPI(epi, (small_bwd_apply_kernel<TT, kGS, kVEC, kEPI><<<grid_of(gm, chunks), kThreads, 0, st>>>(
                                                                                  DWT_IN(x), DWT_IN(dout), DWT_OUT(dx), gm, coef, mean, w, gamma, beta)))));
}

}  // namespace dwt

// Shared device-side pieces of the DWT hot path: argument blocks, reductions, the
// "last CTA of a group finalizes it" protocol, and the small dense algebra that turns
// reduced moments into whitening matrices (forward) or gradient coefficients (backward).
//
// Reference semantics restated here (paths relative to /root/reference):
//   utils/whitening.py:47-53,57-59   covariance -> shrink -> inverse(cholesky) -> EMA
//   utils/batch_norm.py:66-69        F.batch_norm: biased var normalises, unbiased var -> EMA
//   backward: closed form of SURVEY.md §8a (autograd through whitening.py:41-55)
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../../include/dwt_b200.h"

namespace dwt {

constexpr int kThreads = 256;          // every norm kernel runs 256-thread CTAs
constexpr int kWarps = kThreads / 32;

// ---------------------------------------------------------------------------------------------
// argument blocks (passed by value to kernels)
// ---------------------------------------------------------------------------------------------
struct Geom {
  int N;        // images per domain
  int C;        // channels
  int HW;       // pixels per image
  int GS;       // group size (1 for batch norm)
  int G;        // C / GS
  int D;        // domains
  int nchunks;  // CTAs cooperating on one (domain, group)
  int ppc;      // (domain, group) problems served by one CTA (register-resident path; 1, 2, 4 or 8)
  float M;      // N * HW as float
  int cw = 0;   // channels-last kernels: float4 columns per CTA slab (set by their launchers, norm_cl.cu)
  int ls = 0;   // channels-last kernels: threads per row lane, >= cw (set by their launchers, norm_cl.cu)
};

struct FwdFin {
  float a, b;            // S = a * cov + b * I   (whitening: 1-eps, eps ; batch norm: 1, eps)
  float momentum;        // EMA weight of the new statistic
  float unbias;          // factor on the covariance going into the EMA (M/(M-1) for batch norm)
  int update_running;
  int aliased;           // 1: every domain updates the SAME running buffers (ordered EMA collapses to a closed form)
                         // 0: all distinct (independent updates); -1: mixed (ordered, domain by domain)
  float* save_mean;      // [D][C]
  float* save_w;         // [D][G][GS*GS]
  float* save_cov;       // [D][G][GS*GS] workspace: batch covariance, read back for the ordered EMA
  float* rmean[DWT_MAX_DOMAINS];
  float* rcov[DWT_MAX_DOMAINS];
  int* dom_counter;      // [G]
  int* status;
  int* bad;              // [D][G] scratch: 1 when the batch covariance of (d, g) was not positive definite -- the
                         // reference raises from torch.cholesky before its EMA lines (whitening.py:53 vs :57-59), so
                         // that domain's update of the (possibly shared) running buffers is skipped
};

struct BwdFin {
  float a;               // shrink factor on the covariance (1-eps, or 1 for batch norm)
  int mode;              // DWT_MODE_*
  int epi;               // DWT_EPI_*
  const float* save_mean;  // [D][C]
  const float* save_w;     // [D][G][GS*GS]
  const float* gamma;      // [C] or null
  float* coef;           // [D][G][2*GS*GS + GS] : A1 | Bm | cvec   (dx = A1 dz + Bm x + cvec)
  float* dgb_part;       // [D][2][C] per-domain dgamma / dbeta
  float* dgamma;         // [C] or null
  float* dbeta;          // [C] or null
  int* dom_counter;      // [G]
};

__host__ __device__ inline int coef_stride(int GS) { return 2 * GS * GS + GS; }

// ---------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Activation storage of the register-resident kernels (norm_small.cu, norm_cl.cu): float, or __nv_bfloat16
// (DWT_DTYPE_BF16).  Four consecutive elements are one float4 or 8 bytes of bf16: bf16 widens to fp32 exactly as it
// loads and rounds to nearest-even as it stores, so everything between a load and a store is the fp32 code.
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld4(const float* p) { return ldg4(p); }
__device__ __forceinline__ float4 ld4(const __nv_bfloat16* p) {
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));          // bf16 -> fp32 is exact: the high half of the word
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
__device__ __forceinline__ void st4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__nv_bfloat16* p, const float4& v) {
  const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
  *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const unsigned*>(&a), *reinterpret_cast<const unsigned*>(&b));
}
// one element, widened
__device__ __forceinline__ float ld1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld1(const __nv_bfloat16* p) {
  return __uint_as_float((unsigned)__ldg(reinterpret_cast<const unsigned short*>(p)) << 16);
}

// All threads call. Returns true in every thread of the CTA that arrived last on `counter`
// (expected arrivals = n); the counter is reset by that CTA so the workspace stays reusable.
__device__ __forceinline__ bool arrive_is_last(int* counter, int n, int* s_flag) {
  if (n == 1) return true;
  __threadfence();            // publish this CTA's global writes
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = atomicAdd(counter, 1);
    int last = (t == n - 1);
    if (last) atomicExch(counter, 0);
    *s_flag = last;
  }
  __syncthreads();
  bool last = (*s_flag != 0);
  if (last) __threadfence();  // acquire the other CTAs' writes
  return last;
}

// Pilot shift K of the NCHW one-pass moments, per channel: the mean of up to 32 pixels from the middle of image 0,
// unless they sit far from the rest of the domain.  E[(x-K)^2] - (mean-K)^2 loses digits in proportion to
// (K - mean)^2 / var: an image 0 whose pilot window sat 30 sigma off cost 0.28 of the covariance on the tensor-core
// path at the microbench size (test_nchw_fp64.py).  So 32 samples spread over the domain are read as well (flattened
// sample (2k+1) M / 64 + the middle pixel: for N a multiple of 64, the middle pixel of images spread across N), and
// where their mean lies more than 20 of their standard deviations from K, K moves to it -- the rule of the
// channels-last cl_stats_kernel, whose threshold real activations stay below, so ordinary inputs keep K bit for bit.
// 32 samples rather than cl_stats' 8: with 8, about 1 % of channels estimate their spread 1.5x too wide and keep a K
// 30 sigma off, which still cost 4.3e-3 of the microbench covariance on the tensor-core path.  Every CTA of a
// (domain, group) computes the same K from the same loads, so partial sums stay directly addable.  The reference is
// two-pass (whitening.py:41-47).
constexpr int kPilotSpread = 32;

// element offset, from image 0's channel, of spread sample k (0..31) of a domain of N images.  M = N * HW < 2^31
// (make_plan checks N * C * HW), and the sample index below stays under 2M: 32-bit division, no modulo.
__device__ __forceinline__ size_t pilot_spread_offset(int k, int N, int HW, size_t img_stride) {
  const unsigned M = (unsigned)N * (unsigned)HW;
  unsigned m = (unsigned)((2ull * k + 1) * M / (2 * kPilotSpread)) + (unsigned)HW / 2 + (unsigned)sqrtf((float)HW) / 2;
  if (m >= M) m -= M;
  const unsigned n = m / (unsigned)HW;
  return (size_t)n * img_stride + (m - n * (unsigned)HW);
}

// s1, s2: sum and sum of squares of (spread sample - K) over the spread samples
__device__ __forceinline__ float pilot_refine(float K, float s1, float s2) {
  constexpr float inv = 1.f / kPilotSpread;            // exact
  const float dk = s1 * inv;                           // spread mean - K; spread variance = s2 / 32 - dk^2
  return 401.f * dk * dk > 400.f * (s2 * inv) ? K + dk : K;      // dk^2 > 400 * spread variance
}

__device__ __forceinline__ void pilot_shift(const float* xg /* image 0, first channel of group */,
                                            int GS, int N, int HW, size_t img_stride, float* sK) {
  const int np = HW < 32 ? HW : 32;
  const int p0 = ((HW - np) / 2) & ~3;
  const bool spread = (long long)N * HW > kPilotSpread;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t so = spread && lane < kPilotSpread ? pilot_spread_offset(lane, N, HW, img_stride) : 0;
  for (int c = warp; c < GS; c += kWarps) {
    float v = lane < np ? __ldg(xg + (size_t)c * HW + p0 + lane) : 0.f;
    const float s = spread && lane < kPilotSpread ? __ldg(xg + (size_t)c * HW + so) : 0.f;
    v = warp_sum(v);
    const float K = v / (float)np;
    const float e = spread && lane < kPilotSpread ? s - K : 0.f;
    const float s1 = warp_sum(e), s2 = warp_sum(e * e);
    if (lane == 0) sK[c] = spread ? pilot_refine(K, s1, s2) : K;
  }
}

// Fixed-order (deterministic) sum over the per-CTA partials of one (domain, group).
// partial layout: [nchunks][nacc]; result into s_acc[nacc].
__device__ __forceinline__ void reduce_partials(const float* partial, int nchunks, int nacc, float* s_acc) {
  for (int i = threadIdx.x; i < nacc; i += blockDim.x) {
    double s = 0.0;
    for (int c = 0; c < nchunks; ++c) s += (double)__ldcg(partial + (size_t)c * nacc + i);
    s_acc[i] = (float)s;
  }
}

// ---------------------------------------------------------------------------------------------
// forward finalize: (mean, cov) of one (domain, group)  ->  W, saved stats, running-stat EMA
//   sMean [GS], sCov [GS*LD] (full symmetric, leading dimension LD = GS+1), sL/sW scratch [GS*LD]
// ---------------------------------------------------------------------------------------------
__device__ inline void fwd_factor_block(const Geom& gm, const FwdFin& f, int d, int g, const float* sMean,
                                        const float* sCov, float* sL, float* sW, bool store_cov) {
  const int GS = gm.GS, LD = GS + 1, tid = threadIdx.x, nt = blockDim.x;
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  for (int i = tid; i < GS; i += nt) f.save_mean[(size_t)d * gm.C + g * GS + i] = sMean[i];
  for (int e = tid; e < GS * GS; e += nt) {
    int i = e / GS, j = e - i * GS;
    float c = sCov[i * LD + j];
    if (store_cov) f.save_cov[gbase + e] = c;
    sL[i * LD + j] = f.a * c + (i == j ? f.b : 0.f);
    sW[i * LD + j] = 0.f;
  }
  __syncthreads();
  // right-looking Cholesky, lower triangle of sL in place
  bool bad = false;                                 // meaningful in thread 0
  for (int k = 0; k < GS; ++k) {
    if (tid == 0) {
      float piv = sL[k * LD + k];
      bad |= !(piv > 0.f);
      sL[k * LD + k] = sqrtf(piv);
    }
    __syncthreads();
    const float inv = 1.f / sL[k * LD + k];
    for (int i = k + 1 + tid; i < GS; i += nt) sL[i * LD + k] *= inv;
    __syncthreads();
    const int r = GS - k - 1;
    for (int e = tid; e < r * r; e += nt) {
      int i = k + 1 + e / r, j = k + 1 + e % r;
      if (j <= i) sL[i * LD + j] -= sL[i * LD + k] * sL[j * LD + k];
    }
    __syncthreads();
  }
  // W = L^{-1} by forward substitution, one thread per column
  for (int j = tid; j < GS; j += nt) {
    sW[j * LD + j] = 1.f / sL[j * LD + j];
    for (int i = j + 1; i < GS; ++i) {
      float acc = 0.f;
      for (int k = j; k < i; ++k) acc = fmaf(sL[i * LD + k], sW[k * LD + j], acc);
      sW[i * LD + j] = -acc / sL[i * LD + i];
    }
  }
  __syncthreads();
  for (int e = tid; e < GS * GS; e += nt) {
    int i = e / GS, j = e - i * GS;
    f.save_w[gbase + e] = sW[i * LD + j];
  }
  if (tid == 0) {
    if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
    if (store_cov) f.bad[d * gm.G + g] = bad ? 1 : 0;
  }
}

// EMA of the running buffers, domain by domain in order so that aliased buffers end as
// r' = (1-m)^D r + ... exactly like D sequential module calls (SURVEY.md H5).
__device__ inline void fwd_ema_block(const Geom& gm, const FwdFin& f, int g, int* s_flag) {
  if (!f.update_running) return;
  if (!arrive_is_last(f.dom_counter + g, gm.D, s_flag)) return;
  const int GS = gm.GS, tid = threadIdx.x, nt = blockDim.x;
  const float m = f.momentum, k = 1.f - f.momentum;
  for (int e = tid; e < GS * GS + GS; e += nt) {
    for (int d = 0; d < gm.D; ++d) {
      if (__ldcg(f.bad + d * gm.G + g)) continue;
      if (e < GS * GS) {
        float c = __ldcg(f.save_cov + ((size_t)d * gm.G + g) * GS * GS + e) * f.unbias;
        float* p = f.rcov[d] + (size_t)g * GS * GS + e;
        *p = m * c + k * (*p);
      } else {
        int i = e - GS * GS;
        float mu = __ldcg(f.save_mean + (size_t)d * gm.C + g * GS + i);
        float* p = f.rmean[d] + g * GS + i;
        *p = m * mu + k * (*p);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// backward finalize: R = sum dz xc^T, sdz = sum dz of one (domain, group) -> A1, Bm, cvec
//   sR [GS*LD], sSdz [GS]; scratch sW, sT1, sT2 [GS*LD] each, sVec [3*GS]
// ---------------------------------------------------------------------------------------------
__device__ inline void bwd_finalize_block(const Geom& gm, const BwdFin& f, int d, int g, const float* sR,
                                          const float* sSdz, float* sW, float* sT1, float* sT2, float* sVec,
                                          int* s_flag) {
  const int GS = gm.GS, LD = GS + 1, tid = threadIdx.x, nt = blockDim.x;
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  const int c0 = g * GS;
  float* sG = sVec;            // gamma (or 1)
  float* sMu = sVec + GS;      // mean
  const bool affine = (f.epi & DWT_EPI_AFFINE) != 0;
  const bool train = f.mode == DWT_MODE_TRAIN;
  for (int e = tid; e < GS * GS; e += nt) {
    int i = e / GS, j = e - i * GS;
    sW[i * LD + j] = f.save_w[gbase + e];
  }
  for (int i = tid; i < GS; i += nt) {
    sG[i] = affine ? f.gamma[c0 + i] : 1.f;
    sMu[i] = f.save_mean[(size_t)d * gm.C + c0 + i];
  }
  __syncthreads();
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  float* cA1 = coef;
  float* cBm = coef + GS * GS;
  float* cVec = coef + 2 * GS * GS;
  if (affine) {
    // dgamma_i = sum_m dz_i y_i = sum_j W_ij R_ij ; dbeta_i = sum_m dz_i
    for (int i = tid; i < GS; i += nt) {
      float s = 0.f;
      for (int j = 0; j <= i; ++j) s = fmaf(sW[i * LD + j], sR[i * LD + j], s);
      f.dgb_part[((size_t)d * 2 + 0) * gm.C + c0 + i] = s;
      f.dgb_part[((size_t)d * 2 + 1) * gm.C + c0 + i] = sSdz[i];
    }
  }
  if (train) {
    // P = Phi(Q), Q = -dW W^T, dW = diag(gamma) R
    for (int e = tid; e < GS * GS; e += nt) {
      int i = e / GS, j = e - i * GS;
      float q = 0.f;
      if (j <= i) {
        for (int k = 0; k <= j; ++k) q = fmaf(sR[i * LD + k], sW[j * LD + k], q);
        q *= -sG[i] * (i == j ? 0.5f : 1.f);
      }
      sT1[i * LD + j] = q;
    }
    __syncthreads();
    // T = W^T P
    for (int e = tid; e < GS * GS; e += nt) {
      int i = e / GS, j = e - i * GS;
      float t = 0.f;
      for (int k = (i > j ? i : j); k < GS; ++k) t = fmaf(sW[k * LD + i], sT1[k * LD + j], t);
      sT2[i * LD + j] = t;
    }
    __syncthreads();
    // S' = T W
    for (int e = tid; e < GS * GS; e += nt) {
      int i = e / GS, j = e - i * GS;
      float s = 0.f;
      for (int k = j; k < GS; ++k) s = fmaf(sT2[i * LD + k], sW[k * LD + j], s);
      sT1[i * LD + j] = s;
    }
    __syncthreads();
  }
  const float sc = f.a / gm.M;
  for (int e = tid; e < GS * GS; e += nt) {
    int i = e / GS, j = e - i * GS;
    float bm = train ? sc * (sT1[i * LD + j] + sT1[j * LD + i]) : 0.f;   // (2a/M) sym(S')
    float a1 = (j >= i) ? sW[j * LD + i] * sG[j] : 0.f;                  // W^T diag(gamma)
    cBm[e] = bm;
    cA1[e] = a1;
    sT2[i * LD + j] = bm;
  }
  __syncthreads();
  for (int i = tid; i < GS; i += nt) {
    float c = 0.f;
    if (train) {
      for (int j = i; j < GS; ++j) c = fmaf(sW[j * LD + i] * sG[j], sSdz[j] / gm.M, c);
      for (int j = 0; j < GS; ++j) c = fmaf(sT2[i * LD + j], sMu[j], c);
      c = -c;
    }
    cVec[i] = c;
  }
  if (affine && f.dgamma != nullptr) {
    if (!arrive_is_last(f.dom_counter + g, gm.D, s_flag)) return;
    for (int i = tid; i < GS; i += nt) {
      float sg = 0.f, sb = 0.f;
      for (int dd = 0; dd < gm.D; ++dd) {
        sg += __ldcg(f.dgb_part + ((size_t)dd * 2 + 0) * gm.C + c0 + i);
        sb += __ldcg(f.dgb_part + ((size_t)dd * 2 + 1) * gm.C + c0 + i);
      }
      f.dgamma[c0 + i] = sg;
      f.dbeta[c0 + i] = sb;
    }
  }
}

}  // namespace dwt

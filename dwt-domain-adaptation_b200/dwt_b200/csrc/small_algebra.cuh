// Thread-level building blocks shared by the register-resident kernels of both memory layouts
// (norm_small.cu: NCHW, norm_cl.cu: channels-last): vector loads (fp32, or bf16 widened), the group's forward map, and the
// single-thread dense algebra for group sizes <= 4 (Cholesky, triangular inverse, EMA, backward
// coefficients), everything in registers.
#pragma once
#include "dwt_common.cuh"

namespace dwt {
namespace {

template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = __ldg(p);
  }
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    *p = v[0];
  }
}
// bf16 activations: 8-byte vectors only (the C ABI takes NCHW bf16 at HW % 4 == 0 with 8-byte-aligned tensors)
template <int VEC>
__device__ __forceinline__ void load_vec(const __nv_bfloat16* p, float (&v)[VEC]) {
  static_assert(VEC == 4, "bf16 rows are read as 8-byte vectors");
  const float4 t = ld4(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <int VEC>
__device__ __forceinline__ void store_vec(__nv_bfloat16* p, const float (&v)[VEC]) {
  static_assert(VEC == 4, "bf16 rows are written as 8-byte vectors");
  st4(p, make_float4(v[0], v[1], v[2], v[3]));
}

// VEC elements of one row held in registers from their load to their use: fp32 values, or the 8 loaded bytes of bf16,
// widened (exactly) where each value is read -- a prefetched bf16 batch then takes the registers of its bytes
template <class T, int VEC> struct HeldVec {
  float v[VEC];
  __device__ __forceinline__ void load(const float* p) { load_vec<VEC>(p, v); }
  __device__ __forceinline__ float operator[](int e) const { return v[e]; }
};
template <int VEC> struct HeldVec<__nv_bfloat16, VEC> {
  static_assert(VEC == 4, "bf16 rows are read as 8-byte vectors");
  uint2 u;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { u = __ldg(reinterpret_cast<const uint2*>(p)); }
  __device__ __forceinline__ float operator[](int e) const {
    const unsigned w = e < 2 ? u.x : u.y;
    return __uint_as_float((e & 1) ? (w & 0xFFFF0000u) : (w << 16));
  }
};

// out_c = bp_c + sum_{j<=c} Wp[c][j] x_j : W is lower-triangular (Cholesky basis, SURVEY H1).
// One fixed FMA order, shared by forward apply and the backward's ReLU-mask recompute so
// both see bit-identical pre-activations.
template <int GS>
__device__ __forceinline__ void apply_group(const float (&Wp)[GS * (GS + 1) / 2], const float (&bp)[GS],
                                            const float (&x)[GS], float (&out)[GS]) {
#pragma unroll
  for (int c = 0; c < GS; ++c) {
    float acc = bp[c];
#pragma unroll
    for (int j = 0; j <= c; ++j) acc = fmaf(Wp[c * (c + 1) / 2 + j], x[j], acc);
    out[c] = acc;
  }
}

// Per-thread copy of the group's forward map: Wp = diag(gamma) W, bp = gamma (-W mean) + beta.
template <int GS, int EPI>
__device__ __forceinline__ void load_forward_map(const float* save_w_g, const float* mean_g, const float* gamma_g,
                                                 const float* beta_g, float (&Wp)[GS * (GS + 1) / 2],
                                                 float (&bp)[GS]) {
#pragma unroll
  for (int c = 0; c < GS; ++c) {
    float b = 0.f;
#pragma unroll
    for (int j = 0; j <= c; ++j) {
      float w = __ldg(save_w_g + c * GS + j);
      b = fmaf(-w, __ldg(mean_g + j), b);
      Wp[c * (c + 1) / 2 + j] = w;
    }
    bp[c] = b;
  }
  if constexpr ((EPI & DWT_EPI_AFFINE) != 0) {
#pragma unroll
    for (int c = 0; c < GS; ++c) {
      const float ga = __ldg(gamma_g + c), be = __ldg(beta_g + c);
#pragma unroll
      for (int j = 0; j <= c; ++j) Wp[c * (c + 1) / 2 + j] *= ga;
      bp[c] = fmaf(ga, bp[c], be);
    }
  }
}

// ------------------------------------------------------------------------------------------
// single-thread finalize steps (GS <= 4, everything in registers)
// ------------------------------------------------------------------------------------------
template <int GS>
__device__ __forceinline__ bool factor_thread(const Geom& gm, const FwdFin& f, int d, int g, const float (&mean)[GS],
                                              const float (&cov)[GS][GS], bool store_cov) {
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  float L[GS][GS], W[GS][GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    f.save_mean[(size_t)d * gm.C + g * GS + i] = mean[i];
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      if (store_cov) f.save_cov[gbase + i * GS + j] = cov[i][j];
      L[i][j] = f.a * cov[i][j] + (i == j ? f.b : 0.f);
      W[i][j] = 0.f;
    }
  }
  bool bad = false;
#pragma unroll
  for (int k = 0; k < GS; ++k) {
    bad |= !(L[k][k] > 0.f);
    L[k][k] = sqrtf(L[k][k]);
    const float inv = 1.f / L[k][k];
#pragma unroll
    for (int i = k + 1; i < GS; ++i) L[i][k] *= inv;
#pragma unroll
    for (int i = k + 1; i < GS; ++i)
#pragma unroll
      for (int j = k + 1; j <= i; ++j) L[i][j] -= L[i][k] * L[j][k];
  }
  if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
  if (store_cov) f.bad[d * gm.G + g] = bad ? 1 : 0;
#pragma unroll
  for (int j = 0; j < GS; ++j) {
    W[j][j] = 1.f / L[j][j];
#pragma unroll
    for (int i = j + 1; i < GS; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int k = j; k < i; ++k) acc = fmaf(L[i][k], W[k][j], acc);
      W[i][j] = -acc / L[i][i];
    }
  }
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) f.save_w[gbase + i * GS + j] = W[i][j];
  return bad;
}

// EMA of the running buffers by one thread, domains in order (SURVEY.md H5).  With several
// domains the thread that finalizes the LAST domain of group g applies all D updates.
template <int GS>
__device__ __forceinline__ void ema_thread(const Geom& gm, const FwdFin& f, int d_self, int g,
                                           const float (&mean)[GS], const float (&cov)[GS][GS], bool bad_self) {
  if (!f.update_running) return;
  const float m = f.momentum, k = 1.f - f.momentum;
  if (gm.D == 1 || f.aliased == 0) {
    // this domain owns its buffers: update them directly from registers, no cross-CTA traffic
    if (bad_self) return;
    float* rc = f.rcov[d_self] + (size_t)g * GS * GS;
    float* rm = f.rmean[d_self] + g * GS;
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      rm[i] = m * mean[i] + k * rm[i];
#pragma unroll
      for (int j = 0; j < GS; ++j) rc[i * GS + j] = m * (cov[i][j] * f.unbias) + k * rc[i * GS + j];
    }
    return;
  }
  // shared buffers: the thread that finalizes the LAST domain of group g applies all D updates
  __threadfence();
  const int t = atomicAdd(f.dom_counter + g, 1);
  if (t != gm.D - 1) return;
  atomicExch(f.dom_counter + g, 0);
  __threadfence();
  if (f.aliased == 1) {
    // r' = k^D r + m * sum_d k^(D-1-d) s_d  ==  D sequential updates of one buffer (SURVEY.md H5)
    float* rc = f.rcov[0] + (size_t)g * GS * GS;
    float* rm = f.rmean[0] + g * GS;
    float c[GS * GS], u[GS];
#pragma unroll
    for (int e = 0; e < GS * GS; ++e) c[e] = rc[e];
#pragma unroll
    for (int e = 0; e < GS; ++e) u[e] = rm[e];
    for (int d = 0; d < gm.D; ++d) {
      if (__ldcg(f.bad + d * gm.G + g)) continue;
      const float* cv = f.save_cov + ((size_t)d * gm.G + g) * GS * GS;
      const float* mu = f.save_mean + (size_t)d * gm.C + g * GS;
#pragma unroll
      for (int e = 0; e < GS * GS; ++e) c[e] = m * (__ldcg(cv + e) * f.unbias) + k * c[e];
#pragma unroll
      for (int e = 0; e < GS; ++e) u[e] = m * __ldcg(mu + e) + k * u[e];
    }
#pragma unroll
    for (int e = 0; e < GS * GS; ++e) rc[e] = c[e];
#pragma unroll
    for (int e = 0; e < GS; ++e) rm[e] = u[e];
    return;
  }
  for (int d = 0; d < gm.D; ++d) {       // mixed aliasing: plain ordered read-modify-write
    if (__ldcg(f.bad + d * gm.G + g)) continue;
    const float* cv = f.save_cov + ((size_t)d * gm.G + g) * GS * GS;
    const float* mu = f.save_mean + (size_t)d * gm.C + g * GS;
    float* rc = f.rcov[d] + (size_t)g * GS * GS;
    float* rm = f.rmean[d] + g * GS;
    for (int e = 0; e < GS * GS; ++e) rc[e] = m * (__ldcg(cv + e) * f.unbias) + k * rc[e];
    for (int e = 0; e < GS; ++e) rm[e] = m * __ldcg(mu + e) + k * rm[e];
  }
}

// Plain read-modify-write EMA of domain d's buffers from registers.  Correct for ANY aliasing pattern when one
// thread (or threads ordered by a barrier) applies the domains in order.
template <int GS>
__device__ __forceinline__ void ema_direct(const Geom& gm, const FwdFin& f, int d, int g, const float* mean,
                                           const float* cov /* [GS*GS] row-major */) {
  const float m = f.momentum, k = 1.f - f.momentum;
  float* rc = f.rcov[d] + (size_t)g * GS * GS;
  float* rm = f.rmean[d] + g * GS;
#pragma unroll
  for (int i = 0; i < GS; ++i) rm[i] = m * mean[i] + k * rm[i];
#pragma unroll
  for (int e = 0; e < GS * GS; ++e) rc[e] = m * (cov[e] * f.unbias) + k * rc[e];
}

template <int GS>
__device__ __forceinline__ void bwd_finalize_thread(const Geom& gm, const BwdFin& f, int d, int g,
                                                    const float (&R)[GS][GS], const float (&sdz)[GS],
                                                    bool combine_domains = true) {
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  const int c0 = g * GS;
  const bool affine = (f.epi & DWT_EPI_AFFINE) != 0, train = f.mode == DWT_MODE_TRAIN;
  float W[GS][GS], ga[GS], mu[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    ga[i] = affine ? f.gamma[c0 + i] : 1.f;
    mu[i] = f.save_mean[(size_t)d * gm.C + c0 + i];
#pragma unroll
    for (int j = 0; j < GS; ++j) W[i][j] = f.save_w[gbase + i * GS + j];
  }
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  if (affine) {
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j <= i; ++j) s = fmaf(W[i][j], R[i][j], s);
      f.dgb_part[((size_t)d * 2 + 0) * gm.C + c0 + i] = s;
      f.dgb_part[((size_t)d * 2 + 1) * gm.C + c0 + i] = sdz[i];
    }
  }
  float Bm[GS][GS];
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) Bm[i][j] = 0.f;
  if (train) {
    float P[GS][GS], T[GS][GS], S[GS][GS];
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j < GS; ++j) {
        float q = 0.f;
        if (j <= i) {
#pragma unroll
          for (int k = 0; k <= j; ++k) q = fmaf(R[i][k], W[j][k], q);
          q *= -ga[i] * (i == j ? 0.5f : 1.f);
        }
        P[i][j] = q;
      }
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j < GS; ++j) {
        float t = 0.f;
#pragma unroll
        for (int k = (i > j ? i : j); k < GS; ++k) t = fmaf(W[k][i], P[k][j], t);
        T[i][j] = t;
      }
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j < GS; ++j) {
        float s = 0.f;
#pragma unroll
        for (int k = j; k < GS; ++k) s = fmaf(T[i][k], W[k][j], s);
        S[i][j] = s;
      }
    const float sc = f.a / gm.M;
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j < GS; ++j) Bm[i][j] = sc * (S[i][j] + S[j][i]);
  }
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    float c = 0.f;
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      const float a1 = (j >= i) ? W[j][i] * ga[j] : 0.f;
      coef[i * GS + j] = a1;
      coef[GS * GS + i * GS + j] = Bm[i][j];
      if (train) {
        c = fmaf(a1, sdz[j] / gm.M, c);
        c = fmaf(Bm[i][j], mu[j], c);
      }
    }
    coef[2 * GS * GS + i] = -c;
  }
  if (combine_domains && affine && f.dgamma != nullptr) {
    if (gm.D > 1) {
      __threadfence();
      const int t = atomicAdd(f.dom_counter + g, 1);
      if (t != gm.D - 1) return;
      atomicExch(f.dom_counter + g, 0);
      __threadfence();
    }
#pragma unroll
    for (int i = 0; i < GS; ++i) {
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


}  // namespace
}  // namespace dwt

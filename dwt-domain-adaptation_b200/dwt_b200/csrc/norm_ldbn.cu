// Latent-domain batch norm (dwt_bn_latent_*, include/dwt_b200.h): batch norm by the statistics of up to 8 domains whose
// membership is a weight per image.  Every quantity of the layer comes from per-(image, channel) sums, so the kernels are
// four bandwidth passes over rows of one (image, channel) -- statistics, apply, backward reduction, backward apply --
// and two small finalize kernels over channels.  Every reduction runs in a fixed order (no float atomics): reruns are
// bit-identical.
//
// Work split.  A row of M = HW pixels is cut into S segments of P pixels (ldbn_plan): NCHW a warp per (row, segment),
// channels-last a CTA per (image, channel slab, segment) whose threads read 4 channels (one float4 or 8 bytes of bf16)
// of a pixel.  The reductions write one partial per (image, segment, channel); the finalize kernels add the S partials
// in order.  The plan depends on the shape and layout only, never on the dtype: bf16 runs the fp32 schedule on widened
// loads and rounds its stores, so every bf16 output is the fp32 kernels' output on x.float(), rounded.
//
// Finalize kernels: a CTA per 32 channels, lane = channel, warp w takes images w, w + 8, ...; the eight warps' sums are
// added in warp order through shared memory (block_sum).
#include "norm_launch.h"

namespace dwt {
namespace {

constexpr int kLdbnMaxD = 8;
static_assert(DWT_MAX_LATENT_DOMAINS <= kLdbnMaxD, "latent-domain batch norm: raise kLdbnMaxD with the header limit");

// segment partials of one row: the sum of d and the sum of d*d (forward: d = x - K about the pilot K = the row's first
// pixel) or the sum of dy and of dy (x - K) (backward: K = the saved centre)
struct Acc { float a, b; };

template <bool BWD>
__device__ __forceinline__ void acc1(Acc& s, float x, float dy, float K) {
  const float d = x - K;
  if (BWD) { s.a += dy; s.b = fmaf(dy, d, s.b); }
  else { s.a += d; s.b = fmaf(d, d, s.b); }
}
template <bool BWD>
__device__ __forceinline__ void acc4(Acc& s, const float4& x, const float4& dy, float K) {
  acc1<BWD>(s, x.x, dy.x, K); acc1<BWD>(s, x.y, dy.y, K); acc1<BWD>(s, x.z, dy.z, K); acc1<BWD>(s, x.w, dy.w, K);
}

__device__ __forceinline__ void st1(float* p, float v) { *p = v; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// NCHW reduction: a warp per (row, segment).  VEC: HW % 4 == 0, segments of whole float4s.
template <bool BWD, bool VEC, class T>
__global__ void __launch_bounds__(kThreads) ldbn_reduce_nchw(const T* __restrict__ x, const T* __restrict__ dy,
                                                             LdbnGeom g, const float* __restrict__ centre,
                                                             float* __restrict__ pa, float* __restrict__ pb,
                                                             float* __restrict__ pilot) {
  const long long wid = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)g.N * g.C;
  if (wid >= rows * g.S) return;
  const long long row = wid / g.S;
  const int s = (int)(wid - row * g.S);
  const size_t base = (size_t)row * g.HW;
  const float K = BWD ? centre[row] : ld1(x + base);
  const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
  Acc a{0.f, 0.f};
  if (VEC) {
#pragma unroll 4
    for (int p = p0 + 4 * lane; p < p1; p += 128)
      acc4<BWD>(a, ld4(x + base + p), BWD ? ld4(dy + base + p) : float4{}, K);
  } else {
#pragma unroll 4
    for (int p = p0 + lane; p < p1; p += 32) acc1<BWD>(a, ld1(x + base + p), BWD ? ld1(dy + base + p) : 0.f, K);
  }
  a.a = warp_sum(a.a);
  a.b = warp_sum(a.b);
  if (lane == 0) {
    const int n = (int)(row / g.C), c = (int)(row - (long long)n * g.C);
    const size_t o = ((size_t)n * g.S + s) * g.C + c;
    pa[o] = a.a;
    pb[o] = a.b;
    if (!BWD && s == 0) pilot[row] = K;
  }
}

// channels-last reduction: CTA (slab, segment, image) of g.qc float4 columns x g.pr pixel rows; the rows are added in
// order through shared memory
template <bool BWD, class T>
__global__ void __launch_bounds__(kThreads) ldbn_reduce_nhwc(const T* __restrict__ x, const T* __restrict__ dy,
                                                             LdbnGeom g, const float* __restrict__ centre,
                                                             float* __restrict__ pa, float* __restrict__ pb,
                                                             float* __restrict__ pilot) {
  __shared__ float4 sa[kThreads], sb[kThreads];
  const int slabs = (g.C / 4 + g.qc - 1) / g.qc;
  int b = blockIdx.x;
  const int slab = b % slabs; b /= slabs;
  const int s = b % g.S;
  const int n = b / g.S;
  const int q = threadIdx.x % g.qc, r = threadIdx.x / g.qc;
  const int c4 = slab * g.qc + q;
  const bool on = r < g.pr && c4 < g.C / 4;
  float4 va{0.f, 0.f, 0.f, 0.f}, vb{0.f, 0.f, 0.f, 0.f};
  if (on) {
    const size_t img = (size_t)n * g.HW * g.C + 4 * c4;
    const float4 K = BWD ? *reinterpret_cast<const float4*>(centre + (size_t)n * g.C + 4 * c4) : ld4(x + img);
    Acc ax{0.f, 0.f}, ay{0.f, 0.f}, az{0.f, 0.f}, aw{0.f, 0.f};
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
#pragma unroll 4
    for (int p = p0 + r; p < p1; p += g.pr) {
      const float4 v = ld4(x + img + (size_t)p * g.C);
      const float4 d = BWD ? ld4(dy + img + (size_t)p * g.C) : float4{};
      acc1<BWD>(ax, v.x, d.x, K.x); acc1<BWD>(ay, v.y, d.y, K.y);
      acc1<BWD>(az, v.z, d.z, K.z); acc1<BWD>(aw, v.w, d.w, K.w);
    }
    va = make_float4(ax.a, ay.a, az.a, aw.a);
    vb = make_float4(ax.b, ay.b, az.b, aw.b);
    if (!BWD && s == 0 && r == 0) *reinterpret_cast<float4*>(pilot + (size_t)n * g.C + 4 * c4) = K;
  }
  sa[threadIdx.x] = va;
  sb[threadIdx.x] = vb;
  __syncthreads();
  if (on && r == 0) {
    for (int k = 1; k < g.pr; ++k) {
      const float4 ta = sa[k * g.qc + q], tb = sb[k * g.qc + q];
      va.x += ta.x; va.y += ta.y; va.z += ta.z; va.w += ta.w;
      vb.x += tb.x; vb.y += tb.y; vb.z += tb.z; vb.w += tb.w;
    }
    const size_t o = ((size_t)n * g.S + s) * g.C + 4 * c4;
    *reinterpret_cast<float4*>(pa + o) = va;
    *reinterpret_cast<float4*>(pb + o) = vb;
  }
}

// The eight warps' values v[0..cnt) of each lane, added in warp order; the sums land in warp 0 (others: unchanged).
template <int CNT>
__device__ __forceinline__ void block_sum(double (&v)[CNT], double* sm /* [kWarps][8][32] */) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int base = 0; base < CNT; base += 8) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (base + k < CNT) sm[(w * 8 + k) * 32 + lane] = v[base + k];
    __syncthreads();
    if (w == 0) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (base + k < CNT) {
          double t = sm[k * 32 + lane];
          for (int j = 1; j < kWarps; ++j) t += sm[(j * 8 + k) * 32 + lane];
          v[base + k] = t;
        }
    }
  }
  __syncthreads();
}

// s_d = sum_n w_nd of every domain into s (shared): warp d adds its lanes' images in order and then across the lanes in a
// fixed butterfly; a weight of exactly 0 is skipped.  Every thread of the CTA calls.
__device__ __forceinline__ void domain_mass(const LdbnFin& f, double* s) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (w < f.D) {
    double t = 0.0;
    for (int n = lane; n < f.N; n += 32) {
      const float wt = __ldg(f.weights + (size_t)n * f.D + w);
      if (wt != 0.f) t += wt;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) s[w] = t;
  }
  __syncthreads();
}

// per (domain, channel) of the CTA's 32 channels, shared between the passes of a finalize kernel
struct DomSm {
  float mu[kLdbnMaxD][32], var[kLdbnMaxD][32], r[kLdbnMaxD][32];
  double s[kLdbnMaxD];         // s_d
  double red[kWarps * 8 * 32];
};

// Forward finalize.  Train: per image m_n, v_n from the segment partials about the pilot; per domain
// s_d, mu_d, sigma2_d about image 0's mean (fp64); r_d, EMA.  Eval: mu_d, sigma2_d from the running buffers.  Then per
// image a_n, b_n and the apply's alpha = gamma a_n, beta' = gamma b_n + beta.
__global__ void __launch_bounds__(kThreads) ldbn_fwd_finalize(LdbnFin f, const float* __restrict__ pa,
                                                              const float* __restrict__ pb,
                                                              const float* __restrict__ pilot,
                                                              float* __restrict__ alpha, float* __restrict__ shift) {
  __shared__ DomSm sm;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const bool on = c < f.C;
  const int N = f.N, C = f.C, D = f.D, S = f.S;
  float* save_m = f.save;
  float* save_v = f.save + (size_t)N * C;
  float* save_a = f.save + (size_t)2 * N * C;
  float* save_b = f.save + (size_t)3 * N * C;
  float* save_mu = f.save + (size_t)4 * N * C;
  float* save_var = save_mu + (size_t)D * C;
  float* save_r = save_var + (size_t)D * C;
  const double* s = sm.s;
  domain_mass(f, sm.s);
  const double M = f.M;
  if (f.train) {
    // image moments; domain sums about ref = image 0's mean: sum w, sum w (m - ref), sum w (v + (m - ref)^2)
    double acc[2 * kLdbnMaxD];
#pragma unroll
    for (int k = 0; k < 2 * kLdbnMaxD; ++k) acc[k] = 0.0;
    double ref = 0.0;
    if (on) {
      double s1 = 0.0;
      for (int j = 0; j < S; ++j) s1 += pa[(size_t)j * C + c];
      ref = (double)pilot[c] + s1 / M;
    }
    for (int n = w; n < N; n += kWarps) {
      if (!on) break;
      double s1 = 0.0, s2 = 0.0;
      for (int j = 0; j < S; ++j) {
        const size_t o = ((size_t)n * S + j) * C + c;
        s1 += pa[o];
        s2 += pb[o];
      }
      const double dm = s1 / M;
      const double m = (double)pilot[(size_t)n * C + c] + dm;
      const double v = fmax(s2 / M - dm * dm, 0.0);
      save_m[(size_t)n * C + c] = (float)m;
      save_v[(size_t)n * C + c] = (float)v;
      const double e = m - ref;
#pragma unroll
      for (int d = 0; d < kLdbnMaxD; ++d)
        if (d < D) {
          const float wt = __ldg(f.weights + (size_t)n * D + d);
          if (wt != 0.f) {
            acc[d] += wt * e;
            acc[kLdbnMaxD + d] += wt * (v + e * e);
          }
        }
    }
    block_sum(acc, sm.red);
    if (w == 0) {
      bool bad = false;
#pragma unroll
      for (int d = 0; d < kLdbnMaxD; ++d) {
        if (d >= D) break;
        float mu = 0.f, var = 0.f, r = 0.f;
        if (s[d] != 0.0) {
          const double e = acc[d] / s[d];
          const double mud = ref + e, var2 = acc[kLdbnMaxD + d] / s[d] - e * e;
          mu = (float)mud; var = (float)var2;
          const bool good = s[d] > 0.0 && isfinite(mud) && isfinite(var2) && (double)var + (double)f.eps > 0.0;
          r = good ? rsqrtf(var + f.eps) : __int_as_float(0x7fc00000);
          if (on) {
            bad |= !good;
            const double ms = M * s[d];
            if (good && f.update_running && ms > 1.0) {
              float* rm = f.rmean + (size_t)d * C + c;
              float* rv = f.rvar + (size_t)d * C + c;
              *rm = (1.f - f.momentum) * *rm + f.momentum * mu;
              *rv = (1.f - f.momentum) * *rv + f.momentum * (float)(var2 * (ms / (ms - 1.0)));
            }
          }
        }
        sm.mu[d][lane] = mu; sm.var[d][lane] = var; sm.r[d][lane] = r;
        if (on) {
          save_mu[(size_t)d * C + c] = mu; save_var[(size_t)d * C + c] = var; save_r[(size_t)d * C + c] = r;
        }
      }
      if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
    }
  } else if (w == 0) {
    bool bad = false;
#pragma unroll
    for (int d = 0; d < kLdbnMaxD; ++d) {
      if (d >= D) break;
      float mu = 0.f, var = 0.f, r = 0.f;
      if (on && s[d] != 0.0) {
        mu = f.rmean[(size_t)d * C + c];
        var = f.rvar[(size_t)d * C + c];
        const bool good = s[d] > 0.0 && isfinite(mu) && isfinite(var) && (double)var + (double)f.eps > 0.0;
        r = good ? rsqrtf(var + f.eps) : __int_as_float(0x7fc00000);
        bad |= !good;
      }
      sm.mu[d][lane] = mu; sm.var[d][lane] = var; sm.r[d][lane] = r;
      if (on) {
        save_mu[(size_t)d * C + c] = mu; save_var[(size_t)d * C + c] = var; save_r[(size_t)d * C + c] = r;
      }
    }
    if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
  }
  __syncthreads();
  if (!on) return;
  const float gam = f.gamma ? f.gamma[c] : 1.f, bet = f.beta ? f.beta[c] : 0.f;
  bool bad = false;
  for (int n = w; n < N; n += kWarps) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int d = 0; d < kLdbnMaxD; ++d)
      if (d < D && s[d] != 0.0) {
        const float wt = __ldg(f.weights + (size_t)n * D + d);
        if (wt != 0.f) {
          const float wr = wt * sm.r[d][lane];
          a += wr;
          b = fmaf(-wr, sm.mu[d][lane], b);
        }
      }
    if (!(a > 0.f && isfinite(a) && isfinite(b))) {
      a = __int_as_float(0x7fc00000); b = 0.f;
      bad = true;
    }
    const size_t o = (size_t)n * C + c;
    save_a[o] = a;
    save_b[o] = b;
    // eval: the backward's centre, the mix of the domains' means this image is normalised about (train: m_n)
    if (!f.train) save_m[o] = a == a ? -b / a : 0.f;
    alpha[o] = gam * a;
    shift[o] = fmaf(gam, b, bet);
  }
  if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
}

// Backward finalize: per image G_n, H_n from the segment partials (sums of dy, about the centre K_n = save_m); per
// domain A_d, B_d (fp64, over the images in order); dgamma, dbeta; per image the dx coefficients
// dx = alpha dy + p (x - K_n) + q and each channel's share of dweights, summed over the CTA's 32 channels in lane order.
__global__ void __launch_bounds__(kThreads) ldbn_bwd_finalize(LdbnFin f, const float* __restrict__ pa,
                                                              const float* __restrict__ pb, float* __restrict__ ca,
                                                              float* __restrict__ cp, float* __restrict__ cq,
                                                              float* __restrict__ dwpart) {
  __shared__ DomSm sm;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  const bool on = c < f.C;
  const int N = f.N, C = f.C, D = f.D, S = f.S;
  const float* save_m = f.save;
  const float* save_v = f.save + (size_t)N * C;
  const float* save_a = f.save + (size_t)2 * N * C;
  const float* save_b = f.save + (size_t)3 * N * C;
  const float* save_mu = f.save + (size_t)4 * N * C;
  const float* save_var = save_mu + (size_t)D * C;
  const float* save_r = save_var + (size_t)D * C;
  const double* s = sm.s;
  domain_mass(f, sm.s);
  if (w == 0) {
#pragma unroll
    for (int d = 0; d < kLdbnMaxD; ++d)
      if (d < D) {
        sm.mu[d][lane] = on ? save_mu[(size_t)d * C + c] : 0.f;
        sm.var[d][lane] = on ? save_var[(size_t)d * C + c] : 0.f;
        sm.r[d][lane] = on ? save_r[(size_t)d * C + c] : 0.f;
      }
  }
  __syncthreads();
  const float gam = (on && f.gamma) ? f.gamma[c] : 1.f;
  // acc: A_d | B_d | sum dy | sum dy zhat
  double acc[2 * kLdbnMaxD + 2];
#pragma unroll
  for (int k = 0; k < 2 * kLdbnMaxD + 2; ++k) acc[k] = 0.0;
  for (int n = w; n < N; n += kWarps) {
    if (!on) break;
    float G = 0.f, H = 0.f;
    for (int j = 0; j < S; ++j) {
      const size_t o = ((size_t)n * S + j) * C + c;
      G += pa[o];
      H += pb[o];
    }
    const size_t o = (size_t)n * C + c;
    const float K = save_m[o], a = save_a[o], b = save_b[o];
    acc[2 * kLdbnMaxD] += G;
    acc[2 * kLdbnMaxD + 1] += (double)a * H + ((double)a * K + b) * G;
    if (f.train) {
      const float Gg = gam * G, Hg = gam * H;
#pragma unroll
      for (int d = 0; d < kLdbnMaxD; ++d)
        if (d < D && s[d] != 0.0) {
          const float wt = __ldg(f.weights + (size_t)n * D + d);
          if (wt != 0.f) {
            acc[d] += (double)wt * Gg;
            acc[kLdbnMaxD + d] += (double)wt * fmaf(Gg, K - sm.mu[d][lane], Hg);
          }
        }
    }
  }
  block_sum(acc, sm.red);
  // per domain: cA = r A / (M s), cB = r^3 B / (M s), broadcast through shared memory (sm.red is free again)
  float* sA = reinterpret_cast<float*>(sm.red);
  float* sB = sA + kLdbnMaxD * 32;
  if (w == 0) {
    if (on && f.dgamma) {
      f.dbeta[c] = (float)acc[2 * kLdbnMaxD];
      f.dgamma[c] = (float)acc[2 * kLdbnMaxD + 1];
    }
#pragma unroll
    for (int d = 0; d < kLdbnMaxD; ++d)
      if (d < D) {
        float A = 0.f, B = 0.f;
        if (f.train && s[d] != 0.0) {
          const float r = sm.r[d][lane], ims = (float)(1.0 / (f.M * s[d]));
          A = (float)acc[d] * r * ims;
          B = (float)acc[kLdbnMaxD + d] * r * r * r * ims;
        }
        sA[d * 32 + lane] = A;
        sB[d * 32 + lane] = B;
      }
  }
  __syncthreads();
  for (int n = w; n < N; n += kWarps) {
    float G = 0.f, H = 0.f, K = 0.f, v = 0.f, a = 0.f;
    if (on) {
      for (int j = 0; j < S; ++j) {
        const size_t o = ((size_t)n * S + j) * C + c;
        G += pa[o];
        H += pb[o];
      }
      const size_t o = (size_t)n * C + c;
      K = save_m[o]; a = save_a[o];
      if (f.train) v = save_v[o];
    }
    const float Gg = gam * G, Hg = gam * H;
    float p = 0.f, q = 0.f;
#pragma unroll
    for (int d = 0; d < kLdbnMaxD; ++d) {
      if (d >= D) break;
      float t = 0.f;
      if (on && s[d] != 0.0) {
        const float r = sm.r[d][lane], e = K - sm.mu[d][lane];
        t = r * fmaf(Gg, e, Hg);
        if (f.train) {
          const float A = sA[d * 32 + lane], B = sB[d * 32 + lane];
          const float wt = __ldg(f.weights + (size_t)n * D + d);
          if (wt != 0.f) {
            p = fmaf(-wt, B, p);
            q = fmaf(-wt, fmaf(B, e, A), q);
          }
          // (1/s)[r A e + r^3 B (v + e^2 - sigma2) / 2] with r A = M A', r^3 B = M B'
          const float Ms = (float)f.M;
          t -= Ms * (A * e + 0.5f * B * (v + e * e - sm.var[d][lane]));
        }
      }
      if (dwpart) {
        t = warp_sum(t);
        if (lane == 0) dwpart[((size_t)n * D + d) * gridDim.x + blockIdx.x] = t;
      }
    }
    if (on) {
      const size_t o = (size_t)n * C + c;
      ca[o] = gam * a;
      cp[o] = p;
      cq[o] = q;
    }
  }
}

// dweights[n][d] = the CTAs' shares in order
__global__ void __launch_bounds__(kThreads) ldbn_dw(const float* __restrict__ dwpart, int ND, int nblk,
                                                    float* __restrict__ dweights) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= ND) return;
  double t = 0.0;
  for (int k = 0; k < nblk; ++k) t += dwpart[(size_t)i * nblk + k];
  dweights[i] = (float)t;
}

// Apply passes.  Forward y = alpha x + beta' ; backward dx = alpha dy + p (x - K) + q; coefficients per (image, channel).
template <bool BWD>
__device__ __forceinline__ float apply1(float x, float dy, int i, const float* ca, const float* cb, const float* cq,
                                        const float* K) {
  if (BWD) return fmaf(__ldg(ca + i), dy, fmaf(__ldg(cb + i), x - __ldg(K + i), __ldg(cq + i)));
  return fmaf(__ldg(ca + i), x, __ldg(cb + i));
}

// NCHW: VEC -- a thread per 4 pixels of a row (HW % 4 == 0); else a thread per element
template <bool BWD, bool VEC, class T>
__global__ void __launch_bounds__(kThreads) ldbn_apply_nchw(const T* __restrict__ x, const T* __restrict__ dy,
                                                            T* __restrict__ out, LdbnGeom g, const float* __restrict__ ca,
                                                            const float* __restrict__ cb, const float* __restrict__ cq,
                                                            const float* __restrict__ K) {
  const unsigned total = (unsigned)((size_t)g.N * g.C * g.HW / (VEC ? 4 : 1));
  for (unsigned e = blockIdx.x * kThreads + threadIdx.x; e < total; e += gridDim.x * kThreads) {
    if (VEC) {
      const unsigned i = 4 * e, row = i / (unsigned)g.HW;
      const float4 v = ld4(x + i), d = BWD ? ld4(dy + i) : float4{};
      st4(out + i, make_float4(apply1<BWD>(v.x, d.x, row, ca, cb, cq, K), apply1<BWD>(v.y, d.y, row, ca, cb, cq, K),
                               apply1<BWD>(v.z, d.z, row, ca, cb, cq, K), apply1<BWD>(v.w, d.w, row, ca, cb, cq, K)));
    } else {
      const unsigned row = e / (unsigned)g.HW;
      st1(out + e, apply1<BWD>(ld1(x + e), BWD ? ld1(dy + e) : 0.f, row, ca, cb, cq, K));
    }
  }
}

// channels-last: a thread per 4 channels of a pixel
template <bool BWD, class T>
__global__ void __launch_bounds__(kThreads) ldbn_apply_nhwc(const T* __restrict__ x, const T* __restrict__ dy,
                                                            T* __restrict__ out, LdbnGeom g, const float* __restrict__ ca,
                                                            const float* __restrict__ cb, const float* __restrict__ cq,
                                                            const float* __restrict__ K) {
  const unsigned C4 = (unsigned)g.C / 4, per_img = (unsigned)g.HW * C4;
  const unsigned total = (unsigned)g.N * per_img;
  for (unsigned e = blockIdx.x * kThreads + threadIdx.x; e < total; e += gridDim.x * kThreads) {
    const unsigned n = e / per_img, c = 4 * (e % C4), o = n * (unsigned)g.C + c;
    const float4 v = ld4(x + 4 * (size_t)e), d = BWD ? ld4(dy + 4 * (size_t)e) : float4{};
    st4(out + 4 * (size_t)e, make_float4(apply1<BWD>(v.x, d.x, o, ca, cb, cq, K), apply1<BWD>(v.y, d.y, o + 1, ca, cb, cq, K),
                                         apply1<BWD>(v.z, d.z, o + 2, ca, cb, cq, K),
                                         apply1<BWD>(v.w, d.w, o + 3, ca, cb, cq, K)));
  }
}

int sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess
        || n <= 0)
      n = 132;
  }
  return n;
}

int ew_blocks(size_t work) {
  const size_t want = (work + kThreads - 1) / kThreads, cap = (size_t)sms() * 16;
  return (int)(want < cap ? (want < 1 ? 1 : want) : cap);
}

template <bool BWD, class T>
void reduce(const void* x, const void* dy, const LdbnGeom& g, const float* centre, float* pa, float* pb, float* pilot,
            cudaStream_t st) {
  const T* xt = static_cast<const T*>(x);
  const T* dt = static_cast<const T*>(dy);
  if (g.nhwc) {
    const int slabs = (g.C / 4 + g.qc - 1) / g.qc;
    ldbn_reduce_nhwc<BWD, T><<<(unsigned)((size_t)slabs * g.S * g.N), kThreads, 0, st>>>(xt, dt, g, centre, pa, pb, pilot);
  } else {
    const size_t warps = (size_t)g.N * g.C * g.S;
    const unsigned blocks = (unsigned)((warps + kWarps - 1) / kWarps);
    if (g.HW % 4 == 0) ldbn_reduce_nchw<BWD, true, T><<<blocks, kThreads, 0, st>>>(xt, dt, g, centre, pa, pb, pilot);
    else ldbn_reduce_nchw<BWD, false, T><<<blocks, kThreads, 0, st>>>(xt, dt, g, centre, pa, pb, pilot);
  }
}

template <bool BWD, class T>
void apply(const void* x, const void* dy, void* out, const LdbnGeom& g, const float* ca, const float* cb, const float* cq,
           const float* K, cudaStream_t st) {
  const T* xt = static_cast<const T*>(x);
  const T* dt = static_cast<const T*>(dy);
  T* ot = static_cast<T*>(out);
  const size_t n = (size_t)g.N * g.C * g.HW;
  if (g.nhwc) ldbn_apply_nhwc<BWD, T><<<ew_blocks(n / 4), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K);
  else if (g.HW % 4 == 0) ldbn_apply_nchw<BWD, true, T><<<ew_blocks(n / 4), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K);
  else ldbn_apply_nchw<BWD, false, T><<<ew_blocks(n), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K);
}

}  // namespace

LdbnGeom ldbn_plan(int N, int C, int HW, int D, bool nhwc, bool bf16) {
  LdbnGeom g{};
  g.N = N; g.C = C; g.HW = HW; g.D = D; g.nhwc = nhwc; g.bf16 = bf16;
  auto cdiv = [](long long a, long long b) { return (a + b - 1) / b; };
  long long S;
  if (nhwc) {
    const int C4 = C / 4;
    g.qc = C4 < 64 ? C4 : 64;
    g.pr = kThreads / g.qc;
    const long long ctas = (long long)N * cdiv(C4, g.qc), want = 8LL * sms();
    S = cdiv(want, ctas);
    const long long cap = cdiv(HW, 4LL * g.pr);              // at least 4 pixels per thread and segment
    if (S > cap) S = cap;
    if (S < 1) S = 1;
    g.P = (int)cdiv(HW, S);
  } else {
    g.qc = g.pr = 0;
    const long long rows = (long long)N * C, want = 64LL * sms();   // one full load of warps
    S = cdiv(want, rows);
    const long long cap = cdiv(HW, 256);                      // at least 256 pixels per warp and segment
    if (S > cap) S = cap;
    if (S < 1) S = 1;
    g.P = (int)(cdiv(cdiv(HW, S), 4) * 4);                   // whole float4s
  }
  g.S = (int)cdiv(HW, g.P);
  return g;
}

size_t ldbn_scratch_floats(const LdbnGeom& g, size_t* part, size_t* nc, size_t* dw) {
  *part = (size_t)g.N * g.S * g.C;
  *nc = (size_t)g.N * g.C;
  *dw = (size_t)g.N * g.D * ldbn_finalize_ctas(g.C);
  return 2 * *part + 4 * *nc + *dw;
}

int ldbn_finalize_ctas(int C) { return (C + 31) / 32; }

void ldbn_stats(const void* x, const LdbnGeom& g, float* pa, float* pb, float* pilot, cudaStream_t st) {
  if (g.bf16) reduce<false, __nv_bfloat16>(x, nullptr, g, nullptr, pa, pb, pilot, st);
  else reduce<false, float>(x, nullptr, g, nullptr, pa, pb, pilot, st);
}

void ldbn_fwd_finalize(const LdbnFin& f, const float* pa, const float* pb, const float* pilot, float* alpha, float* shift,
                       cudaStream_t st) {
  ldbn_fwd_finalize<<<ldbn_finalize_ctas(f.C), kThreads, 0, st>>>(f, pa, pb, pilot, alpha, shift);
}

void ldbn_apply(const void* x, void* y, const LdbnGeom& g, const float* alpha, const float* shift, cudaStream_t st) {
  if (g.bf16) apply<false, __nv_bfloat16>(x, nullptr, y, g, alpha, shift, nullptr, nullptr, st);
  else apply<false, float>(x, nullptr, y, g, alpha, shift, nullptr, nullptr, st);
}

void ldbn_bwd_reduce(const void* x, const void* dy, const LdbnGeom& g, const float* centre, float* pa, float* pb,
                     cudaStream_t st) {
  if (g.bf16) reduce<true, __nv_bfloat16>(x, dy, g, centre, pa, pb, nullptr, st);
  else reduce<true, float>(x, dy, g, centre, pa, pb, nullptr, st);
}

void ldbn_bwd_finalize(const LdbnFin& f, const float* pa, const float* pb, float* ca, float* cp, float* cq, float* dwpart,
                       float* dweights, cudaStream_t st) {
  const int nblk = ldbn_finalize_ctas(f.C);
  ldbn_bwd_finalize<<<nblk, kThreads, 0, st>>>(f, pa, pb, ca, cp, cq, dweights ? dwpart : nullptr);
  if (dweights) {
    const int nd = f.N * f.D;
    ldbn_dw<<<(nd + kThreads - 1) / kThreads, kThreads, 0, st>>>(dwpart, nd, nblk, dweights);
  }
}

void ldbn_bwd_apply(const void* x, const void* dy, void* dx, const LdbnGeom& g, const float* ca, const float* cp,
                    const float* cq, const float* centre, cudaStream_t st) {
  if (g.bf16) apply<true, __nv_bfloat16>(x, dy, dx, g, ca, cp, cq, centre, st);
  else apply<true, float>(x, dy, dx, g, ca, cp, cq, centre, st);
}

}  // namespace dwt

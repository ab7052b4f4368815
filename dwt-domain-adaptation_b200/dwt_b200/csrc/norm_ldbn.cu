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
//
// Latent-domain whitening at group sizes 1, 2, 4 (dwt_whiten_latent_small_*, the lds_* kernels below) runs on the same
// plan and passes, a group of GS channels in place of one channel.
#include <type_traits>

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

// Site epilogue E (DWT_EPI_* bits; 0: the plain layer).  RC: the backward recomputes the ReLU mask from x (a ReLU
// without a residual); MK: the channels-last residual's byte map.
template <int E> constexpr bool kEpiRc = (E & DWT_EPI_RELU) && !(E & DWT_EPI_RESIDUAL);
template <int E> constexpr bool kEpiMk = (E & DWT_EPI_RESIDUAL) != 0;

// ReLU as torch.relu and its gradient as threshold_backward: a NaN pre-activation stays NaN and passes its gradient,
// so a bad image's NaN (the layers' edge rules) survives the site
__device__ __forceinline__ bool relu_pass(float z) { return !(z <= 0.f); }

// the forward's output of a site: z (+ r), bit k of bits = relu_pass(that), then the ReLU
template <int E>
__device__ __forceinline__ float site_out(float z, float r, unsigned& bits, int k) {
  if (E & DWT_EPI_RESIDUAL) {
    z += r;
    bits |= (relu_pass(z) ? 1u : 0u) << k;
  }
  return (E & DWT_EPI_RELU) ? (z != z ? z : fmaxf(z, 0.f)) : z;
}

// batch norm: the forward's apply coefficients of (image, channel) o, channel c -- alpha = gamma a_n, shift = gamma b_n +
// beta, the finalize's arithmetic, so a recomputed pre-activation is the forward's bit for bit
__device__ __forceinline__ float2 ldbn_fwd_coef(const LdEpi& ep, size_t o, int c) {
  const float gam = __ldg(ep.gamma + c);
  return make_float2(gam * __ldg(ep.p0 + o), fmaf(gam, __ldg(ep.p1 + o), __ldg(ep.beta + c)));
}
__device__ __forceinline__ float relu_dy(float x, float dy, float2 k) { return relu_pass(fmaf(k.x, x, k.y)) ? dy : 0.f; }
__device__ __forceinline__ float bit_dy(unsigned bits, int k, float dy) { return (bits >> k) & 1u ? dy : 0.f; }

// NCHW reduction: a warp per (row, segment).  VEC: HW % 4 == 0, segments of whole float4s.
template <bool BWD, bool VEC, class T, int E = 0>
__global__ void __launch_bounds__(kThreads) ldbn_reduce_nchw(const T* __restrict__ x, const T* __restrict__ dy,
                                                             LdbnGeom g, const float* __restrict__ centre,
                                                             float* __restrict__ pa, float* __restrict__ pb,
                                                             float* __restrict__ pilot, LdEpi ep) {
  static_assert(!kEpiMk<E>, "an NCHW residual's backward runs on dz without the epilogue");
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
  if constexpr (kEpiRc<E>) {
    const float2 k = ldbn_fwd_coef(ep, (size_t)row, (int)(row % g.C));
    if (VEC) {
#pragma unroll 4
      for (int p = p0 + 4 * lane; p < p1; p += 128) {
        const float4 v = ld4(x + base + p), d = ld4(dy + base + p);
        acc4<BWD>(a, v, make_float4(relu_dy(v.x, d.x, k), relu_dy(v.y, d.y, k), relu_dy(v.z, d.z, k),
                                    relu_dy(v.w, d.w, k)), K);
      }
    } else {
#pragma unroll 4
      for (int p = p0 + lane; p < p1; p += 32) {
        const float v = ld1(x + base + p);
        acc1<BWD>(a, v, relu_dy(v, ld1(dy + base + p), k), K);
      }
    }
  } else if (VEC) {
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
// order through shared memory.  MK: dy masked by the byte map, written to ep.dz.
template <bool BWD, class T, int E = 0>
__global__ void __launch_bounds__(kThreads) ldbn_reduce_nhwc(const T* __restrict__ x, const T* __restrict__ dy,
                                                             LdbnGeom g, const float* __restrict__ centre,
                                                             float* __restrict__ pa, float* __restrict__ pb,
                                                             float* __restrict__ pilot, LdEpi ep) {
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
    if constexpr (kEpiRc<E> || kEpiMk<E>) {
      float2 k[4];
      if constexpr (kEpiRc<E>) {
#pragma unroll
        for (int j = 0; j < 4; ++j) k[j] = ldbn_fwd_coef(ep, (size_t)n * g.C + 4 * c4 + j, 4 * c4 + j);
      }
      const unsigned C4 = (unsigned)g.C / 4;
#pragma unroll 4
      for (int p = p0 + r; p < p1; p += g.pr) {
        const float4 v = ld4(x + img + (size_t)p * g.C);
        float4 d = ld4(dy + img + (size_t)p * g.C);
        if constexpr (kEpiMk<E>) {
          const unsigned bits = __ldg(ep.mask + ((size_t)n * g.HW + p) * C4 + c4);
          d = make_float4(bit_dy(bits, 0, d.x), bit_dy(bits, 1, d.y), bit_dy(bits, 2, d.z), bit_dy(bits, 3, d.w));
          st4(static_cast<T*>(ep.dz) + img + (size_t)p * g.C, d);
        } else {
          d = make_float4(relu_dy(v.x, d.x, k[0]), relu_dy(v.y, d.y, k[1]), relu_dy(v.z, d.z, k[2]),
                          relu_dy(v.w, d.w, k[3]));
        }
        acc1<BWD>(ax, v.x, d.x, K.x); acc1<BWD>(ay, v.y, d.y, K.y);
        acc1<BWD>(az, v.z, d.z, K.z); acc1<BWD>(aw, v.w, d.w, K.w);
      }
    } else {
#pragma unroll 4
    for (int p = p0 + r; p < p1; p += g.pr) {
      const float4 v = ld4(x + img + (size_t)p * g.C);
      const float4 d = BWD ? ld4(dy + img + (size_t)p * g.C) : float4{};
      acc1<BWD>(ax, v.x, d.x, K.x); acc1<BWD>(ay, v.y, d.y, K.y);
      acc1<BWD>(az, v.z, d.z, K.z); acc1<BWD>(aw, v.w, d.w, K.w);
    }
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

// NCHW: VEC -- a thread per 4 pixels of a row (HW % 4 == 0); else a thread per element.  E: forward the site's residual
// and ReLU on the output, backward (RC) dy masked by the recomputed pre-activation.
template <bool BWD, bool VEC, class T, int E = 0>
__global__ void __launch_bounds__(kThreads) ldbn_apply_nchw(const T* __restrict__ x, const T* __restrict__ dy,
                                                            T* __restrict__ out, LdbnGeom g, const float* __restrict__ ca,
                                                            const float* __restrict__ cb, const float* __restrict__ cq,
                                                            const float* __restrict__ K, LdEpi ep) {
  static_assert(!BWD || !kEpiMk<E>, "a residual's backward apply reads dz without the epilogue");
  const unsigned total = (unsigned)((size_t)g.N * g.C * g.HW / (VEC ? 4 : 1));
  for (unsigned e = blockIdx.x * kThreads + threadIdx.x; e < total; e += gridDim.x * kThreads) {
    if constexpr (E != 0) {
      const T* res = static_cast<const T*>(ep.res);
      unsigned bits = 0;
      if (VEC) {
        const unsigned i = 4 * e, row = i / (unsigned)g.HW;
        const float4 v = ld4(x + i);
        float4 d = BWD ? ld4(dy + i) : float4{};
        if constexpr (BWD) {
          const float2 k = ldbn_fwd_coef(ep, row, (int)(row % (unsigned)g.C));
          d = make_float4(relu_dy(v.x, d.x, k), relu_dy(v.y, d.y, k), relu_dy(v.z, d.z, k), relu_dy(v.w, d.w, k));
          st4(out + i, make_float4(apply1<true>(v.x, d.x, row, ca, cb, cq, K), apply1<true>(v.y, d.y, row, ca, cb, cq, K),
                                   apply1<true>(v.z, d.z, row, ca, cb, cq, K), apply1<true>(v.w, d.w, row, ca, cb, cq, K)));
        } else {
          const float4 rv = kEpiMk<E> ? ld4(res + i) : float4{};
          st4(out + i, make_float4(site_out<E>(apply1<false>(v.x, 0.f, row, ca, cb, cq, K), rv.x, bits, 0),
                                   site_out<E>(apply1<false>(v.y, 0.f, row, ca, cb, cq, K), rv.y, bits, 1),
                                   site_out<E>(apply1<false>(v.z, 0.f, row, ca, cb, cq, K), rv.z, bits, 2),
                                   site_out<E>(apply1<false>(v.w, 0.f, row, ca, cb, cq, K), rv.w, bits, 3)));
        }
      } else {
        const unsigned row = e / (unsigned)g.HW;
        const float v = ld1(x + e);
        if constexpr (BWD) {
          const float d = relu_dy(v, ld1(dy + e), ldbn_fwd_coef(ep, row, (int)(row % (unsigned)g.C)));
          st1(out + e, apply1<true>(v, d, row, ca, cb, cq, K));
        } else {
          st1(out + e, site_out<E>(apply1<false>(v, 0.f, row, ca, cb, cq, K), kEpiMk<E> ? ld1(res + e) : 0.f, bits, 0));
        }
      }
    } else if (VEC) {
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

// channels-last: a thread per 4 channels of a pixel.  E as ldbn_apply_nchw; a residual's forward writes the byte map.
template <bool BWD, class T, int E = 0>
__global__ void __launch_bounds__(kThreads) ldbn_apply_nhwc(const T* __restrict__ x, const T* __restrict__ dy,
                                                            T* __restrict__ out, LdbnGeom g, const float* __restrict__ ca,
                                                            const float* __restrict__ cb, const float* __restrict__ cq,
                                                            const float* __restrict__ K, LdEpi ep) {
  static_assert(!BWD || !kEpiMk<E>, "a residual's backward apply reads dz without the epilogue");
  const unsigned C4 = (unsigned)g.C / 4, per_img = (unsigned)g.HW * C4;
  const unsigned total = (unsigned)g.N * per_img;
  for (unsigned e = blockIdx.x * kThreads + threadIdx.x; e < total; e += gridDim.x * kThreads) {
    const unsigned n = e / per_img, c = 4 * (e % C4), o = n * (unsigned)g.C + c;
    if constexpr (E != 0) {
      const float4 v = ld4(x + 4 * (size_t)e);
      if constexpr (BWD) {
        float4 d = ld4(dy + 4 * (size_t)e);
        d = make_float4(relu_dy(v.x, d.x, ldbn_fwd_coef(ep, o, c)), relu_dy(v.y, d.y, ldbn_fwd_coef(ep, o + 1, c + 1)),
                        relu_dy(v.z, d.z, ldbn_fwd_coef(ep, o + 2, c + 2)),
                        relu_dy(v.w, d.w, ldbn_fwd_coef(ep, o + 3, c + 3)));
        st4(out + 4 * (size_t)e, make_float4(apply1<true>(v.x, d.x, o, ca, cb, cq, K),
                                             apply1<true>(v.y, d.y, o + 1, ca, cb, cq, K),
                                             apply1<true>(v.z, d.z, o + 2, ca, cb, cq, K),
                                             apply1<true>(v.w, d.w, o + 3, ca, cb, cq, K)));
      } else {
        const float4 rv = kEpiMk<E> ? ld4(static_cast<const T*>(ep.res) + 4 * (size_t)e) : float4{};
        unsigned bits = 0;
        st4(out + 4 * (size_t)e, make_float4(site_out<E>(apply1<false>(v.x, 0.f, o, ca, cb, cq, K), rv.x, bits, 0),
                                             site_out<E>(apply1<false>(v.y, 0.f, o + 1, ca, cb, cq, K), rv.y, bits, 1),
                                             site_out<E>(apply1<false>(v.z, 0.f, o + 2, ca, cb, cq, K), rv.z, bits, 2),
                                             site_out<E>(apply1<false>(v.w, 0.f, o + 3, ca, cb, cq, K), rv.w, bits, 3)));
        if constexpr (kEpiMk<E>) ep.mask[e] = (uint8_t)bits;
      }
      continue;
    }
    const float4 v = ld4(x + 4 * (size_t)e), d = BWD ? ld4(dy + 4 * (size_t)e) : float4{};
    st4(out + 4 * (size_t)e, make_float4(apply1<BWD>(v.x, d.x, o, ca, cb, cq, K), apply1<BWD>(v.y, d.y, o + 1, ca, cb, cq, K),
                                         apply1<BWD>(v.z, d.z, o + 2, ca, cb, cq, K),
                                         apply1<BWD>(v.w, d.w, o + 3, ca, cb, cq, K)));
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// Latent-domain whitening at group sizes 1, 2, 4 (dwt_whiten_latent_small_*): the same four bandwidth passes on the same
// segments, a group of GS channels in place of one channel.  The reductions keep per group the GS sums and the
// GS(GS+1)/2 lower cross-products about the pilot (forward), or g_n = sum dy and the full R_n = sum dy (x - m_n)^T
// (backward); the apply passes hold their group's coefficients in registers for a whole segment.  The finalize
// kernels give every (image, group) its own thread and every (domain, group) its own warp (a domain's 14 forward and 20
// backward fp64 sums at GS 4 do not fit LDBN's per-lane layout, and one thread walking every image is latency-bound);
// all sums run in a fixed order, the domain moments in fp64 about image 0's mean.
// ------------------------------------------------------------------------------------------------------------------------
template <int GS> struct LdsDim {
  static constexpr int T = GS * (GS + 1) / 2;            // lower triangle
  static constexpr int NF = GS + T;                      // forward partial: sums | lower cross-products
  static constexpr int NB = GS + GS * GS;                // backward partial: g | R row-major
  static constexpr int REC = GS * GS + GS;               // a save_stats record: (cov, mean)
  static constexpr int NCF = T + GS;                     // forward apply: A lower | -A m~
  static constexpr int NCB = T + GS * GS + 2 * GS;       // backward apply: A lower | B | c | m
  static constexpr int PER4 = 4 / GS;                    // whole groups in a float4 of channels
};

// NCHW: four float4 loads of x in flight per lane and iteration, as ldbn_reduce_nchw's unrolled loop
template <int GS> constexpr int kLdsVecUnroll = 4 / GS;

__device__ __forceinline__ float lane4(const float4& v, int e) { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }

// one pixel of one group into its partials at a[o..]: forward d = x - K, the sums of d_i, then d_i d_j (j <= i) row by
// row; backward d = x - K (K: the image mean), the sums of dy_i, then dy_i d_j row-major
template <int GS, bool BWD, int NA>
__device__ __forceinline__ void lds_acc(float (&a)[NA], int o, const float (&x)[GS], const float (&dy)[GS],
                                        const float (&K)[GS]) {
  float d[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) d[i] = x[i] - K[i];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    if (BWD) {
      a[o + i] += dy[i];
#pragma unroll
      for (int j = 0; j < GS; ++j) a[o + GS + i * GS + j] = fmaf(dy[i], d[j], a[o + GS + i * GS + j]);
    } else {
      a[o + i] += d[i];
#pragma unroll
      for (int j = 0; j <= i; ++j) a[o + GS + i * (i + 1) / 2 + j] = fmaf(d[i], d[j], a[o + GS + i * (i + 1) / 2 + j]);
    }
  }
}

// a group's apply coefficients into cf[o..]: forward A_n's lower triangle and bp = -A_n m~_n; backward the finalize's
// A_n lower | B_n | c_n | m_n.  gi = n G + group.
template <int GS, bool BWD, int NC>
__device__ __forceinline__ void lds_load(float (&cf)[NC], int o, size_t gi, const float* save_mean, const float* save_w,
                                         const float* coef) {
  using Dm = LdsDim<GS>;
  if (BWD) {
#pragma unroll
    for (int k = 0; k < Dm::NCB; ++k) cf[o + k] = __ldg(coef + gi * Dm::NCB + k);
  } else {
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      float b = 0.f;
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const float w = __ldg(save_w + gi * GS * GS + i * GS + j);
        b = fmaf(-w, __ldg(save_mean + gi * GS + j), b);
        cf[o + i * (i + 1) / 2 + j] = w;
      }
      cf[o + Dm::T + i] = b;
    }
  }
}

// a site's forward coefficients: lds_load's with diag(gamma) folded into A_n's rows and beta into the bias (c0: the
// group's first channel).  The forward apply and both backward passes load them here, so a recomputed pre-activation
// is the forward's bit for bit.
template <int GS, int NC>
__device__ __forceinline__ void lds_site_load(float (&cf)[NC], int o, size_t gi, int c0, const LdEpi& ep) {
  lds_load<GS, false>(cf, o, gi, ep.p0, ep.p1, nullptr);
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    const float gam = __ldg(ep.gamma + c0 + i);
#pragma unroll
    for (int j = 0; j <= i; ++j) cf[o + i * (i + 1) / 2 + j] *= gam;
    cf[o + LdsDim<GS>::T + i] = fmaf(gam, cf[o + LdsDim<GS>::T + i], __ldg(ep.beta + c0 + i));
  }
}

// forward y_i = bp_i + sum_{j<=i} A_ij x_j;  backward dx_i = c_i + sum_j B_ij (x_j - m_j) + sum_{j>=i} A_ji dy_j
template <int GS, bool BWD, int NC>
__device__ __forceinline__ void lds_map(const float (&cf)[NC], int o, const float (&x)[GS], const float (&dy)[GS],
                                        float (&out)[GS]) {
  constexpr int T = LdsDim<GS>::T;
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    float acc;
    if (BWD) {
      acc = cf[o + T + GS * GS + i];
#pragma unroll
      for (int j = 0; j < GS; ++j) acc = fmaf(cf[o + T + i * GS + j], x[j] - cf[o + T + GS * GS + GS + j], acc);
#pragma unroll
      for (int j = i; j < GS; ++j) acc = fmaf(cf[o + j * (j + 1) / 2 + i], dy[j], acc);
    } else {
      acc = cf[o + T + i];
#pragma unroll
      for (int j = 0; j <= i; ++j) acc = fmaf(cf[o + i * (i + 1) / 2 + j], x[j], acc);
    }
    out[i] = acc;
  }
}

// a site's ReLU mask recomputed on one pixel of a group: dy_i = 0 where the forward's pre-activation is <= 0
template <int GS, int NC>
__device__ __forceinline__ void lds_relu_dy(const float (&fc)[NC], int o, const float (&x)[GS], float (&dy)[GS]) {
  float z[GS];
  lds_map<GS, false>(fc, o, x, dy, z);
#pragma unroll
  for (int i = 0; i < GS; ++i) dy[i] = relu_pass(z[i]) ? dy[i] : 0.f;
}

// NCHW reduction: a warp per (image, group, segment) over the group's GS rows.  VEC: HW % 4 == 0.  stats: save_stats
// (backward: the image means are the centre).  E (backward): RC masks dy by the recomputed pre-activation.
template <int GS, bool BWD, bool VEC, class T, int E = 0>
__global__ void __launch_bounds__(kThreads, 1) lds_reduce_nchw(const T* __restrict__ x, const T* __restrict__ dy, LdbnGeom g,
                                                            const float* __restrict__ stats, float* __restrict__ part,
                                                            float* __restrict__ pilot, LdEpi ep) {
  static_assert(!kEpiMk<E>, "an NCHW residual's backward runs on dz without the epilogue");
  using Dm = LdsDim<GS>;
  constexpr int NA = BWD ? Dm::NB : Dm::NF;
  const long long wid = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int G = g.C / GS;
  const long long rows = (long long)g.N * G;
  if (wid >= rows * g.S) return;
  const long long row = wid / g.S;                       // n G + group
  const int s = (int)(wid - row * g.S);
  const size_t base = (size_t)row * GS * g.HW;
  float K[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) K[i] = BWD ? stats[row * Dm::REC + GS * GS + i] : ld1(x + base + (size_t)i * g.HW);
  const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
  float a[NA];
#pragma unroll
  for (int k = 0; k < NA; ++k) a[k] = 0.f;
  float fc[kEpiRc<E> ? Dm::NCF : 1];
  if constexpr (kEpiRc<E>) lds_site_load<GS>(fc, 0, (size_t)row, (int)(row % G) * GS, ep);
  float xv[GS], dv[GS];
  if (VEC) {
#pragma unroll kLdsVecUnroll<GS>
    for (int p = p0 + 4 * lane; p < p1; p += 128) {
      float4 v[GS], d[GS];
#pragma unroll
      for (int i = 0; i < GS; ++i) {
        v[i] = ld4(x + base + (size_t)i * g.HW + p);
        d[i] = BWD ? ld4(dy + base + (size_t)i * g.HW + p) : float4{};
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
#pragma unroll
        for (int i = 0; i < GS; ++i) { xv[i] = lane4(v[i], e); dv[i] = lane4(d[i], e); }
        if constexpr (kEpiRc<E>) lds_relu_dy<GS>(fc, 0, xv, dv);
        lds_acc<GS, BWD>(a, 0, xv, dv, K);
      }
    }
  } else {
#pragma unroll 4
    for (int p = p0 + lane; p < p1; p += 32) {
#pragma unroll
      for (int i = 0; i < GS; ++i) {
        xv[i] = ld1(x + base + (size_t)i * g.HW + p);
        dv[i] = BWD ? ld1(dy + base + (size_t)i * g.HW + p) : 0.f;
      }
      if constexpr (kEpiRc<E>) lds_relu_dy<GS>(fc, 0, xv, dv);
      lds_acc<GS, BWD>(a, 0, xv, dv, K);
    }
  }
#pragma unroll
  for (int k = 0; k < NA; ++k) a[k] = warp_sum(a[k]);
  if (lane == 0) {
    const long long n = row / G;
    float* o = part + (((size_t)n * g.S + s) * G + (size_t)(row - n * G)) * NA;
#pragma unroll
    for (int k = 0; k < NA; ++k) o[k] = a[k];
    if (!BWD && s == 0) {
#pragma unroll
      for (int i = 0; i < GS; ++i) pilot[row * GS + i] = K[i];
    }
  }
}

// channels-last reduction: ldbn_reduce_nhwc's CTA (slab, segment, image); a thread's 4 channels are 4/GS groups, the
// pixel rows added in order through shared memory.  E (backward): RC as lds_reduce_nchw; MK masks dy by the byte map and
// writes it to ep.dz.
template <int GS, bool BWD, class T, int E = 0>
__global__ void __launch_bounds__(kThreads, 1) lds_reduce_nhwc(const T* __restrict__ x, const T* __restrict__ dy, LdbnGeom g,
                                                            const float* __restrict__ stats, float* __restrict__ part,
                                                            float* __restrict__ pilot, LdEpi ep) {
  using Dm = LdsDim<GS>;
  constexpr int NA = BWD ? Dm::NB : Dm::NF, NV = Dm::PER4 * NA;
  __shared__ float sm[NV * kThreads];
  const int slabs = (g.C / 4 + g.qc - 1) / g.qc;
  int b = blockIdx.x;
  const int slab = b % slabs; b /= slabs;
  const int s = b % g.S;
  const int n = b / g.S;
  const int q = threadIdx.x % g.qc, r = threadIdx.x / g.qc;
  const int c4 = slab * g.qc + q;
  const int G = g.C / GS;
  const bool on = r < g.pr && c4 < g.C / 4;
  float a[NV];
#pragma unroll
  for (int k = 0; k < NV; ++k) a[k] = 0.f;
  if (on) {
    const size_t img = (size_t)n * g.HW * g.C + 4 * c4;
    float K[4];
    if (BWD) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ch = 4 * c4 + j;
        K[j] = stats[((size_t)n * G + ch / GS) * Dm::REC + GS * GS + ch % GS];
      }
    } else {
      const float4 k = ld4(x + img);
      K[0] = k.x; K[1] = k.y; K[2] = k.z; K[3] = k.w;
    }
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
    float fc[kEpiRc<E> ? Dm::PER4 * Dm::NCF : 1];
    if constexpr (kEpiRc<E>) {
#pragma unroll
      for (int t = 0; t < Dm::PER4; ++t)
        lds_site_load<GS>(fc, t * Dm::NCF, (size_t)n * G + 4 * c4 / GS + t, 4 * c4 + t * GS, ep);
    }
#pragma unroll 4
    for (int p = p0 + r; p < p1; p += g.pr) {
      const float4 v = ld4(x + img + (size_t)p * g.C);
      float4 d = BWD ? ld4(dy + img + (size_t)p * g.C) : float4{};
      if constexpr (kEpiMk<E>) {
        const unsigned bits = __ldg(ep.mask + ((size_t)n * g.HW + p) * (g.C / 4) + c4);
        d = make_float4(bit_dy(bits, 0, d.x), bit_dy(bits, 1, d.y), bit_dy(bits, 2, d.z), bit_dy(bits, 3, d.w));
        st4(static_cast<T*>(ep.dz) + img + (size_t)p * g.C, d);
      }
#pragma unroll
      for (int t = 0; t < Dm::PER4; ++t) {
        float xv[GS], dv[GS], kv[GS];
#pragma unroll
        for (int i = 0; i < GS; ++i) { xv[i] = lane4(v, t * GS + i); dv[i] = lane4(d, t * GS + i); kv[i] = K[t * GS + i]; }
        if constexpr (kEpiRc<E>) lds_relu_dy<GS>(fc, t * Dm::NCF, xv, dv);
        lds_acc<GS, BWD>(a, t * NA, xv, dv, kv);
      }
    }
    if (!BWD && s == 0 && r == 0)
      *reinterpret_cast<float4*>(pilot + (size_t)n * g.C + 4 * c4) = make_float4(K[0], K[1], K[2], K[3]);
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) sm[k * kThreads + threadIdx.x] = a[k];
  __syncthreads();
  if (on && r == 0) {
    for (int rr = 1; rr < g.pr; ++rr)
#pragma unroll
      for (int k = 0; k < NV; ++k) a[k] += sm[k * kThreads + rr * g.qc + q];
    float* o = part + (((size_t)n * g.S + s) * G + 4 * c4 / GS) * NA;
#pragma unroll
    for (int k = 0; k < NV; ++k) o[k] = a[k];
  }
}

// A site pixel of one group in the apply passes.  Forward: the folded map, the residual r and the ReLU (bit t GS + i of
// bits: out > 0).  Backward: dy masked by the recomputed pre-activation (RC), times gamma, through the backward map.
template <int GS, bool BWD, int E, int NC, int NF>
__device__ __forceinline__ void lds_site_px(const float (&cf)[NC], const float (&fc)[NF], int o, int of, const float (&gam)[4],
                                            int t, const float (&x)[GS], float (&dy)[GS], const float* r, float (&out)[GS],
                                            unsigned& bits) {
  if constexpr (BWD) {
    if constexpr (kEpiRc<E>) lds_relu_dy<GS>(fc, of, x, dy);
#pragma unroll
    for (int i = 0; i < GS; ++i) dy[i] *= gam[t * GS + i];
    lds_map<GS, true>(cf, o, x, dy, out);
  } else {
    lds_map<GS, false>(cf, o, x, dy, out);
#pragma unroll
    for (int i = 0; i < GS; ++i) out[i] = site_out<E>(out[i], r[i], bits, t * GS + i);
  }
}

// NCHW apply: the reduction's warps, the group's coefficients held for the segment.  E: a site (lds_site_px; an NCHW
// residual's forward reads it, no byte map).
template <int GS, bool BWD, bool VEC, class T, int E = 0>
__global__ void __launch_bounds__(kThreads, 1) lds_apply_nchw(const T* __restrict__ x, const T* __restrict__ dy,
                                                           T* __restrict__ out, LdbnGeom g, const float* __restrict__ save_mean,
                                                           const float* __restrict__ save_w, const float* __restrict__ coef,
                                                           LdEpi ep) {
  using Dm = LdsDim<GS>;
  constexpr int NC = BWD ? Dm::NCB : Dm::NCF;
  const long long wid = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long rows = (long long)g.N * (g.C / GS);
  if (wid >= rows * g.S) return;
  const long long row = wid / g.S;
  const int s = (int)(wid - row * g.S);
  const size_t base = (size_t)row * GS * g.HW;
  float cf[NC];
  if constexpr (E != 0) {
    static_assert((E & DWT_EPI_AFFINE) && !(BWD && kEpiMk<E>), "a site has AFFINE; a residual's backward reads dz");
    const int c0 = (int)(row % (g.C / GS)) * GS;
    float fc[BWD && kEpiRc<E> ? Dm::NCF : 1], gam[4] = {1.f, 1.f, 1.f, 1.f};
    if constexpr (BWD) {
      lds_load<GS, true>(cf, 0, (size_t)row, save_mean, save_w, coef);
      if constexpr (kEpiRc<E>) lds_site_load<GS>(fc, 0, (size_t)row, c0, ep);
#pragma unroll
      for (int i = 0; i < GS; ++i) gam[i] = __ldg(ep.gamma + c0 + i);
    } else {
      lds_site_load<GS>(cf, 0, (size_t)row, c0, ep);
    }
    const T* res = static_cast<const T*>(ep.res);
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
    float xv[GS], dv[GS], rv[GS], ov[GS];
    unsigned bits = 0;
#pragma unroll
    for (int i = 0; i < GS; ++i) rv[i] = 0.f;
    if (VEC) {
#pragma unroll kLdsVecUnroll<GS>
      for (int p = p0 + 4 * lane; p < p1; p += 128) {
        float4 v[GS], d[GS], r4[GS];
        float o4[GS][4];
#pragma unroll
        for (int i = 0; i < GS; ++i) {
          v[i] = ld4(x + base + (size_t)i * g.HW + p);
          d[i] = BWD ? ld4(dy + base + (size_t)i * g.HW + p) : float4{};
          r4[i] = (!BWD && kEpiMk<E>) ? ld4(res + base + (size_t)i * g.HW + p) : float4{};
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
#pragma unroll
          for (int i = 0; i < GS; ++i) { xv[i] = lane4(v[i], e); dv[i] = lane4(d[i], e); rv[i] = lane4(r4[i], e); }
          lds_site_px<GS, BWD, E>(cf, fc, 0, 0, gam, 0, xv, dv, rv, ov, bits);
#pragma unroll
          for (int i = 0; i < GS; ++i) o4[i][e] = ov[i];
        }
#pragma unroll
        for (int i = 0; i < GS; ++i)
          st4(out + base + (size_t)i * g.HW + p, make_float4(o4[i][0], o4[i][1], o4[i][2], o4[i][3]));
      }
    } else {
#pragma unroll 4
      for (int p = p0 + lane; p < p1; p += 32) {
#pragma unroll
        for (int i = 0; i < GS; ++i) {
          xv[i] = ld1(x + base + (size_t)i * g.HW + p);
          dv[i] = BWD ? ld1(dy + base + (size_t)i * g.HW + p) : 0.f;
          if (!BWD && kEpiMk<E>) rv[i] = ld1(res + base + (size_t)i * g.HW + p);
        }
        lds_site_px<GS, BWD, E>(cf, fc, 0, 0, gam, 0, xv, dv, rv, ov, bits);
#pragma unroll
        for (int i = 0; i < GS; ++i) st1(out + base + (size_t)i * g.HW + p, ov[i]);
      }
    }
  } else {
    lds_load<GS, BWD>(cf, 0, (size_t)row, save_mean, save_w, coef);
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
    float xv[GS], dv[GS], ov[GS];
    if (VEC) {
  #pragma unroll kLdsVecUnroll<GS>
      for (int p = p0 + 4 * lane; p < p1; p += 128) {
        float4 v[GS], d[GS];
        float o4[GS][4];
  #pragma unroll
        for (int i = 0; i < GS; ++i) {
          v[i] = ld4(x + base + (size_t)i * g.HW + p);
          d[i] = BWD ? ld4(dy + base + (size_t)i * g.HW + p) : float4{};
        }
  #pragma unroll
        for (int e = 0; e < 4; ++e) {
  #pragma unroll
          for (int i = 0; i < GS; ++i) { xv[i] = lane4(v[i], e); dv[i] = lane4(d[i], e); }
          lds_map<GS, BWD>(cf, 0, xv, dv, ov);
  #pragma unroll
          for (int i = 0; i < GS; ++i) o4[i][e] = ov[i];
        }
  #pragma unroll
        for (int i = 0; i < GS; ++i)
          st4(out + base + (size_t)i * g.HW + p, make_float4(o4[i][0], o4[i][1], o4[i][2], o4[i][3]));
      }
    } else {
  #pragma unroll 4
      for (int p = p0 + lane; p < p1; p += 32) {
  #pragma unroll
        for (int i = 0; i < GS; ++i) {
          xv[i] = ld1(x + base + (size_t)i * g.HW + p);
          dv[i] = BWD ? ld1(dy + base + (size_t)i * g.HW + p) : 0.f;
        }
        lds_map<GS, BWD>(cf, 0, xv, dv, ov);
  #pragma unroll
        for (int i = 0; i < GS; ++i) st1(out + base + (size_t)i * g.HW + p, ov[i]);
      }
    }
  }
}

// channels-last apply: the reduction's CTAs, a thread's 4/GS groups' coefficients held for the segment.  E: a site
// (lds_site_px); a residual's forward writes the byte map.
template <int GS, bool BWD, class T, int E = 0>
__global__ void __launch_bounds__(kThreads, 1) lds_apply_nhwc(const T* __restrict__ x, const T* __restrict__ dy,
                                                           T* __restrict__ out, LdbnGeom g, const float* __restrict__ save_mean,
                                                           const float* __restrict__ save_w, const float* __restrict__ coef,
                                                           LdEpi ep) {
  using Dm = LdsDim<GS>;
  constexpr int NC = BWD ? Dm::NCB : Dm::NCF;
  const int slabs = (g.C / 4 + g.qc - 1) / g.qc;
  int b = blockIdx.x;
  const int slab = b % slabs; b /= slabs;
  const int s = b % g.S;
  const int n = b / g.S;
  const int q = threadIdx.x % g.qc, r = threadIdx.x / g.qc;
  const int c4 = slab * g.qc + q;
  if (r >= g.pr || c4 >= g.C / 4) return;
  float cf[Dm::PER4 * NC];
  if constexpr (E != 0) {
    static_assert((E & DWT_EPI_AFFINE) && !(BWD && kEpiMk<E>), "a site has AFFINE; a residual's backward reads dz");
    float fc[BWD && kEpiRc<E> ? Dm::PER4 * Dm::NCF : 1], gam[4];
#pragma unroll
    for (int t = 0; t < Dm::PER4; ++t) {
      const size_t gi = (size_t)n * (g.C / GS) + 4 * c4 / GS + t;
      if constexpr (BWD) {
        lds_load<GS, true>(cf, t * NC, gi, save_mean, save_w, coef);
        if constexpr (kEpiRc<E>) lds_site_load<GS>(fc, t * Dm::NCF, gi, 4 * c4 + t * GS, ep);
      } else {
        lds_site_load<GS>(cf, t * NC, gi, 4 * c4 + t * GS, ep);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) gam[j] = BWD ? __ldg(ep.gamma + 4 * c4 + j) : 1.f;
    const size_t img = (size_t)n * g.HW * g.C + 4 * c4;
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
#pragma unroll 4
    for (int p = p0 + r; p < p1; p += g.pr) {
      const size_t at = img + (size_t)p * g.C;
      const float4 v = ld4(x + at);
      const float4 d = BWD ? ld4(dy + at) : float4{};
      const float4 rr = (!BWD && kEpiMk<E>) ? ld4(static_cast<const T*>(ep.res) + at) : float4{};
      float o[4];
      unsigned bits = 0;
#pragma unroll
      for (int t = 0; t < Dm::PER4; ++t) {
        float xv[GS], dv[GS], rv[GS], ov[GS];
#pragma unroll
        for (int i = 0; i < GS; ++i) {
          xv[i] = lane4(v, t * GS + i); dv[i] = lane4(d, t * GS + i); rv[i] = lane4(rr, t * GS + i);
        }
        lds_site_px<GS, BWD, E>(cf, fc, t * NC, t * Dm::NCF, gam, t, xv, dv, rv, ov, bits);
#pragma unroll
        for (int i = 0; i < GS; ++i) o[t * GS + i] = ov[i];
      }
      st4(out + at, make_float4(o[0], o[1], o[2], o[3]));
      if constexpr (!BWD && kEpiMk<E>) ep.mask[at / 4] = (uint8_t)bits;
    }
  } else {
  #pragma unroll
    for (int t = 0; t < Dm::PER4; ++t)
      lds_load<GS, BWD>(cf, t * NC, (size_t)n * (g.C / GS) + 4 * c4 / GS + t, save_mean, save_w, coef);
    const size_t img = (size_t)n * g.HW * g.C + 4 * c4;
    const int p0 = s * g.P, p1 = min(p0 + g.P, g.HW);
  #pragma unroll 4
    for (int p = p0 + r; p < p1; p += g.pr) {
      const float4 v = ld4(x + img + (size_t)p * g.C);
      const float4 d = BWD ? ld4(dy + img + (size_t)p * g.C) : float4{};
      float o[4];
  #pragma unroll
      for (int t = 0; t < Dm::PER4; ++t) {
        float xv[GS], dv[GS], ov[GS];
  #pragma unroll
        for (int i = 0; i < GS; ++i) { xv[i] = lane4(v, t * GS + i); dv[i] = lane4(d, t * GS + i); }
        lds_map<GS, BWD>(cf, t * NC, xv, dv, ov);
  #pragma unroll
        for (int i = 0; i < GS; ++i) o[t * GS + i] = ov[i];
      }
      st4(out + img + (size_t)p * g.C, make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

// save_stats of dwt_whiten_latent_*: [N][G] records (C_n, m_n), [K][G] records (Sigma_k, mu_k), [K][G][GS*GS] W_k, [K] s_k
template <int GS> struct LdsLayout {
  float* base;
  int N, G, K;
  __device__ LdsLayout(const LdsFin& f) : base(f.save_stats), N(f.N), G(f.G), K(f.K) {}
  __device__ float* img(size_t gi) const { return base + gi * LdsDim<GS>::REC; }
  __device__ float* dom(int k, int g) const { return base + ((size_t)(N + k) * G + g) * LdsDim<GS>::REC; }
  __device__ float* w(int k, int g) const { return base + ((size_t)(N + K) * G * LdsDim<GS>::REC) + ((size_t)k * G + g) * GS * GS; }
  __device__ float* mass() const { return base + (size_t)(N + K) * G * LdsDim<GS>::REC + (size_t)K * G * GS * GS; }
};

// per (image, group): the segment partials added in order (fp64) into the image's mean and biased covariance about the
// pilot; save_stats' image record and im (fp64: m | C lower)
template <int GS>
__global__ void __launch_bounds__(kThreads) lds_fwd_image(const LdsFin f, const float* __restrict__ part,
                                                          const float* __restrict__ pilot, double* __restrict__ im) {
  using Dm = LdsDim<GS>;
  const int gi = blockIdx.x * kThreads + threadIdx.x;
  if (gi >= f.N * f.G) return;
  const int n = gi / f.G, grp = gi - n * f.G;
  double s1[GS], s2[Dm::T];
#pragma unroll
  for (int i = 0; i < GS; ++i) s1[i] = 0.0;
#pragma unroll
  for (int t = 0; t < Dm::T; ++t) s2[t] = 0.0;
  for (int j = 0; j < f.S; ++j) {
    const float* p = part + (((size_t)n * f.S + j) * f.G + grp) * Dm::NF;
#pragma unroll
    for (int i = 0; i < GS; ++i) s1[i] += p[i];
#pragma unroll
    for (int t = 0; t < Dm::T; ++t) s2[t] += p[GS + t];
  }
  const LdsLayout<GS> L(f);
  float* rec = L.img(gi);
  double* o = im + (size_t)gi * Dm::NF;
  double dm[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    dm[i] = s1[i] / f.M;
    const double m = (double)pilot[(size_t)gi * GS + i] + dm[i];
    o[i] = m;
    rec[GS * GS + i] = (float)m;
  }
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      const double c = s2[i * (i + 1) / 2 + j] / f.M - dm[i] * dm[j];
      o[GS + i * (i + 1) / 2 + j] = c;
      rec[i * GS + j] = (float)c;
      rec[j * GS + i] = (float)c;
    }
}

// the sum of v over the warp by a fixed butterfly: every lane ends with the same, rerun-identical value
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// a warp per (domain, group): s_k (fp64, lane l takes images l, l + 32, ..., zero weights skipped, the lanes added by
// warp_sum_d); train: mu_k, Sigma_k by the law of total covariance about image 0's mean, eval: the running buffers; then
// lane 0: S_k = a Sigma_k + b I = L L^T, W_k = L^-1 (fp32) and the EMA.  s_k == 0: skipped (no W_k, no status, no EMA);
// s_k < 0 or NaN, non-finite statistics or S_k not positive definite: W_k = NaN, DWT_STATUS_NOT_PD, no EMA.
template <int GS>
__global__ void __launch_bounds__(kThreads) lds_fwd_domain(const LdsFin f, const double* __restrict__ im) {
  using Dm = LdsDim<GS>;
  const int idx = (blockIdx.x * kThreads + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (idx >= f.K * f.G) return;
  const int k = idx / f.G, grp = idx - k * f.G;
  const LdsLayout<GS> L(f);
  double ref[GS], a1[GS], a2[Dm::T], s = 0.0;
#pragma unroll
  for (int i = 0; i < GS; ++i) { ref[i] = im[(size_t)grp * Dm::NF + i]; a1[i] = 0.0; }
#pragma unroll
  for (int t = 0; t < Dm::T; ++t) a2[t] = 0.0;
  for (int n = lane; n < f.N; n += 32) {
    const float w = __ldg(f.weights + (size_t)n * f.K + k);
    if (w == 0.f) continue;
    s += (double)w;
    if (!f.train) continue;
    const double* r = im + ((size_t)n * f.G + grp) * Dm::NF;
    const double dw = (double)w;
    double e[GS];
#pragma unroll
    for (int i = 0; i < GS; ++i) { e[i] = r[i] - ref[i]; a1[i] += dw * e[i]; }
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) a2[i * (i + 1) / 2 + j] += dw * (r[GS + i * (i + 1) / 2 + j] + e[i] * e[j]);
  }
  s = warp_sum_d(s);
#pragma unroll
  for (int i = 0; i < GS; ++i) a1[i] = warp_sum_d(a1[i]);
#pragma unroll
  for (int t = 0; t < Dm::T; ++t) a2[t] = warp_sum_d(a2[t]);
  if (lane != 0) return;
  const float sf = (float)s;
  if (grp == 0) L.mass()[k] = sf;
  float mu[GS], sig[GS][GS];
  if (f.train) {
    const double inv = s != 0.0 ? 1.0 / s : 0.0;
    double mi[GS];
#pragma unroll
    for (int i = 0; i < GS; ++i) { mi[i] = a1[i] * inv; mu[i] = s != 0.0 ? (float)(ref[i] + mi[i]) : 0.f; }
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const float v = s != 0.0 ? (float)(a2[i * (i + 1) / 2 + j] * inv - mi[i] * mi[j]) : 0.f;
        sig[i][j] = v; sig[j][i] = v;
      }
  } else {
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      mu[i] = f.rmean[(size_t)k * f.C + grp * GS + i];
#pragma unroll
      for (int j = 0; j < GS; ++j) sig[i][j] = f.rcov[((size_t)k * f.G + grp) * GS * GS + i * GS + j];
    }
  }
  float* dr = L.dom(k, grp);
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    dr[GS * GS + i] = mu[i];
#pragma unroll
    for (int j = 0; j < GS; ++j) dr[i * GS + j] = sig[i][j];
  }
  if (sf == 0.f) return;
  bool bad = !(sf > 0.f);
  float Lm[GS][GS], W[GS][GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    bad = bad || !isfinite(mu[i]);
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      Lm[i][j] = f.a * sig[i][j] + (i == j ? f.b : 0.f);
      bad = bad || !isfinite(Lm[i][j]);
      W[i][j] = 0.f;
    }
  }
#pragma unroll
  for (int c = 0; c < GS; ++c) {
    bad = bad || !(Lm[c][c] > 0.f);
    Lm[c][c] = sqrtf(Lm[c][c]);
    const float inv = 1.f / Lm[c][c];
#pragma unroll
    for (int i = c + 1; i < GS; ++i) Lm[i][c] *= inv;
#pragma unroll
    for (int i = c + 1; i < GS; ++i)
#pragma unroll
      for (int j = c + 1; j <= i; ++j) Lm[i][j] -= Lm[i][c] * Lm[j][c];
  }
#pragma unroll
  for (int j = 0; j < GS; ++j) {
    W[j][j] = 1.f / Lm[j][j];
#pragma unroll
    for (int i = j + 1; i < GS; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int c = j; c < i; ++c) acc = fmaf(Lm[i][c], W[c][j], acc);
      W[i][j] = -acc / Lm[i][i];
    }
  }
  float* wr = L.w(k, grp);
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) wr[i * GS + j] = bad ? __int_as_float(0x7fc00000) : W[i][j];
  if (bad) { atomicOr(f.status, DWT_STATUS_NOT_PD); return; }
  if (!f.train || !f.update_running) return;
  const float m = f.momentum, km = 1.f - f.momentum;    // dwt_whiten_fwd's EMA on the unshrunk, biased moments
  float* rc = f.rcov + ((size_t)k * f.G + grp) * GS * GS;
  float* rm = f.rmean + (size_t)k * f.C + grp * GS;
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    rm[i] = fmaf(km, rm[i], __fmul_rn(m, mu[i]));
#pragma unroll
    for (int j = 0; j < GS; ++j) rc[i * GS + j] = m * sig[i][j] + km * rc[i * GS + j];
  }
}

// per (image, group): A_n = sum_k w_nk W_k and b_n = sum_k w_nk W_k mu_k over the domains in order (skipping w_nk == 0
// and s_k == 0), A_n m~_n = b_n by forward substitution.  A diagonal entry that is not positive and finite, or a
// non-finite A_n or m~_n: A_n = NaN, m~_n = 0, DWT_STATUS_NOT_PD.
template <int GS>
__global__ void __launch_bounds__(kThreads) lds_fwd_mix(const LdsFin f) {
  const int gi = blockIdx.x * kThreads + threadIdx.x;
  if (gi >= f.N * f.G) return;
  const int n = gi / f.G, grp = gi - n * f.G;
  const LdsLayout<GS> L(f);
  float A[GS][GS], b[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    b[i] = 0.f;
#pragma unroll
    for (int j = 0; j < GS; ++j) A[i][j] = 0.f;
  }
  for (int k = 0; k < f.K; ++k) {
    const float w = __ldg(f.weights + (size_t)n * f.K + k);
    if (w == 0.f || L.mass()[k] == 0.f) continue;
    const float* Wk = L.w(k, grp);
    const float* mk = L.dom(k, grp) + GS * GS;
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      float v = 0.f;
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const float wij = Wk[i * GS + j];
        A[i][j] = fmaf(w, wij, A[i][j]);
        v = fmaf(wij, mk[j], v);
      }
      b[i] = fmaf(w, v, b[i]);
    }
  }
  bool bad = false;
  float z[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    float r = b[i];
#pragma unroll
    for (int j = 0; j < i; ++j) {
      r = fmaf(-A[i][j], z[j], r);
      bad = bad || !isfinite(A[i][j]);
    }
    bad = bad || !(A[i][i] > 0.f && A[i][i] < INFINITY);
    z[i] = r / A[i][i];
    bad = bad || !isfinite(z[i]);
  }
  float* sw = f.save_w + (size_t)gi * GS * GS;
  float* sm = f.save_mean + (size_t)gi * GS;
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    sm[i] = bad ? 0.f : z[i];
#pragma unroll
    for (int j = 0; j < GS; ++j) sw[i * GS + j] = bad ? __int_as_float(0x7fc00000) : (j <= i ? A[i][j] : 0.f);
  }
  if (bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
}

// per (image, group): the backward segment partials added in order (fp64) into red = g_n | R_n.  AFF (a site): the
// partials are those of dz, the gradient of gamma zhat + beta; with zhat = A_n (x - m~_n) the image's shares
//   dgamma_i = sum_{j<=i} A_ij Rz_ij + [A_n (m_n - m~_n)]_i gz_i,   dbeta_i = gz_i
// go to pgb ([2][N][C]), and red gets the sums of the whitened value's gradient gamma dz: g_n = gamma gz, R_n's rows
// scaled by gamma.
template <int GS, bool AFF = false>
__global__ void __launch_bounds__(kThreads) lds_bwd_image(const LdsFin f, const float* __restrict__ part,
                                                          float* __restrict__ red, const float* __restrict__ gamma,
                                                          float* __restrict__ pgb) {
  using Dm = LdsDim<GS>;
  const int gi = blockIdx.x * kThreads + threadIdx.x;
  if (gi >= f.N * f.G) return;
  const int n = gi / f.G, grp = gi - n * f.G;
  double acc[Dm::NB];
#pragma unroll
  for (int k = 0; k < Dm::NB; ++k) acc[k] = 0.0;
  for (int j = 0; j < f.S; ++j) {
    const float* p = part + (((size_t)n * f.S + j) * f.G + grp) * Dm::NB;
#pragma unroll
    for (int k = 0; k < Dm::NB; ++k) acc[k] += p[k];
  }
  if constexpr (AFF) {
    const float* A = f.save_w + (size_t)gi * GS * GS;
    const float* mt = f.save_mean + (size_t)gi * GS;
    const float* m = f.save_stats + (size_t)gi * Dm::REC + GS * GS;
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      double dg = 0.0, off = 0.0;
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const double a = A[i * GS + j];
        dg += a * acc[GS + i * GS + j];
        off += a * ((double)m[j] - (double)mt[j]);
      }
      const int c = grp * GS + i;
      pgb[(size_t)n * f.C + c] = (float)(dg + off * acc[i]);
      pgb[((size_t)f.N + n) * f.C + c] = (float)acc[i];
      const double gam = gamma[c];
      acc[i] *= gam;
#pragma unroll
      for (int j = 0; j < GS; ++j) acc[GS + i * GS + j] *= gam;
    }
  }
#pragma unroll
  for (int k = 0; k < Dm::NB; ++k) red[(size_t)gi * Dm::NB + k] = (float)acc[k];
}

// a site's dgamma[c], dbeta[c]: the images' shares in order (fp64)
__global__ void __launch_bounds__(kThreads) lds_site_dgb(const float* __restrict__ pgb, int N, int C,
                                                         float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  double tg = 0.0, tb = 0.0;
  for (int n = 0; n < N; ++n) {
    tg += pgb[(size_t)n * C + c];
    tb += pgb[((size_t)N + n) * C + c];
  }
  dgamma[c] = (float)tg;
  dbeta[c] = (float)tb;
}

// a warp per (domain, group), train, s_k != 0: Wbar_k = sum_n w_nk [R_n + g_n (m_n - mu_k)^T] and sum_n w_nk g_n (fp64,
// lane l takes images l, l + 32, ..., zero weights skipped, the lanes added by warp_sum_d); then lane 0: the Cholesky
// backward P_k = a sym(W^T Phi(-Wbar W^T) W) and mubar_k = -W_k^T sum_n w_nk g_n into pd, <P_k, Sigma_k> into pc
template <int GS>
__global__ void __launch_bounds__(kThreads) lds_bwd_domain(const LdsFin f, const float* __restrict__ red,
                                                           float* __restrict__ pd, float* __restrict__ pc) {
  using Dm = LdsDim<GS>;
  const int idx = (blockIdx.x * kThreads + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (idx >= f.K * f.G) return;
  const int k = idx / f.G, grp = idx - k * f.G;
  const LdsLayout<GS> L(f);
  if (L.mass()[k] == 0.f) return;
  const float* dr = L.dom(k, grp);
  double wb[GS][GS], gs[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    gs[i] = 0.0;
#pragma unroll
    for (int j = 0; j < GS; ++j) wb[i][j] = 0.0;
  }
  for (int n = lane; n < f.N; n += 32) {
    const float w = __ldg(f.weights + (size_t)n * f.K + k);
    if (w == 0.f) continue;
    const size_t gi = (size_t)n * f.G + grp;
    const float* r = red + gi * Dm::NB;
    const float* mn = L.img(gi) + GS * GS;
    const double dw = (double)w;
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      const double gi_ = r[i];
      gs[i] += dw * gi_;
#pragma unroll
      for (int j = 0; j < GS; ++j)
        wb[i][j] += dw * ((double)r[GS + i * GS + j] + gi_ * ((double)mn[j] - (double)dr[GS * GS + j]));
    }
  }
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    gs[i] = warp_sum_d(gs[i]);
#pragma unroll
    for (int j = 0; j < GS; ++j) wb[i][j] = warp_sum_d(wb[i][j]);
  }
  if (lane != 0) return;
  float W[GS][GS], P1[GS][GS], T[GS][GS], S[GS][GS];
  const float* Wk = L.w(k, grp);
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) W[i][j] = j <= i ? Wk[i * GS + j] : 0.f;
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      float q = 0.f;
      if (j <= i) {
#pragma unroll
        for (int l = 0; l <= j; ++l) q = fmaf((float)wb[i][l], W[j][l], q);
        q *= i == j ? -0.5f : -1.f;
      }
      P1[i][j] = q;
    }
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      float t = 0.f;
#pragma unroll
      for (int l = (i > j ? i : j); l < GS; ++l) t = fmaf(W[l][i], P1[l][j], t);
      T[i][j] = t;
    }
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      float t = 0.f;
#pragma unroll
      for (int l = j; l < GS; ++l) t = fmaf(T[i][l], W[l][j], t);
      S[i][j] = t;
    }
  float* o = pd + (size_t)idx * Dm::REC;
  const float h = 0.5f * f.a;
  float c = 0.f;
#pragma unroll
  for (int i = 0; i < GS; ++i)
#pragma unroll
    for (int j = 0; j < GS; ++j) {
      const float p = h * (S[i][j] + S[j][i]);
      o[i * GS + j] = p;
      c = fmaf(p, dr[i * GS + j], c);
    }
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    float v = 0.f;
#pragma unroll
    for (int j = i; j < GS; ++j) v = fmaf(W[j][i], (float)gs[j], v);
    o[GS * GS + i] = -v;
  }
  pc[idx] = c;
}

// per (image, group), the domains in order (skipping s_k == 0; the terms of dx also skip w_nk == 0, dweights does not),
// with u_k = m_n - mu_k:  coef = A_n (lower) | B_n = train (2/M) sum_k (w_nk/s_k) P_k |
// c_n = train (1/M) sum_k (w_nk/s_k) [mubar_k + 2 P_k u_k] | m_n, and
// dwpart[k] = <W_k, R_n + g_n u_k^T> + train [<mubar_k, u_k> + <P_k, C_n + u_k u_k^T> - <P_k, Sigma_k>] / s_k
template <int GS>
__global__ void __launch_bounds__(kThreads) lds_bwd_coef(const LdsFin f, const float* __restrict__ red,
                                                         const float* __restrict__ pd, const float* __restrict__ pc,
                                                         float* __restrict__ coef, float* __restrict__ dwpart) {
  using Dm = LdsDim<GS>;
  const int gi = blockIdx.x * kThreads + threadIdx.x;
  if (gi >= f.N * f.G) return;
  const int n = gi / f.G, grp = gi - n * f.G;
  const LdsLayout<GS> L(f);
  const float* rec = L.img(gi);
  const float* r = red + (size_t)gi * Dm::NB;
  float m[GS], B[GS][GS], kv[GS];
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    m[i] = rec[GS * GS + i];
    kv[i] = 0.f;
#pragma unroll
    for (int j = 0; j < GS; ++j) B[i][j] = 0.f;
  }
  for (int k = 0; k < f.K; ++k) {
    const float sk = L.mass()[k];
    float dw = 0.f;
    if (sk != 0.f) {
      const float rs = 1.f / sk, w = __ldg(f.weights + (size_t)n * f.K + k);
      const float* dr = L.dom(k, grp);
      const float* Wk = L.w(k, grp);
      float u[GS];
#pragma unroll
      for (int i = 0; i < GS; ++i) u[i] = m[i] - dr[GS * GS + i];
#pragma unroll
      for (int i = 0; i < GS; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) dw = fmaf(Wk[i * GS + j], fmaf(r[i], u[j], r[GS + i * GS + j]), dw);
      if (f.train) {
        const float* P = pd + ((size_t)k * f.G + grp) * Dm::REC;
        const float wr = w * rs;
        float t = -pc[(size_t)k * f.G + grp];
#pragma unroll
        for (int i = 0; i < GS; ++i) {
          float pu = 0.f;
#pragma unroll
          for (int j = 0; j < GS; ++j) {
            const float p = P[i * GS + j];
            pu = fmaf(p, u[j], pu);
            t = fmaf(p, fmaf(u[i], u[j], rec[i * GS + j]), t);
            if (w != 0.f) B[i][j] = fmaf(wr, p, B[i][j]);
          }
          t = fmaf(P[GS * GS + i], u[i], t);
          if (w != 0.f) kv[i] = fmaf(wr, fmaf(2.f, pu, P[GS * GS + i]), kv[i]);
        }
        dw = fmaf(rs, t, dw);
      }
    }
    if (dwpart) dwpart[(size_t)gi * kLdsMaxDomains + k] = dw;
  }
  float* cf = coef + (size_t)gi * Dm::NCB;
  const float* A = f.save_w + (size_t)gi * GS * GS;
  const float invM = (float)(1.0 / f.M);
#pragma unroll
  for (int i = 0; i < GS; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) cf[i * (i + 1) / 2 + j] = A[i * GS + j];
#pragma unroll
    for (int j = 0; j < GS; ++j) cf[Dm::T + i * GS + j] = 2.f * invM * B[i][j];
    cf[Dm::T + GS * GS + i] = kv[i] * invM;
    cf[Dm::T + GS * GS + GS + i] = m[i];
  }
}

// dweights[n][k] = the groups' shares in order (fp64)
__global__ void __launch_bounds__(kThreads) lds_dw(const float* __restrict__ dwpart, int N, int G, int K,
                                                   float* __restrict__ dweights) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N * K) return;
  const int n = i / K, k = i - n * K;
  double t = 0.0;
  for (int g = 0; g < G; ++g) t += dwpart[((size_t)n * G + g) * kLdsMaxDomains + k];
  dweights[i] = (float)t;
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

template <bool BWD, class T, int E = 0>
void reduce(const void* x, const void* dy, const LdbnGeom& g, const float* centre, float* pa, float* pb, float* pilot,
            cudaStream_t st, const LdEpi& ep = LdEpi{}) {
  const T* xt = static_cast<const T*>(x);
  const T* dt = static_cast<const T*>(dy);
  if (g.nhwc) {
    const int slabs = (g.C / 4 + g.qc - 1) / g.qc;
    ldbn_reduce_nhwc<BWD, T, E><<<(unsigned)((size_t)slabs * g.S * g.N), kThreads, 0, st>>>(xt, dt, g, centre, pa, pb,
                                                                                             pilot, ep);
  } else if constexpr (!kEpiMk<E>) {
    const size_t warps = (size_t)g.N * g.C * g.S;
    const unsigned blocks = (unsigned)((warps + kWarps - 1) / kWarps);
    if (g.HW % 4 == 0) ldbn_reduce_nchw<BWD, true, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, g, centre, pa, pb, pilot, ep);
    else ldbn_reduce_nchw<BWD, false, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, g, centre, pa, pb, pilot, ep);
  }
}

template <bool BWD, class T, int E = 0>
void apply(const void* x, const void* dy, void* out, const LdbnGeom& g, const float* ca, const float* cb, const float* cq,
           const float* K, cudaStream_t st, const LdEpi& ep = LdEpi{}) {
  const T* xt = static_cast<const T*>(x);
  const T* dt = static_cast<const T*>(dy);
  T* ot = static_cast<T*>(out);
  const size_t n = (size_t)g.N * g.C * g.HW;
  if (g.nhwc) ldbn_apply_nhwc<BWD, T, E><<<ew_blocks(n / 4), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K, ep);
  else if (g.HW % 4 == 0)
    ldbn_apply_nchw<BWD, true, T, E><<<ew_blocks(n / 4), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K, ep);
  else ldbn_apply_nchw<BWD, false, T, E><<<ew_blocks(n), kThreads, 0, st>>>(xt, dt, ot, g, ca, cb, cq, K, ep);
}

// a site's epilogue bits -> the kernels' E: forward RELU or RELU|RESIDUAL; backward RELU (recomputed mask) or
// RELU|RESIDUAL (channels-last byte map, reduction only); AFFINE alone (in the coefficients) or none runs the plain kernels
#define DWT_LD_SITE(EPI, ...)                                                                                          \
  do {                                                                                                                 \
    const int e_ = (EPI) & (DWT_EPI_RELU | DWT_EPI_RESIDUAL);                                                          \
    if (e_ == (DWT_EPI_RELU | DWT_EPI_RESIDUAL)) { constexpr int E = DWT_EPI_RELU | DWT_EPI_RESIDUAL; __VA_ARGS__; }   \
    else if (e_ == DWT_EPI_RELU) { constexpr int E = DWT_EPI_RELU; __VA_ARGS__; }                                      \
    else { constexpr int E = 0; __VA_ARGS__; }                                                                         \
  } while (0)

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

void ldbn_apply(const void* x, void* y, const LdbnGeom& g, const float* alpha, const float* shift, int epi,
                const LdEpi& ep, cudaStream_t st) {
  DWT_LD_SITE(epi, {
    if (g.bf16) apply<false, __nv_bfloat16, E>(x, nullptr, y, g, alpha, shift, nullptr, nullptr, st, ep);
    else apply<false, float, E>(x, nullptr, y, g, alpha, shift, nullptr, nullptr, st, ep);
  });
}

void ldbn_bwd_reduce(const void* x, const void* dy, const LdbnGeom& g, const float* centre, float* pa, float* pb, int epi,
                     const LdEpi& ep, cudaStream_t st) {
  DWT_LD_SITE(epi, {
    if (g.bf16) reduce<true, __nv_bfloat16, E>(x, dy, g, centre, pa, pb, nullptr, st, ep);
    else reduce<true, float, E>(x, dy, g, centre, pa, pb, nullptr, st, ep);
  });
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

// only a ReLU without a residual recomputes its mask here; the residual's backward apply reads dz: the plain kernels
void ldbn_bwd_apply(const void* x, const void* dy, void* dx, const LdbnGeom& g, const float* ca, const float* cp,
                    const float* cq, const float* centre, int epi, const LdEpi& ep, cudaStream_t st) {
  if ((epi & (DWT_EPI_RELU | DWT_EPI_RESIDUAL)) == DWT_EPI_RELU) {
    if (g.bf16) apply<true, __nv_bfloat16, DWT_EPI_RELU>(x, dy, dx, g, ca, cp, cq, centre, st, ep);
    else apply<true, float, DWT_EPI_RELU>(x, dy, dx, g, ca, cp, cq, centre, st, ep);
  } else if (g.bf16) {
    apply<true, __nv_bfloat16>(x, dy, dx, g, ca, cp, cq, centre, st);
  } else {
    apply<true, float>(x, dy, dx, g, ca, cp, cq, centre, st);
  }
}

namespace {

// grid of the bandwidth passes: NCHW a warp per (image, group, segment), channels-last a CTA per (slab, segment, image)
unsigned lds_blocks(const LdbnGeom& g, int GS) {
  if (g.nhwc) return (unsigned)((size_t)((g.C / 4 + g.qc - 1) / g.qc) * g.S * g.N);
  const size_t warps = (size_t)g.N * (g.C / GS) * g.S;
  return (unsigned)((warps + kWarps - 1) / kWarps);
}

// PASS 0: forward statistics, 1: forward apply, 2: backward reduction, 3: backward apply.  NCHW bf16 runs at HW % 4 == 0.
// E: the kernels' epilogue (lds_site_pass).
template <int GS, int PASS, class T, int E = 0>
void lds_launch(const void* x, const void* dy, void* out, const LdbnGeom& g, const float* p0, const float* p1,
                const float* p2, float* part, float* pilot, cudaStream_t st, const LdEpi& ep = LdEpi{}) {
  constexpr bool BWD = PASS >= 2, APPLY = PASS == 1 || PASS == 3;
  const T* xt = static_cast<const T*>(x);
  const T* dt = static_cast<const T*>(dy);
  T* ot = static_cast<T*>(out);
  const unsigned blocks = lds_blocks(g, GS);
  if (g.nhwc) {
    if constexpr (APPLY) lds_apply_nhwc<GS, BWD, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, ot, g, p0, p1, p2, ep);
    else lds_reduce_nhwc<GS, BWD, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, g, p0, part, pilot, ep);
    return;
  }
  if constexpr (!APPLY && kEpiMk<E>) return;
  else if (g.HW % 4 == 0) {
    if constexpr (APPLY) lds_apply_nchw<GS, BWD, true, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, ot, g, p0, p1, p2, ep);
    else lds_reduce_nchw<GS, BWD, true, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, g, p0, part, pilot, ep);
  } else if constexpr (std::is_same<T, float>::value) {
    if constexpr (APPLY) lds_apply_nchw<GS, BWD, false, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, ot, g, p0, p1, p2, ep);
    else lds_reduce_nchw<GS, BWD, false, T, E><<<blocks, kThreads, 0, st>>>(xt, dt, g, p0, part, pilot, ep);
  }
}

template <int PASS, int E = 0>
void lds_pass(const void* x, const void* dy, void* out, const LdbnGeom& g, int GS, const float* p0, const float* p1,
              const float* p2, float* part, float* pilot, cudaStream_t st, const LdEpi& ep = LdEpi{}) {
#define DWT_LDS_GS(G_)                                                                                                   \
  if (GS == G_) {                                                                                                        \
    if (g.bf16) lds_launch<G_, PASS, __nv_bfloat16, E>(x, dy, out, g, p0, p1, p2, part, pilot, st, ep);                  \
    else lds_launch<G_, PASS, float, E>(x, dy, out, g, p0, p1, p2, part, pilot, st, ep);                                 \
  }
  DWT_LDS_GS(1) else DWT_LDS_GS(2) else DWT_LDS_GS(4)
#undef DWT_LDS_GS
}

// a pass under the epilogue bits epi (0: the layer) as that pass's kernels take them -- the backward reduction without
// a ReLU and the backward apply of a residual (which reads dz) need only gamma, the reduction none of it
template <int PASS>
void lds_site_pass(const void* x, const void* dy, void* out, const LdbnGeom& g, int GS, const float* p0, const float* p1,
                   const float* p2, float* part, int epi, const LdEpi& ep, cudaStream_t st) {
  constexpr int A = DWT_EPI_AFFINE, AR = A | DWT_EPI_RELU, ARR = AR | DWT_EPI_RESIDUAL;
  if (PASS == 2 && !(epi & DWT_EPI_RELU)) epi = 0;
  if (PASS == 3 && (epi & DWT_EPI_RESIDUAL)) epi = A;
  if (epi == ARR) { if constexpr (PASS != 3) lds_pass<PASS, ARR>(x, dy, out, g, GS, p0, p1, p2, part, nullptr, st, ep); }
  else if (epi == AR) lds_pass<PASS, AR>(x, dy, out, g, GS, p0, p1, p2, part, nullptr, st, ep);
  else if (epi == A) { if constexpr (PASS != 2) lds_pass<PASS, A>(x, dy, out, g, GS, p0, p1, p2, part, nullptr, st, ep); }
  else lds_pass<PASS>(x, dy, out, g, GS, p0, p1, p2, part, nullptr, st);
}

unsigned lds_grid(int work) { return (unsigned)((work + kThreads - 1) / kThreads); }

template <int GS>
void lds_fwd_fin(const LdsFin& f, const float* part, const float* pilot, double* im, cudaStream_t st) {
  lds_fwd_image<GS><<<lds_grid(f.N * f.G), kThreads, 0, st>>>(f, part, pilot, im);
  lds_fwd_domain<GS><<<lds_grid(32 * f.K * f.G), kThreads, 0, st>>>(f, im);
  lds_fwd_mix<GS><<<lds_grid(f.N * f.G), kThreads, 0, st>>>(f);
}

// gamma (a site's AFFINE) folds into the per-image sums; dgamma / dbeta when asked
template <int GS>
void lds_bwd_fin(const LdsFin& f, const float* part, float* red, float* pd, float* pc, float* coef, float* dwpart,
                 float* dweights, const float* gamma, float* pgb, float* dgamma, float* dbeta, cudaStream_t st) {
  if (gamma) lds_bwd_image<GS, true><<<lds_grid(f.N * f.G), kThreads, 0, st>>>(f, part, red, gamma, pgb);
  else lds_bwd_image<GS><<<lds_grid(f.N * f.G), kThreads, 0, st>>>(f, part, red, nullptr, nullptr);
  if (f.train) lds_bwd_domain<GS><<<lds_grid(32 * f.K * f.G), kThreads, 0, st>>>(f, red, pd, pc);
  lds_bwd_coef<GS><<<lds_grid(f.N * f.G), kThreads, 0, st>>>(f, red, pd, pc, coef, dweights ? dwpart : nullptr);
  if (dweights) lds_dw<<<lds_grid(f.N * f.K), kThreads, 0, st>>>(dwpart, f.N, f.G, f.K, dweights);
  if (dgamma) lds_site_dgb<<<lds_grid(f.C), kThreads, 0, st>>>(pgb, f.N, f.C, dgamma, dbeta);
}

}  // namespace

LdbnGeom lds_plan(int N, int C, int HW, int GS, int K, bool nhwc, bool bf16) {
  LdbnGeom g = ldbn_plan(N, nhwc ? C : C / GS, HW, K, nhwc, bf16);
  g.C = C;
  return g;
}

int lds_partial_floats(int GS) { return GS + GS * GS; }   // the backward's g | R; the forward's GS + GS(GS+1)/2 fits

int lds_coef_floats(int GS) { return GS * (GS + 1) / 2 + GS * GS + 2 * GS; }

void lds_stats(const void* x, const LdbnGeom& g, int GS, float* part, float* pilot, cudaStream_t st) {
  lds_pass<0>(x, nullptr, nullptr, g, GS, nullptr, nullptr, nullptr, part, pilot, st);
}

void lds_fwd_finalize(const LdsFin& f, const float* part, const float* pilot, double* im, cudaStream_t st) {
  if (f.GS == 1) lds_fwd_fin<1>(f, part, pilot, im, st);
  else if (f.GS == 2) lds_fwd_fin<2>(f, part, pilot, im, st);
  else lds_fwd_fin<4>(f, part, pilot, im, st);
}

void lds_apply(const void* x, void* y, const LdbnGeom& g, int GS, int epi, const LdEpi& ep, cudaStream_t st) {
  lds_site_pass<1>(x, nullptr, y, g, GS, ep.p0, ep.p1, nullptr, nullptr, epi, ep, st);
}

void lds_bwd_reduce(const void* x, const void* dy, const LdbnGeom& g, int GS, const float* save_stats, float* part, int epi,
                    const LdEpi& ep, cudaStream_t st) {
  lds_site_pass<2>(x, dy, nullptr, g, GS, save_stats, nullptr, nullptr, part, epi, ep, st);
}

void lds_bwd_finalize(const LdsFin& f, const float* part, float* red, float* pd, float* pc, float* coef, float* dwpart,
                      float* dweights, const float* gamma, float* pgb, float* dgamma, float* dbeta, cudaStream_t st) {
  if (f.GS == 1) lds_bwd_fin<1>(f, part, red, pd, pc, coef, dwpart, dweights, gamma, pgb, dgamma, dbeta, st);
  else if (f.GS == 2) lds_bwd_fin<2>(f, part, red, pd, pc, coef, dwpart, dweights, gamma, pgb, dgamma, dbeta, st);
  else lds_bwd_fin<4>(f, part, red, pd, pc, coef, dwpart, dweights, gamma, pgb, dgamma, dbeta, st);
}

void lds_bwd_apply(const void* x, const void* dy, void* dx, const LdbnGeom& g, int GS, const float* coef, int epi,
                   const LdEpi& ep, cudaStream_t st) {
  lds_site_pass<3>(x, dy, dx, g, GS, nullptr, nullptr, coef, nullptr, epi, ep, st);
}

}  // namespace dwt

// Channels-last (NHWC) register-resident path for group sizes 1, 2, 4.
//
// cuDNN's tensor-core convolutions are NHWC kernels: fed NCHW fp32 tensors they bracket every
// convolution with nchwToNhwc / nhwcToNchw copies.  Running the whole model channels-last removes those copies,
// provided the normalisation layers in between read and write NHWC natively -- this file.
//
// Layout: x[(n*HW + p)*C + c].  One float4 = 4 consecutive channels of one pixel = one whitening
// group (gs = 4), two groups (gs = 2) or four batch-norm channels (gs = 1).  A thread owns one float4
// COLUMN q (channels 4q..4q+3) and walks down the rows (pixels); a warp therefore reads 512
// contiguous bytes per step, and a thread's accumulators always belong to the same channels.
// A CTA covers CW = min(C/4, 256) columns x a contiguous range of rows; 256/CW threads share a column
// and are summed in shared memory.  Per-CTA partial moments go to global memory; one small finalize launch
// (a warp per float4 column and domain) adds them in fixed order and does the dense algebra
// (small_algebra.cuh) and the ordered running-statistic EMA -- no atomics.
//
//   cl_stats -> cl_fwd_finalize -> cl_apply          (forward, 12 B/element)
//   cl_bwd_reduce -> cl_bwd_finalize -> cl_bwd_apply (backward, 20 B/element)
//
// Two-site tail (template flag DS): the residual tail of a downsampling Bottleneck,
// relu(site3(x3) + site_d(xd)) with site_d = gamma_d W_d (xd - mu_d) + beta_d.  Both sites share N, C, HW, gs and D;
// the statistics run per site, the finalize launches serve both sites (grid.y = site) and the elementwise and
// backward-reduction kernels sweep x3 and xd together, so the identity tensor is never written and the backward
// gradient of the downsample site's output (the masked dz) is read from the same pass as the tail's.
//
// Sweep order (round 2).  The tensor a pass reads was touched a moment ago: x was just WRITTEN front to back
// by the producing convolution, and the second pass of a site re-reads what the first pass just read.  The newest
// tens of MB of it are still in L2 (50 MB on H100) -- but only if the kernel gets to them before its own misses evict
// them.  So every kernel is a persistent grid of CTAs
// that together sweep the tensor as ONE moving window of consecutive 32-row chunks (chunk c -> CTA c mod grid):
// the two reductions sweep from the END of the tensor to its start (newest bytes first, domains D-1..0 one
// after the other), the two elementwise passes from the START to the end (where the reduction just finished).
// A CTA's partial sums are still a fixed set added in a fixed order: results stay deterministic.
//
// The residual tail relu(z + identity) (resnet50_dwt_mec_officehome.py:239-240): the forward apply leaves one
// byte per float4 with the four (out > 0) bits; the backward reduction masks dout with it (the pre-activation cannot
// be recomputed without the residual) and writes the masked gradient dz, which is also the gradient of the identity
// branch; bwd_apply then reads x and dz only (the plain AFFINE apply with dout = dz).
// Such a site's output is used twice by the next block (first convolution and identity branch): the two gradients
// arrive as dout and dout2 and are summed where they are read (template flag D2; dwt_b200.h, functional.fork_for_sum)
// instead of by an elementwise kernel in between.
//
// Reference semantics: utils/whitening.py:37-61, utils/batch_norm.py:54-69 (/root/reference).
#include <stdlib.h>

#include "dwt_common.cuh"
#include "norm_launch.h"
#include "small_algebra.cuh"

namespace dwt {
namespace {

constexpr int kT = 256;

// Programmatic dependent launch (PDL).  The three launches of a pass form a chain reduction -> finalize -> elementwise.
// With DWT_PDL=1 the finalize and elementwise kernels are launched with programmaticStreamSerialization: they may become
// resident while their predecessor is still draining, run their prologue (index arithmetic, parameter loads that do not
// depend on the predecessor) and block in griddepcontrol.wait until the predecessor grid has completed and flushed.
// Kernels launched the ordinary way see both instructions as no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <int GS> struct ClShape {
  static constexpr int NSUB = 4 / GS;                       // problems per float4 column
  static constexpr int NM = GS * (GS + 1) / 2;
  static constexpr int FWD1 = GS + NM;                      // forward accumulators per problem
  static constexpr int BWD1 = GS * GS + GS;                 // backward accumulators per problem
  static constexpr int FWD = NSUB * FWD1;
  static constexpr int BWD = NSUB * BWD1;
};

// Thread placement inside the CTA.
struct ClThread {
  int C4, CW, rpi, col, rsub, q;
  __device__ __forceinline__ ClThread(const Geom& gm) {
    C4 = gm.C >> 2;
    CW = C4 < kT ? C4 : kT;
    rpi = kT / CW;
    col = threadIdx.x % CW;
    rsub = threadIdx.x / CW;
    q = blockIdx.y * CW + col;
  }
};

// The CTAs of grid.x sweep the rows of one domain as a moving window of chunks of rpi*UNROLL consecutive rows:
// chunk c belongs to CTA c mod gridDim.x; DESC walks from the last chunk to the first.  body(r) gets the first
// row of the calling thread inside the chunk (its rows are r + u*rpi, u < UNROLL, to be guarded by r < rows).
template <int UNROLL, bool DESC, class F>
__device__ __forceinline__ void sweep_rows(const ClThread& t, unsigned rows, F&& body) {
  const unsigned krows = (unsigned)t.rpi * UNROLL, nch = (rows + krows - 1) / krows;
  for (unsigned i = blockIdx.x; i < nch; i += gridDim.x) body((DESC ? nch - 1 - i : i) * krows + t.rsub);
}
// Domains served by this CTA: all of them one after the other (gridDim.z == 1) or one (gridDim.z == D).
#define CL_FOR_DOMAINS(d, gm, DESC) \
  for (int di_ = blockIdx.z, d = (DESC) ? (gm).D - 1 - di_ : di_; di_ < (gm).D; di_ += gridDim.z, d = (DESC) ? (gm).D - 1 - di_ : di_)

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Sum the per-thread accumulators of the rpi threads that share a column; thread rsub == 0 of every column
// then holds the CTA total.  sRed must hold kT * NACC floats.
template <int NACC>
__device__ __forceinline__ void column_reduce(const ClThread& t, float (&acc)[NACC], float* sRed) {
  if (t.rpi == 1) return;
#pragma unroll
  for (int i = 0; i < NACC; ++i) sRed[i * kT + threadIdx.x] = acc[i];
  __syncthreads();
  if (t.rsub == 0) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) {
      float s = acc[i];
      for (int r = 1; r < t.rpi; ++r) s += sRed[i * kT + r * t.CW + t.col];
      acc[i] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------
// forward statistics: partial[d][cta][q][FWD] ; CTA (0, y, d) also publishes the pilot shift
// ------------------------------------------------------------------------------------------
template <int GS>
__global__ void __launch_bounds__(kT, 3) cl_stats_kernel(const float* __restrict__ x, const Geom gm,
                                                         float* __restrict__ partial, float* __restrict__ shift) {
  using S = ClShape<GS>;
  constexpr int UNROLL = 8;
  __shared__ float sRed[kT * S::FWD];
  const ClThread t(gm);
  const unsigned rows = (unsigned)gm.N * gm.HW;
  pdl_launch_dependents();
  CL_FOR_DOMAINS(d, gm, true) {
    const float* xd = x + (size_t)d * rows * gm.C + 4 * t.q;
    // pilot shift K, per channel (every thread of a column agrees): the mean of the first <= 8 rows of the domain,
    // unless they sit far from the rest of it.  The one-pass moments lose digits in proportion to (K - mean)^2 / var:
    // a first image whose top row sat 30 sigma off cost 1.1e-4 of the stem site's covariance at the benchmark's size
    // (test_channels_last_fp64.py).  So 8 rows spread over the domain are read as well (the middle pixel, for square
    // images, of the image at row (2k+1) * rows / 16: never the same border pixel of 8 images), and where their mean
    // lies more than 20 of their standard deviations from K, K moves to it.  The threshold sits above what real
    // activations show (at most 14 over the sites of 20 training steps), so they keep the first rows' K and their
    // statistics bit for bit.
    float K[4] = {0.f, 0.f, 0.f, 0.f};
    {
      const unsigned np = rows < 8 ? rows : 8;
      for (unsigned r = 0; r < np; ++r) {
        const float4 v = ldg4(xd + (size_t)r * gm.C);
        K[0] += v.x; K[1] += v.y; K[2] += v.z; K[3] += v.w;
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) K[c] /= (float)np;
      if (rows > 8) {
        float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};   // moments of the spread rows around K
        const size_t mid = (size_t)gm.HW / 2 + (size_t)sqrtf((float)gm.HW) / 2;
        for (unsigned k = 0; k < 8; ++k) {
          const float4 v = ldg4(xd + ((2 * (size_t)k + 1) * rows / 16 + mid) % rows * gm.C);
          const float e[4] = {v.x - K[0], v.y - K[1], v.z - K[2], v.w - K[3]};
#pragma unroll
          for (int c = 0; c < 4; ++c) { s1[c] += e[c]; s2[c] = fmaf(e[c], e[c], s2[c]); }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float dk = s1[c] * 0.125f;                      // spread mean - K; spread variance = s2 / 8 - dk^2
          if (401.f * dk * dk > 400.f * (s2[c] * 0.125f)) K[c] += dk;   // dk^2 > 400 * spread variance
        }
      }
      if (blockIdx.x == 0 && t.rsub == 0) *reinterpret_cast<float4*>(shift + (size_t)d * gm.C + 4 * t.q) = make_float4(K[0], K[1], K[2], K[3]);
    }
    float acc[S::FWD];
#pragma unroll
    for (int i = 0; i < S::FWD; ++i) acc[i] = 0.f;
    sweep_rows<UNROLL, true>(t, rows, [&](unsigned r) {
      float4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const unsigned rr = r + u * t.rpi;
        v[u] = rr < rows ? ldg4(xd + (size_t)rr * gm.C) : make_float4(K[0], K[1], K[2], K[3]);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const float e[4] = {v[u].x - K[0], v[u].y - K[1], v[u].z - K[2], v[u].w - K[3]};
#pragma unroll
        for (int s = 0; s < S::NSUB; ++s) {
#pragma unroll
          for (int c = 0; c < GS; ++c) {
            acc[s * S::FWD1 + c] += e[s * GS + c];
#pragma unroll
            for (int j = 0; j <= c; ++j)
              acc[s * S::FWD1 + GS + c * (c + 1) / 2 + j] = fmaf(e[s * GS + c], e[s * GS + j], acc[s * S::FWD1 + GS + c * (c + 1) / 2 + j]);
          }
        }
      }
    });
    column_reduce<S::FWD>(t, acc, sRed);
    if (t.rsub == 0) {
      float* dst = partial + (((size_t)d * gridDim.x + blockIdx.x) * t.C4 + t.q) * S::FWD;
#pragma unroll
      for (int i = 0; i < S::FWD; ++i) dst[i] = acc[i];
    }
    if (gridDim.z == 1) __syncthreads();             // sRed is reused by the next domain
  }
}

// index of accumulator a of group g inside a W-vector
template <int GS, int PER>
__device__ __forceinline__ int acc_index(int g, int a) {
  constexpr int NSUB = 4 / GS;
  return (g / NSUB) * (NSUB * PER) + (g % NSUB) * PER + a;
}

// Finalize launches (one per pass, between the reduction and the elementwise kernel).  blockDim = (32, kFinQ columns,
// D domains): ONE WARP serves one (float4 column, domain).  Lane l adds the per-CTA partial rows l, l+32, ... of its
// column in ascending order (independent 8-byte loads, several rows in flight), five xor-shuffles add the lanes in a
// fixed tree, and lane 0 does the dense algebra of the column's 4/gs groups in registers.  This replaced a many-CTA
// `vec_reduce` launch plus a finalize launch in which one thread per (group, domain) walked the reduced rows itself --
// a chain of ~30 dependent L2 round trips, 212 launches per step.  The running-statistic EMA follows
// the aliasing class found on the host: all domains on ONE buffer pair (the shipped models) -> one closed-form
// read-modify-write r' = k^D r + m sum_d k^(D-1-d) s_d; all distinct -> every domain's warp updates its own buffers;
// mixed -> the d == 0 warp applies the domains in order.  No atomics, fixed summation order.
constexpr int kFinQ = 2;   // few columns per block: many small blocks pull the partial rows from L2 in parallel

template <int NACC>
__device__ __forceinline__ void column_row_sum(const float* __restrict__ col, int nrows, int W, float (&a)[NACC]) {
  static_assert(NACC % 2 == 0, "accumulators are read as float2");
#pragma unroll
  for (int i = 0; i < NACC; ++i) a[i] = 0.f;
#pragma unroll 4
  for (int r = threadIdx.x; r < nrows; r += 32) {
    const float2* p = reinterpret_cast<const float2*>(col + (size_t)r * W);
#pragma unroll
    for (int i = 0; i < NACC / 2; ++i) {
      const float2 v = __ldcg(p + i);
      a[2 * i] += v.x; a[2 * i + 1] += v.y;
    }
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1)
#pragma unroll
    for (int i = 0; i < NACC; ++i) a[i] += __shfl_xor_sync(0xffffffffu, a[i], o);
}

// After column_row_sum every lane holds the column's NSUB * PER totals; lane s < NSUB takes the PER values of group s
// (selected with predicated moves: the NSUB groups of a column are then finalized by NSUB lanes in parallel, not one
// after the other by lane 0 -- for batch norm, NSUB = 4, that was four dependent sqrt / divide / read-modify-write chains).
template <int NSUB, int PER>
__device__ __forceinline__ void take_group(const float (&a)[NSUB * PER], int s, float (&v)[PER]) {
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    v[i] = a[i];
#pragma unroll
    for (int k = 1; k < NSUB; ++k)
      if (s == k) v[i] = a[k * PER + i];
  }
}

template <int GS>
__device__ __forceinline__ void cl_fwd_finalize_site(const float* __restrict__ partial, int nrows, const float* __restrict__ shift,
                                                     const Geom& gm, const FwdFin& fin) {
  using SH = ClShape<GS>;
  constexpr int NST = GS + GS * GS;
  __shared__ float sStat[DWT_MAX_DOMAINS][kFinQ][SH::NSUB][NST + 1];
  __shared__ unsigned char sBad[DWT_MAX_DOMAINS][kFinQ][SH::NSUB];
  const int s = threadIdx.x, ql = threadIdx.y, d = threadIdx.z, q = blockIdx.x * blockDim.y + ql;
  const int W = (gm.C >> 2) * SH::FWD;
  const float invM = 1.f / gm.M;
  const bool lead = s < SH::NSUB;                          // lane s finalizes group q * NSUB + s
  const int g = q * SH::NSUB + (lead ? s : 0);
  const bool direct = gm.D == 1 || fin.aliased == 0;       // this domain owns its buffers
  // the running buffers this lane will update are fetched first: their (DRAM) latency hides behind the row sums
  const int dbuf = direct ? d : 0;
  const bool upd = fin.update_running && lead && (direct || (fin.aliased == 1 && d == 0));
  float rc_old[GS * GS], rm_old[GS];
  if (upd) {
#pragma unroll
    for (int e = 0; e < GS * GS; ++e) rc_old[e] = fin.rcov[dbuf][(size_t)g * GS * GS + e];
#pragma unroll
    for (int e = 0; e < GS; ++e) rm_old[e] = fin.rmean[dbuf][g * GS + e];
  }
  pdl_launch_dependents();
  pdl_wait();                                       // the reduction's partial rows and pilot shifts are complete
  float a[SH::FWD];
  column_row_sum<SH::FWD>(partial + (size_t)d * nrows * W + (size_t)q * SH::FWD, nrows, W, a);
  if (lead) {
    float v[SH::FWD1];
    take_group<SH::NSUB, SH::FWD1>(a, s, v);
    float mean[GS], cov[GS][GS];
#pragma unroll
    for (int i = 0; i < GS; ++i) mean[i] = shift[(size_t)d * gm.C + g * GS + i] + v[i] * invM;
#pragma unroll
    for (int i = 0; i < GS; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        const float c = v[GS + i * (i + 1) / 2 + j] * invM - (v[i] * invM) * (v[j] * invM);
        cov[i][j] = c; cov[j][i] = c;
      }
    const bool bad = factor_thread<GS>(gm, fin, d, g, mean, cov, false);
    if (fin.update_running) {
      if (direct) {
        if (!bad) {
          const float m = fin.momentum, kk = 1.f - fin.momentum;
#pragma unroll
          for (int i = 0; i < GS; ++i) {
            fin.rmean[d][g * GS + i] = m * mean[i] + kk * rm_old[i];
#pragma unroll
            for (int j = 0; j < GS; ++j)
              fin.rcov[d][(size_t)g * GS * GS + i * GS + j] = m * (cov[i][j] * fin.unbias) + kk * rc_old[i * GS + j];
          }
        }
      } else {
        sBad[d][ql][s] = bad ? 1 : 0;
#pragma unroll
        for (int i = 0; i < GS; ++i) {
          sStat[d][ql][s][i] = mean[i];
#pragma unroll
          for (int j = 0; j < GS; ++j) sStat[d][ql][s][GS + i * GS + j] = cov[i][j];
        }
      }
    }
  }
  if (!fin.update_running || direct) return;
  __syncthreads();
  if (!(lead && d == 0)) return;
  if (fin.aliased == 1) {
    // one shared buffer pair: the D sequential updates collapse to one read-modify-write
    const float m = fin.momentum, kk = 1.f - fin.momentum;
    float* rc = fin.rcov[0] + (size_t)g * GS * GS;
    float* rm = fin.rmean[0] + g * GS;
    for (int dd = 0; dd < gm.D; ++dd) {
      if (sBad[dd][ql][s]) continue;
#pragma unroll
      for (int e = 0; e < GS * GS; ++e) rc_old[e] = m * (sStat[dd][ql][s][GS + e] * fin.unbias) + kk * rc_old[e];
#pragma unroll
      for (int e = 0; e < GS; ++e) rm_old[e] = m * sStat[dd][ql][s][e] + kk * rm_old[e];
    }
#pragma unroll
    for (int e = 0; e < GS * GS; ++e) rc[e] = rc_old[e];
#pragma unroll
    for (int e = 0; e < GS; ++e) rm[e] = rm_old[e];
  } else {
    for (int dd = 0; dd < gm.D; ++dd)               // mixed aliasing: plain ordered read-modify-write
      if (!sBad[dd][ql][s]) ema_direct<GS>(gm, fin, dd, g, &sStat[dd][ql][s][0], &sStat[dd][ql][s][GS]);
  }
}

// grid.y = sites: site 1 (two-site tail) reads its partial rows at partial + pstride and its shifts at shift + sstride
template <int GS>
__global__ void __launch_bounds__(32 * kFinQ * DWT_MAX_DOMAINS) cl_fwd_finalize_kernel(const float* __restrict__ partial, size_t pstride, int nrows,
                                                                                      const float* __restrict__ shift, size_t sstride, const Geom gm,
                                                                                      const __grid_constant__ FwdFin fin, const __grid_constant__ FwdFin fin2) {
  const bool second = blockIdx.y != 0;
  cl_fwd_finalize_site<GS>(partial + (second ? pstride : 0), nrows, shift + (second ? sstride : 0), gm, second ? fin2 : fin);
}

// ------------------------------------------------------------------------------------------
// apply
// ------------------------------------------------------------------------------------------
// DS (two-site tail, EPI = AFFINE|RELU|RESIDUAL): `res` is the downsample site's INPUT xd and the residual is its
// output gamma_d W_d (xd - mu_d) + beta_d, formed in registers exactly as the downsample site's own apply would.
template <int GS, int EPI, bool DS>
__global__ void __launch_bounds__(kT, 3) cl_apply_kernel(const float* __restrict__ x, float* __restrict__ y, const Geom gm,
                                                         const float* __restrict__ save_mean, const float* __restrict__ save_w,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                                         const float* __restrict__ res, uint8_t* __restrict__ mask,
                                                         const float* __restrict__ save_mean_d, const float* __restrict__ save_w_d,
                                                         const float* __restrict__ gamma_d, const float* __restrict__ beta_d) {
  using S = ClShape<GS>;
  constexpr bool RES = (EPI & DWT_EPI_RESIDUAL) != 0;
  static_assert(!DS || RES, "the two-site tail is a residual epilogue");
  // rows per thread and step (the grid shape comes from cl_plan either way): two sites' maps need the registers
  constexpr int UNROLL = DS ? 2 : (RES ? 4 : 8);
  const ClThread t(gm);
  const unsigned rows = (unsigned)gm.N * gm.HW;
  pdl_wait();                                       // save_mean / save_w of the finalize launch are complete
  CL_FOR_DOMAINS(d, gm, false) {
    float Wp[S::NSUB][S::NM], bp[S::NSUB][GS], Wd[DS ? S::NSUB : 1][S::NM], bd[DS ? S::NSUB : 1][GS];
#pragma unroll
    for (int s = 0; s < S::NSUB; ++s) {
      const int g = t.q * S::NSUB + s;
      load_forward_map<GS, EPI>(save_w + ((size_t)d * gm.G + g) * GS * GS, save_mean + (size_t)d * gm.C + g * GS,
                                gamma + g * GS, beta + g * GS, Wp[s], bp[s]);
      if constexpr (DS)
        load_forward_map<GS, DWT_EPI_AFFINE>(save_w_d + ((size_t)d * gm.G + g) * GS * GS, save_mean_d + (size_t)d * gm.C + g * GS,
                                             gamma_d + g * GS, beta_d + g * GS, Wd[s], bd[s]);
    }
    const size_t base = (size_t)d * rows * gm.C + 4 * t.q;
    const float* xd = x + base;
    const float* rd = res + base;
    float* yd = y + base;
    uint8_t* md = mask + (size_t)d * rows * t.C4 + t.q;          // one byte per float4: the four (out > 0) bits
    sweep_rows<UNROLL, false>(t, rows, [&](unsigned r) {
      float4 v[UNROLL], rs[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const unsigned rr = r + u * t.rpi;
        if (rr < rows) {
          v[u] = ldg4(xd + (size_t)rr * gm.C);
          if constexpr (RES) rs[u] = ldg4(rd + (size_t)rr * gm.C);
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const unsigned rr = r + u * t.rpi;
        if (rr < rows) {
          const float e[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
          float o[4], ra[4] = {0.f, 0.f, 0.f, 0.f};
          if constexpr (RES) { ra[0] = rs[u].x; ra[1] = rs[u].y; ra[2] = rs[u].z; ra[3] = rs[u].w; }
          unsigned bits = 0;
#pragma unroll
          for (int s = 0; s < S::NSUB; ++s) {
            float xi[GS], oi[GS];
            if constexpr (DS) {
              float xdi[GS], odi[GS];
#pragma unroll
              for (int c = 0; c < GS; ++c) xdi[c] = ra[s * GS + c];
              apply_group<GS>(Wd[s], bd[s], xdi, odi);
#pragma unroll
              for (int c = 0; c < GS; ++c) ra[s * GS + c] = odi[c];
            }
#pragma unroll
            for (int c = 0; c < GS; ++c) xi[c] = e[s * GS + c];
            apply_group<GS>(Wp[s], bp[s], xi, oi);
#pragma unroll
            for (int c = 0; c < GS; ++c) {
              const float z = RES ? oi[c] + ra[s * GS + c] : oi[c];
              if constexpr (RES) bits |= (z > 0.f ? 1u : 0u) << (s * GS + c);
              o[s * GS + c] = (EPI & DWT_EPI_RELU) ? fmaxf(z, 0.f) : z;
            }
          }
          *reinterpret_cast<float4*>(yd + (size_t)rr * gm.C) = make_float4(o[0], o[1], o[2], o[3]);
          if constexpr (RES) { if (mask != nullptr) md[(size_t)rr * t.C4] = (uint8_t)bits; }
        }
      }
    });
  }
}

// ------------------------------------------------------------------------------------------
// backward reduce: partial[d][cta][q][BWD]  (per problem: R row-major, then sdz)
// ------------------------------------------------------------------------------------------
// one row's contribution to a problem's backward accumulators: R += dz (x - mu)^T, sdz += dz
template <int GS>
__device__ __forceinline__ void bwd_accumulate(float* acc, const float (&dz)[GS], const float (&xi)[GS], const float* mu) {
#pragma unroll
  for (int i = 0; i < GS; ++i) {
    acc[GS * GS + i] += dz[i];
#pragma unroll
    for (int j = 0; j < GS; ++j) acc[i * GS + j] = fmaf(dz[i], xi[j] - mu[j], acc[i * GS + j]);
  }
}

// MASK (residual tail): the masked gradient dz -- also the gradient of the identity branch -- is written to dzout.
// DS (two-site tail): the downsample site's input xd is swept alongside x; its gradient is the same dz, so its
// accumulators (R_d, sdz) go to a second set of partial rows at partial + pstride.
template <int GS, int EPI, bool D2, bool DS>
__global__ void __launch_bounds__(kT, 2) cl_bwd_reduce_kernel(const float* __restrict__ x, const float* __restrict__ dout, const float* __restrict__ dout2,
                                                              const Geom gm, const float* __restrict__ save_mean,
                                                              const float* __restrict__ save_w, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, const uint8_t* __restrict__ mask,
                                                              float* __restrict__ dzout, float* __restrict__ partial,
                                                              const float* __restrict__ xds, const float* __restrict__ save_mean_d,
                                                              size_t pstride) {
  using S = ClShape<GS>;
  constexpr int UNROLL = 4;
  constexpr bool MASK = (EPI & DWT_EPI_RESIDUAL) != 0;          // ReLU mask saved by the forward (residual tail)
  constexpr bool RELU = (EPI & DWT_EPI_RELU) != 0 && !MASK;     // ReLU mask recomputed from x
  static_assert(!DS || MASK, "the two-site tail is a residual epilogue");
  constexpr int NS = DS ? 2 : 1;
  __shared__ float sRed[kT * S::BWD];
  const ClThread t(gm);
  const unsigned rows = (unsigned)gm.N * gm.HW;
  pdl_launch_dependents();
  CL_FOR_DOMAINS(d, gm, true) {
    float Wp[S::NSUB][S::NM], bp[S::NSUB][GS], mu[NS][4];
#pragma unroll
    for (int s = 0; s < S::NSUB; ++s) {
      const int g = t.q * S::NSUB + s;
      if constexpr (RELU)
        load_forward_map<GS, EPI>(save_w + ((size_t)d * gm.G + g) * GS * GS, save_mean + (size_t)d * gm.C + g * GS,
                                  gamma + g * GS, beta + g * GS, Wp[s], bp[s]);
    }
#pragma unroll
    for (int k = 0; k < NS; ++k) {
      const float4 m4 = ldg4((k ? save_mean_d : save_mean) + (size_t)d * gm.C + 4 * t.q);
      mu[k][0] = m4.x; mu[k][1] = m4.y; mu[k][2] = m4.z; mu[k][3] = m4.w;
    }
    float acc[NS][S::BWD];
#pragma unroll
    for (int k = 0; k < NS; ++k)
#pragma unroll
      for (int i = 0; i < S::BWD; ++i) acc[k][i] = 0.f;
    const size_t base = (size_t)d * rows * gm.C + 4 * t.q;
    const float* xp[NS];
    xp[0] = x + base;
    if constexpr (DS) xp[NS - 1] = xds + base;
    const float* gd = dout + base;
    const float* gd2 = D2 ? dout2 + base : nullptr;        // second addend of the incoming gradient (see dwt_b200.h)
    float* zd = MASK ? dzout + base : nullptr;
    const uint8_t* md = mask + (size_t)d * rows * t.C4 + t.q;
    // rows per load batch: all of the chunk's rows, or (two sites) half of them, so that both sites' accumulators stay
    // in registers.  The rows are accumulated in the same order either way.
    constexpr int H = DS ? UNROLL / 2 : UNROLL;
    sweep_rows<UNROLL, true>(t, rows, [&](unsigned r0) {
#pragma unroll
     for (int h = 0; h < UNROLL; h += H) {
      const unsigned r = r0 + h * t.rpi;
      float4 v[NS][H], q[H], q2[D2 ? H : 1];
      unsigned mb[H];
#pragma unroll
      for (int u = 0; u < H; ++u) {                            // every load of the batch first: nothing waits on another
        const unsigned rr = r + u * t.rpi;
        if (rr < rows) {
#pragma unroll
          for (int k = 0; k < NS; ++k) v[k][u] = ldg4(xp[k] + (size_t)rr * gm.C);
          q[u] = ldg4(gd + (size_t)rr * gm.C);
          if constexpr (MASK) mb[u] = __ldg(md + (size_t)rr * t.C4);
          if constexpr (D2) q2[u] = ldg4(gd2 + (size_t)rr * gm.C);
        } else {
#pragma unroll
          for (int k = 0; k < NS; ++k) v[k][u] = make_float4(mu[k][0], mu[k][1], mu[k][2], mu[k][3]);
          q[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if constexpr (MASK) mb[u] = 0u;
          if constexpr (D2) q2[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      if constexpr (D2) {
#pragma unroll
        for (int u = 0; u < H; ++u) { q[u].x += q2[u].x; q[u].y += q2[u].y; q[u].z += q2[u].z; q[u].w += q2[u].w; }
      }
#pragma unroll
      for (int u = 0; u < H; ++u) {
        const float ge[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
        const float e[4] = {v[0][u].x, v[0][u].y, v[0][u].z, v[0][u].w};
        const float ed[4] = {v[NS - 1][u].x, v[NS - 1][u].y, v[NS - 1][u].z, v[NS - 1][u].w};
        float zm[4];
#pragma unroll
        for (int s = 0; s < S::NSUB; ++s) {
          float xi[GS], dz[GS];
#pragma unroll
          for (int c = 0; c < GS; ++c) { xi[c] = e[s * GS + c]; dz[c] = ge[s * GS + c]; }
          if constexpr (RELU) {
            float oi[GS];
            apply_group<GS>(Wp[s], bp[s], xi, oi);
#pragma unroll
            for (int c = 0; c < GS; ++c) dz[c] = oi[c] > 0.f ? dz[c] : 0.f;
          }
          if constexpr (MASK) {
#pragma unroll
            for (int c = 0; c < GS; ++c) { dz[c] = ((mb[u] >> (s * GS + c)) & 1u) ? dz[c] : 0.f; zm[s * GS + c] = dz[c]; }
          }
          bwd_accumulate<GS>(acc[0] + s * S::BWD1, dz, xi, &mu[0][s * GS]);
          if constexpr (DS) {
#pragma unroll
            for (int c = 0; c < GS; ++c) xi[c] = ed[s * GS + c];
            bwd_accumulate<GS>(acc[NS - 1] + s * S::BWD1, dz, xi, &mu[NS - 1][s * GS]);
          }
        }
        if constexpr (MASK) {
          const unsigned rr = r + u * t.rpi;
          if (rr < rows) *reinterpret_cast<float4*>(zd + (size_t)rr * gm.C) = make_float4(zm[0], zm[1], zm[2], zm[3]);
        }
      }
     }
    });
#pragma unroll
    for (int k = 0; k < NS; ++k) {
      if (k) __syncthreads();                          // sRed is reused by the second site
      column_reduce<S::BWD>(t, acc[k], sRed);
      if (t.rsub == 0) {
        float* dst = partial + k * pstride + (((size_t)d * gridDim.x + blockIdx.x) * t.C4 + t.q) * S::BWD;
#pragma unroll
        for (int i = 0; i < S::BWD; ++i) dst[i] = acc[k][i];
      }
    }
    if (gridDim.z == 1) __syncthreads();             // sRed is reused by the next domain
  }
}

// Same arrangement as the forward finalize (one warp per (float4 column, domain)); dgamma / dbeta are summed over the
// domains by the d == 0 warp after the barrier.
template <int GS>
__device__ __forceinline__ void cl_bwd_finalize_site(const float* __restrict__ partial, int nrows, const Geom& gm, const BwdFin& fin) {
  using SH = ClShape<GS>;
  const int s = threadIdx.x, d = threadIdx.z, q = blockIdx.x * blockDim.y + threadIdx.y;
  const int W = (gm.C >> 2) * SH::BWD;
  pdl_launch_dependents();
  pdl_wait();                                       // the backward reduction's partial rows are complete
  float a[SH::BWD];
  column_row_sum<SH::BWD>(partial + (size_t)d * nrows * W + (size_t)q * SH::BWD, nrows, W, a);
  if (s < SH::NSUB) {                               // lane s finalizes group q * NSUB + s
    float v[SH::BWD1], R[GS][GS], sdz[GS];
    take_group<SH::NSUB, SH::BWD1>(a, s, v);
#pragma unroll
    for (int i = 0; i < SH::BWD1; ++i) {
      if (i < GS * GS) R[i / GS][i % GS] = v[i]; else sdz[i - GS * GS] = v[i];
    }
    bwd_finalize_thread<GS>(gm, fin, d, q * SH::NSUB + s, R, sdz, false);
  }
  if (!((fin.epi & DWT_EPI_AFFINE) && fin.dgamma != nullptr)) return;
  __syncthreads();                                  // the block's dgb_part writes (global) are visible block-wide
  if (d == 0 && s < 4) {                            // lane i sums channel 4q + i over the domains
    const int ch = 4 * q + s;
    float sg = 0.f, sb = 0.f;
    for (int dd = 0; dd < gm.D; ++dd) {
      sg += fin.dgb_part[((size_t)dd * 2 + 0) * gm.C + ch];
      sb += fin.dgb_part[((size_t)dd * 2 + 1) * gm.C + ch];
    }
    fin.dgamma[ch] = sg;
    fin.dbeta[ch] = sb;
  }
}

// grid.y = sites, as for the forward finalize
template <int GS>
__global__ void __launch_bounds__(32 * kFinQ * DWT_MAX_DOMAINS) cl_bwd_finalize_kernel(const float* __restrict__ partial, size_t pstride, int nrows,
                                                                                      const Geom gm, const __grid_constant__ BwdFin fin,
                                                                                      const __grid_constant__ BwdFin fin2) {
  const bool second = blockIdx.y != 0;
  cl_bwd_finalize_site<GS>(partial + (second ? pstride : 0), nrows, gm, second ? fin2 : fin);
}

// ------------------------------------------------------------------------------------------
// backward apply
// ------------------------------------------------------------------------------------------
// Per-thread copy of a problem's backward coefficients (dx = A1 dz + Bm x + cvec; A1 upper-, Bm full symmetric,
// both kept as packed lower triangles)
template <int GS>
struct BwdCoef {
  float A1[GS * (GS + 1) / 2], Bm[GS * (GS + 1) / 2], cv[GS];
  __device__ __forceinline__ void load(const float* cf) {
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      cv[i] = __ldg(cf + 2 * GS * GS + i);
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        A1[i * (i + 1) / 2 + j] = __ldg(cf + j * GS + i);
        Bm[i * (i + 1) / 2 + j] = __ldg(cf + GS * GS + i * GS + j);
      }
    }
  }
  __device__ __forceinline__ void apply(const float (&dz)[GS], const float (&xi)[GS], float* o) const {
#pragma unroll
    for (int i = 0; i < GS; ++i) {
      float a = cv[i];
#pragma unroll
      for (int j = i; j < GS; ++j) a = fmaf(A1[j * (j + 1) / 2 + i], dz[j], a);
#pragma unroll
      for (int j = 0; j < GS; ++j) {
        const int hi = i > j ? i : j, lo = i > j ? j : i;
        a = fmaf(Bm[hi * (hi + 1) / 2 + lo], xi[j], a);
      }
      o[i] = a;
    }
  }
};

// The residual tail's apply is the AFFINE one with dout = the masked dz its reduction wrote.  DS (two-site tail):
// the same dz is the downsample site's output gradient, so the pass also reads xd and writes dxd with the downsample
// site's coefficients (coef_d).
template <int GS, int EPI, bool D2, bool DS>
__global__ void __launch_bounds__(kT, 2) cl_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dout, const float* __restrict__ dout2,
                                                             float* __restrict__ dx, const Geom gm, const float* __restrict__ coef,
                                                             const float* __restrict__ save_mean, const float* __restrict__ save_w,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             const float* __restrict__ xds, float* __restrict__ dxds,
                                                             const float* __restrict__ coef_d) {
  using S = ClShape<GS>;
  constexpr int UNROLL = 4;
  constexpr bool RELU = (EPI & DWT_EPI_RELU) != 0;
  static_assert((EPI & DWT_EPI_RESIDUAL) == 0, "the residual tail's apply runs with EPI = AFFINE on dz");
  static_assert(!DS || (!D2 && !RELU), "the two-site tail's apply reads dz");
  constexpr int NS = DS ? 2 : 1;
  const ClThread t(gm);
  const unsigned rows = (unsigned)gm.N * gm.HW;
  pdl_wait();                                       // the coefficients of the backward finalize launch are complete
  CL_FOR_DOMAINS(d, gm, false) {
    float Wp[S::NSUB][S::NM], bp[S::NSUB][GS];
    BwdCoef<GS> cf[NS][S::NSUB];
#pragma unroll
    for (int s = 0; s < S::NSUB; ++s) {
      const int g = t.q * S::NSUB + s;
      if constexpr (RELU)
        load_forward_map<GS, EPI>(save_w + ((size_t)d * gm.G + g) * GS * GS, save_mean + (size_t)d * gm.C + g * GS,
                                  gamma + g * GS, beta + g * GS, Wp[s], bp[s]);
#pragma unroll
      for (int k = 0; k < NS; ++k) cf[k][s].load((k ? coef_d : coef) + ((size_t)d * gm.G + g) * coef_stride(GS));
    }
    const size_t base = (size_t)d * rows * gm.C + 4 * t.q;
    const float* xp[NS];
    float* op[NS];
    xp[0] = x + base; op[0] = dx + base;
    if constexpr (DS) { xp[NS - 1] = xds + base; op[NS - 1] = dxds + base; }
    const float* gd = dout + base;
    const float* gd2 = D2 ? dout2 + base : nullptr;        // second addend of the incoming gradient (see dwt_b200.h)
    sweep_rows<UNROLL, false>(t, rows, [&](unsigned r) {
      float4 v[NS][UNROLL], q[UNROLL], q2[D2 ? UNROLL : 1];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const unsigned rr = r + u * t.rpi;
        if (rr < rows) {
#pragma unroll
          for (int k = 0; k < NS; ++k) v[k][u] = ldg4(xp[k] + (size_t)rr * gm.C);
          q[u] = ldg4(gd + (size_t)rr * gm.C);
          if constexpr (D2) q2[u] = ldg4(gd2 + (size_t)rr * gm.C);
        }
      }
      if constexpr (D2) {
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
          if (r + u * t.rpi < rows) { q[u].x += q2[u].x; q[u].y += q2[u].y; q[u].z += q2[u].z; q[u].w += q2[u].w; }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const unsigned rr = r + u * t.rpi;
        if (rr < rows) {
          const float ge[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
#pragma unroll
          for (int k = 0; k < NS; ++k) {
            const float e[4] = {v[k][u].x, v[k][u].y, v[k][u].z, v[k][u].w};
            float o[4];
#pragma unroll
            for (int s = 0; s < S::NSUB; ++s) {
              float xi[GS], dz[GS];
#pragma unroll
              for (int c = 0; c < GS; ++c) { xi[c] = e[s * GS + c]; dz[c] = ge[s * GS + c]; }
              if constexpr (RELU) {
                float oi[GS];
                apply_group<GS>(Wp[s], bp[s], xi, oi);
#pragma unroll
                for (int c = 0; c < GS; ++c) dz[c] = oi[c] > 0.f ? dz[c] : 0.f;
              }
              cf[k][s].apply(dz, xi, o + s * GS);
            }
            *reinterpret_cast<float4*>(op[k] + (size_t)rr * gm.C) = make_float4(o[0], o[1], o[2], o[3]);
          }
        }
      }
    });
  }
}

#define CL_GS(GS_, ...)                                  \
  switch (GS_) {                                         \
    case 1: { constexpr int kGS = 1; __VA_ARGS__; break; } \
    case 2: { constexpr int kGS = 2; __VA_ARGS__; break; } \
    case 4: { constexpr int kGS = 4; __VA_ARGS__; break; } \
    default: break;                                      \
  }
#define CL_EPI(E_, ...)                                                   \
  if ((E_) == 3) { constexpr int kEPI = 3; __VA_ARGS__; }                 \
  else if ((E_) == 1) { constexpr int kEPI = 1; __VA_ARGS__; }            \
  else { constexpr int kEPI = 0; __VA_ARGS__; }
// backward reduction: 7 = AFFINE with the ReLU mask of the residual tail read from the forward's byte map
#define CL_EPI_BWD(E_, ...)                                               \
  if ((E_) == 7) { constexpr int kEPI = 7; __VA_ARGS__; }                 \
  else CL_EPI(E_, __VA_ARGS__)
#define CL_D2(P_, ...)                                                    \
  if (P_) { constexpr bool kD2 = true; __VA_ARGS__; }                     \
  else { constexpr bool kD2 = false; __VA_ARGS__; }

inline bool use_pdl() {
  static const bool on = [] { const char* v = getenv("DWT_PDL"); return v != nullptr && v[0] == '1'; }();
  return on;
}

// ordinary launch, or (pdl) with programmatic stream serialization: see pdl_wait() above
template <class... KArgs, class... Args>
inline void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// grid.x = CTAs sweeping one domain, grid.y = column slabs, grid.z = 1 (domains one after the other) or D
inline dim3 cl_grid(const Geom& gm, int nctas, int gz) {
  const int C4 = gm.C / 4, CW = C4 < kT ? C4 : kT;
  return dim3(nctas, C4 / CW, gz);
}

}  // namespace

// C/4 must be a power of two (every thread keeps one float4 column for the whole kernel)
bool cl_supports(int C, int GS) {
  if (!(GS == 1 || GS == 2 || GS == 4) || C % 4 != 0) return false;
  const int c4 = C / 4;
  return (c4 & (c4 - 1)) == 0 && c4 <= 16384;
}
int cl_fwd_width(int C, int GS) { return (C / 4) * (4 / GS) * (GS + GS * (GS + 1) / 2); }
int cl_bwd_width(int C, int GS) { return (C / 4) * (4 / GS) * (GS * GS + GS); }


void cl_stats(const float* x, const Geom& gm, int nctas, int gz, float* partial, float* shift, cudaStream_t st) {
  CL_GS(gm.GS, (cl_stats_kernel<kGS><<<cl_grid(gm, nctas, gz), kT, 0, st>>>(x, gm, partial, shift)));
}
inline dim3 fin_block(const Geom& gm) { const int c4 = gm.C / 4; return dim3(32, c4 < kFinQ ? c4 : kFinQ, gm.D); }
void cl_fwd_finalize(const float* partial, int nrows, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st,
                     const FwdFin* fin2, size_t pstride, size_t sstride) {
  const dim3 b = fin_block(gm), g((gm.C / 4) / b.y, fin2 ? 2 : 1);
  CL_GS(gm.GS, (launch_k(cl_fwd_finalize_kernel<kGS>, g, b, st, use_pdl(), partial, pstride, nrows, shift, sstride, gm, fin, fin2 ? *fin2 : fin)));
}
void cl_apply(const float* x, float* y, const Geom& gm, int nctas, int gz, int epi, const float* mean, const float* w,
              const float* gamma, const float* beta, const float* residual, uint8_t* mask, cudaStream_t st) {
  const float* nul = nullptr;
  if (epi == 7) {
    CL_GS(gm.GS, (launch_k(cl_apply_kernel<kGS, 7, false>, cl_grid(gm, nctas, gz), dim3(kT), st, use_pdl(), x, y, gm, mean, w, gamma, beta, residual, mask,
                           nul, nul, nul, nul)));
    return;
  }
  CL_GS(gm.GS, CL_EPI(epi, (launch_k(cl_apply_kernel<kGS, kEPI, false>, cl_grid(gm, nctas, gz), dim3(kT), st, use_pdl(), x, y, gm, mean, w, gamma, beta,
                                     nul, (uint8_t*)nullptr, nul, nul, nul, nul))));
}
void cl_tail2_apply(const float* x, const float* xd, float* y, const Geom& gm, int nctas, int gz, const float* mean, const float* w,
                    const float* gamma, const float* beta, const float* mean_d, const float* w_d, const float* gamma_d,
                    const float* beta_d, uint8_t* mask, cudaStream_t st) {
  CL_GS(gm.GS, (launch_k(cl_apply_kernel<kGS, 7, true>, cl_grid(gm, nctas, gz), dim3(kT), st, use_pdl(), x, y, gm, mean, w, gamma, beta, xd, mask,
                         mean_d, w_d, gamma_d, beta_d)));
}
void cl_bwd_reduce(const float* x, const float* dout, const float* dout2, const Geom& gm, int nctas, int gz, int epi, const float* mean, const float* w,
                   const float* gamma, const float* beta, const uint8_t* mask, float* dz, float* partial, cudaStream_t st) {
  const float* nul = nullptr;
  CL_GS(gm.GS, CL_D2(dout2, CL_EPI_BWD(epi, (cl_bwd_reduce_kernel<kGS, kEPI, kD2, false><<<cl_grid(gm, nctas, gz), kT, 0, st>>>(
                                                x, dout, dout2, gm, mean, w, gamma, beta, mask, dz, partial, nul, nul, 0)))));
}
void cl_tail2_bwd_reduce(const float* x, const float* xd, const float* dout, const float* dout2, const Geom& gm, int nctas, int gz,
                         const float* mean, const float* mean_d, const uint8_t* mask, float* dz, float* partial, size_t pstride,
                         cudaStream_t st) {
  const float* nul = nullptr;
  CL_GS(gm.GS, CL_D2(dout2, (cl_bwd_reduce_kernel<kGS, 7, kD2, true><<<cl_grid(gm, nctas, gz), kT, 0, st>>>(
                                x, dout, dout2, gm, mean, nul, nul, nul, mask, dz, partial, xd, mean_d, pstride))));
}
void cl_bwd_finalize(const float* partial, int nrows, const Geom& gm, const BwdFin& fin, cudaStream_t st, const BwdFin* fin2, size_t pstride) {
  const dim3 b = fin_block(gm), g((gm.C / 4) / b.y, fin2 ? 2 : 1);
  CL_GS(gm.GS, (launch_k(cl_bwd_finalize_kernel<kGS>, g, b, st, use_pdl(), partial, pstride, nrows, gm, fin, fin2 ? *fin2 : fin)));
}
void cl_bwd_apply(const float* x, const float* dout, const float* dout2, float* dx, const Geom& gm, int nctas, int gz, int epi, const float* coef,
                  const float* mean, const float* w, const float* gamma, const float* beta, cudaStream_t st) {
  const float* nul = nullptr;
  CL_GS(gm.GS, CL_D2(dout2, CL_EPI(epi, (launch_k(cl_bwd_apply_kernel<kGS, kEPI, kD2, false>, cl_grid(gm, nctas, gz), dim3(kT), st, use_pdl(), x, dout,
                                                  dout2, dx, gm, coef, mean, w, gamma, beta, nul, (float*)nullptr, nul)))));
}
void cl_tail2_bwd_apply(const float* x, const float* xd, const float* dz, float* dx, float* dxd, const Geom& gm, int nctas, int gz,
                        const float* coef, const float* coef_d, cudaStream_t st) {
  const float* nul = nullptr;
  CL_GS(gm.GS, (launch_k(cl_bwd_apply_kernel<kGS, 1, false, true>, cl_grid(gm, nctas, gz), dim3(kT), st, use_pdl(), x, dz, nul, dx, gm, coef,
                         nul, nul, nul, nul, xd, dxd, coef_d)));
}

}  // namespace dwt

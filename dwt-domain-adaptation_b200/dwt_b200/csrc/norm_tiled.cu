// Shared-memory tiled path for any group size up to 64 (the general-shape path: group
// sizes the register-resident kernels do not cover, and shapes the TMA/wgmma kernels
// cannot take, e.g. H*W not a multiple of 4).
//
// The flattened sample axis m = n*HW + p is cut into tiles of TP samples; a CTA stages a
// [GS x TP] tile in shared memory (global reads coalesced along p, next tile prefetched
// into registers while the current one is consumed) and every thread owns a 4x4 register
// block of the small dense product:
//   stats       G  = sum (x-K)(x-K)^T            tile stored sample-major  (float4 = 4 channels)
//   bwd_reduce  R  = sum dy (x-mean)^T           two sample-major tiles
//   apply       y  = W x + b                     tile stored channel-major (float4 = 4 samples)
//   bwd_apply   dx = A1 dy + Bm x + cvec         two channel-major tiles
// Finalize steps are the shared block-cooperative routines of dwt_common.cuh.
//
// Reference: utils/whitening.py:37-61 (/root/reference).
#include "dwt_common.cuh"
#include "norm_launch.h"

namespace dwt {
namespace {

constexpr int TP = 128;            // samples per tile
constexpr int kPre = TP * DWT_MAX_GROUP_SIZE / kThreads;   // prefetch registers per thread (32)

__device__ __forceinline__ int round4(int v) { return (v + 3) & ~3; }

// global address of channel c (within the group), flattened sample m
struct TileSrc {
  const float* base;   // domain + group base
  int HW;
  size_t img_stride;   // C*HW
  __device__ __forceinline__ const float* at(int c, unsigned m) const {
    unsigned n = m / (unsigned)HW, p = m - n * (unsigned)HW;
    return base + (size_t)n * img_stride + (size_t)c * HW + p;
  }
};

// Prefetch one [GS x TP] tile into registers.  VEC=4: thread slots are float4 (4 samples).
template <int VEC>
__device__ __forceinline__ void tile_prefetch(const TileSrc& src, int GS, int GSP, unsigned m0, unsigned Mtot,
                                              float fill_unused, float (&pre)[kPre]) {
  constexpr int SLOTS = kPre / VEC;
  const int per_row = TP / VEC;
#pragma unroll
  for (int k = 0; k < SLOTS; ++k) {
    const int idx = threadIdx.x + k * kThreads;
    const int c = idx / per_row, q = idx - c * per_row;
    const unsigned m = m0 + q * VEC;
    if (c < GSP) {
      if (c < GS && m < Mtot) {
        if constexpr (VEC == 4) {
          float4 t = __ldg(reinterpret_cast<const float4*>(src.at(c, m)));
          pre[k * 4 + 0] = t.x; pre[k * 4 + 1] = t.y; pre[k * 4 + 2] = t.z; pre[k * 4 + 3] = t.w;
        } else {
          pre[k] = __ldg(src.at(c, m));
        }
      } else {
#pragma unroll
        for (int e = 0; e < VEC; ++e) pre[k * VEC + e] = fill_unused;
      }
    }
  }
}

// Store the prefetched tile sample-major: sT[m][c] = pre - shift[c] (0 outside the valid range).
template <int VEC>
__device__ __forceinline__ void tile_store_sample_major(float* sT, int LDT, const float* sShift, int GS, int GSP,
                                                        unsigned m0, unsigned Mtot, const float (&pre)[kPre]) {
  constexpr int SLOTS = kPre / VEC;
  const int per_row = TP / VEC;
#pragma unroll
  for (int k = 0; k < SLOTS; ++k) {
    const int idx = threadIdx.x + k * kThreads;
    const int c = idx / per_row, q = idx - c * per_row;
    if (c < GSP) {
      const float sh = (c < GS && sShift != nullptr) ? sShift[c] : 0.f;
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const unsigned m = m0 + q * VEC + e;
        sT[(q * VEC + e) * LDT + c] = (c < GS && m < Mtot) ? pre[k * VEC + e] - sh : 0.f;
      }
    }
  }
}

// Store channel-major: sX[c][m] = pre (0 outside).
template <int VEC>
__device__ __forceinline__ void tile_store_channel_major(float* sX, int LDX, int GS, int GSP, unsigned m0,
                                                         unsigned Mtot, const float (&pre)[kPre]) {
  constexpr int SLOTS = kPre / VEC;
  const int per_row = TP / VEC;
#pragma unroll
  for (int k = 0; k < SLOTS; ++k) {
    const int idx = threadIdx.x + k * kThreads;
    const int c = idx / per_row, q = idx - c * per_row;
    if (c < GSP) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const unsigned m = m0 + q * VEC + e;
        sX[c * LDX + q * VEC + e] = (c < GS && m < Mtot) ? pre[k * VEC + e] : 0.f;
      }
    }
  }
}

// acc[a][b] += sum_p A[p][4bi+a] * B[p][4bj+b] over this thread's sample slice
__device__ __forceinline__ void outer_accumulate(const float* sA, const float* sB, int LDT, int bi, int bj, int slice,
                                                 int nslices, float (&acc)[4][4], float (&rowsum)[4], bool do_sum) {
  for (int p = slice; p < TP; p += nslices) {
    const float4 a = *reinterpret_cast<const float4*>(sA + p * LDT + 4 * bi);
    const float4 b = *reinterpret_cast<const float4*>(sB + p * LDT + 4 * bj);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (do_sum) rowsum[i] += av[i];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
}

// Shared layout (floats) used by both reduction kernels; finalize scratch aliases the tiles.
struct ReduceSmem {
  int GSP, LDT, nB, nblk, nslices;
  __device__ ReduceSmem(int GS) {
    GSP = round4(GS); LDT = GSP + 4; nB = GSP / 4; nblk = nB * nB;
    nslices = kThreads / nblk; if (nslices < 1) nslices = 1;
  }
};

// Sum the per-thread 4x4 blocks over sample slices in a fixed order and emit the CTA's
// partial row: [GS*GS matrix | GS vector].  sScratch must hold nslices*(GSP*GSP+GSP) floats.
__device__ __forceinline__ void emit_partial(const ReduceSmem& L, int GS, const float (&acc)[4][4],
                                             const float (&rowsum)[4], bool active, int bi, int bj, int slice,
                                             float* sScratch, float* prow) {
  const int GSP = L.GSP, per = GSP * GSP + GSP;
  __syncthreads();     // tiles no longer needed; scratch may alias them
  if (active) {
    float* dst = sScratch + slice * per;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int j = 0; j < 4; ++j) dst[(4 * bi + i) * GSP + 4 * bj + j] = acc[i][j];
      if (bj == 0) dst[GSP * GSP + 4 * bi + i] = rowsum[i];
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < GS * GS + GS; e += kThreads) {
    int src;
    if (e < GS * GS) { int i = e / GS, j = e - i * GS; src = i * GSP + j; }
    else src = GSP * GSP + (e - GS * GS);
    float t = 0.f;
    for (int s = 0; s < L.nslices; ++s) t += sScratch[s * per + src];
    prow[e] = t;
  }
}

// ------------------------------------------------------------------------------------------
// stats
// ------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(kThreads) tiled_stats_kernel(const float* __restrict__ x, Geom gm, FwdFin fin,
                                                                float* __restrict__ partial, int* counters) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float sK[DWT_MAX_GROUP_SIZE];
  __shared__ int sFlag;
  const int GS = gm.GS, g = blockIdx.y, d = blockIdx.z, tid = threadIdx.x;
  const ReduceSmem L(GS);
  const TileSrc src{x + ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW, gm.HW, (size_t)gm.C * gm.HW};
  pilot_shift(src.base, GS, gm.HW, sK);
  __syncthreads();
  const unsigned Mtot = (unsigned)gm.N * gm.HW, ntiles = (Mtot + TP - 1) / TP;
  const int blk = tid % L.nblk, slice = tid / L.nblk;
  const bool active = slice < L.nslices;
  const int bi = blk / L.nB, bj = blk % L.nB;
  float acc[4][4] = {}, rowsum[4] = {};
  float pre[kPre];
  float* sT = smem;
  unsigned t = blockIdx.x;
  if (t < ntiles) tile_prefetch<VEC>(src, GS, L.GSP, t * TP, Mtot, 0.f, pre);
  for (; t < ntiles; t += gridDim.x) {
    tile_store_sample_major<VEC>(sT, L.LDT, sK, GS, L.GSP, t * TP, Mtot, pre);
    __syncthreads();
    if (t + gridDim.x < ntiles) tile_prefetch<VEC>(src, GS, L.GSP, (t + gridDim.x) * TP, Mtot, 0.f, pre);
    if (active) outer_accumulate(sT, sT, L.LDT, bi, bj, slice, L.nslices, acc, rowsum, bj == 0);
    __syncthreads();
  }
  const int nacc = GS * GS + GS;
  float* prow = partial + (((size_t)d * gm.G + g) * gm.nchunks + blockIdx.x) * nacc;
  emit_partial(L, GS, acc, rowsum, active, bi, bj, slice, smem, prow);
  if (!arrive_is_last(counters + d * gm.G + g, gm.nchunks, &sFlag)) return;

  const int LD = GS + 1;
  float* sAcc = smem;                 // [GS*GS + GS]
  float* sMean = sAcc + nacc;         // [GS]
  float* sCov = sMean + GS;           // [GS*LD]
  float* sL = sCov + GS * LD;
  float* sW = sL + GS * LD;
  __syncthreads();
  reduce_partials(partial + ((size_t)d * gm.G + g) * gm.nchunks * nacc, gm.nchunks, nacc, sAcc);
  __syncthreads();
  const float invM = 1.f / gm.M;
  for (int i = tid; i < GS; i += kThreads) sMean[i] = sK[i] + sAcc[GS * GS + i] * invM;
  for (int e = tid; e < GS * GS; e += kThreads) {
    int i = e / GS, j = e - i * GS;
    // the two triangles were accumulated in different orders; use the lower one for both
    int hi = i > j ? i : j, lo = i > j ? j : i;
    sCov[i * LD + j] = sAcc[hi * GS + lo] * invM - (sAcc[GS * GS + i] * invM) * (sAcc[GS * GS + j] * invM);
  }
  __syncthreads();
  fwd_factor_block(gm, fin, d, g, sMean, sCov, sL, sW, true);
  fwd_ema_block(gm, fin, g, &sFlag);
}

__global__ void __launch_bounds__(kThreads) tiled_eval_prep_kernel(Geom gm, FwdFin fin) {
  extern __shared__ __align__(16) float smem[];
  const int GS = gm.GS, LD = GS + 1, g = blockIdx.y, d = blockIdx.z, tid = threadIdx.x;
  float* sMean = smem;
  float* sCov = sMean + GS;
  float* sL = sCov + GS * LD;
  float* sW = sL + GS * LD;
  for (int i = tid; i < GS; i += kThreads) sMean[i] = fin.rmean[d][g * GS + i];
  for (int e = tid; e < GS * GS; e += kThreads) sCov[(e / GS) * LD + e % GS] = fin.rcov[d][(size_t)g * GS * GS + e];
  __syncthreads();
  fwd_factor_block(gm, fin, d, g, sMean, sCov, sL, sW, false);
}

// ------------------------------------------------------------------------------------------
// backward reduce:  R = sum dy (x - mean)^T ,  sdz = sum dy
// ------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(kThreads) tiled_bwd_reduce_kernel(const float* __restrict__ x,
                                                                     const float* __restrict__ dout, Geom gm,
                                                                     BwdFin fin, float* __restrict__ partial,
                                                                     int* counters) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float sMu[DWT_MAX_GROUP_SIZE];
  __shared__ int sFlag;
  const int GS = gm.GS, g = blockIdx.y, d = blockIdx.z, tid = threadIdx.x;
  const ReduceSmem L(GS);
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const TileSrc srcx{x + base, gm.HW, (size_t)gm.C * gm.HW}, srcg{dout + base, gm.HW, (size_t)gm.C * gm.HW};
  for (int i = tid; i < GS; i += kThreads) sMu[i] = fin.save_mean[(size_t)d * gm.C + g * GS + i];
  __syncthreads();
  const unsigned Mtot = (unsigned)gm.N * gm.HW, ntiles = (Mtot + TP - 1) / TP;
  const int blk = tid % L.nblk, slice = tid / L.nblk;
  const bool active = slice < L.nslices;
  const int bi = blk / L.nB, bj = blk % L.nB;
  float acc[4][4] = {}, rowsum[4] = {};
  float prex[kPre], preg[kPre];
  float* sX = smem;
  float* sG = smem + TP * L.LDT;
  unsigned t = blockIdx.x;
  if (t < ntiles) {
    tile_prefetch<VEC>(srcx, GS, L.GSP, t * TP, Mtot, 0.f, prex);
    tile_prefetch<VEC>(srcg, GS, L.GSP, t * TP, Mtot, 0.f, preg);
  }
  for (; t < ntiles; t += gridDim.x) {
    tile_store_sample_major<VEC>(sX, L.LDT, sMu, GS, L.GSP, t * TP, Mtot, prex);
    tile_store_sample_major<VEC>(sG, L.LDT, nullptr, GS, L.GSP, t * TP, Mtot, preg);
    __syncthreads();
    if (t + gridDim.x < ntiles) {
      tile_prefetch<VEC>(srcx, GS, L.GSP, (t + gridDim.x) * TP, Mtot, 0.f, prex);
      tile_prefetch<VEC>(srcg, GS, L.GSP, (t + gridDim.x) * TP, Mtot, 0.f, preg);
    }
    if (active) outer_accumulate(sG, sX, L.LDT, bi, bj, slice, L.nslices, acc, rowsum, bj == 0);
    __syncthreads();
  }
  const int nacc = GS * GS + GS;
  float* prow = partial + (((size_t)d * gm.G + g) * gm.nchunks + blockIdx.x) * nacc;
  emit_partial(L, GS, acc, rowsum, active, bi, bj, slice, smem, prow);
  if (!arrive_is_last(counters + d * gm.G + g, gm.nchunks, &sFlag)) return;

  const int LD = GS + 1;
  float* sAcc = smem;
  float* sR = sAcc + nacc;
  float* sSdz = sR + GS * LD;
  float* sW = sSdz + GS;
  float* sT1 = sW + GS * LD;
  float* sT2 = sT1 + GS * LD;
  float* sVec = sT2 + GS * LD;
  __syncthreads();
  reduce_partials(partial + ((size_t)d * gm.G + g) * gm.nchunks * nacc, gm.nchunks, nacc, sAcc);
  __syncthreads();
  for (int e = tid; e < GS * GS; e += kThreads) sR[(e / GS) * LD + e % GS] = sAcc[e];
  for (int i = tid; i < GS; i += kThreads) sSdz[i] = sAcc[GS * GS + i];
  __syncthreads();
  bwd_finalize_block(gm, fin, d, g, sR, sSdz, sW, sT1, sT2, sVec, &sFlag);
}

__global__ void __launch_bounds__(kThreads) tiled_bwd_prep_kernel(Geom gm, BwdFin fin) {
  extern __shared__ __align__(16) float smem[];
  __shared__ int sFlag;
  const int GS = gm.GS, LD = GS + 1;
  float* sR = smem;
  float* sSdz = sR + GS * LD;
  float* sW = sSdz + GS;
  float* sT1 = sW + GS * LD;
  float* sT2 = sT1 + GS * LD;
  float* sVec = sT2 + GS * LD;
  for (int e = threadIdx.x; e < GS * LD + GS; e += kThreads) smem[e] = 0.f;
  __syncthreads();
  bwd_finalize_block(gm, fin, blockIdx.z, blockIdx.y, sR, sSdz, sW, sT1, sT2, sVec, &sFlag);
}

// ------------------------------------------------------------------------------------------
// apply kernels: out[c][m] = bias[c] + sum_j M1[c][j] in1[j][m] (+ sum_j M2[c][j] in2[j][m])
// Each thread owns 4 channels x 4 samples; matrices are kept transposed in shared memory
// (sMt[j][c]) so the 4 channel weights of one input row are a single float4.
// ------------------------------------------------------------------------------------------
template <int VEC, bool TWO>
__device__ __forceinline__ void tile_matmul_store(const float* sM1t, const float* sM2t, const float* sBias,
                                                  const float* sX1, const float* sX2, int LDM, int LDX, int GS,
                                                  int GSP, bool lower1, const TileSrc& dst_like, float* out_base,
                                                  unsigned m0, unsigned Mtot) {
  const int nB = GSP / 4, nq = TP / 4;
  for (int item = threadIdx.x; item < nB * nq; item += kThreads) {
    const int cb = item / nq, pq = item - cb * nq;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float b = sBias[4 * cb + i];
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][e] = b;
    }
    // M1 is triangular: lower1 -> columns j <= c ; else (upper) columns j >= c
    const int j1lo = lower1 ? 0 : 4 * cb, j1hi = lower1 ? 4 * cb + 4 : GSP;
    for (int j = j1lo; j < j1hi; ++j) {
      const float4 w = *reinterpret_cast<const float4*>(sM1t + j * LDM + 4 * cb);
      const float4 v = *reinterpret_cast<const float4*>(sX1 + j * LDX + 4 * pq);
      const float wv[4] = {w.x, w.y, w.z, w.w}, xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][e] = fmaf(wv[i], xv[e], acc[i][e]);
    }
    if constexpr (TWO) {
      for (int j = 0; j < GSP; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(sM2t + j * LDM + 4 * cb);
        const float4 v = *reinterpret_cast<const float4*>(sX2 + j * LDX + 4 * pq);
        const float wv[4] = {w.x, w.y, w.z, w.w}, xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[i][e] = fmaf(wv[i], xv[e], acc[i][e]);
      }
    }
    const unsigned m = m0 + 4 * pq;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = 4 * cb + i;
      if (c < GS) {
        if (VEC == 4) {
          if (m < Mtot) {
            float* p = out_base + (dst_like.at(c, m) - dst_like.base);
            *reinterpret_cast<float4*>(p) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
          }
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (m + e < Mtot) out_base[dst_like.at(c, m + e) - dst_like.base] = acc[i][e];
        }
      }
    }
  }
}

// load a GSxGS row-major global matrix transposed into shared (sMt[j][c] = M[c][j]), zero padded
__device__ __forceinline__ void load_matrix_T(const float* gM, float* sMt, int GS, int GSP, int LDM) {
  for (int e = threadIdx.x; e < GSP * GSP; e += kThreads) {
    int c = e / GSP, j = e - c * GSP;
    sMt[j * LDM + c] = (c < GS && j < GS) ? __ldg(gM + c * GS + j) : 0.f;
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads) tiled_apply_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                Geom gm, const float* __restrict__ save_mean,
                                                                const float* __restrict__ save_w) {
  extern __shared__ __align__(16) float smem[];
  const int GS = gm.GS, GSP = round4(GS), LDM = GSP + 4, LDX = TP + 4;
  const int g = blockIdx.y, d = blockIdx.z, tid = threadIdx.x;
  float* sWt = smem;                 // [GSP][LDM]
  float* sBias = sWt + GSP * LDM;    // [GSP]
  float* sX = sBias + GSP;           // [GSP][LDX]
  const float* wg = save_w + ((size_t)d * gm.G + g) * GS * GS;
  const float* mg = save_mean + (size_t)d * gm.C + g * GS;
  load_matrix_T(wg, sWt, GS, GSP, LDM);
  for (int c = tid; c < GSP; c += kThreads) {
    float b = 0.f;
    if (c < GS)
      for (int j = 0; j <= c; ++j) b = fmaf(-__ldg(wg + c * GS + j), __ldg(mg + j), b);
    sBias[c] = b;
  }
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const TileSrc src{x + base, gm.HW, (size_t)gm.C * gm.HW};
  const unsigned Mtot = (unsigned)gm.N * gm.HW, ntiles = (Mtot + TP - 1) / TP;
  float pre[kPre];
  unsigned t = blockIdx.x;
  if (t < ntiles) tile_prefetch<VEC>(src, GS, GSP, t * TP, Mtot, 0.f, pre);
  for (; t < ntiles; t += gridDim.x) {
    __syncthreads();     // previous tile fully consumed (also orders the sWt/sBias fill)
    tile_store_channel_major<VEC>(sX, LDX, GS, GSP, t * TP, Mtot, pre);
    __syncthreads();
    if (t + gridDim.x < ntiles) tile_prefetch<VEC>(src, GS, GSP, (t + gridDim.x) * TP, Mtot, 0.f, pre);
    tile_matmul_store<VEC, false>(sWt, nullptr, sBias, sX, nullptr, LDM, LDX, GS, GSP, true, src, y + base, t * TP,
                                  Mtot);
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads) tiled_bwd_apply_kernel(const float* __restrict__ x,
                                                                    const float* __restrict__ dout,
                                                                    float* __restrict__ dx, Geom gm,
                                                                    const float* __restrict__ coef) {
  extern __shared__ __align__(16) float smem[];
  const int GS = gm.GS, GSP = round4(GS), LDM = GSP + 4, LDX = TP + 4;
  const int g = blockIdx.y, d = blockIdx.z, tid = threadIdx.x;
  float* sA1t = smem;
  float* sBmt = sA1t + GSP * LDM;
  float* sBias = sBmt + GSP * LDM;
  float* sG = sBias + GSP;           // dy tile, channel-major
  float* sX = sG + GSP * LDX;
  const float* cf = coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  load_matrix_T(cf, sA1t, GS, GSP, LDM);
  load_matrix_T(cf + GS * GS, sBmt, GS, GSP, LDM);
  for (int c = tid; c < GSP; c += kThreads) sBias[c] = c < GS ? __ldg(cf + 2 * GS * GS + c) : 0.f;
  const size_t base = ((size_t)d * gm.N * gm.C + (size_t)g * GS) * gm.HW;
  const TileSrc srcx{x + base, gm.HW, (size_t)gm.C * gm.HW}, srcg{dout + base, gm.HW, (size_t)gm.C * gm.HW};
  const unsigned Mtot = (unsigned)gm.N * gm.HW, ntiles = (Mtot + TP - 1) / TP;
  float prex[kPre], preg[kPre];
  unsigned t = blockIdx.x;
  if (t < ntiles) {
    tile_prefetch<VEC>(srcx, GS, GSP, t * TP, Mtot, 0.f, prex);
    tile_prefetch<VEC>(srcg, GS, GSP, t * TP, Mtot, 0.f, preg);
  }
  for (; t < ntiles; t += gridDim.x) {
    __syncthreads();
    tile_store_channel_major<VEC>(sX, LDX, GS, GSP, t * TP, Mtot, prex);
    tile_store_channel_major<VEC>(sG, LDX, GS, GSP, t * TP, Mtot, preg);
    __syncthreads();
    if (t + gridDim.x < ntiles) {
      tile_prefetch<VEC>(srcx, GS, GSP, (t + gridDim.x) * TP, Mtot, 0.f, prex);
      tile_prefetch<VEC>(srcg, GS, GSP, (t + gridDim.x) * TP, Mtot, 0.f, preg);
    }
    tile_matmul_store<VEC, true>(sA1t, sBmt, sBias, sG, sX, LDM, LDX, GS, GSP, false, srcx, dx + base, t * TP, Mtot);
  }
}

// shared memory sizing ---------------------------------------------------------------------
int reduce_smem_floats(int GS, int ntile_bufs) {
  const int GSP = (GS + 3) & ~3, LDT = GSP + 4, LD = GS + 1;
  int nblk = (GSP / 4) * (GSP / 4);
  int nslices = kThreads / nblk; if (nslices < 1) nslices = 1;
  int tiles = ntile_bufs * TP * LDT;
  int scratch = nslices * (GSP * GSP + GSP);
  int fin_fwd = (GS * GS + GS) + GS + 3 * GS * LD;
  int fin_bwd = (GS * GS + GS) + 4 * GS * LD + GS + 3 * GS;
  int m = tiles;
  if (scratch > m) m = scratch;
  if (fin_fwd > m) m = fin_fwd;
  if (fin_bwd > m) m = fin_bwd;
  return m;
}
int apply_smem_floats(int GS, int nmat) {
  const int GSP = (GS + 3) & ~3, LDM = GSP + 4, LDX = TP + 4;
  return nmat * GSP * LDM + GSP + nmat * GSP * LDX;
}

}  // namespace

int tiled_init() {
  const int big = 200 * 1024;
  cudaError_t e = cudaSuccess;
#define DWT_SET(k) if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, big)
  DWT_SET(tiled_stats_kernel<1>); DWT_SET(tiled_stats_kernel<4>);
  DWT_SET(tiled_bwd_reduce_kernel<1>); DWT_SET(tiled_bwd_reduce_kernel<4>);
  DWT_SET(tiled_apply_kernel<1>); DWT_SET(tiled_apply_kernel<4>);
  DWT_SET(tiled_bwd_apply_kernel<1>); DWT_SET(tiled_bwd_apply_kernel<4>);
  DWT_SET(tiled_eval_prep_kernel); DWT_SET(tiled_bwd_prep_kernel);
#undef DWT_SET
  return (int)e;
}

void tiled_stats(const float* x, const Geom& gm, int vec, const FwdFin& fin, float* partial, int* counters,
                 cudaStream_t st) {
  const size_t sm = sizeof(float) * reduce_smem_floats(gm.GS, 1);
  dim3 grid(gm.nchunks, gm.G, gm.D);
  if (vec == 4) tiled_stats_kernel<4><<<grid, kThreads, sm, st>>>(x, gm, fin, partial, counters);
  else tiled_stats_kernel<1><<<grid, kThreads, sm, st>>>(x, gm, fin, partial, counters);
}

void tiled_eval_prep(const Geom& gm, const FwdFin& fin, cudaStream_t st) {
  const size_t sm = sizeof(float) * reduce_smem_floats(gm.GS, 0);
  tiled_eval_prep_kernel<<<dim3(1, gm.G, gm.D), kThreads, sm, st>>>(gm, fin);
}

void tiled_apply(const float* x, float* y, const Geom& gm, int vec, int chunks, const float* mean, const float* w,
                 cudaStream_t st) {
  const size_t sm = sizeof(float) * apply_smem_floats(gm.GS, 1);
  dim3 grid(chunks, gm.G, gm.D);
  if (vec == 4) tiled_apply_kernel<4><<<grid, kThreads, sm, st>>>(x, y, gm, mean, w);
  else tiled_apply_kernel<1><<<grid, kThreads, sm, st>>>(x, y, gm, mean, w);
}

void tiled_bwd_reduce(const float* x, const float* dout, const Geom& gm, int vec, const BwdFin& fin, float* partial,
                      int* counters, cudaStream_t st) {
  const size_t sm = sizeof(float) * reduce_smem_floats(gm.GS, 2);
  dim3 grid(gm.nchunks, gm.G, gm.D);
  if (vec == 4) tiled_bwd_reduce_kernel<4><<<grid, kThreads, sm, st>>>(x, dout, gm, fin, partial, counters);
  else tiled_bwd_reduce_kernel<1><<<grid, kThreads, sm, st>>>(x, dout, gm, fin, partial, counters);
}

void tiled_bwd_prep(const Geom& gm, const BwdFin& fin, cudaStream_t st) {
  const size_t sm = sizeof(float) * reduce_smem_floats(gm.GS, 0);
  tiled_bwd_prep_kernel<<<dim3(1, gm.G, gm.D), kThreads, sm, st>>>(gm, fin);
}

void tiled_bwd_apply(const float* x, const float* dout, float* dx, const Geom& gm, int vec, int chunks,
                     const float* coef, cudaStream_t st) {
  const size_t sm = sizeof(float) * apply_smem_floats(gm.GS, 2);
  dim3 grid(chunks, gm.G, gm.D);
  if (vec == 4) tiled_bwd_apply_kernel<4><<<grid, kThreads, sm, st>>>(x, dout, dx, gm, coef);
  else tiled_bwd_apply_kernel<1><<<grid, kThreads, sm, st>>>(x, dout, dx, gm, coef);
}

}  // namespace dwt

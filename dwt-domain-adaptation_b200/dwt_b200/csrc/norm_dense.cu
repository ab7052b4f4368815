// Dense per-group algebra for large groups (8 <= gs <= 64) as separate, latency-tuned launches
// behind the tensor-core contraction:
//
//   partial_reduce   sum the per-CTA partial Gram matrices of a 64-channel super-block in fixed
//                    chunk order, spread over many CTAs (a single "last CTA" doing this alone would idle
//                    the rest of the grid)
//   fwd_factor       per group: mean, covariance, S = a*cov + b*I, Cholesky S = L L^T, W = L^-1,
//                    running-statistic EMA (domains in order: one CTA owns all domains of its group)
//   bwd_coef         per (domain, group): A1 = W^T, Bm = (2a/M) sym(W^T Phi(-R W^T) W), cvec
//
// All three keep a 64x64 problem in ONE 256-thread CTA arranged 16x16, each thread owning a 4x4
// register block.  fwd_factor runs the Cholesky factorisation AND the triangular inverse as one blocked
// right-looking sweep of 16 panel steps (one block barrier each): the matrices live in registers, shared
// memory only carries the 4-column panel of L and the 4-row panel of W of the current step.
//
// Reference: utils/whitening.py:47-53,57-59 (/root/reference); backward: SURVEY.md §8a.
#ifdef DWT_PROF_DENSE
#include <cstdio>
#endif
#include "dwt_common.cuh"
#include "norm_launch.h"

namespace dwt {
namespace {

constexpr int kSB = 64;                         // super-block edge
constexpr int kNacc = kSB * kSB + kSB;          // Gram + row sums
constexpr int LDS = kSB + 1;                    // padded leading dimension in shared memory
constexpr int kMat = kSB * LDS;                 // floats per shared matrix

// development: -DDWT_PROF_DENSE prints the clock of every phase of CTA 0 (build.py, DWT_NVCC_EXTRA)
#ifdef DWT_PROF_DENSE
#define PROF_DECL long long pt_[24]; int pn_ = 0
#define PROF_MARK() do { if (threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.z == 0 && pn_ < 24) pt_[pn_++] = clock64(); } while (0)
#define PROF_DUMP(name) do { if (threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.z == 0) { printf(name ":"); for (int q_ = 1; q_ < pn_; ++q_) printf(" %lld", pt_[q_] - pt_[q_ - 1]); printf("\n"); } } while (0)
#define PROF_ARGS , long long (&pt_)[24], int& pn_
#define PROF_PASS , pt_, pn_
#else
#define PROF_DECL
#define PROF_MARK()
#define PROF_DUMP(name)
#define PROF_ARGS
#define PROF_PASS
#endif

// ------------------------------------------------------------------------------------------
// partial_reduce: out[p][e] = sum_c partial[p][c][e]   (p = domain*SB + sb, fixed order over c)
// grid (ceil(kNacc/64), problems), 256 threads = 4 chunk-quarters x 64 elements
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) partial_reduce_kernel(const float* __restrict__ partial, int nchunks,
                                                             float* __restrict__ out) {
  __shared__ float sQ[4][64];
  const int l = threadIdx.x & 63, q = threadIdx.x >> 6;
  const int e = blockIdx.x * 64 + l, p = blockIdx.y;
  const float* base = partial + (size_t)p * nchunks * kNacc;
  const int c0 = (nchunks * q) / 4, c1 = (nchunks * (q + 1)) / 4;
  float acc = 0.f;
  if (e < kNacc) {
    int c = c0;
    for (; c + 4 <= c1; c += 4) {
      const float v0 = __ldcg(base + (size_t)(c + 0) * kNacc + e), v1 = __ldcg(base + (size_t)(c + 1) * kNacc + e);
      const float v2 = __ldcg(base + (size_t)(c + 2) * kNacc + e), v3 = __ldcg(base + (size_t)(c + 3) * kNacc + e);
      acc = (((acc + v0) + v1) + v2) + v3;
    }
    for (; c < c1; ++c) acc += __ldcg(base + (size_t)c * kNacc + e);
  }
  sQ[q][l] = acc;
  __syncthreads();
  if (q == 0 && e < kNacc) out[(size_t)p * kNacc + e] = ((sQ[0][l] + sQ[1][l]) + sQ[2][l]) + sQ[3][l];
}

// ------------------------------------------------------------------------------------------
// register-blocked helpers (256 threads as 16 x 16, thread (bi,bj) owns rows 4bi.., cols 4bj..)
// ------------------------------------------------------------------------------------------
struct Blk {
  int bi, bj;
  bool act;
  __device__ Blk(int GS) : bi(threadIdx.x >> 4), bj(threadIdx.x & 15) { act = 4 * bi < GS && 4 * bj < GS; }
};

// C = op(A) * op(B) on GS x GS matrices in shared memory (leading dimension LDS), result in registers.
// TA: use A^T ; TB: use B^T.  Structural zeros are simply stored zeros.
template <bool TA, bool TB>
__device__ __forceinline__ void mm_block(const float* A, const float* B, int GS, const Blk& t, float (&c)[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) c[r][s] = 0.f;
  if (!t.act) return;
  for (int k = 0; k < GS; ++k) {
    float a[4], b[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) a[r] = TA ? A[k * LDS + 4 * t.bi + r] : A[(4 * t.bi + r) * LDS + k];
#pragma unroll
    for (int s = 0; s < 4; ++s) b[s] = TB ? B[(4 * t.bj + s) * LDS + k] : B[k * LDS + 4 * t.bj + s];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) c[r][s] = fmaf(a[r], b[s], c[r][s]);
  }
}

__device__ __forceinline__ void store_block(float* M, const Blk& t, const float (&c)[4][4]) {
  if (!t.act) return;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) M[(4 * t.bi + r) * LDS + 4 * t.bj + s] = c[r][s];
}

// Blocked right-looking sweep: S = L L^T and W = L^-1 together, 4 columns per step, ONE block barrier per step.
//
//   a[r][s]  the SPD matrix, blocks held TRANSPOSED: element (i = 4*bj + s, j = 4*bi + r) -- for the symmetric input
//            the same numbers as the (bi, bj) block, so the caller fills it as if it were untransposed.  The 16 owners
//            of a COLUMN block (fixed bi) are one half-warp.
//   b[r][s]  the running inverse, element (i = 4*bi + r, j = 4*bj + s); starts as I, ends as W.  The 16 owners of a ROW
//            block are the same half-warp.
//
// Step k, in the half-warp bi == k: the diagonal thread factors its 4 x 4 block (4 square roots in one thread) and
// hands L11 and 1/diag to the other 15 by shuffle; every thread solves its 4 x 4 block of the panel L21 = A21 L11^-T and
// of the finished row block W_k = L11^-1 B_k and publishes both to shared memory (double-buffered).  After the barrier
// every thread applies the rank-4 updates  A -= L21 L21^T  (blocks at or below the diagonal of the trailing matrix)
// and  B -= L21 W_k  (rows below the panel, columns up to it).  16 steps replace 64 single-column steps (sqrt,
// reciprocal, broadcast and barrier per column) plus a separate recursive-doubling inverse through shared memory.
// Returns false on a non-positive pivot.
struct PanelSmem {
  float L[2][kSB][4];      // L[i][4k + p] of the current panel, 0 for rows i < 4k + 4
  float W[2][4][kSB];      // W[4k + p][j], the finished row block
};

__device__ __forceinline__ bool factor_and_invert(float (&a)[4][4], float (&b)[4][4], int GS, const Blk& t, PanelSmem& sp) {
  bool ok = true;
  const unsigned hmask = (threadIdx.x & 16) ? 0xFFFF0000u : 0x0000FFFFu;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) b[r][s] = (t.act && t.bi == t.bj && r == s) ? 1.f : 0.f;
  const int nsteps = GS >> 2;
  for (int k = 0; k < nsteps; ++k) {
    const int buf = k & 1;
    if (t.bi == k) {                                  // half-warp uniform
      // --- diagonal block: unblocked 4 x 4 Cholesky in the thread bj == k.  The other 15 run the same instructions on
      //     the identity (no divergence before the shuffles, and no special-case slow path of the square root on the
      //     arbitrary numbers of an off-diagonal block -- that cost 2000 cycles per step).  Only 1/diag(L11) is ever
      //     used (L itself is not an output): reciprocal square root + one Newton step, no square root, no division.
      float l[4][4], inv[4];                          // l[i][j], i >= j
      const bool diag = t.bj == k;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) l[i][j] = diag ? a[j][i] : (i == j ? 1.f : 0.f);
      bool pos = true;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const float x = l[p][p];
        pos = pos && (x > 0.f);
        const float y = rsqrtf(x);
        inv[p] = y * fmaf(-0.5f * x * y, y, 1.5f);   // y (3 - x y^2) / 2
#pragma unroll
        for (int i = p + 1; i < 4; ++i) l[i][p] *= inv[p];
#pragma unroll
        for (int j = p + 1; j < 4; ++j)
#pragma unroll
          for (int i = j; i < 4; ++i) l[i][j] = fmaf(-l[i][p], l[j][p], l[i][j]);
      }
      const int src = k;                              // lane of the diagonal thread inside the half-warp
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        inv[i] = __shfl_sync(hmask, inv[i], src, 16);
#pragma unroll
        for (int j = 0; j < i; ++j) l[i][j] = __shfl_sync(hmask, l[i][j], src, 16);
      }
      pos = __shfl_sync(hmask, pos ? 1 : 0, src, 16) != 0;
      ok = ok && pos;
      // --- panel of L: rows 4*bj + s, x L11^T = a  (forward substitution along the 4 columns)
      const bool below = t.bj > k;
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        float x0 = a[0][s] * inv[0];
        float x1 = fmaf(-x0, l[1][0], a[1][s]) * inv[1];
        float x2 = fmaf(-x1, l[2][1], fmaf(-x0, l[2][0], a[2][s])) * inv[2];
        float x3 = fmaf(-x2, l[3][2], fmaf(-x1, l[3][1], fmaf(-x0, l[3][0], a[3][s]))) * inv[3];
        if (!below) { x0 = x1 = x2 = x3 = 0.f; }
        *reinterpret_cast<float4*>(&sp.L[buf][4 * t.bj + s][0]) = make_float4(x0, x1, x2, x3);
      }
      // --- finished row block of W: L11 x = b  (columns 4*bj + s; zero right of the diagonal block by construction)
      float w[4][4];
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        w[0][s] = b[0][s] * inv[0];
        w[1][s] = fmaf(-l[1][0], w[0][s], b[1][s]) * inv[1];
        w[2][s] = fmaf(-l[2][1], w[1][s], fmaf(-l[2][0], w[0][s], b[2][s])) * inv[2];
        w[3][s] = fmaf(-l[3][2], w[2][s], fmaf(-l[3][1], w[1][s], fmaf(-l[3][0], w[0][s], b[3][s]))) * inv[3];
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int s = 0; s < 4; ++s) b[r][s] = w[r][s];
        *reinterpret_cast<float4*>(&sp.W[buf][r][4 * t.bj]) = make_float4(w[r][0], w[r][1], w[r][2], w[r][3]);
      }
    }
    __syncthreads();
    if (t.act && t.bi > k) {
      float li[4][4];                                 // panel rows 4*bi + r
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 v = *reinterpret_cast<const float4*>(&sp.L[buf][4 * t.bi + r][0]);
        li[r][0] = v.x; li[r][1] = v.y; li[r][2] = v.z; li[r][3] = v.w;
      }
      if (t.bj >= t.bi) {                             // a(i = 4bj+s, j = 4bi+r) -= sum_p L[i][p] L[j][p]
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const float4 v = *reinterpret_cast<const float4*>(&sp.L[buf][4 * t.bj + s][0]);
#pragma unroll
          for (int r = 0; r < 4; ++r)
            a[r][s] = fmaf(-v.w, li[r][3], fmaf(-v.z, li[r][2], fmaf(-v.y, li[r][1], fmaf(-v.x, li[r][0], a[r][s]))));
        }
      }
      if (t.bj <= k) {                                // b(i = 4bi+r, j = 4bj+s) -= sum_p L[i][p] W[p][j]
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float4 v = *reinterpret_cast<const float4*>(&sp.W[buf][p][4 * t.bj]);
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            b[r][0] = fmaf(-li[r][p], v.x, b[r][0]);
            b[r][1] = fmaf(-li[r][p], v.y, b[r][1]);
            b[r][2] = fmaf(-li[r][p], v.z, b[r][2]);
            b[r][3] = fmaf(-li[r][p], v.w, b[r][3]);
          }
        }
      }
    }
  }
  return ok;
}

// ------------------------------------------------------------------------------------------
// fwd_factor: grid (G), 256 threads; loops over the domains in order (EMA sequence, SURVEY H5)
//   gram  [D][SB][kNacc]  reduced moments around the pilot shift (null: take the running buffers = eval)
//   shift [D][SB*64]
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) fwd_factor_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                         const Geom gm, const FwdFin f) {
  __shared__ __align__(16) PanelSmem sp;
  __shared__ float sC[kMat];       // un-shrunk covariance (for the EMA)
  __shared__ float sMean[kSB], sRow[kSB];
  __shared__ int sBad, sBadDom;
  const int g = blockIdx.x, GS = gm.GS, nb = kSB / GS, sb = g / nb, o = (g % nb) * GS;
  const Blk t(GS);
  const int SB = (gm.C + kSB - 1) / kSB;
  const float invM = 1.f / gm.M;
  if (threadIdx.x == 0) sBad = 0;
  PROF_DECL;
  PROF_MARK();
  for (int d = 0; d < gm.D; ++d) {
    const float* G = gram ? gram + ((size_t)d * SB + sb) * kNacc : nullptr;
    const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
    // every global load of this domain is issued before the first dependent instruction: the Gram block, the row
    // sums, and the running buffers the EMA needs at the very end (their latency hides behind the factorisation;
    // the previous domain's stores precede this point by a block barrier, so aliased buffers still see the ordered
    // sequence)
    float graw[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        float v = 0.f;
        if (t.act) {
          const int i = 4 * t.bi + r, j = 4 * t.bj + s, hi = i > j ? i : j, lo = i > j ? j : i;
          v = G ? __ldcg(G + (o + hi) * kSB + o + lo) : f.rcov[d][(size_t)g * GS * GS + i * GS + j];
        }
        graw[r][s] = v;
      }
    float rowsum = 0.f, shf = 0.f;
    if ((int)threadIdx.x < GS) {
      if (G) { rowsum = __ldcg(G + kSB * kSB + o + threadIdx.x); shf = shift[((size_t)d * SB + sb) * kSB + o + threadIdx.x]; }
      else shf = f.rmean[d][g * GS + threadIdx.x];
    }
    constexpr int kEmaPer = kSB * kSB / 256;
    float rc_old[kEmaPer], rm_old = 0.f;
    const bool ema = G != nullptr && f.update_running;
    if (ema) {
#pragma unroll
      for (int n = 0; n < kEmaPer; ++n) {
        const int e = threadIdx.x + 256 * n;
        rc_old[n] = e < GS * GS ? f.rcov[d][(size_t)g * GS * GS + e] : 0.f;
      }
      if ((int)threadIdx.x < GS) rm_old = f.rmean[d][g * GS + threadIdx.x];
    }
    if ((int)threadIdx.x < GS) {
      const float mu = G ? shf + rowsum * invM : shf;
      sMean[threadIdx.x] = mu;
      sRow[threadIdx.x] = rowsum * invM;              // mean of the shifted samples
      f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x] = mu;
    }
    if (threadIdx.x == 0) sBadDom = 0;
    __syncthreads();
    float a[4][4], w[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        float v = 0.f;
        if (t.act) {
          const int i = 4 * t.bi + r, j = 4 * t.bj + s;
          float cov = graw[r][s];
          if (G) {
            cov = cov * invM - sRow[i] * sRow[j];
            sC[i * LDS + j] = cov;
          }
          v = f.a * cov + (i == j ? f.b : 0.f);
        }
        a[r][s] = v;
      }
    PROF_MARK();
    if (!factor_and_invert(a, w, GS, t, sp)) { sBad = 1; sBadDom = 1; }
    PROF_MARK();
    if (t.act) {                                      // w[r][s] = W(4bi + r, 4bj + s): straight from the registers
#pragma unroll
      for (int r = 0; r < 4; ++r)
        *reinterpret_cast<float4*>(f.save_w + gbase + (size_t)(4 * t.bi + r) * GS + 4 * t.bj) =
            make_float4(w[r][0], w[r][1], w[r][2], w[r][3]);
    }
    __syncthreads();                                  // sC complete, sBadDom final
    if (ema && !sBadDom) {                            // a non-PD batch covariance never reaches the running buffers
      const float m = f.momentum, k = 1.f - f.momentum;
#pragma unroll
      for (int n = 0; n < kEmaPer; ++n) {
        const int e = threadIdx.x + 256 * n;
        if (e < GS * GS) f.rcov[d][(size_t)g * GS * GS + e] = m * (sC[(e / GS) * LDS + e % GS] * f.unbias) + k * rc_old[n];
      }
      if ((int)threadIdx.x < GS) f.rmean[d][g * GS + threadIdx.x] = m * sMean[threadIdx.x] + k * rm_old;
    }
    __syncthreads();      // also orders this domain's buffer writes before the next domain's reads (aliasing)
    PROF_MARK();
  }
  PROF_DUMP("fwd_factor load|factor+invert|save+ema");
  if (threadIdx.x == 0 && sBad) atomicOr(f.status, DWT_STATUS_NOT_PD);
}

// ------------------------------------------------------------------------------------------
// bwd_coef: grid (G, 1, D), 256 threads.  rgram [D][SB][kNacc] = (R = sum dy xc^T | sdz = sum dy).
// coef[d][g] = A1 | Bm | cvec  with  dx = A1 dy + Bm x + cvec   (no affine epilogue on this path)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bwd_coef_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f,
                                                       float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sR = sW + kMat;
  float* sT1 = sR + kMat;
  float* sT2 = sT1 + kMat;
  __shared__ float sSdz[kSB], sMu[kSB];
  const int g = blockIdx.x, d = blockIdx.z, GS = gm.GS, nb = kSB / GS, sb = g / nb, o = (g % nb) * GS;
  const Blk t(GS);
  const int SB = (gm.C + kSB - 1) / kSB;
  const bool train = f.mode == DWT_MODE_TRAIN;
  const float* G = rgram ? rgram + ((size_t)d * SB + sb) * kNacc : nullptr;
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  PROF_DECL;
  PROF_MARK();
  // all global loads first (interleaved with their shared-memory stores the compiler kept them in order: 16 dependent
  // round trips, 17.7 k of this kernel's 44 k cycles at gs = 64); GS is a power of two: shifts, not divisions
  const int gsh = __ffs(GS) - 1;
  const float invM = 1.f / gm.M;
  constexpr int kPer = kSB * kSB / 256;
  float wv[kPer], rv[kPer];
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    const bool in = e < GS * GS;
    wv[n] = in ? f.save_w[gbase + e] : 0.f;
    rv[n] = (in && G && train) ? __ldcg(G + (o + i) * kSB + o + j) : 0.f;
  }
  float sdz = 0.f, mu = 0.f;
  if ((int)threadIdx.x < GS) {
    sdz = (G && train) ? __ldcg(G + kSB * kSB + o + threadIdx.x) : 0.f;
    mu = f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x];
  }
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    if (e < GS * GS) { sW[i * LDS + j] = wv[n]; sR[i * LDS + j] = rv[n]; }
  }
  if ((int)threadIdx.x < GS) {
    sSdz[threadIdx.x] = sdz * invM;                   // mean_M dy (0 in eval mode)
    sMu[threadIdx.x] = mu;
    if (dybar) dybar[((size_t)d * SB + sb) * kSB + o + threadIdx.x] = sdz * invM;
  }
  __syncthreads();
  PROF_MARK();
  float c[4][4];
  if (train) {
    mm_block<false, true>(sR, sW, GS, t, c);               // R W^T ; P = Phi(-R W^T)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const int i = 4 * t.bi + r, j = 4 * t.bj + s;
        c[r][s] = (i > j) ? -c[r][s] : ((i == j) ? -0.5f * c[r][s] : 0.f);
      }
    store_block(sT1, t, c);
    __syncthreads();
    PROF_MARK();
    mm_block<true, false>(sW, sT1, GS, t, c);              // T = W^T P
    store_block(sT2, t, c);
    __syncthreads();
    PROF_MARK();
    mm_block<false, false>(sT2, sW, GS, t, c);             // S' = T W
    store_block(sT1, t, c);
    __syncthreads();
    PROF_MARK();
  }
  const float sc = f.a * invM;
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    if (e < GS * GS) {
      const float bm = train ? sc * (sT1[i * LDS + j] + sT1[j * LDS + i]) : 0.f;
      coef[e] = (j >= i) ? sW[j * LDS + i] : 0.f;          // A1 = W^T
      coef[GS * GS + e] = bm;
      sT2[i * LDS + j] = bm;
    }
  }
  __syncthreads();
  // cvec_i = -(sum_j W_ji mean(dy)_j + sum_j Bm_ij mu_j): 4 threads per row, partial sums met by shuffle
  {
    const int i = threadIdx.x >> 2, q = threadIdx.x & 3;
    float cv = 0.f;
    if (train && i < GS) {
      for (int j = q; j < GS; j += 4) cv = fmaf(sW[j * LDS + i], sSdz[j], fmaf(sT2[i * LDS + j], sMu[j], cv));   // W_ji = 0 for j < i
    }
    cv += __shfl_xor_sync(0xffffffffu, cv, 1);
    cv += __shfl_xor_sync(0xffffffffu, cv, 2);
    if (q == 0 && i < GS) coef[2 * GS * GS + i] = -cv;
  }
  PROF_MARK();
  PROF_DUMP("bwd_coef load|mm1|mm2|mm3|tail");
}

constexpr size_t kFactorSmem = 0;   // fwd_factor: static shared memory only (panel buffers + covariance)
constexpr size_t kCoefSmem = sizeof(float) * 4 * kMat;

}  // namespace

int dense_init() {
  cudaError_t e = cudaFuncSetAttribute(fwd_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFactorSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(bwd_coef_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kCoefSmem);
  return (int)e;
}

// partial [problems][nchunks][kNacc] -> gram [problems][kNacc]
void dense_partial_reduce(const float* partial, int nchunks, int problems, float* gram, cudaStream_t st) {
  partial_reduce_kernel<<<dim3((kNacc + 63) / 64, problems), 256, 0, st>>>(partial, nchunks, gram);
}

// gram == nullptr: eval mode (running buffers -> W)
void dense_fwd_factor(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st) {
  fwd_factor_kernel<<<gm.G, 256, kFactorSmem, st>>>(gram, shift, gm, fin);
}

// rgram == nullptr: eval mode without affine (A1 = W^T only)
void dense_bwd_coef(const float* rgram, const Geom& gm, const BwdFin& fin, float* dybar, cudaStream_t st) {
  bwd_coef_kernel<<<dim3(gm.G, 1, gm.D), 256, kCoefSmem, st>>>(rgram, gm, fin, dybar);
}

}  // namespace dwt

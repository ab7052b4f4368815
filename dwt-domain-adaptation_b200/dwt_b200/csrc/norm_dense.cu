// Dense per-group algebra for large groups (8 <= gs <= 64) as separate, latency-tuned launches
// behind the tensor-core contraction:
//
//   partial_reduce   sum the per-CTA partial Gram matrices of a 64-channel super-block in fixed
//                    chunk order, spread over many CTAs (a single "last CTA" doing this alone would idle
//                    the rest of the grid)
//   fwd_factor       per group: mean, covariance, S = a*cov + b*I, Cholesky S = L L^T, W = L^-1,
//                    running-statistic EMA (domains in order: one CTA owns all domains of its group)
//   bwd_coef         per (domain, group): A1 = W^T, Bm = (2a/M) sym(W^T Phi(-R W^T) W), cvec
//   fwd_zca/bwd_zca  the same two steps in the ZCA basis (dwt_whiten_zca_*): W = P_T / sqrt(tr S) by T Newton-Schulz
//                    iterations on shared-memory operands, and the reverse of that recursion
//   fwd_eigh/bwd_eigh  the exact ZCA basis (dwt_whiten_eigh_*): W = U diag(lambda^-1/2) U^T by a cyclic Jacobi
//                    eigensolver in shared memory, and the Daleckii-Krein backward
//   fwd_factor<COLOR>, bwd_color  colouring (dwt_whiten_color_*): fwd_factor also writes color W; bwd_color runs bwd_coef's
//                    algebra on color^T R, domains in order in one CTA per group, and sums dcolor and dbias over them
//   fwd_instance     instance whitening (dwt_whiten_instance_*): fwd_factor's statistics and factorisation, one CTA per
//                    (image, group), no EMA; its backward is bwd_coef as it is, with the images as the domains
//   sw_*             switchable whitening (dwt_whiten_switch_*): per-image and batch moments (sw_stats), the mixture and
//                    fwd_instance's factorisation (sw_fwd_factor); backward: dL/dcov_hat and dL/dm per (image, group)
//                    (sw_bwd_coef), their fixed-order sums over the images (sw_bwd_sum, sw_dmix) and tc_bwd_apply's
//                    coefficients (sw_bwd_apply_coef)
//   ld_*             latent-domain whitening (dwt_whiten_latent_*): each latent domain's weighted moments from the per-image
//                    ones (ld_stats), fwd_instance's factorisation + EMA per (domain, group) (ld_fwd_factor), the per-image
//                    mix A_n = sum_k w_nk W_k and its centre (ld_mix); backward: per-domain sums and the Cholesky backward
//                    (ld_bwd_sum, ld_bwd_dom), tc_bwd_apply's coefficients and the dweights terms per (image, group)
//                    (ld_bwd_coef) and their fixed-order sum over the groups (ld_dw)
//
// All three keep a 64x64 problem in ONE 256-thread CTA arranged 16x16, each thread owning a 4x4
// register block.  fwd_factor runs the Cholesky factorisation AND the triangular inverse as one blocked
// right-looking sweep of 16 panel steps (one block barrier each): the matrices live in registers, shared
// memory only carries the 4-column panel of L and the 4-row panel of W of the current step.
//
// The forward kernels are built from shared pieces: fwd_domains (the domain loop of fwd_factor, fwd_zca and fwd_eigh:
// domain_stats, the barriers, the EMA of an accepted domain (domain_ema) and DWT_STATUS_NOT_PD; a basis adds only its
// step from S to W and its saved matrices) and image_factor_tail (factorisation, W or NaN and the status bit of
// fwd_instance and sw_fwd_factor).  ema_cov / ema_mean are the one EMA formula of domain_ema and sw_fwd_factor.
//
// The backward kernels are built from shared pieces: load_operands / store_operands (W, R = sum dy xc^T, sum dy and a
// basis' third matrix; bwd_coef, bwd_zca, bwd_eigh, sw_bwd_coef), chol_bwd_core (the Cholesky basis' three products;
// bwd_coef, bwd_color, sw_bwd_coef) and coef_tail (A1 | Bm | cvec from dL/dS; bwd_coef, bwd_color, bwd_zca, bwd_eigh).
// A basis' backward kernel adds only its own dL/dS between them.
//
// Group size 128 runs fwd_factor128 / bwd_coef128 (one 1024-thread CTA per group on the generic shared-memory routines
// of dwt_common.cuh); partial_reduce serves it unchanged (its problems are 64 x 64 blocks).
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

// this thread's 4 x 4 block to a dense GS x GS matrix in global memory
__device__ __forceinline__ void store_block_global(float* M, int GS, const Blk& t, const float (&c)[4][4]) {
  if (!t.act) return;
#pragma unroll
  for (int r = 0; r < 4; ++r)
    *reinterpret_cast<float4*>(M + (size_t)(4 * t.bi + r) * GS + 4 * t.bj) = make_float4(c[r][0], c[r][1], c[r][2], c[r][3]);
}

// The NaN a problem that cannot be whitened writes into W or A1 | Bm: the quiet NaN the apply's TF32 split keeps (an
// arithmetic NaN, 0x7fffffff, would round to -0 there and leave a finite, wrong result)
constexpr int kApplyNaN = 0x7fc00000;

// this thread's block of W to save_w (dense GS x GS), or NaN in full when the problem is bad
__device__ __forceinline__ void store_w_or_nan(float* save_w, size_t problem, int GS, const Blk& t, const float (&w)[4][4], bool bad) {
  if (!t.act) return;
  float* M = save_w + problem * GS * GS;
  const float q = __int_as_float(kApplyNaN);
#pragma unroll
  for (int r = 0; r < 4; ++r)
    *reinterpret_cast<float4*>(M + (size_t)(4 * t.bi + r) * GS + 4 * t.bj) =
        bad ? make_float4(q, q, q, q) : make_float4(w[r][0], w[r][1], w[r][2], w[r][3]);
}

// Where group g sits in the 64-channel super-blocks the tensor-core passes reduce: super-block sb of SB, first
// channel o inside it
struct GroupPos {
  int GS, sb, o, SB;
};

__device__ __forceinline__ GroupPos group_pos(const Geom& gm, int g) {
  const int nb = kSB / gm.GS;
  return {gm.GS, g / nb, (g % nb) * gm.GS, (gm.C + kSB - 1) / kSB};
}

// sum of v over the CTA (256 threads) in one fixed order: warp trees, then the 8 warp totals in order; every thread
// gets it.  Two block barriers, the first so that sRed is free however the caller used it last.
__device__ __forceinline__ float block_sum(float v, float* sRed) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += sRed[w];
  return s;
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
// The domain loop of the per-group forward kernels (fwd_factor, fwd_zca, fwd_eigh): every basis sees the same S, writes
// the same save_mean and applies the same running-buffer update, bit for bit.
//   gram  [D][SB][kNacc]  reduced moments around the pilot shift (null: take the running buffers = eval)
//   shift [D][SB*64]
// ------------------------------------------------------------------------------------------
constexpr int kPer = kSB * kSB / 256;   // elements of a 64 x 64 matrix per thread: e = threadIdx.x + 256 n

struct EmaOld {            // the running buffers as the domain's EMA finds them (loaded with the moments)
  float rc[kPer], rm;
  bool on;                 // train with update_running
};

// Loads domain d's moments G (null: eval, the running buffers), writes save_mean, and leaves this thread's block of
// S = a cov + b I in a[r][s] = S(4bi + r, 4bj + s); train: the un-shrunk covariance in sC.  Contains one block barrier.
__device__ __forceinline__ void domain_stats(const float* G, const float* __restrict__ shift, int d, int g, int sb, int o,
                                             int SB, float invM, const Geom& gm, const FwdFin& f, const Blk& t, float* sC,
                                             float* sMean, float* sRow, int& sBadDom, float (&a)[4][4], EmaOld& old) {
  const int GS = gm.GS;
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
  old.rm = 0.f;
  old.on = G != nullptr && f.update_running;
  if (old.on) {
#pragma unroll
    for (int n = 0; n < kPer; ++n) {
      const int e = threadIdx.x + 256 * n;
      old.rc[n] = e < GS * GS ? f.rcov[d][(size_t)g * GS * GS + e] : 0.f;
    }
    if ((int)threadIdx.x < GS) old.rm = f.rmean[d][g * GS + threadIdx.x];
  }
  if ((int)threadIdx.x < GS) {
    const float mu = G ? shf + rowsum * invM : shf;
    sMean[threadIdx.x] = mu;
    sRow[threadIdx.x] = rowsum * invM;              // mean of the shifted samples
    f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x] = mu;
  }
  if (threadIdx.x == 0) sBadDom = 0;
  __syncthreads();
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
}

// One element of the running-statistic EMA (m = momentum, k = 1 - m), for every gs 8-64 forward, so that their running
// buffers agree bit for bit: the covariance contracted by the compiler, the mean by the contraction fwd_factor has always
// used, fma(1 - m, old, m * stat)
__device__ __forceinline__ float ema_cov(float m, float k, float stat, float old) { return m * stat + k * old; }
__device__ __forceinline__ float ema_mean(float m, float k, float stat, float old) { return fmaf(k, old, __fmul_rn(m, stat)); }

// The EMA of domain d (train, update_running, batch covariance accepted): sC and sMean complete behind a block barrier.
__device__ __forceinline__ void domain_ema(int d, int g, const Geom& gm, const FwdFin& f, const float* sC, const float* sMean,
                                           const EmaOld& old) {
  const int GS = gm.GS;
  const float m = f.momentum, k = 1.f - f.momentum;
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n;
    if (e < GS * GS) f.rcov[d][(size_t)g * GS * GS + e] = ema_cov(m, k, sC[(e / GS) * LDS + e % GS] * f.unbias, old.rc[n]);
  }
  if ((int)threadIdx.x < GS) f.rmean[d][g * GS + threadIdx.x] = ema_mean(m, k, sMean[threadIdx.x], old.rm);
}

// fwd_domains' shared memory: domain_stats' outputs (sC [kMat], sMean, sRow [kSB]) and the bad flags of the group and of
// the current domain.  Each kernel declares them as separate arrays: one __shared__ struct of them made ptxas schedule
// fwd_factor's sweep differently and measurably slower.
struct DomainSmem {
  float *C, *mean, *row;
  int &bad, &bad_dom;
};

// A basis' step flags the current domain: DWT_STATUS_NOT_PD at the end, and no EMA for the domain
__device__ __forceinline__ void mark_bad(const DomainSmem& sd) { sd.bad = 1; sd.bad_dom = 1; }

struct NoAfter { __device__ void operator()(size_t, const Blk&) const {} };

// The domain loop of fwd_factor, fwd_zca and fwd_eigh: the CTA of group blockIdx.x runs the domains in order (EMA
// sequence, SURVEY H5).  Per domain: domain_stats; the basis' step(d, gbase, a, t) with this thread's block of S in a,
// which writes save_w + gbase and the basis' saved matrices and may call mark_bad; a block barrier; after(gbase, t),
// which may read what the step left in shared memory; the EMA unless the domain was marked bad.
template <class Step, class After = NoAfter>
__device__ __forceinline__ void fwd_domains(const float* __restrict__ gram, const float* __restrict__ shift, const Geom& gm,
                                            const FwdFin& f, const DomainSmem& sd PROF_ARGS, Step step, After after = {}) {
  const int g = blockIdx.x;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const float invM = 1.f / gm.M;
  if (threadIdx.x == 0) sd.bad = 0;
  PROF_MARK();
  for (int d = 0; d < gm.D; ++d) {
    const float* G = gram ? gram + ((size_t)d * SB + sb) * kNacc : nullptr;
    const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
    float a[4][4];
    EmaOld old;
    domain_stats(G, shift, d, g, sb, o, SB, invM, gm, f, t, sd.C, sd.mean, sd.row, sd.bad_dom, a, old);
    step(d, gbase, a, t);
    __syncthreads();                                  // sC complete, sBadDom final
    after(gbase, t);
    if (old.on && !sd.bad_dom) domain_ema(d, g, gm, f, sd.C, sd.mean, old);   // a non-PD batch covariance never reaches the running buffers
    __syncthreads();      // also orders this domain's buffer writes before the next domain's reads (aliasing)
    PROF_MARK();
  }
  if (threadIdx.x == 0 && sd.bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
}

// ------------------------------------------------------------------------------------------
// fwd_factor: grid (G), 256 threads, fwd_domains with the blocked Cholesky + inverse as its step.  A domain that is not
// positive definite keeps the W the sweep left (not NaN'd).
// COLOR: also gw [D][G][gs*gs] = color[g] W (color [G][gs*gs]), for the apply in place of W; dynamic shared memory holds
// color and W (kColorFwdSmem)
// ------------------------------------------------------------------------------------------
template <bool COLOR>
__global__ void __launch_bounds__(256) fwd_factor_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                         const Geom gm, const FwdFin f, const float* __restrict__ color,
                                                         float* __restrict__ gw) {
  __shared__ __align__(16) PanelSmem sp;
  __shared__ float sC[kMat], sMean[kSB], sRow[kSB];
  __shared__ int sBad, sBadDom;
  const DomainSmem sd{sC, sMean, sRow, sBad, sBadDom};
  extern __shared__ __align__(16) float dsm[];
  float* sGam = dsm;                                  // COLOR: color[g], then W of the domain
  float* sWd = dsm + kMat;
  const int GS = gm.GS;
  if constexpr (COLOR) {                              // published by domain_stats' barrier
    for (int e = threadIdx.x; e < GS * GS; e += 256) sGam[(e / GS) * LDS + e % GS] = color[(size_t)blockIdx.x * GS * GS + e];
  }
  PROF_DECL;
  fwd_domains(gram, shift, gm, f, sd PROF_PASS, [&](int, size_t gbase, float (&a)[4][4], const Blk& t) {
    float w[4][4];
    PROF_MARK();
    if (!factor_and_invert(a, w, GS, t, sp)) mark_bad(sd);
    PROF_MARK();
    store_block_global(f.save_w + gbase, GS, t, w);  // w[r][s] = W(4bi + r, 4bj + s): straight from the registers
    if constexpr (COLOR) store_block(sWd, t, w);
  }, [&](size_t gbase, const Blk& t) {
    if constexpr (COLOR) {
      float c[4][4];
      mm_block<false, false>(sGam, sWd, GS, t, c);
      store_block_global(gw + gbase, GS, t, c);
    }
  });
  PROF_DUMP("fwd_factor load|factor+invert|save+ema");
}

// ------------------------------------------------------------------------------------------
// Backward pieces shared by the per-group backward kernels (gs 8..64)
// ------------------------------------------------------------------------------------------
// One (domain, group) problem's backward operands in registers: this thread's elements of W, of R = sum dy xc^T and,
// with HAS_X, of a third GS x GS matrix X; and sum dy of channel threadIdx.x.
struct Operands {
  float w[kPer], r[kPer], x[kPer];
  float sdz;
};

// Issues the loads of W (w: the problem's save_w), of R and sum dy (G: the problem's reduced block [kNacc], channel o of
// the super-block) and of X (x).  on false (eval): R, X and sdz are zeros, and G and x are not read.  Every global load
// goes out before the first shared-memory store: interleaved with their stores, the compiler kept the loads in order (16
// dependent round trips, 17.7 k of bwd_coef's 44 k cycles at gs = 64).  So a caller issues its own per-channel loads
// between load_operands and store_operands.  GS is a power of two: shifts, not divisions.
template <bool HAS_X>
__device__ __forceinline__ void load_operands(Operands& op, const float* w, const float* G, const float* x, bool on, int GS,
                                              int gsh, int o) {
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    const bool in = e < GS * GS;
    op.w[n] = in ? w[e] : 0.f;
    op.r[n] = (in && on) ? __ldcg(G + (o + i) * kSB + o + j) : 0.f;
    if constexpr (HAS_X) op.x[n] = (in && on) ? x[e] : 0.f;
  }
  op.sdz = 0.f;
  if ((int)threadIdx.x < GS) op.sdz = on ? __ldcg(G + kSB * kSB + o + threadIdx.x) : 0.f;
}

template <bool HAS_X>
__device__ __forceinline__ void store_operands(const Operands& op, float* sW, float* sR, float* sX, int GS, int gsh) {
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    if (e < GS * GS) {
      sW[i * LDS + j] = op.w[n];
      sR[i * LDS + j] = op.r[n];
      if constexpr (HAS_X) sX[i * LDS + j] = op.x[n];
    }
  }
}

// The Cholesky basis' backward: from R = sum dL/dy xc^T (sR) and W (sW), S' = W^T Phi(-R W^T) W into sT1 (sT2: scratch;
// it may be sR, which is read only before the first barrier), Bm = (a/M)(S' + S'^T).  Ends with a block barrier.
__device__ __forceinline__ void chol_bwd_core(const float* sR, const float* sW, float* sT1, float* sT2, int GS, const Blk& t PROF_ARGS) {
  float c[4][4];
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

// The coefficients tc_bwd_apply reads, coef = A1 | Bm | cvec with dx = A1 dy + Bm x + cvec, from the matrix sA whose
// transpose is A1 and, in training, G = dL/dS (sG):
//   A1 = sA^T, in full, or TRI: its upper triangle and zeros below (a Cholesky W of a group that is not positive
//        definite can hold NaN above its diagonal, 0 x NaN from a NaN 1/diag)
//   Bm = (a/M)(G + G^T) = sc (G + G^T), also into the scratch sBm; 0 in eval
//   cvec_i = -(sum_j A1_ij mean(dy)_j + sum_j Bm_ij mu_j): 4 threads per row, partial sums met by shuffle; 0 in eval
// One block barrier.
template <bool TRI>
__device__ __forceinline__ void coef_tail(const float* sA, const float* sG, float* sBm, const float* sSdz, const float* sMu,
                                          bool train, float sc, int GS, int gsh, float* coef) {
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    if (e < GS * GS) {
      const float bm = train ? sc * (sG[i * LDS + j] + sG[j * LDS + i]) : 0.f;
      coef[e] = (!TRI || j >= i) ? sA[j * LDS + i] : 0.f;
      coef[GS * GS + e] = bm;
      sBm[i * LDS + j] = bm;
    }
  }
  __syncthreads();
  const int i = threadIdx.x >> 2, q = threadIdx.x & 3;
  float cv = 0.f;
  if (train && i < GS) {
    for (int j = q; j < GS; j += 4) cv = fmaf(sA[j * LDS + i], sSdz[j], fmaf(sBm[i * LDS + j], sMu[j], cv));
  }
  cv += __shfl_xor_sync(0xffffffffu, cv, 1);
  cv += __shfl_xor_sync(0xffffffffu, cv, 2);
  if (q == 0 && i < GS) coef[2 * GS * GS + i] = -cv;
}

// ------------------------------------------------------------------------------------------
// bwd_coef: grid (G, 1, D), 256 threads.  rgram [D][SB][kNacc] = (R = sum dy xc^T | sdz = sum dy).
// coef[d][g] = A1 | Bm | cvec  with  dx = A1 dy + Bm x + cvec   (no affine epilogue on this path), A1 = W^T
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bwd_coef_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f,
                                                       float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sR = sW + kMat;
  float* sT1 = sR + kMat;
  float* sT2 = sT1 + kMat;
  __shared__ float sSdz[kSB], sMu[kSB];
  const int g = blockIdx.x, d = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const bool train = f.mode == DWT_MODE_TRAIN;
  const float* G = rgram ? rgram + ((size_t)d * SB + sb) * kNacc : nullptr;
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  const int gsh = __ffs(GS) - 1;
  const float invM = 1.f / gm.M;
  PROF_DECL;
  PROF_MARK();
  Operands op;
  load_operands<false>(op, f.save_w + ((size_t)d * gm.G + g) * GS * GS, G, nullptr, G && train, GS, gsh, o);
  float mu = 0.f;
  if ((int)threadIdx.x < GS) mu = f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x];
  store_operands<false>(op, sW, sR, nullptr, GS, gsh);
  if ((int)threadIdx.x < GS) {
    sSdz[threadIdx.x] = op.sdz * invM;                // mean_M dy (0 in eval mode)
    sMu[threadIdx.x] = mu;
    if (dybar) dybar[((size_t)d * SB + sb) * kSB + o + threadIdx.x] = op.sdz * invM;
  }
  __syncthreads();
  PROF_MARK();
  if (train) chol_bwd_core(sR, sW, sT1, sT2, GS, t PROF_PASS);
  coef_tail<true>(sW, sT1, sT2, sSdz, sMu, train, f.a * invM, GS, gsh, coef);
  PROF_MARK();
  PROF_DUMP("bwd_coef load|mm1|mm2|mm3|tail");
}

// ------------------------------------------------------------------------------------------
// bwd_color: grid (G), 256 threads, the domains of a group in order.  y = color W xc + bias: with dy_hat = color^T dy, per domain
//   train: bwd_coef's algebra on R_hat = color^T R, A1 = W^T color^T (full), dybar = mean_M dy (tc_bwd_apply: A1 (dy - dybar))
//   eval:  A1 = W^T color^T, Bm = 0, dybar = 0
// and, when dcolor is given (rgram given), dcolor[g] = sum_d R_d W_d^T, dbias[g] = sum_d sum_m dy, summed in domain order in
// registers: deterministic.  In eval R comes from the contraction without pilot shift (tc_bwd_reduce, pilot = false).
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bwd_color_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f,
                                                        const float* __restrict__ color, float* __restrict__ dcolor,
                                                        float* __restrict__ dbias, float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sR = sW + kMat;           // R, then R_hat
  float* sT1 = sR + kMat;
  float* sT2 = sT1 + kMat;
  float* sGam = sT2 + kMat;        // color[g]
  float* sGW = sGam + kMat;        // color W = A1^T
  __shared__ float sSdz[kSB], sMu[kSB];
  const int g = blockIdx.x;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const bool train = f.mode == DWT_MODE_TRAIN;
  const int gsh = __ffs(GS) - 1;
  const float invM = 1.f / gm.M;
  for (int e = threadIdx.x; e < GS * GS; e += 256) sGam[(e >> gsh) * LDS + (e & (GS - 1))] = color[(size_t)g * GS * GS + e];
  PROF_DECL;
  float dg[4][4], db = 0.f;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) dg[r][s] = 0.f;
  for (int d = 0; d < gm.D; ++d) {
    const float* G = rgram ? rgram + ((size_t)d * SB + sb) * kNacc : nullptr;
    const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
    float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
#pragma unroll
    for (int n = 0; n < kPer; ++n) {
      const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
      if (e < GS * GS) {
        sW[i * LDS + j] = f.save_w[gbase + e];
        sR[i * LDS + j] = G ? __ldcg(G + (o + i) * kSB + o + j) : 0.f;
      }
    }
    if ((int)threadIdx.x < GS) {
      const float sdz = G ? __ldcg(G + kSB * kSB + o + threadIdx.x) : 0.f;
      db += sdz;
      sSdz[threadIdx.x] = train ? sdz * invM : 0.f;   // mean_M dy
      sMu[threadIdx.x] = f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x];
      if (dybar) dybar[((size_t)d * SB + sb) * kSB + o + threadIdx.x] = train ? sdz * invM : 0.f;
    }
    __syncthreads();
    float c[4][4], gw[4][4];
    if (dcolor) {
      mm_block<false, true>(sR, sW, GS, t, c);        // R W^T
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) dg[r][s] += c[r][s];
    }
    mm_block<false, false>(sGam, sW, GS, t, gw);      // color W
    if (train) mm_block<true, false>(sGam, sR, GS, t, c);   // R_hat = color^T R
    __syncthreads();                                  // every read of sR is done
    if (train) store_block(sR, t, c);
    store_block(sGW, t, gw);
    __syncthreads();
    if (train) chol_bwd_core(sR, sW, sT1, sT2, GS, t PROF_PASS);
    coef_tail<false>(sGW, sT1, sT2, sSdz, sMu, train, f.a * invM, GS, gsh, coef);   // A1 = (color W)^T
    __syncthreads();                                  // the next domain overwrites every shared matrix
  }
  if (dcolor) {
    store_block_global(dcolor + (size_t)g * GS * GS, GS, t, dg);
    if ((int)threadIdx.x < GS) dbias[g * GS + threadIdx.x] = db;
  }
}

// ------------------------------------------------------------------------------------------
// ZCA basis (dwt_whiten_zca_*): W = S^-1/2 by T steps of the Newton-Schulz iteration instead of W = L^-1
//   t = tr S,  N = S / t,  P_0 = I,  P_k = (3 P_{k-1} - P_{k-1}^3 N) / 2  (k = 1..T),  W = P_T / sqrt(t)
// W is NOT symmetrised: it is P_T / sqrt(t) as computed, symmetric in exact arithmetic only, and both apply kernels use
// exactly the saved W (A1 = W^T in full).  save_p [D][G][T][GS*GS]: slot 0 holds S, slot k holds P_k (k = 1..T-1).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_block(const float* M, const Blk& t, float (&c)[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) c[r][s] = t.act ? M[(4 * t.bi + r) * LDS + 4 * t.bj + s] : 0.f;
}

// tr M of a shared matrix, in one fixed order (fwd_zca and bwd_zca form the same t from the same S); ends with a barrier
__device__ __forceinline__ float trace_of(const float* M, int GS, float* sRed) {
  if (threadIdx.x < 32) {
    const int l = threadIdx.x;
    float v = (l < GS ? M[l * LDS + l] : 0.f) + (l + 32 < GS ? M[(l + 32) * LDS + l + 32] : 0.f);
    v = warp_sum(v);
    if (l == 0) sRed[0] = v;
  }
  __syncthreads();
  return sRed[0];
}

// fwd_zca: grid (G), 256 threads, fwd_domains with the Newton-Schulz iteration as its step.  Three products per
// iteration (P P, (P P) P, (P P P) N) on shared-memory operands; each thread keeps its block of P in registers.
// A non-finite or non-positive t, or a non-finite W, flags the domain as a non-positive pivot does in fwd_factor
// (DWT_STATUS_NOT_PD, no EMA).  An indefinite S whose iteration stays finite is not detected: batch statistics are
// positive semi-definite and shrunk, so only running buffers a user supplied (eval) can be indefinite.
__global__ void __launch_bounds__(256) fwd_zca_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                      const Geom gm, const FwdFin f, int T, float* __restrict__ save_p) {
  extern __shared__ __align__(16) float dsm[];
  float* sN = dsm;                 // S, then N = S / t
  float* sP = sN + kMat;
  float* sT1 = sP + kMat;          // P P
  float* sT2 = sT1 + kMat;         // P P P
  __shared__ float sC[kMat], sMean[kSB], sRow[kSB];
  __shared__ int sBad, sBadDom;
  const DomainSmem sd{sC, sMean, sRow, sBad, sBadDom};
  __shared__ float sRed[1];
  const int GS = gm.GS;
  PROF_DECL;
  fwd_domains(gram, shift, gm, f, sd PROF_PASS, [&](int, size_t gbase, float (&a)[4][4], const Blk& t) {
    float* pd = save_p + gbase * T;
    float p[4][4], c[4][4];
    store_block(sN, t, a);
    store_block_global(pd, GS, t, a);                 // slot 0: S
    __syncthreads();
    const float tr = trace_of(sN, GS, sRed);
    if (threadIdx.x == 0 && !(tr > 0.f && tr < INFINITY)) mark_bad(sd);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        a[r][s] = a[r][s] / tr;
        p[r][s] = (t.act && t.bi == t.bj && r == s) ? 1.f : 0.f;
      }
    store_block(sN, t, a);                            // own block: every read of S was before trace_of's barrier
    store_block(sP, t, p);
    __syncthreads();
    PROF_MARK();
    for (int k = 1; k <= T; ++k) {
      mm_block<false, false>(sP, sP, GS, t, c);
      store_block(sT1, t, c);
      __syncthreads();
      mm_block<false, false>(sT1, sP, GS, t, c);
      store_block(sT2, t, c);
      __syncthreads();
      mm_block<false, false>(sT2, sN, GS, t, c);      // nothing reads sP in this phase: P_k replaces P_{k-1} in place
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) p[r][s] = 0.5f * (3.f * p[r][s] - c[r][s]);
      if (k < T) {
        store_block(sP, t, p);
        store_block_global(pd + (size_t)k * GS * GS, GS, t, p);
      }
      __syncthreads();
    }
    PROF_MARK();
    const float rs = 1.f / sqrtf(tr);
    bool finite = true;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        p[r][s] *= rs;
        finite = finite && isfinite(p[r][s]);
      }
    store_block_global(f.save_w + gbase, GS, t, p);
    if (!finite) mark_bad(sd);
  });
  PROF_DUMP("fwd_zca load|iterate|save+ema");
}

// bwd_zca: grid (G, 1, D), 256 threads.  The reverse of fwd_zca's recursion from dL/dW = R = sum dy xc^T:
//   Q_T = R / sqrt(t),  tbar = -<R, P_T> t^-3/2 / 2 = -<R, W> / (2 t),  Nbar = 0
//   k = T..1, P = P_{k-1}:  Nbar -= P^3 Q_k / 2,  Q_{k-1} = 3 Q_k / 2 - (Q_k N P^2 + P Q_k N P + P^2 Q_k N) / 2
//   G = dL/dS = Nbar / t + (tbar - <Nbar, N> / t) I,   Bm = (a/M)(G + G^T),   A1 = W^T (full),   cvec
// Step k = 1 has P_0 = I: Nbar -= Q_1 / 2, and Q_0 is not needed.  Steps k >= 2 run eight products in three phases.
// coef[d][g] = A1 | Bm | cvec where tc_bwd_apply reads them; eval (rgram null): A1 = W^T, Bm = 0.
__global__ void __launch_bounds__(256) bwd_zca_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f, int T,
                                                      const float* __restrict__ save_p, float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sN = sW + kMat;           // S, then N = S / t
  float* sQ = sN + kMat;           // R, then Q_k
  float* sP = sQ + kMat;           // P_{k-1}
  float* sPP = sP + kMat;          // P^2; at the end Bm
  float* sQN = sPP + kMat;         // Q N
  float* sP3 = sQN + kMat;         // P^3
  float* sT = sP3 + kMat;          // P Q N; at the end G
  __shared__ float sSdz[kSB], sMu[kSB], sRed[8];
  const int g = blockIdx.x, d = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const bool train = f.mode == DWT_MODE_TRAIN && rgram != nullptr;
  const float* G = train ? rgram + ((size_t)d * SB + sb) * kNacc : nullptr;
  const size_t gbase = ((size_t)d * gm.G + g) * GS * GS;
  const float* pd = save_p + gbase * T;
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  const int gsh = __ffs(GS) - 1;
  const float invM = 1.f / gm.M;
  PROF_DECL;
  PROF_MARK();
  Operands op;
  load_operands<true>(op, f.save_w + gbase, G, pd, train, GS, gsh, o);   // X = S (save_p slot 0)
  float mu = 0.f;
  if ((int)threadIdx.x < GS) mu = f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x];
  store_operands<true>(op, sW, sQ, sN, GS, gsh);
  float rw = 0.f;                                     // this thread's share of <R, W>
#pragma unroll
  for (int n = 0; n < kPer; ++n) rw = fmaf(op.r[n], op.w[n], rw);
  if ((int)threadIdx.x < GS) {
    sSdz[threadIdx.x] = op.sdz * invM;                // mean_M dy (0 in eval mode)
    sMu[threadIdx.x] = mu;
    if (dybar) dybar[((size_t)d * SB + sb) * kSB + o + threadIdx.x] = op.sdz * invM;
  }
  __syncthreads();
  PROF_MARK();
  if (train) {
    const float tr = trace_of(sN, GS, sRed);          // fwd_zca's t, bit for bit
    const float rs = 1.f / sqrtf(tr);
    const float tbar = -0.5f * block_sum(rw, sRed) / tr;
    float q[4][4], nbar[4][4], c[4][4], acc[4][4];
    load_block(sN, t, c);
    load_block(sQ, t, q);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        c[r][s] = c[r][s] / tr;
        q[r][s] *= rs;
        nbar[r][s] = 0.f;
      }
    store_block(sN, t, c);                            // own blocks only
    store_block(sQ, t, q);
    for (int k = T; k >= 2; --k) {
      const float* pk = pd + (size_t)(k - 1) * GS * GS;
#pragma unroll
      for (int n = 0; n < kPer; ++n) {
        const int e = threadIdx.x + 256 * n;
        if (e < GS * GS) sP[(e >> gsh) * LDS + (e & (GS - 1))] = pk[e];
      }
      __syncthreads();
      mm_block<false, false>(sP, sP, GS, t, c);       // P^2
      store_block(sPP, t, c);
      mm_block<false, false>(sQ, sN, GS, t, c);       // Q N
      store_block(sQN, t, c);
      __syncthreads();
      mm_block<false, false>(sPP, sP, GS, t, c);      // P^3
      store_block(sP3, t, c);
      mm_block<false, false>(sP, sQN, GS, t, c);      // P Q N
      store_block(sT, t, c);
      mm_block<false, false>(sQN, sPP, GS, t, acc);   // Q N P^2
      mm_block<false, false>(sPP, sQN, GS, t, c);     // P^2 Q N
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) acc[r][s] += c[r][s];
      __syncthreads();
      mm_block<false, false>(sP3, sQ, GS, t, c);      // P^3 Q
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) nbar[r][s] = fmaf(-0.5f, c[r][s], nbar[r][s]);
      mm_block<false, false>(sT, sP, GS, t, c);       // P Q N P
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) q[r][s] = 1.5f * q[r][s] - 0.5f * (acc[r][s] + c[r][s]);
      __syncthreads();                                // every read of sQ and sP of this step is done
      store_block(sQ, t, q);
    }
    // k = 1 (P_0 = I), then G = Nbar / t + (tbar - <Nbar, N> / t) I
    float nn = 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        nbar[r][s] = fmaf(-0.5f, q[r][s], nbar[r][s]);
        if (t.act) nn = fmaf(nbar[r][s], sN[(4 * t.bi + r) * LDS + 4 * t.bj + s], nn);
      }
    const float diag = tbar - block_sum(nn, sRed) / tr;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) c[r][s] = nbar[r][s] / tr + ((t.bi == t.bj && r == s) ? diag : 0.f);
    store_block(sT, t, c);
    __syncthreads();
  }
  PROF_MARK();
  coef_tail<false>(sW, sT, sPP, sSdz, sMu, train, f.a * invM, GS, gsh, coef);
  PROF_MARK();
  PROF_DUMP("bwd_zca load|iterate|tail");
}

// ------------------------------------------------------------------------------------------
// Exact ZCA basis (dwt_whiten_eigh_*): W = U diag(lambda^-1/2) U^T from S = U diag(lambda) U^T
// Cyclic two-sided Jacobi in shared memory: one sweep is GS - 1 steps of the round-robin (circle) ordering, each step
// GS/2 disjoint rotations at once with Rutishauser's formulas, U accumulates the rotations.  A rotation is skipped when
// |a_pq| <= kJacobiTol sqrt(|a_pp a_qq|) (the relative criterion of positive definite Jacobi); the solver stops after
// the first sweep that skips every rotation, or after kJacobiSweeps.  Every decision is a fixed function of the data:
// reruns are bit-identical.  save_e [D][G][GS + 1][GS]: rows 0..GS-1 hold U (column j the eigenvector of lambda_j),
// row GS holds lambda, in the order the sweeps leave them.
// ------------------------------------------------------------------------------------------
constexpr float kJacobiTol = 1.2e-7f;   // about FLT_EPSILON
constexpr int kJacobiSweeps = 16;

// pair k of step r of the circle method on n = GS indices: index n - 1 stays, the other n - 1 rotate; p < q
__device__ __forceinline__ void jacobi_pair(int n, int r, int k, int& p, int& q) {
  const int m = n - 1;
  const int a = k == 0 ? r : (r + k) % m, b = k == 0 ? m : (r - k + m) % m;
  p = a < b ? a : b;
  q = a < b ? b : a;
}

struct JacobiSmem {
  int p[kSB / 2], q[kSB / 2];
  float c[kSB / 2], s[kSB / 2], t[kSB / 2];
  int rot[2];                      // a rotation happened in the sweep of this parity
};

// Diagonalises the symmetric GS x GS matrix in sA in place (its diagonal ends as lambda) and leaves U in sU.  The
// caller has published sA behind a block barrier; ends with one.
__device__ void jacobi_eigh(float* sA, float* sU, int GS, JacobiSmem& js) {
  const int np = GS >> 1, lnp = __ffs(np) - 1, lgs = __ffs(GS) - 1;
  for (int e = threadIdx.x; e < GS * GS; e += blockDim.x) sU[(e >> lgs) * LDS + (e & (GS - 1))] = (e >> lgs) == (e & (GS - 1)) ? 1.f : 0.f;
  if (threadIdx.x < 2) js.rot[threadIdx.x] = 0;
  __syncthreads();
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    const int par = sweep & 1;
    for (int r = 0; r < GS - 1; ++r) {
      if ((int)threadIdx.x < np) {                    // the rotations of this step
        int p, q;
        jacobi_pair(GS, r, threadIdx.x, p, q);
        const float app = sA[p * LDS + p], aqq = sA[q * LDS + q], apq = sA[p * LDS + q];
        float c = 1.f, s = 0.f, tt = 0.f;
        if (!(fabsf(apq) <= kJacobiTol * sqrtf(fabsf(app * aqq)))) {
          const float theta = 0.5f * (aqq - app) / apq;
          tt = copysignf(1.f, theta) / (fabsf(theta) + sqrtf(fmaf(theta, theta, 1.f)));   // the smaller root: |angle| <= pi/4
          c = 1.f / sqrtf(fmaf(tt, tt, 1.f));
          s = tt * c;
          js.rot[par] = 1;
        }
        js.p[threadIdx.x] = p; js.q[threadIdx.x] = q;
        js.c[threadIdx.x] = c; js.s[threadIdx.x] = s; js.t[threadIdx.x] = tt;
      }
      __syncthreads();
      if (r == 0 && threadIdx.x == 0) js.rot[par ^ 1] = 0;   // every thread read it before the barrier above
      // A <- J^T A J on the 2 x 2 blocks (pair k rows, pair l columns): disjoint, so in place
      for (int b = threadIdx.x; b < np * np; b += blockDim.x) {
        const int k = b >> lnp, l = b & (np - 1);
        const int pk = js.p[k], qk = js.q[k], pl = js.p[l], ql = js.q[l];
        const float ck = js.c[k], sk = js.s[k];
        if (k == l) {                                 // Rutishauser: a_pp -= t a_pq, a_qq += t a_pq, a_pq = 0
          if (sk == 0.f) continue;
          const float apq = sA[pk * LDS + qk], tk = js.t[k];
          sA[pk * LDS + pk] = fmaf(-tk, apq, sA[pk * LDS + pk]);
          sA[qk * LDS + qk] = fmaf(tk, apq, sA[qk * LDS + qk]);
          sA[pk * LDS + qk] = 0.f;
          sA[qk * LDS + pk] = 0.f;
          continue;
        }
        const float cl = js.c[l], sl = js.s[l];
        const float a00 = sA[pk * LDS + pl], a01 = sA[pk * LDS + ql], a10 = sA[qk * LDS + pl], a11 = sA[qk * LDS + ql];
        const float x00 = ck * a00 - sk * a10, x01 = ck * a01 - sk * a11;        // rows
        const float x10 = sk * a00 + ck * a10, x11 = sk * a01 + ck * a11;
        sA[pk * LDS + pl] = cl * x00 - sl * x01;                                 // columns
        sA[pk * LDS + ql] = sl * x00 + cl * x01;
        sA[qk * LDS + pl] = cl * x10 - sl * x11;
        sA[qk * LDS + ql] = sl * x10 + cl * x11;
      }
      // U <- U J
      for (int e = threadIdx.x; e < GS * np; e += blockDim.x) {
        const int i = e & (GS - 1), k = e >> lgs;
        const float sk = js.s[k];
        if (sk == 0.f) continue;
        const int pk = js.p[k], qk = js.q[k];
        const float ck = js.c[k], up = sU[i * LDS + pk], uq = sU[i * LDS + qk];
        sU[i * LDS + pk] = ck * up - sk * uq;
        sU[i * LDS + qk] = sk * up + ck * uq;
      }
      __syncthreads();
    }
    if (!js.rot[par]) break;                          // final since the last barrier: every thread leaves together
  }
}

// fwd_eigh: grid (G), 256 threads, fwd_domains with the Jacobi solve as its step.  A non-finite S skips the solver;
// a non-finite or non-positive eigenvalue (an indefinite running buffer in eval, too) flags the domain as a
// non-positive pivot does in fwd_factor (DWT_STATUS_NOT_PD, no EMA).  W = V V^T with V = U diag(lambda^-1/4):
// symmetric bit for bit.
__global__ void __launch_bounds__(256) fwd_eigh_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                       const Geom gm, const FwdFin f, float* __restrict__ save_e) {
  extern __shared__ __align__(16) float dsm[];
  float* sA = dsm;                 // S, then diag(lambda) + rounding, then V
  float* sU = sA + kMat;
  __shared__ float sC[kMat], sMean[kSB], sRow[kSB];
  __shared__ int sBad, sBadDom;
  const DomainSmem sd{sC, sMean, sRow, sBad, sBadDom};
  __shared__ float sLam[kSB];
  __shared__ JacobiSmem js;
  const int GS = gm.GS, lgs = __ffs(GS) - 1;
  PROF_DECL;
  fwd_domains(gram, shift, gm, f, sd PROF_PASS, [&](int d, size_t gbase, float (&a)[4][4], const Blk& t) {
    float* ed = save_e + ((size_t)d * gm.G + blockIdx.x) * (GS + 1) * GS;
    float c[4][4];
    bool finite = true;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) finite = finite && isfinite(a[r][s]);
    store_block(sA, t, a);
    if (!finite) mark_bad(sd);
    __syncthreads();
    PROF_MARK();
    if (!sd.bad_dom) jacobi_eigh(sA, sU, GS, js);     // block-uniform
    PROF_MARK();
    if ((int)threadIdx.x < GS) {
      const float lam = sA[threadIdx.x * LDS + threadIdx.x];
      sLam[threadIdx.x] = lam;
      ed[GS * GS + threadIdx.x] = lam;
      if (!(lam > 0.f && lam < INFINITY)) mark_bad(sd);
    }
    __syncthreads();
    for (int e = threadIdx.x; e < GS * GS; e += blockDim.x) {
      const int i = e >> lgs, j = e & (GS - 1);
      const float u = sd.bad_dom ? NAN : sU[i * LDS + j];   // a skipped solver left no U
      ed[e] = u;
      sA[i * LDS + j] = u / sqrtf(sqrtf(sLam[j]));    // V = U lambda^-1/4
    }
    __syncthreads();
    mm_block<false, true>(sA, sA, GS, t, c);          // W = V V^T
    store_block_global(f.save_w + gbase, GS, t, c);
  });
  PROF_DUMP("fwd_eigh load|solve|save+ema");
}

// bwd_eigh: grid (G, 1, D), 256 threads.  From dL/dW = R = sum dy xc^T by the Daleckii-Krein formula:
//   G = dL/dS = U [(U^T R U) o F] U^T,  F_ij = -1 / (sqrt(l_i) sqrt(l_j) (sqrt(l_i) + sqrt(l_j)))
// F is the divided difference of l^-1/2 without its cancellation: finite at equal eigenvalues (-l^-3/2 / 2).  Then as
// bwd_zca: Bm = (a/M)(G + G^T), A1 = W^T (full), cvec; eval (rgram null): A1 = W^T, Bm = 0.  Four products.
__global__ void __launch_bounds__(256) bwd_eigh_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f,
                                                       const float* __restrict__ save_e, float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sU = sW + kMat;
  float* sR = sU + kMat;           // R; at the end G
  float* sT1 = sR + kMat;          // R U, then U H
  float* sH = sT1 + kMat;          // H = (U^T R U) o F; at the end Bm
  __shared__ float sSdz[kSB], sMu[kSB], sRl[kSB];
  const int g = blockIdx.x, d = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const bool train = f.mode == DWT_MODE_TRAIN && rgram != nullptr;
  const float* G = train ? rgram + ((size_t)d * SB + sb) * kNacc : nullptr;
  const float* ed = save_e + ((size_t)d * gm.G + g) * (GS + 1) * GS;
  float* coef = f.coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  const int gsh = __ffs(GS) - 1;
  const float invM = 1.f / gm.M;
  PROF_DECL;
  PROF_MARK();
  Operands op;
  load_operands<true>(op, f.save_w + ((size_t)d * gm.G + g) * GS * GS, G, ed, train, GS, gsh, o);   // X = U
  float mu = 0.f, lam = 1.f;
  if ((int)threadIdx.x < GS) {
    mu = f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x];
    if (train) lam = ed[GS * GS + threadIdx.x];
  }
  store_operands<true>(op, sW, sR, sU, GS, gsh);
  if ((int)threadIdx.x < GS) {
    sSdz[threadIdx.x] = op.sdz * invM;                // mean_M dy (0 in eval mode)
    sMu[threadIdx.x] = mu;
    sRl[threadIdx.x] = sqrtf(lam);
    if (dybar) dybar[((size_t)d * SB + sb) * kSB + o + threadIdx.x] = op.sdz * invM;
  }
  __syncthreads();
  PROF_MARK();
  if (train) {
    float c[4][4];
    mm_block<false, false>(sR, sU, GS, t, c);         // R U
    store_block(sT1, t, c);
    __syncthreads();
    mm_block<true, false>(sU, sT1, GS, t, c);         // U^T R U, times F
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const float ri = sRl[4 * t.bi + r], rj = sRl[4 * t.bj + s];
        c[r][s] = -c[r][s] / (ri * rj * (ri + rj));
      }
    store_block(sH, t, c);
    __syncthreads();
    mm_block<false, false>(sU, sH, GS, t, c);         // U H (every read of sT1 was before the barrier above)
    store_block(sT1, t, c);
    __syncthreads();
    mm_block<false, true>(sT1, sU, GS, t, c);         // G = U H U^T (R is dead)
    store_block(sR, t, c);
    __syncthreads();
  }
  PROF_MARK();
  coef_tail<false>(sW, sR, sH, sSdz, sMu, train, f.a * invM, GS, gsh, coef);
  PROF_MARK();
  PROF_DUMP("bwd_eigh load|solve|tail");
}

// ------------------------------------------------------------------------------------------
// group size 128: one 1024-thread CTA per group runs the shared-memory routines of dwt_common.cuh (fwd_factor_block:
// right-looking Cholesky + forward-substitution inverse; bwd_finalize_block: P, T = W^T P, S' = T W, A1, Bm) on the
// whole 128 x 128 matrix, assembled from the 64 x 64 blocks the tensor-core contractions reduced.  Three matrices of
// 128 x 129 floats: 194 KB of shared memory.
// ------------------------------------------------------------------------------------------
constexpr int kGS2 = 2 * kSB, kLD2 = kGS2 + 1, kMat2 = kGS2 * kLD2;
constexpr int kThreads2 = 1024;
constexpr size_t kFactor2Smem = sizeof(float) * (3 * kMat2 + kGS2);
constexpr size_t kCoef2Smem = sizeof(float) * (3 * kMat2 + 3 * kGS2);

// fwd_factor at 128: grid (G), domains in order (EMA sequence).  gram [D][SB][kNacc] holds the diagonal blocks and the
// row sums (super-blocks 2g, 2g + 1), goff [D][SB/2][kNacc] the off-diagonal block G10 of group g; null: eval.
__global__ void __launch_bounds__(kThreads2) fwd_factor128_kernel(const float* __restrict__ gram, const float* __restrict__ goff,
                                                                  const float* __restrict__ shift, const Geom gm, const FwdFin f) {
  extern __shared__ __align__(16) float dsm2[];
  float* sCov = dsm2;
  float* sL = sCov + kMat2;
  float* sW = sL + kMat2;
  float* sMean = sW + kMat2;
  __shared__ float sRow[kGS2];
  const int g = blockIdx.x, tid = threadIdx.x, SB = gm.C / kSB;
  const float invM = 1.f / gm.M;
  for (int d = 0; d < gm.D; ++d) {
    const float* Gd = gram ? gram + ((size_t)d * SB + 2 * g) * kNacc : nullptr;
    const float* Go = gram ? goff + ((size_t)d * (SB / 2) + g) * kNacc : nullptr;
    if (tid < kGS2) {
      float mu;
      if (Gd) {
        const float rs = __ldcg(Gd + (tid >> 6) * kNacc + kSB * kSB + (tid & 63));
        mu = shift[((size_t)d * SB + 2 * g) * kSB + tid] + rs * invM;
        sRow[tid] = rs * invM;                        // mean of the shifted samples
      } else {
        mu = f.rmean[d][g * kGS2 + tid];
      }
      sMean[tid] = mu;
    }
    __syncthreads();
    // lower triangle (i >= j) of the Gram from its block, mirrored: the covariance is exactly symmetric
    for (int e = tid; e < kGS2 * kGS2; e += kThreads2) {
      const int i = e >> 7, j = e & 127, hi = i > j ? i : j, lo = i > j ? j : i;
      float c;
      if (Gd) {
        const float raw = (hi >> 6) == (lo >> 6) ? __ldcg(Gd + (hi >> 6) * kNacc + (hi & 63) * kSB + (lo & 63))
                                                 : __ldcg(Go + (hi & 63) * kSB + lo);
        c = raw * invM - sRow[i] * sRow[j];
      } else {
        c = f.rcov[d][(size_t)g * kGS2 * kGS2 + e];
      }
      sCov[i * kLD2 + j] = c;
    }
    __syncthreads();
    fwd_factor_block(gm, f, d, g, sMean, sCov, sL, sW, Gd != nullptr);   // save_mean, save_w, status; train: bad[d][g]
    __syncthreads();
    if (Gd && f.update_running && !__ldcg(f.bad + d * gm.G + g)) {     // a non-PD batch covariance never reaches the EMA
      const float m = f.momentum, k = 1.f - f.momentum;
      for (int e = tid; e < kGS2 * kGS2; e += kThreads2) {
        float* rc = f.rcov[d] + (size_t)g * kGS2 * kGS2 + e;
        *rc = m * (sCov[(e >> 7) * kLD2 + (e & 127)] * f.unbias) + k * *rc;
      }
      if (tid < kGS2) f.rmean[d][g * kGS2 + tid] = m * sMean[tid] + k * f.rmean[d][g * kGS2 + tid];
    }
    __syncthreads();      // this domain's buffer writes before the next domain's reads (aliasing)
  }
}

// bwd_coef at 128: grid (G, 1, D).  rgram [D][2 SB][kNacc]: block (r, c) of group g's R = sum dy xc^T at 4 g + 2 r + c,
// the dy row sums of rows r in block (r, r).
__global__ void __launch_bounds__(kThreads2) bwd_coef128_kernel(const float* __restrict__ rgram, const Geom gm, const BwdFin f,
                                                                float* __restrict__ dybar) {
  extern __shared__ __align__(16) float dsm2[];
  float* sW = dsm2;
  float* sR = sW + kMat2;
  float* sT1 = sR + kMat2;
  float* sVec = sT1 + kMat2;                         // gamma | mean (bwd_finalize_block)
  float* sSdz = sVec + 2 * kGS2;
  __shared__ int s_flag;
  const int g = blockIdx.x, d = blockIdx.z, tid = threadIdx.x, SB = gm.C / kSB;
  const bool train = f.mode == DWT_MODE_TRAIN;
  const float* G = (rgram && train) ? rgram + ((size_t)d * 2 * SB + 4 * g) * kNacc : nullptr;
  for (int e = tid; e < kGS2 * kGS2; e += kThreads2) {
    const int i = e >> 7, j = e & 127;
    sR[i * kLD2 + j] = G ? __ldcg(G + (2 * (i >> 6) + (j >> 6)) * kNacc + (i & 63) * kSB + (j & 63)) : 0.f;
  }
  if (tid < kGS2) {
    const float sdz = G ? __ldcg(G + 3 * (tid >> 6) * kNacc + kSB * kSB + (tid & 63)) : 0.f;
    sSdz[tid] = sdz;
    if (dybar) dybar[((size_t)d * SB + 2 * g) * kSB + tid] = sdz * (1.f / gm.M);   // mean_M dy (0 in eval mode)
  }
  // bwd_finalize_block's barrier after loading W publishes sR and sSdz; R is dead once P is formed, so its buffer
  // doubles as the T scratch
  bwd_finalize_block(gm, f, d, g, sR, sSdz, sW, sT1, sR, sVec, &s_flag);
}

// ------------------------------------------------------------------------------------------
// The end of the per-image forward kernels (fwd_instance, sw_fwd_factor) and of ld_fwd_factor: this thread's block of S
// (a) factored and inverted, the CTA's OR of bad (S or the mean not finite) and of a non-positive pivot, W to save_w, or
// NaN in full for a bad problem, and DWT_STATUS_NOT_PD.  Returns that OR (the same in every thread).
__device__ __forceinline__ bool image_factor_tail(float (&a)[4][4], bool bad, size_t problem, int GS, const Blk& t,
                                                  PanelSmem& sp, float* save_w, int* status) {
  float w[4][4];
  const bool ok = factor_and_invert(a, w, GS, t, sp);
  bad = __syncthreads_or(bad || !ok) != 0;
  store_w_or_nan(save_w, problem, GS, t, w, bad);
  if (threadIdx.x == 0 && bad) atomicOr(status, DWT_STATUS_NOT_PD);
  return bad;
}

// fwd_instance: instance whitening (dwt_whiten_instance_fwd), grid (G, 1, D), 256 threads, one CTA per (image, group):
// the Geom's domains are the images (N = 1, M = HW).  fwd_factor's statistics prologue and blocked Cholesky + inverse,
// without the EMA and without its loop over the domains: fwd_factor serialises them in one CTA per group, which at
// hundreds of images would leave all but G CTAs of the H100 idle.  A group whose S is not positive definite (or not
// finite) gets W = NaN in full, so that image's whole group reads NaN, and sets DWT_STATUS_NOT_PD.
__global__ void __launch_bounds__(256) fwd_instance_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                           const Geom gm, const FwdFin f) {
  __shared__ __align__(16) PanelSmem sp;
  __shared__ float sC[kMat];       // written by domain_stats, not read (no EMA)
  __shared__ float sMean[kSB], sRow[kSB];
  __shared__ int sBadDom;          // cleared by domain_stats, not read
  const int g = blockIdx.x, d = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const float* G = gram + ((size_t)d * SB + sb) * kNacc;
  float a[4][4];
  EmaOld old;                      // f.update_running is 0: domain_stats reads no running buffer
  domain_stats(G, shift, d, g, sb, o, SB, 1.f / gm.M, gm, f, t, sC, sMean, sRow, sBadDom, a, old);
  image_factor_tail(a, false, (size_t)d * gm.G + g, GS, t, sp, f.save_w, f.status);
}

// ------------------------------------------------------------------------------------------
// Switchable whitening (dwt_whiten_switch_*): the Geom's domains are the images (N = 1, M = HW), as for fwd_instance.
// A group's statistics record is rec = gs*gs + gs floats (covariance, then mean); save_stats holds [D + 1][G] of them, the
// images' own and then the batch's.  mix = (a_b, a_i, w_bw, w_iw, w_bn, w_in).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int sw_rec(int GS) { return GS * GS + GS; }

// sw_stats: grid (ceil(rec / 256), G), 256 threads, one record element per thread.  Each image's own covariance and mean
// into save_stats rows 0..D-1 (fp32, fwd_instance's arithmetic).  Train: the batch moments into row D by the law of total
// covariance, cov_b = mean_n cov_n + cov_n(mu_n), accumulated in fp64 over the images in order about image 0's mean (no
// second pass over x; bit-identical reruns).  Eval: row D is a copy of the running buffers.
__global__ void __launch_bounds__(256) sw_stats_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                       const Geom gm, const SwFin f) {
  const int g = blockIdx.y;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const int rec = sw_rec(GS), e = blockIdx.x * 256 + threadIdx.x;
  if (e >= rec) return;
  const int D = gm.D;
  const float invM = 1.f / gm.M;
  const double invMd = 1.0 / (double)gm.M;
  const bool cov = e < GS * GS;
  const int i = cov ? e / GS : e - GS * GS, j = cov ? e % GS : i, hi = i > j ? i : j, lo = i > j ? j : i;
  float* out = f.save_stats + (size_t)g * rec + e;
  const size_t ostride = (size_t)gm.G * rec;
  const float* G0 = gram + (size_t)sb * kNacc;
  const float* S0 = shift + (size_t)sb * kSB + o;
  const double ci = (double)S0[i] + (double)__ldcg(G0 + kSB * kSB + o + i) * invMd;   // image 0's mean: the common shift
  const double cj = (double)S0[j] + (double)__ldcg(G0 + kSB * kSB + o + j) * invMd;
  double acc = 0.0, accm = 0.0, acci = 0.0, accj = 0.0;
#pragma unroll 4
  for (int d = 0; d < D; ++d) {
    const float* Gd = G0 + (size_t)d * SB * kNacc;
    const float* Sd = S0 + (size_t)d * SB * kSB;
    const float ri = __ldcg(Gd + kSB * kSB + o + i), si = Sd[i];
    if (cov) {
      const float graw = __ldcg(Gd + (o + hi) * kSB + o + lo), rj = __ldcg(Gd + kSB * kSB + o + j), sj = Sd[j];
      const float ri_m = ri * invM, rj_m = rj * invM;
      out[(size_t)d * ostride] = graw * invM - ri_m * rj_m;
      if (f.train) {
        const double dri = (double)ri * invMd, drj = (double)rj * invMd;
        const double mi = ((double)si + dri) - ci, mj = ((double)sj + drj) - cj;
        acc += (double)graw * invMd - dri * drj;
        accm = fma(mi, mj, accm);
        acci += mi;
        accj += mj;
      }
    } else {
      out[(size_t)d * ostride] = si + ri * invM;
      if (f.train) acci += ((double)si + (double)ri * invMd) - ci;
    }
  }
  float b;
  if (f.train) {
    const double invD = 1.0 / (double)D, mi = acci * invD, mj = accj * invD;
    b = cov ? (float)(acc * invD + (accm * invD - mi * mj)) : (float)(ci + mi);
  } else {
    b = cov ? f.rcov[(size_t)g * GS * GS + e] : f.rmean[g * GS + i];
  }
  out[(size_t)D * ostride] = b;
}

// sw_fwd_factor: grid (G, 1, D), 256 threads, one CTA per (image, group): the mixed mean m = a_b mu_b + a_i mu_n into
// save_mean, the mixed covariance, S = a cov_hat + b I and fwd_instance's blocked Cholesky + inverse.  An (image, group)
// whose S is not positive definite, or whose S or m is not finite, gets W = NaN in full and sets DWT_STATUS_NOT_PD.
// The CTAs of image 0 also run the EMA of their group's batch moments (train, update_running), skipped with
// DWT_STATUS_NOT_PD when those are not finite.
__global__ void __launch_bounds__(256) sw_fwd_factor_kernel(const Geom gm, const SwFin f) {
  __shared__ __align__(16) PanelSmem sp;
  const int g = blockIdx.x, d = blockIdx.z, GS = gm.GS, rec = sw_rec(GS);
  const Blk t(GS);
  const float* sn = f.save_stats + ((size_t)d * gm.G + g) * rec;
  const float* sbt = f.save_stats + ((size_t)gm.D * gm.G + g) * rec;
  const float a_b = f.mix[0], a_i = f.mix[1], w_bw = f.mix[2], w_iw = f.mix[3], w_bn = f.mix[4], w_in = f.mix[5];
  bool bad = false;
  float a[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      float v = 0.f;
      if (t.act) {
        const int i = 4 * t.bi + r, j = 4 * t.bj + s;
        const float cn = sn[i * GS + j], cb = sbt[i * GS + j];
        float c = fmaf(w_iw, cn, w_bw * cb);
        if (i == j) c = fmaf(w_in, cn, fmaf(w_bn, cb, c));
        v = f.a * c + (i == j ? f.b : 0.f);
        bad = bad || !isfinite(v);
      }
      a[r][s] = v;
    }
  if ((int)threadIdx.x < GS) {
    const float m = fmaf(a_i, sn[GS * GS + threadIdx.x], a_b * sbt[GS * GS + threadIdx.x]);
    f.save_mean[(size_t)d * gm.C + g * GS + threadIdx.x] = m;
    bad = bad || !isfinite(m);
  }
  image_factor_tail(a, bad, (size_t)d * gm.G + g, GS, t, sp, f.save_w, f.status);
  if (d != 0 || !f.train || !f.update_running) return;
  constexpr int kRecPer = (kSB * kSB + kSB + 255) / 256;
  float old[kRecPer], stat[kRecPer];
  bool fin = true;
#pragma unroll
  for (int n = 0; n < kRecPer; ++n) {
    const int e = threadIdx.x + 256 * n;
    stat[n] = e < rec ? sbt[e] : 0.f;
    old[n] = e < GS * GS ? f.rcov[(size_t)g * GS * GS + e] : (e < rec ? f.rmean[g * GS + e - GS * GS] : 0.f);
    fin = fin && isfinite(stat[n]);
  }
  if (!__syncthreads_or(!fin)) {        // dwt_whiten_fwd's EMA on the unshrunk batch moments
    const float m = f.momentum, k = 1.f - f.momentum;
#pragma unroll
    for (int n = 0; n < kRecPer; ++n) {
      const int e = threadIdx.x + 256 * n;
      if (e < GS * GS) f.rcov[(size_t)g * GS * GS + e] = ema_cov(m, k, stat[n], old[n]);
      else if (e < rec) f.rmean[g * GS + e - GS * GS] = ema_mean(m, k, stat[n], old[n]);
    }
  } else if (threadIdx.x == 0) {
    atomicOr(f.status, DWT_STATUS_NOT_PD);
  }
}

// sw_bwd_coef: grid (G, 1, D), 256 threads, one CTA per (image, group).  rgram [D][SB][kNacc] = (R = sum dy (x - m)^T |
// sum dy).  P = a sym(W^T Phi(-R W^T) W) (dL/dcov_hat) and dm = -W^T sum dy (dL/dm) into pd [D][G][rec], and the image's
// six dmix terms (<dm, mu_b>, <dm, mu_n>, <P, cov_b>, <P, cov_n>, <diag P, cov_b>, <diag P, cov_n>) into part [D][G][8].
__global__ void __launch_bounds__(256) sw_bwd_coef_kernel(const float* __restrict__ rgram, const Geom gm, const SwFin f,
                                                          float* __restrict__ pd, float* __restrict__ part) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sR = sW + kMat;
  float* sT = sR + kMat;
  __shared__ float sSdz[kSB], sRed[8];
  const int g = blockIdx.x, d = blockIdx.z, rec = sw_rec(gm.GS);
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const Blk t(GS);
  const int gsh = __ffs(GS) - 1;
  const float* G = rgram + ((size_t)d * SB + sb) * kNacc;
  const float* sn = f.save_stats + ((size_t)d * gm.G + g) * rec;
  const float* sbt = f.save_stats + ((size_t)gm.D * gm.G + g) * rec;
  float* out = pd + ((size_t)d * gm.G + g) * rec;
  PROF_DECL;
  Operands op;
  load_operands<false>(op, f.save_w + ((size_t)d * gm.G + g) * GS * GS, G, nullptr, true, GS, gsh, o);
  store_operands<false>(op, sW, sR, nullptr, GS, gsh);
  if ((int)threadIdx.x < GS) sSdz[threadIdx.x] = op.sdz;
  __syncthreads();
  chol_bwd_core(sR, sW, sT, sR, GS, t PROF_PASS);       // T' = W^T Phi(-R W^T) W into sT
  const float h = 0.5f * f.a;
  float p_bw = 0.f, p_iw = 0.f, p_bn = 0.f, p_in = 0.f;
#pragma unroll
  for (int n = 0; n < kPer; ++n) {
    const int e = threadIdx.x + 256 * n, i = e >> gsh, j = e & (GS - 1);
    if (e < GS * GS) {
      const float p = h * (sT[i * LDS + j] + sT[j * LDS + i]);
      out[e] = p;
      const float cb = sbt[e], cn = sn[e];
      p_bw = fmaf(p, cb, p_bw);
      p_iw = fmaf(p, cn, p_iw);
      if (i == j) { p_bn = fmaf(p, cb, p_bn); p_in = fmaf(p, cn, p_in); }
    }
  }
  // dm_i = -sum_j W_ji sdz_j: 4 threads per row, partial sums met by shuffle
  float t_b = 0.f, t_i = 0.f;
  {
    const int i = threadIdx.x >> 2, q = threadIdx.x & 3;
    float v = 0.f;
    if (i < GS)
      for (int j = q; j < GS; j += 4) v = fmaf(sW[j * LDS + i], sSdz[j], v);   // W_ji = 0 for j < i
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (q == 0 && i < GS) {
      out[GS * GS + i] = -v;
      t_b = -v * sbt[GS * GS + i];
      t_i = -v * sn[GS * GS + i];
    }
  }
  const float terms[6] = {t_b, t_i, p_bw, p_iw, p_bn, p_in};
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const float s = block_sum(terms[k], sRed);
    if (threadIdx.x == 0) part[((size_t)d * gm.G + g) * 8 + k] = s;
  }
}

// sw_bwd_sum: grid (ceil(rec / 256), G), 256 threads: sums [G][rec] = sum over the images, in order and in fp64, of pd
// (sum_n P_n | sum_n dm_n).
__global__ void __launch_bounds__(256) sw_bwd_sum_kernel(const float* __restrict__ pd, const Geom gm, float* __restrict__ sums) {
  const int g = blockIdx.y, rec = sw_rec(gm.GS), e = blockIdx.x * 256 + threadIdx.x;
  if (e >= rec) return;
  const float* p = pd + (size_t)g * rec + e;
  const size_t stride = (size_t)gm.G * rec;
  double acc = 0.0;
#pragma unroll 8
  for (int d = 0; d < gm.D; ++d) acc += (double)__ldcg(p + (size_t)d * stride);
  sums[(size_t)g * rec + e] = (float)acc;
}

// sw_dmix: one CTA of 256 threads: dmix[k] = the sum over every (image, group) of part[.][.][k], in a fixed order in fp64.
__global__ void __launch_bounds__(256) sw_dmix_kernel(const float* __restrict__ part, int problems, float* __restrict__ dmix) {
  __shared__ double sRed[256];
  for (int k = 0; k < 6; ++k) {
    double v = 0.0;
    for (int p = threadIdx.x; p < problems; p += 256) v += (double)__ldcg(part + (size_t)p * 8 + k);
    sRed[threadIdx.x] = v;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
      if ((int)threadIdx.x < h) sRed[threadIdx.x] += sRed[threadIdx.x + h];
      __syncthreads();
    }
    if (threadIdx.x == 0) dmix[k] = (float)sRed[0];
    __syncthreads();
  }
}

// sw_bwd_apply_coef: grid (G, 1, D), 256 threads, one CTA per (image, group): the coefficients of tc_bwd_apply's
// dx = A1 (dy - dybar) + Bm (x - mu) with mu = mu_n (written to mu [D][C]):
//   A1 = W^T,  Bm = (2/M) Q_n + train (2/NM) Q_b,  Q_n = w_iw P_n + w_in diag P_n,  Q_b = w_bw sum P + w_bn diag sum P
//   k = (a_i/M) dm_n + train ((a_b/NM) sum dm + (2/NM) Q_b (mu_n - mu_b)),   dybar = -W^-T k (back substitution; 0 when
//   A1 or Bm is not finite)
__global__ void __launch_bounds__(256) sw_bwd_apply_coef_kernel(const float* __restrict__ pd, const float* __restrict__ sums,
                                                                const Geom gm, const SwFin f, float* __restrict__ coef,
                                                                float* __restrict__ dybar, float* __restrict__ mu) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sQ = sW + kMat;
  __shared__ float sDmu[kSB], sK[kSB];
  const int g = blockIdx.x, d = blockIdx.z, rec = sw_rec(gm.GS);
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const int gsh = __ffs(GS) - 1;
  const float* p = pd + ((size_t)d * gm.G + g) * rec;
  const float* ps = sums + (size_t)g * rec;
  const float* sn = f.save_stats + ((size_t)d * gm.G + g) * rec;
  const float* sbt = f.save_stats + ((size_t)gm.D * gm.G + g) * rec;
  float* cf = coef + ((size_t)d * gm.G + g) * coef_stride(GS);
  const float a_b = f.mix[0], a_i = f.mix[1], w_bw = f.mix[2], w_iw = f.mix[3], w_bn = f.mix[4], w_in = f.mix[5];
  const float invM = 1.f / gm.M, invNM = invM / (float)gm.D;
  const bool train = f.train != 0;                       // eval: the batch terms are constants (sums is not read)
  bool nanc = false;
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    sW[i * LDS + j] = f.save_w[((size_t)d * gm.G + g) * GS * GS + e];
    const float pb = train ? ps[e] : 0.f, pn = p[e], qb = train ? (i == j ? fmaf(w_bn, pb, w_bw * pb) : w_bw * pb) : 0.f;
    const float qn = i == j ? fmaf(w_in, pn, w_iw * pn) : w_iw * pn;
    sQ[i * LDS + j] = qb;
    const float bm = 2.f * fmaf(invM, qn, invNM * qb);
    cf[GS * GS + e] = bm;
    nanc = nanc || !isfinite(bm) || !isfinite(sW[i * LDS + j]);
  }
  if ((int)threadIdx.x < GS) {
    const float mn = sn[GS * GS + threadIdx.x];
    sDmu[threadIdx.x] = mn - sbt[GS * GS + threadIdx.x];
    mu[(size_t)d * gm.C + g * GS + threadIdx.x] = mn;
  }
  nanc = __syncthreads_or(nanc) != 0;
  // a group whose A1 or Bm is not finite gets both as kApplyNaN
  const float q = __int_as_float(kApplyNaN);
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    cf[e] = nanc ? q : ((j >= i) ? sW[j * LDS + i] : 0.f);   // A1 = W^T
    if (nanc) cf[GS * GS + e] = q;
  }
  {
    const int i = threadIdx.x >> 2, q = threadIdx.x & 3;
    float v = 0.f;
    if (i < GS)
      for (int j = q; j < GS; j += 4) v = fmaf(sQ[i * LDS + j], sDmu[j], v);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (q == 0 && i < GS) {
      const float kb = train ? fmaf(a_b * invNM, ps[GS * GS + i], 2.f * invNM * v) : 0.f;
      sK[i] = fmaf(a_i * invM, p[GS * GS + i], kb);
    }
  }
  __syncthreads();
  if (threadIdx.x < 32) {                                 // W^T z = -k, W^T upper triangular: rows i from the bottom
    const int l = threadIdx.x;
    float r0 = l < GS ? -sK[l] : 0.f, r1 = l + 32 < GS ? -sK[l + 32] : 0.f;
    for (int i = GS - 1; i >= 0; --i) {
      const float own = i >= 32 ? r1 : r0;
      const float zi = __shfl_sync(0xffffffffu, own, i & 31) / sW[i * LDS + i];
      if (l == (i & 31)) { if (i >= 32) r1 = zi; else r0 = zi; }
      if (l < i) r0 = fmaf(-sW[i * LDS + l], zi, r0);     // (W^T)_{l i} = W_il
      if (l + 32 < i) r1 = fmaf(-sW[i * LDS + l + 32], zi, r1);
    }
    // a group whose A1 or Bm is not finite (W = NaN from the forward; in training, Q_b of a group with such an image) has
    // a NaN dx through them (above); dybar = 0 keeps that NaN out of the other groups of its super-block
    float* db = dybar + ((size_t)d * SB + sb) * kSB + o;
    if (l < GS) db[l] = nanc ? 0.f : r0;
    if (l + 32 < GS) db[l + 32] = nanc ? 0.f : r1;
  }
}

// ------------------------------------------------------------------------------------------
// Latent-domain whitening (dwt_whiten_latent_*): the Geom's domains are the images (N = 1, M = HW), as for fwd_instance;
// K latent domains k weight image n by w_nk = weights[n][K].  save_stats (rec = gs*gs + gs floats per record):
//   [D][G] records  each image's (C_n, m_n)          [K][G] records  each domain's (Sigma_k, mu_k)
//   [K][G][gs*gs]   W_k = L_k^-1                     [K]             s_k = sum_n w_nk
// A domain with s_k == 0 is skipped everywhere: no W_k, no EMA, no share in any output.  Every sum over the images skips
// a weight that is exactly 0 instead of multiplying by it, so a non-finite domain or image stays out of the others.
// ------------------------------------------------------------------------------------------
struct LdLayout {
  const int GS, rec, G, D, K;
  float* base;
  __device__ LdLayout(const Geom& gm, const LdFin& f)
      : GS(gm.GS), rec(sw_rec(gm.GS)), G(gm.G), D(gm.D), K(f.K), base(f.save_stats) {}
  __device__ float* img(int n, int g) const { return base + ((size_t)n * G + g) * rec; }
  __device__ float* dom(int k, int g) const { return base + ((size_t)(D + k) * G + g) * rec; }
  __device__ float* w_base() const { return base + (size_t)(D + K) * G * rec; }
  __device__ float* mass() const { return w_base() + (size_t)K * G * GS * GS; }
};

// ld_stats: grid (ceil(rec / 256), G, K), 256 threads, one record element of one domain per thread.  The CTAs of domain 0
// write each image's own covariance and mean (sw_stats' fp32 arithmetic).  s_k in fp64 over the images in order.  Train:
// (Sigma_k, mu_k) = the w-weighted moments of the images' pixels by the law of total covariance,
// Sigma_k = sum_n w_nk [C_n + (m_n - mu_k)(m_n - mu_k)^T] / s_k, accumulated in fp64 over the images in order about image
// 0's mean; eval: a copy of domain k's running buffers.
__global__ void __launch_bounds__(256) ld_stats_kernel(const float* __restrict__ gram, const float* __restrict__ shift,
                                                       const Geom gm, const LdFin f) {
  const int g = blockIdx.y, k = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const LdLayout L(gm, f);
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= L.rec) return;
  const int N = gm.D, K = f.K;
  const float invM = 1.f / gm.M;
  const double invMd = 1.0 / (double)gm.M;
  const bool cov = e < GS * GS;
  const int i = cov ? e / GS : e - GS * GS, j = cov ? e % GS : i, hi = i > j ? i : j, lo = i > j ? j : i;
  const float* G0 = gram + (size_t)sb * kNacc;
  const float* S0 = shift + (size_t)sb * kSB + o;
  const double ci = (double)S0[i] + (double)__ldcg(G0 + kSB * kSB + o + i) * invMd;   // image 0's mean: the common shift
  const double cj = (double)S0[j] + (double)__ldcg(G0 + kSB * kSB + o + j) * invMd;
  double s = 0.0, acc = 0.0, accm = 0.0, acci = 0.0, accj = 0.0;
  for (int n = 0; n < N; ++n) {
    const float w = __ldg(f.weights + (size_t)n * K + k);
    if (w != 0.f) s += (double)w;
    const bool use = f.train && w != 0.f;
    if (!use && k != 0) continue;
    const float* Gd = G0 + (size_t)n * SB * kNacc;
    const float* Sd = S0 + (size_t)n * SB * kSB;
    const float ri = __ldcg(Gd + kSB * kSB + o + i), si = Sd[i];
    const double dw = (double)w;
    if (cov) {
      const float graw = __ldcg(Gd + (o + hi) * kSB + o + lo), rj = __ldcg(Gd + kSB * kSB + o + j), sj = Sd[j];
      if (k == 0) L.img(n, g)[e] = graw * invM - (ri * invM) * (rj * invM);
      if (use) {
        const double dri = (double)ri * invMd, drj = (double)rj * invMd;
        const double mi = ((double)si + dri) - ci, mj = ((double)sj + drj) - cj;
        acc += dw * ((double)graw * invMd - dri * drj);
        accm += dw * (mi * mj);
        acci += dw * mi;
        accj += dw * mj;
      }
    } else {
      if (k == 0) L.img(n, g)[e] = si + ri * invM;
      if (use) acci += dw * (((double)si + (double)ri * invMd) - ci);
    }
  }
  if (e == 0 && g == 0) L.mass()[k] = (float)s;
  float v = 0.f;                                    // a zero-mass domain's row is never read
  if (!f.train) {
    v = cov ? f.rcov[((size_t)k * gm.G + g) * GS * GS + e] : f.rmean[(size_t)k * gm.C + g * GS + i];
  } else if (s != 0.0) {
    const double inv = 1.0 / s, mi = acci * inv, mj = accj * inv;
    v = cov ? (float)(acc * inv + (accm * inv - mi * mj)) : (float)(ci + mi);
  }
  L.dom(k, g)[e] = v;
}

// ld_fwd_factor: grid (G, 1, K), 256 threads, one CTA per (domain, group): S_k = a Sigma_k + b I, fwd_instance's blocked
// Cholesky + inverse into W_k, and the EMA of (Sigma_k, mu_k) (train, update_running).  A domain with s_k < 0 or NaN,
// non-finite statistics or an S_k that is not positive definite gets W_k = NaN, sets DWT_STATUS_NOT_PD and skips its
// EMA.  A domain with s_k == 0 is skipped (no W_k, no status, no EMA).
__global__ void __launch_bounds__(256) ld_fwd_factor_kernel(const Geom gm, const LdFin f) {
  __shared__ __align__(16) PanelSmem sp;
  const int g = blockIdx.x, k = blockIdx.z, GS = gm.GS;
  const LdLayout L(gm, f);
  const Blk t(GS);
  const float s = L.mass()[k];
  if (s == 0.f) return;
  const float* st = L.dom(k, g);
  bool bad = !(s > 0.f);
  float a[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float v = 0.f;
      if (t.act) {
        const int i = 4 * t.bi + r, j = 4 * t.bj + c;
        v = f.a * st[i * GS + j] + (i == j ? f.b : 0.f);
        bad = bad || !isfinite(v);
      }
      a[r][c] = v;
    }
  if ((int)threadIdx.x < GS) bad = bad || !isfinite(st[GS * GS + threadIdx.x]);
  bad = image_factor_tail(a, bad, (size_t)k * gm.G + g, GS, t, sp, L.w_base(), f.status);
  if (bad || !f.train || !f.update_running) return;
  const float m = f.momentum, km = 1.f - f.momentum;     // dwt_whiten_fwd's EMA on the unshrunk moments
  float* rc = f.rcov + ((size_t)k * gm.G + g) * GS * GS;
  float* rm = f.rmean + (size_t)k * gm.C + g * GS;
  for (int e = threadIdx.x; e < GS * GS; e += 256) rc[e] = ema_cov(m, km, st[e], rc[e]);
  if ((int)threadIdx.x < GS) rm[threadIdx.x] = ema_mean(m, km, st[GS * GS + threadIdx.x], rm[threadIdx.x]);
}

// ld_mix: grid (G, 1, D), 256 threads, one CTA per (image, group): A_n = sum_k w_nk W_k and b_n = sum_k w_nk W_k mu_k over
// the domains in order (skipping w_nk == 0 and s_k == 0), then A_n m~_n = b_n by forward substitution (A_n is lower
// triangular).  save_w = A_n, save_mean = m~_n; an (image, group) whose A_n has a diagonal entry that is not positive and
// finite, or whose A_n or m~_n is not finite, gets A_n = NaN and m~_n = 0 and sets DWT_STATUS_NOT_PD (a NaN centre would
// reach the other groups of its super-block through the apply's zero blocks).
__global__ void __launch_bounds__(256) ld_mix_kernel(const Geom gm, const LdFin f) {
  __shared__ float sA[kMat], sB[kSB];
  const int g = blockIdx.x, n = blockIdx.z, GS = gm.GS, K = f.K;
  const LdLayout L(gm, f);
  const Blk t(GS);
  const int ri = threadIdx.x >> 2, rq = threadIdx.x & 3;
  float a[4][4], bq = 0.f;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) a[r][c] = 0.f;
  for (int k = 0; k < K; ++k) {
    const float w = __ldg(f.weights + (size_t)n * K + k);
    if (w == 0.f || L.mass()[k] == 0.f) continue;       // CTA-uniform
    const float* Wk = L.w_base() + ((size_t)k * gm.G + g) * GS * GS;
    const float* mk = L.dom(k, g) + GS * GS;
    if (t.act) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 v = *reinterpret_cast<const float4*>(Wk + (size_t)(4 * t.bi + r) * GS + 4 * t.bj);
        a[r][0] = fmaf(w, v.x, a[r][0]); a[r][1] = fmaf(w, v.y, a[r][1]);
        a[r][2] = fmaf(w, v.z, a[r][2]); a[r][3] = fmaf(w, v.w, a[r][3]);
      }
    }
    if (ri < GS) {
      float v = 0.f;
      for (int j = rq; j <= ri; j += 4) v = fmaf(Wk[ri * GS + j], mk[j], v);   // W_k lower triangular
      bq = fmaf(w, v, bq);
    }
  }
  bq += __shfl_xor_sync(0xffffffffu, bq, 1);
  bq += __shfl_xor_sync(0xffffffffu, bq, 2);
  bool bad = false;
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) bad = bad || (t.act && !isfinite(a[r][c]));
  store_block(sA, t, a);
  if (rq == 0 && ri < GS) sB[ri] = bq;
  __syncthreads();
  if (threadIdx.x < 32) {                                 // A z = b, rows i from the top
    const int l = threadIdx.x;
    float r0 = l < GS ? sB[l] : 0.f, r1 = l + 32 < GS ? sB[l + 32] : 0.f;
    for (int i = 0; i < GS; ++i) {
      const float d = sA[i * LDS + i];
      bad = bad || !(d > 0.f && d < INFINITY);
      const float own = i >= 32 ? r1 : r0;
      const float zi = __shfl_sync(0xffffffffu, own, i & 31) / d;
      if (l == (i & 31)) { if (i >= 32) r1 = zi; else r0 = zi; }
      if (l > i && l < GS) r0 = fmaf(-sA[l * LDS + i], zi, r0);
      if (l + 32 > i && l + 32 < GS) r1 = fmaf(-sA[(l + 32) * LDS + i], zi, r1);
    }
    bad = bad || (l < GS && !isfinite(r0)) || (l + 32 < GS && !isfinite(r1));
    sB[l] = r0;                                           // each lane rewrites only its own rows
    sB[l + 32] = r1;
  }
  bad = __syncthreads_or(bad) != 0;
  store_w_or_nan(f.save_w, (size_t)n * gm.G + g, GS, t, a, bad);
  if ((int)threadIdx.x < GS) f.save_mean[(size_t)n * gm.C + g * GS + threadIdx.x] = bad ? 0.f : sB[threadIdx.x];
  if (threadIdx.x == 0 && bad) atomicOr(f.status, DWT_STATUS_NOT_PD);
}

// ld_bwd_sum: grid (ceil(rec / 256), G, K), 256 threads (train).  rgram [D][SB][kNacc] = (R~_n = sum dy (x - m~_n)^T |
// g_n = sum dy).  sums[k][g] = (Wbar_k = sum_n w_nk [R~_n + g_n (m~_n - mu_k)^T] | sum_n w_nk g_n), over the images in
// order in fp64.
__global__ void __launch_bounds__(256) ld_bwd_sum_kernel(const float* __restrict__ rgram, const Geom gm, const LdFin f,
                                                         float* __restrict__ sums) {
  const int g = blockIdx.y, k = blockIdx.z;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const LdLayout L(gm, f);
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= L.rec || L.mass()[k] == 0.f) return;
  const bool cov = e < GS * GS;
  const int i = cov ? e / GS : e - GS * GS, j = cov ? e % GS : 0;
  const double muj = cov ? (double)L.dom(k, g)[GS * GS + j] : 0.0;
  double acc = 0.0;
  for (int n = 0; n < gm.D; ++n) {
    const float w = __ldg(f.weights + (size_t)n * f.K + k);
    if (w == 0.f) continue;
    const float* Gn = rgram + ((size_t)n * SB + sb) * kNacc;
    const double gi = (double)__ldcg(Gn + kSB * kSB + o + i);
    double v = gi;
    if (cov) v = (double)__ldcg(Gn + (o + i) * kSB + o + j) + gi * ((double)f.save_mean[(size_t)n * gm.C + g * GS + j] - muj);
    acc += (double)w * v;
  }
  sums[((size_t)k * gm.G + g) * L.rec + e] = (float)acc;
}

// ld_bwd_dom: grid (G, 1, K), 256 threads (train), one CTA per (domain, group): from Wbar_k (sums) and W_k, the Cholesky
// backward P_k = dL/dSigma_k = a sym(W^T Phi(-Wbar W^T) W) and mubar_k = -W_k^T sum_n w_nk g_n into pd[k][g], and
// c_k = <P_k, Sigma_k> into pc[k][g].
__global__ void __launch_bounds__(256) ld_bwd_dom_kernel(const Geom gm, const LdFin f, const float* __restrict__ sums,
                                                         float* __restrict__ pd, float* __restrict__ pc) {
  extern __shared__ __align__(16) float dsm[];
  float* sW = dsm;
  float* sR = sW + kMat;
  float* sT = sR + kMat;
  __shared__ float sSdz[kSB], sRed[8];
  const int g = blockIdx.x, k = blockIdx.z, GS = gm.GS;
  const LdLayout L(gm, f);
  if (L.mass()[k] == 0.f) return;
  const Blk t(GS);
  const int gsh = __ffs(GS) - 1;
  const float* Wk = L.w_base() + ((size_t)k * gm.G + g) * GS * GS;
  const float* sm = sums + ((size_t)k * gm.G + g) * L.rec;
  const float* st = L.dom(k, g);
  float* out = pd + ((size_t)k * gm.G + g) * L.rec;
  PROF_DECL;
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    sW[i * LDS + j] = Wk[e];
    sR[i * LDS + j] = sm[e];
  }
  if ((int)threadIdx.x < GS) sSdz[threadIdx.x] = sm[GS * GS + threadIdx.x];
  __syncthreads();
  chol_bwd_core(sR, sW, sT, sR, GS, t PROF_PASS);        // T' = W^T Phi(-Wbar W^T) W into sT
  const float h = 0.5f * f.a;
  float c = 0.f;
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    const float p = h * (sT[i * LDS + j] + sT[j * LDS + i]);
    out[e] = p;
    c = fmaf(p, st[e], c);
  }
  {
    const int i = threadIdx.x >> 2, q = threadIdx.x & 3;
    float v = 0.f;
    if (i < GS)
      for (int j = q; j < GS; j += 4) v = fmaf(sW[j * LDS + i], sSdz[j], v);   // W_ji = 0 for j < i
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (q == 0 && i < GS) out[GS * GS + i] = -v;
  }
  c = block_sum(c, sRed);
  if (threadIdx.x == 0) pc[(size_t)k * gm.G + g] = c;
}

// ld_bwd_coef: grid (G, 1, D), 256 threads, one CTA per (image, group), the domains in order (skipping s_k == 0; the
// terms of dx also skip w_nk == 0, dweights does not: its derivative there is not 0).  With u_k = m_n - mu_k and
// v_k = m~_n - mu_k:
//   A1 = A_n^T,  Bm = train (2/M) sum_k (w_nk/s_k) P_k,
//   k_n = train (1/M) sum_k (w_nk/s_k) [mubar_k + 2 P_k u_k],  dybar = -A_n^-T k_n (0 when A1 or Bm is not finite)
//   part[n][g][k] = <W_k, R~_n + g_n v_k^T> + train [<mubar_k, u_k> + <P_k, C_n + u_k u_k^T> - c_k] / s_k
// and mu [D][C] = m_n, the centre of tc_bwd_apply's Bm term.
__global__ void __launch_bounds__(256) ld_bwd_coef_kernel(const float* __restrict__ rgram, const Geom gm, const LdFin f,
                                                          const float* __restrict__ pd, const float* __restrict__ pc,
                                                          float* __restrict__ part, float* __restrict__ coef,
                                                          float* __restrict__ dybar, float* __restrict__ mu) {
  extern __shared__ __align__(16) float dsm[];
  float* sA = dsm;
  float* sR = sA + kMat;
  __shared__ float sU[kLdMaxDomains][kSB], sV[kLdMaxDomains][kSB], sG[kSB], sK[kSB], sRed[8][kLdMaxDomains];
  const int g = blockIdx.x, n = blockIdx.z, K = f.K;
  const auto [GS, sb, o, SB] = group_pos(gm, g);
  const LdLayout L(gm, f);
  const int gsh = __ffs(GS) - 1;
  const bool train = f.train != 0;
  const float invM = 1.f / gm.M;
  const float* Gn = rgram + ((size_t)n * SB + sb) * kNacc;
  const float* cn = L.img(n, g);
  float* cf = coef + ((size_t)n * gm.G + g) * coef_stride(GS);
  float wk[kLdMaxDomains], rs[kLdMaxDomains];                         // w_nk (0: no share in dx), 1/s_k (0: the domain is skipped)
#pragma unroll
  for (int k = 0; k < kLdMaxDomains; ++k) {
    wk[k] = 0.f; rs[k] = 0.f;
    if (k < K) {
      const float s = L.mass()[k];
      if (s != 0.f) { wk[k] = __ldg(f.weights + (size_t)n * K + k); rs[k] = 1.f / s; }
    }
  }
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    sA[i * LDS + j] = f.save_w[((size_t)n * gm.G + g) * GS * GS + e];
    sR[i * LDS + j] = __ldcg(Gn + (o + i) * kSB + o + j);
  }
  if ((int)threadIdx.x < GS) {
    const int i = threadIdx.x;
    const float mn = cn[GS * GS + i], mt = f.save_mean[(size_t)n * gm.C + g * GS + i];
    sG[i] = __ldcg(Gn + kSB * kSB + o + i);
    mu[(size_t)n * gm.C + g * GS + i] = mn;
#pragma unroll
    for (int k = 0; k < kLdMaxDomains; ++k) {
      if (rs[k] == 0.f) continue;
      const float muk = L.dom(k, g)[GS * GS + i];
      sU[k][i] = mn - muk;
      sV[k][i] = mt - muk;
    }
  }
  __syncthreads();
  float dwp[kLdMaxDomains];
#pragma unroll
  for (int k = 0; k < kLdMaxDomains; ++k) dwp[k] = 0.f;
  bool nanc = false;
  for (int e = threadIdx.x; e < GS * GS; e += 256) {
    const int i = e >> gsh, j = e & (GS - 1);
    const float r = sR[i * LDS + j], gi = sG[i], cij = train ? cn[e] : 0.f;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < kLdMaxDomains; ++k) {
      if (rs[k] == 0.f) continue;
      const size_t kg = (size_t)k * gm.G + g;
      dwp[k] = fmaf(L.w_base()[kg * GS * GS + e], fmaf(gi, sV[k][j], r), dwp[k]);
      if (train) {
        const float p = pd[kg * L.rec + e];
        if (wk[k] != 0.f) q = fmaf(wk[k] * rs[k], p, q);
        dwp[k] = fmaf(rs[k] * p, fmaf(sU[k][i], sU[k][j], cij), dwp[k]);
      }
    }
    const float bm = 2.f * invM * q, av = sA[j * LDS + i];
    cf[GS * GS + e] = bm;
    cf[e] = j >= i ? av : 0.f;                            // A1 = A^T (A lower triangular)
    nanc = nanc || !isfinite(bm) || !isfinite(av);
  }
  if (train && (int)threadIdx.x < GS) {                   // <mubar_k, u_k> and -c_k, over s_k
    const int i = threadIdx.x;
#pragma unroll
    for (int k = 0; k < kLdMaxDomains; ++k) {
      if (rs[k] == 0.f) continue;
      const size_t kg = (size_t)k * gm.G + g;
      float v = pd[kg * L.rec + GS * GS + i] * sU[k][i];
      if (i == 0) v -= pc[kg];
      dwp[k] = fmaf(rs[k], v, dwp[k]);
    }
  }
  {                                                       // k_n: 4 threads per row, partial sums met by shuffle
    const int i = threadIdx.x >> 2, qq = threadIdx.x & 3;
    float v = 0.f;
    if (train && i < GS) {
#pragma unroll
      for (int k = 0; k < kLdMaxDomains; ++k) {
        if (wk[k] == 0.f) continue;
        const float* pk = pd + ((size_t)k * gm.G + g) * L.rec;
        float pu = 0.f;
        for (int j = qq; j < GS; j += 4) pu = fmaf(pk[i * GS + j], sU[k][j], pu);
        pu *= 2.f;
        if (qq == 0) pu += pk[GS * GS + i];
        v = fmaf(wk[k] * rs[k], pu, v);
      }
    }
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (qq == 0 && i < GS) sK[i] = v * invM;
  }
#pragma unroll
  for (int k = 0; k < kLdMaxDomains; ++k) {
    const float v = warp_sum(dwp[k]);
    if ((threadIdx.x & 31) == 0) sRed[threadIdx.x >> 5][k] = v;
  }
  nanc = __syncthreads_or(nanc) != 0;
  if ((int)threadIdx.x < K) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += sRed[w][threadIdx.x];
    part[((size_t)n * gm.G + g) * kLdMaxDomains + threadIdx.x] = s;
  }
  // a group whose A1 or Bm is not finite gets both as kApplyNaN
  if (nanc) {
    const float q = __int_as_float(kApplyNaN);
    for (int e = threadIdx.x; e < GS * GS; e += 256) { cf[e] = q; cf[GS * GS + e] = q; }
  }
  if (threadIdx.x < 32) {                                 // A^T z = -k, A^T upper triangular: rows i from the bottom
    const int l = threadIdx.x;
    float r0 = l < GS ? -sK[l] : 0.f, r1 = l + 32 < GS ? -sK[l + 32] : 0.f;
    for (int i = GS - 1; i >= 0; --i) {
      const float own = i >= 32 ? r1 : r0;
      const float zi = __shfl_sync(0xffffffffu, own, i & 31) / sA[i * LDS + i];
      if (l == (i & 31)) { if (i >= 32) r1 = zi; else r0 = zi; }
      if (l < i) r0 = fmaf(-sA[i * LDS + l], zi, r0);     // (A^T)_{l i} = A_il
      if (l + 32 < i) r1 = fmaf(-sA[i * LDS + l + 32], zi, r1);
    }
    float* db = dybar + ((size_t)n * SB + sb) * kSB + o;
    if (l < GS) db[l] = nanc ? 0.f : r0;
    if (l + 32 < GS) db[l + 32] = nanc ? 0.f : r1;
  }
}

// ld_dw: grid (ceil(D K / 256)), 256 threads: dweights[n][k] = the sum over the groups, in order and in fp64, of
// part[n][g][k] (0 for a skipped domain).
__global__ void __launch_bounds__(256) ld_dw_kernel(const float* __restrict__ part, const Geom gm, int K,
                                                    float* __restrict__ dw) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= gm.D * K) return;
  const int n = p / K, k = p % K;
  const float* q = part + (size_t)n * gm.G * kLdMaxDomains + k;
  double acc = 0.0;
  for (int g = 0; g < gm.G; ++g) acc += (double)__ldcg(q + (size_t)g * kLdMaxDomains);
  dw[p] = (float)acc;
}

constexpr size_t kFactorSmem = 0;   // fwd_factor: static shared memory only (panel buffers + covariance)
constexpr size_t kCoefSmem = sizeof(float) * 4 * kMat;
constexpr size_t kZcaFwdSmem = sizeof(float) * 4 * kMat;   // N, P, P^2, P^3 (66.6 KB; + 16.9 KB static)
constexpr size_t kZcaBwdSmem = sizeof(float) * 8 * kMat;   // W, N, Q, P, P^2, Q N, P^3, P Q N (133 KB)
constexpr size_t kEighFwdSmem = sizeof(float) * 2 * kMat;  // S / V, U (33.3 KB; + 17.6 KB static)
constexpr size_t kEighBwdSmem = sizeof(float) * 5 * kMat;  // W, U, R / G, R U / U H, H / Bm (83.2 KB)
constexpr size_t kColorFwdSmem = sizeof(float) * 2 * kMat; // color, W (33.3 KB; + 21.3 KB static)
constexpr size_t kColorBwdSmem = sizeof(float) * 6 * kMat; // W, R / R_hat, T1, T2, color, color W (99.8 KB)
constexpr size_t kSwCoefSmem = sizeof(float) * 3 * kMat;   // switchable backward: W, R / W^T Phi, Phi / T' (49.9 KB)
constexpr size_t kSwApplySmem = sizeof(float) * 2 * kMat;  // switchable backward coefficients: W, Q_b (33.3 KB)

}  // namespace

int dense_init() {
  const struct { const void* kernel; size_t smem; } dynamic_smem[] = {
      {(const void*)fwd_factor_kernel<false>, kFactorSmem},   {(const void*)bwd_coef_kernel, kCoefSmem},
      {(const void*)fwd_factor128_kernel, kFactor2Smem},      {(const void*)bwd_coef128_kernel, kCoef2Smem},
      {(const void*)fwd_zca_kernel, kZcaFwdSmem},             {(const void*)bwd_zca_kernel, kZcaBwdSmem},
      {(const void*)fwd_eigh_kernel, kEighFwdSmem},           {(const void*)bwd_eigh_kernel, kEighBwdSmem},
      {(const void*)fwd_factor_kernel<true>, kColorFwdSmem},  {(const void*)bwd_color_kernel, kColorBwdSmem},
      {(const void*)sw_bwd_coef_kernel, kSwCoefSmem},         {(const void*)ld_bwd_dom_kernel, kSwCoefSmem}};
  for (const auto& k : dynamic_smem) {
    const cudaError_t e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}

// partial [problems][nchunks][kNacc] -> gram [problems][kNacc]
void dense_partial_reduce(const float* partial, int nchunks, int problems, float* gram, cudaStream_t st) {
  partial_reduce_kernel<<<dim3((kNacc + 63) / 64, problems), 256, 0, st>>>(partial, nchunks, gram);
}

// gram == nullptr: eval mode (running buffers -> W).  Group size 128: gram holds [D][SB] diagonal blocks followed by
// [D][SB/2] off-diagonal blocks.
void dense_fwd_factor(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st) {
  if (gm.GS == kGS2) {
    const float* goff = gram ? gram + (size_t)gm.D * (gm.C / kSB) * kNacc : nullptr;
    fwd_factor128_kernel<<<gm.G, kThreads2, kFactor2Smem, st>>>(gram, goff, shift, gm, fin);
    return;
  }
  fwd_factor_kernel<false><<<gm.G, 256, kFactorSmem, st>>>(gram, shift, gm, fin, nullptr, nullptr);
}

// rgram == nullptr: eval mode without affine (A1 = W^T only).  Group size 128: rgram [D][2 SB] blocks.
void dense_bwd_coef(const float* rgram, const Geom& gm, const BwdFin& fin, float* dybar, cudaStream_t st) {
  if (gm.GS == kGS2) {
    bwd_coef128_kernel<<<dim3(gm.G, 1, gm.D), kThreads2, kCoef2Smem, st>>>(rgram, gm, fin, dybar);
    return;
  }
  bwd_coef_kernel<<<dim3(gm.G, 1, gm.D), 256, kCoefSmem, st>>>(rgram, gm, fin, dybar);
}

void dense_fwd_zca(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, int iters, float* save_p,
                   cudaStream_t st) {
  fwd_zca_kernel<<<gm.G, 256, kZcaFwdSmem, st>>>(gram, shift, gm, fin, iters, save_p);
}

void dense_bwd_zca(const float* rgram, const Geom& gm, const BwdFin& fin, int iters, const float* save_p, float* dybar,
                   cudaStream_t st) {
  bwd_zca_kernel<<<dim3(gm.G, 1, gm.D), 256, kZcaBwdSmem, st>>>(rgram, gm, fin, iters, save_p, dybar);
}

void dense_fwd_eigh(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, float* save_e, cudaStream_t st) {
  fwd_eigh_kernel<<<gm.G, 256, kEighFwdSmem, st>>>(gram, shift, gm, fin, save_e);
}

void dense_bwd_eigh(const float* rgram, const Geom& gm, const BwdFin& fin, const float* save_e, float* dybar, cudaStream_t st) {
  bwd_eigh_kernel<<<dim3(gm.G, 1, gm.D), 256, kEighBwdSmem, st>>>(rgram, gm, fin, save_e, dybar);
}

void dense_fwd_color(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, const float* color, float* gw,
                     cudaStream_t st) {
  fwd_factor_kernel<true><<<gm.G, 256, kColorFwdSmem, st>>>(gram, shift, gm, fin, color, gw);
}

void dense_bwd_color(const float* rgram, const Geom& gm, const BwdFin& fin, const float* color, float* dcolor, float* dbias,
                     float* dybar, cudaStream_t st) {
  bwd_color_kernel<<<gm.G, 256, kColorBwdSmem, st>>>(rgram, gm, fin, color, dcolor, dbias, dybar);
}

void dense_fwd_instance(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st) {
  fwd_instance_kernel<<<dim3(gm.G, 1, gm.D), 256, 0, st>>>(gram, shift, gm, fin);
}

void dense_sw_stats(const float* gram, const float* shift, const Geom& gm, const SwFin& fin, cudaStream_t st) {
  sw_stats_kernel<<<dim3((gm.GS * gm.GS + gm.GS + 255) / 256, gm.G), 256, 0, st>>>(gram, shift, gm, fin);
}

void dense_sw_fwd_factor(const Geom& gm, const SwFin& fin, cudaStream_t st) {
  sw_fwd_factor_kernel<<<dim3(gm.G, 1, gm.D), 256, 0, st>>>(gm, fin);
}

void dense_sw_bwd(const float* rgram, const Geom& gm, const SwFin& fin, float* pd, float* part, float* sums, float* dmix,
                  float* coef, float* dybar, float* mu, cudaStream_t st) {
  sw_bwd_coef_kernel<<<dim3(gm.G, 1, gm.D), 256, kSwCoefSmem, st>>>(rgram, gm, fin, pd, part);
  if (fin.train) sw_bwd_sum_kernel<<<dim3((gm.GS * gm.GS + gm.GS + 255) / 256, gm.G), 256, 0, st>>>(pd, gm, sums);
  if (dmix) sw_dmix_kernel<<<1, 256, 0, st>>>(part, gm.D * gm.G, dmix);
  sw_bwd_apply_coef_kernel<<<dim3(gm.G, 1, gm.D), 256, kSwApplySmem, st>>>(pd, sums, gm, fin, coef, dybar, mu);
}

void dense_ld_stats(const float* gram, const float* shift, const Geom& gm, const LdFin& fin, cudaStream_t st) {
  ld_stats_kernel<<<dim3((gm.GS * gm.GS + gm.GS + 255) / 256, gm.G, fin.K), 256, 0, st>>>(gram, shift, gm, fin);
}

void dense_ld_fwd(const Geom& gm, const LdFin& fin, cudaStream_t st) {
  ld_fwd_factor_kernel<<<dim3(gm.G, 1, fin.K), 256, 0, st>>>(gm, fin);
  ld_mix_kernel<<<dim3(gm.G, 1, gm.D), 256, 0, st>>>(gm, fin);
}

// eval: the coefficients and the direct term of dweights only (Sigma_k and mu_k are constants)
void dense_ld_bwd(const float* rgram, const Geom& gm, const LdFin& fin, float* sums, float* pd, float* pc, float* part,
                  float* dweights, float* coef, float* dybar, float* mu, cudaStream_t st) {
  if (fin.train) {
    ld_bwd_sum_kernel<<<dim3((gm.GS * gm.GS + gm.GS + 255) / 256, gm.G, fin.K), 256, 0, st>>>(rgram, gm, fin, sums);
    ld_bwd_dom_kernel<<<dim3(gm.G, 1, fin.K), 256, kSwCoefSmem, st>>>(gm, fin, sums, pd, pc);
  }
  ld_bwd_coef_kernel<<<dim3(gm.G, 1, gm.D), 256, kSwApplySmem, st>>>(rgram, gm, fin, pd, pc, part, coef, dybar, mu);
  if (dweights) ld_dw_kernel<<<(gm.D * fin.K + 255) / 256, 256, 0, st>>>(part, gm, fin.K, dweights);
}

}  // namespace dwt

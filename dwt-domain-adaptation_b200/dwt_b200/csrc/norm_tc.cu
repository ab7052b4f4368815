// Tensor-core path for the two CONTRACTIONS over the flattened N*H*W axis when groups are large
// (group size 8..64, i.e. BASELINE.json config 2: C=256, group_size=64; and 128, see below):
//
//   stats       G = sum_m (x-K)(x-K)^T        per 64-channel super-block (gs x gs diagonal blocks kept)
//   bwd_reduce  R = sum_m dy (x-mean)^T
//
// 2*gs flop per 4 bytes read puts these far below the TF32 tensor ridge: they are HBM-bound.  All three kernels are
// persistent CTAs (two per SM) over a contiguous range of [64 channels x 32 pixels] tiles (TileRange), warp-specialised
// (tc_ring.cuh), and differ only in what a stage holds, the transforms, the products and the last epilogue step:
//
//   produce     warp 8: cp.async.bulk.tensor.3d (box 32 px x 64 ch x 1 image, SWIZZLE_128B) into the Ring of
//               shared-memory stages, mbarrier complete_tx.
//   consume     warps 0-7, two warpgroups taking alternate tiles: the kernel's transform splits the landed tile for the
//               tensor core and names the tile's Products, issued as wgmma.mma_async kind::tf32 (M = 64 channels, K = 8
//               pixels per instruction) into a fresh fp32 accumulator in registers, then the stage is released.  Operands
//               are K-major straight from the swizzled tile (NCHW rows ARE K-major: the reference's transposing copy,
//               whitening.py:46, disappears).
//   cta_sums    the two warpgroups' sums are added in shared memory -> per-CTA partial -> global.  The fixed-order
//               reduction of the partials and the dense algebra (Cholesky / inverse / EMA, or the backward
//               coefficients) run as the small follow-up launches of norm_dense.cu.
//
// stats (tc_gram_kernel) -- SPLIT precision.  The covariance feeds a Cholesky factor whose error is the Gram
// error times the condition number (the eps = 1e-3 shrinkage is absolute and stops helping once activations are
// large), so a single tf32 pass is not enough (y errors of 1e-3..5e-3 at cond >= 1e4).  Each centred sample
// s = x - K is split hi = trunc_tf32(s) and lo = s - hi (exact in fp32; the core keeps its top 11 bits), and
//       G = (S + S^T) / 2,  S = HH + 2 LH      HH = sum hi hi^T,  LH = sum lo hi^T     (lo lo^T ~ 3e-7 G is dropped)
// comes out of two M=64 N=64 K=8 MMAs per 8 pixels: A = the hi tile (written back in place) or the 2 lo tile (a
// per-warpgroup buffer; doubling is exact), B = the hi tile.  ACCUMULATION: each 32-pixel tile's eight MMAs go into a
// fresh accumulator (the first one overwrites it) that is added into an fp32 register sum after the tile.  The tensor
// core's own fp32 accumulation loses about one low bit per instruction, and not at random: with one accumulator per CTA
// (~760 instructions per warpgroup at config 2, ~380 tiles per CTA) the covariance drifted 3.9e-5 from float64, growing
// with the tiles per CTA (8.1e-5 at 760); per tile it stays at 7.5e-7 at every length
// (tests/test_tc_forward_stats_fp64.py).  The row sums the mean needs are summed by the transform.
//
// bwd_reduce (tc_contract_kernel) -- SPLIT precision, dy CENTRED.  A single tf32 pass (RN_tf32(dy) RN_tf32(xc)^T) is
// accurate only for gradients like iid randn.  A per-channel mean c in dy adds about 2^-11 c sigma_x sqrt(M) of error to
// R, although the true R does not depend on c (sum xc = 0); and a dy mostly along y largely cancels in dx, so R's 2^-11
// relative error comes back amplified.  Both are what real networks send back (a following bias, an affine layer's
// dgamma direction): at N*HW = 4096 dx was off by up to 1.1e-2 of fp64.  So dy is centred around a per-(domain, channel)
// pilot shift K of dy (pilot_shift on dout: every CTA of a problem computes the same K), e = dy - K and xc = x - mean are
// both split hi / lo as in the Gram kernel, and  R = Eh Xh^T + El Xh^T + Eh Xl^T  (sum e xc^T is R: sum_m xc = 0 up to the
// rounding of save_mean), each tile into a fresh accumulator added into an fp32 register sum; the row sums are
// sum e + n_valid K, in the CTA epilogue, so the partial layout and everything downstream are unchanged.  dx then lands
// within a small factor of the float32 operator sequence (tools/tf32_contract_accuracy.py,
// tests/test_tc_backward_fp64.py).  Cost at config 2 (DESIGN.md section 8): fp32 +3.4 % on this kernel, fp32 NHWC +13 %,
// bf16 +57 % (NCHW) / +53 % (NHWC): with half the bytes, the split transform rather than HBM bounds the bf16 kernels.
//
// bf16 activations (DWT_DTYPE_BF16): both kernels are templated on the storage type T.  A bf16 box is 32 px x 64 ch of
// 2-byte values, 64-byte rows landed without swizzle (only ld.shared reads it: a warp's 8-byte loads cover whole rows,
// conflict-free).  The transform widens each value to fp32 and writes exactly what it writes in place for an fp32 tile
// -- same values, same SWIZZLE_128B positions -- into a per-warpgroup fp32 staging tile (the Gram kernel: hi there, lo to
// its lo tile; the contraction: the hi parts of xc and dy each to their own, the lo parts to the lo tiles), releases the
// ring stage and issues the unchanged wgmma sequence from the staging tiles.  Grid, tile ranges, warpgroup alternation
// and epilogue are those of the fp32 kernels, so every partial is bit for bit the fp32 kernel's on x.float().
//
// channels-last activations (DWT_LAYOUT_NHWC): both kernels are also templated on the layout.  The tensor map is 3-D
// {C, HW, N*D} with channels innermost; a tile is the same [64 ch x 32 px] block of one image, landed as rows of pixels:
// fp32 two boxes of 32 ch x 32 px (128-byte rows, SWIZZLE_128B), bf16 one box of 64 ch x 32 px (likewise).  TMA zero
// fill past C and past HW keeps the NCHW tile schedule, partial tiles and partial super-blocks included.  wgmma wants K
// (the pixels) contiguous, so the transform reads each thread's (channel, 4-pixel chunk) from the landed [px][ch] tile
// and writes exactly what the NCHW transform writes, at the same swizzled positions, into the per-warpgroup fp32
// staging tiles of the bf16 kernels; the rest is the NCHW kernel, so every partial is bit for bit the NCHW kernel's on
// x.contiguous().  fp32 rings are shallower (Gram 8, contraction 2 stages) to keep two CTAs per SM with the staging.
//
// group size 128 (fp32, both layouts): a group spans the super-blocks 2p and 2p + 1, so its 128 x 128 statistics are
// three 64 x 64 blocks plus the 128 row sums.
//   Gram: the diagonal blocks and row sums are tc_gram_kernel's, unchanged (it never reads the group size); the
//   off-diagonal block G10 = sum s1 s0^T comes from tc_gram_pair_kernel, one launch later: a stage carries the tiles of
//   both super-blocks, each is split hi / lo by split_transform around the same pilot shifts (read back from the diagonal
//   launch), and H1 H0^T + L1 H0^T + H1 L0^T go into a fresh accumulator per tile, added into an fp32 register sum --
//   the hi/lo model of the diagonal kernel over the whole 128-vector (lo lo^T dropped, lo hi^T kept on both sides).
//   Chosen over one CTA holding both super-blocks' tiles and all seven 64 x 64 accumulators (224 registers per thread
//   for one warpgroup, or an uneven split of block rows across warpgroups) because it reuses the diagonal kernel as it is and keeps two CTAs per SM.  Cost: x is read
//   from HBM twice per call (the second pass is a separate launch over an 822 MB tensor at BASELINE config 2, far
//   beyond L2) -- 2x by design, not measured directly; the profile counts the algorithmic bytes once.
//   Contraction: tc_contract_kernel<.., PAIR = true> forms all four blocks of R (it is not symmetric), blockIdx.y =
//   4 p + 2 r + c: dy rows from super-block 2p + r (and their shift K), x columns from 2p + c; x and dy are each read twice (concurrently
//   by the blocks of one wave, so partly from L2; not measured).
//   ptxas (sm_90a): tc_gram_kernel 96 registers in all four instantiations; tc_gram_pair_kernel NCHW 90 / NHWC 88
//   registers; tc_contract_kernel<float, NCHW / NHWC, PAIR> 96 / 94 registers; no spills; dynamic shared memory 97 KB (gram pair) and the contraction's 97 KB as above.
//
// Reference: utils/whitening.py:46-47 of the reference project and its autograd transpose.
#include <cuda.h>
#include <cuda_bf16.h>

#include "dwt_common.cuh"
#include "norm_launch.h"
#include "tc_ring.cuh"

namespace dwt {
namespace {

using namespace tc;

constexpr int kPer = 512 / 128;                         // 16-byte chunks of a tile per consumer thread
constexpr int kTilePx = 32, kTileCh = 64;
constexpr int kTileBytes = kTileCh * kTilePx * 4;       // 8192: one fp32 tile (also a staging tile of the bf16 kernels)
constexpr int kStagesBwd = 4;                           // x + dy per stage: 64 KB + 32 KB lo tiles per CTA (bf16: 32 KB + 64 KB)
constexpr int kNacc = kTileCh * kTileCh + kTileCh;      // per-CTA partial: 64x64 moments + 64 row sums
constexpr int kGramStages = 10;                         // 80 KB ring + 2 x 8 KB lo tiles per CTA (bf16: 40 KB + 32 KB)
// a landed box is kTileCh x kTilePx values of T
template <class T> constexpr int kBoxBytes = kTileCh * kTilePx * (int)sizeof(T);
// Layout NHWC: the transform writes to staging tiles (the bf16 kernels always do).  fp32 NHWC: the staging tiles cost
// 32 KB (Gram) or 64 KB (contraction: hi and lo of xc and dy) per CTA, so the rings are shallower to keep two CTAs per SM
// (Gram 64 + 32 KB, contraction 32 + 64 KB).
template <class T, bool NHWC> constexpr bool kStaged = kBf16<T> || NHWC;
template <class T, bool NHWC> constexpr int kGramStagesOf = (NHWC && !kBf16<T>) ? 8 : kGramStages;
template <class T, bool NHWC> constexpr int kStagesBwdOf = (NHWC && !kBf16<T>) ? 2 : kStagesBwd;
template <bool NHWC> constexpr int kPairStagesOf = NHWC ? 2 : 4;

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// Pixels 4j .. 4j+3 of tile row `row` as fp32.  fp32: the 16-byte chunk q = 8 row + (j ^ (row & 7)) of the SWIZZLE_128B
// tile.  bf16: 8 bytes at row * 64 + 8 j of the unswizzled box, widened (bf16 -> fp32 is exact: the high half of the word).
// NHWC: channel `row` of pixels 4j .. 4j+3 of the landed [px][ch] tile, one load per pixel.
template <class T, bool NHWC>
__device__ __forceinline__ float4 ld_px4(uint32_t tile, int q, int row, int j) {
  if constexpr (NHWC) {
    // landed [px][ch] tile, 128-byte pixel rows, SWIZZLE_128B (fp32: two boxes of 32 channels, 4 KB apart; bf16: one of
    // 64).  Pixel 4j + k is row 4j + k; its 16-byte chunk holding channel `row` is c4 ^ (4 (j & 1) + k) = a ^ k.
    const int c4 = kBf16<T> ? row >> 3 : (row & 31) >> 2, a = c4 ^ ((j & 1) << 2);
    const uint32_t base = tile + 512u * j + (kBf16<T> ? 2u * (row & 7) : 4096u * (row >> 5) + 4u * (row & 3));
    return make_float4(lds_f<T>(base + (a << 4)), lds_f<T>(base + 128u + ((a ^ 1) << 4)),
                       lds_f<T>(base + 256u + ((a ^ 2) << 4)), lds_f<T>(base + 384u + ((a ^ 3) << 4)));
  } else if constexpr (kBf16<T>) {
    uint32_t a, b;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "r"(tile + 64u * row + 8u * j));
    return make_float4(__uint_as_float(a << 16), __uint_as_float(a & 0xFFFF0000u), __uint_as_float(b << 16),
                       __uint_as_float(b & 0xFFFF0000u));
  } else {
    return lds128(tile + 16u * q);
  }
}
template <class T> __device__ __forceinline__ float ldg_f(const T* p) {
  if constexpr (kBf16<T>) return __bfloat162float(__ldg(p));
  else return __ldg(p);
}

// Pilot shift of channel c: the mean of <= 32 mid-image pixels of image 0 of domain d, moved to the mean of 32 samples
// spread over the domain where that lies more than 20 of their standard deviations away (pilot_shift in dwt_common.cuh).
// NHWC reads the same samples: pixel p of image n at (n * HW + p) * C from the channel.
template <class T, bool NHWC>
__device__ __forceinline__ float pilot_shift(const T* __restrict__ x, const Geom& gm, int d, int c) {
  if (c >= gm.C) return 0.f;
  const int np = gm.HW < 32 ? gm.HW : 32, p0 = ((gm.HW - np) / 2) & ~3;
  const T* xc = NHWC ? x + (size_t)d * gm.N * gm.C * gm.HW + c : x + ((size_t)d * gm.N * gm.C + c) * gm.HW;
  float a = 0.f;
  if constexpr (NHWC) for (int k = 0; k < np; ++k) a += ldg_f(xc + (size_t)(p0 + k) * gm.C);
  else for (int k = 0; k < np; ++k) a += ldg_f(xc + p0 + k);
  const float K = a / (float)np;
  if ((long long)gm.N * gm.HW <= kPilotSpread) return K;
  float s1 = 0.f, s2 = 0.f;
  for (int k = 0; k < kPilotSpread; ++k) {
    const size_t o = NHWC ? pilot_spread_offset(k, gm.N, gm.HW, (size_t)gm.HW) * gm.C
                          : pilot_spread_offset(k, gm.N, gm.HW, (size_t)gm.C * gm.HW);
    const float e = ldg_f(xc + o) - K;
    s1 += e;
    s2 = fmaf(e, e, s2);
  }
  return pilot_refine(K, s1, s2);
}

// Split transform of one landed tile by the 128 threads of a consumer warpgroup (thread t): s = v - shift[row] (shared
// memory) inside the
// tensor, 0 outside; hi = trunc_tf32(s) to hi (fp32 NCHW: the tile itself, in place), lo = s - hi (exact) to the
// warpgroup's lo tile at the same swizzled position; returns per-thread row sums of s.  hi is written explicitly so that
// every product sees the same hi whatever rounding the tensor core applies to fp32 words.  Chunk q = t + 128 i (16-byte
// units): row = q >> 3, physical chunk q & 7, logical chunk (q & 7) ^ (row & 7).  Two chunks at a time: the accumulators
// leave few registers at two CTAs per SM.  LO2: the lo tile holds 2 lo (exact), for the Gram kernel's symmetric form.
template <class T, bool NHWC, bool LO2 = false>
__device__ __forceinline__ void split_transform(uint32_t tile, uint32_t hi, uint32_t lo, int t, const float* shift, int px0,
                                                int HW, int ch0, int C, float (&rowsum)[kPer]) {
#pragma unroll
  for (int h = 0; h < kPer; h += 2) {
    float4 v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = t + 128 * (h + i), row = q >> 3;
      if constexpr (!NHWC) v[i] = ld_px4<T, NHWC>(tile, q, row, (q & 7) ^ (row & 7));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = t + 128 * (h + i), row = q >> 3, j = (q & 7) ^ (row & 7);
      if constexpr (NHWC) v[i] = ld_px4<T, NHWC>(tile, q, row, j);
      const int px = px0 + 4 * j;
      const bool rowok = (ch0 + row) < C;
      const float sh = shift[row];
      float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w}, l[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float s = (rowok && (px + k) < HW) ? e[k] - sh : 0.f;
        rowsum[h + i] += s;
        e[k] = __uint_as_float(__float_as_uint(s) & kTf32Mask);
        l[k] = LO2 ? 2.f * (s - e[k]) : s - e[k];
      }
      sts128(hi + 16u * q, e[0], e[1], e[2], e[3]);
      sts128(lo + 16u * q, l[0], l[1], l[2], l[3]);
    }
  }
}

// The 8 consecutive threads that share a tile row (chunk q = t + 128 i, row = q >> 3) add their row sums into s[row].
__device__ __forceinline__ void add_rowsums(float* s, const float (&rowsum)[kPer], int t) {
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    float v = rowsum[i];
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    if ((t & 7) == 0) atomicAdd(s + ((t + 128 * i) >> 3), v);
  }
}

// Adds a warpgroup's [64 x 8*NB] accumulator fragment into a shared [64][pitch] matrix.  wgmma layout: thread (warp w,
// lane l) holds, for every 8-column block j, rows 16w + l/4 and 16w + l/4 + 8 at columns 8j + 2(l%4) and 8j + 2(l%4) + 1.
// At most two warpgroups add into a zeroed entry, so the result does not depend on their order.
template <int NB>
__device__ __forceinline__ void add_fragment(float* s, int pitch, const float (&acc)[4 * NB], int warp, int lane) {
  const int r0 = 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    atomicAdd(s + r0 * pitch + 8 * j + c0, acc[4 * j]);
    atomicAdd(s + r0 * pitch + 8 * j + c0 + 1, acc[4 * j + 1]);
    atomicAdd(s + (r0 + 8) * pitch + 8 * j + c0, acc[4 * j + 2]);
    atomicAdd(s + (r0 + 8) * pitch + 8 * j + c0 + 1, acc[4 * j + 3]);
  }
}

// TMA of one input's tile (channels ch0.., pixels px0.. of image img) into dst: NCHW one box {32 px, 64 ch}; NHWC fp32 two
// boxes {32 ch, 32 px} (channel halves, 4 KB apart), NHWC bf16 one box {64 ch, 32 px}.  Always kBoxBytes<T> bytes.
template <class T, bool NHWC>
__device__ __forceinline__ void tma_tile(uint8_t* dst, const CUtensorMap* map, int ch0, int px0, int img, uint64_t* bar) {
  if constexpr (!NHWC) {
    tma_load_3d(dst, map, px0, ch0, img, bar);
  } else {
    tma_load_3d(dst, map, ch0, px0, img, bar);
    if constexpr (!kBf16<T>) tma_load_3d(dst + 4096, map, ch0 + 32, px0, img, bar);
  }
}

// ---- the pipeline shared by the three kernels

// TMA producer (one thread): tile it of the range goes to stage it % STAGES once the stage's previous phase is released;
// issue(stage, px0, image, full barrier) issues the tile's `bytes`.
template <int STAGES, class Issue>
__device__ __forceinline__ void produce(Ring<STAGES>& ring, const TileRange<kTilePx>& tr, int img0, uint32_t bytes, Issue issue) {
  int n = tr.begin / tr.PB, pb = tr.begin - n * tr.PB;
  for (int it = 0; it < tr.end - tr.begin; ++it) {
    const int s = it % STAGES;
    mbar_wait_relaxed(&ring.empty[s], ((it / STAGES) & 1) ^ 1);
    mbar_arrive_expect_tx(&ring.full[s], bytes);
    issue(s, pb * kTilePx, img0 + n, &ring.full[s]);
    if (++pb == tr.PB) { pb = 0; ++n; }
  }
}

// The MMA chain of one tile: per 8-pixel k-step, D += A_p B_p^T for p = 0 .. N-1 (K-major descriptors of 32-pixel rows)
template <int N> struct Products {
  static constexpr int kN = N;
  uint64_t a[N], b[N];
};

// One consumer warpgroup's tiles.  transform(stage address, px0) splits the landed stage into the operand tiles and
// returns the tile's products; they go into a fresh accumulator (the first MMA overwrites it, see the file header) that
// is then added into tot.  A STAGED stage is released as soon as the transform has read it; an in-place one (fp32 NCHW:
// hi is written over the landed tile) only after the wait on the MMAs.  The operand tiles of a warpgroup are rewritten
// by its next transform, hence the wait before it.
template <bool STAGED, int STAGES, class Transform>
__device__ __forceinline__ void consume(Ring<STAGES>& ring, const TileRange<kTilePx>& tr, uint32_t ring0, uint32_t stage_bytes,
                                        float (&tot)[32], Transform transform) {
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int it = wg; it < tr.end - tr.begin; it += kConsumers) {
    const int s = it % STAGES;
    mbar_wait(&ring.full[s], (it / STAGES) & 1);
    const int tl = tr.begin + it, n = tl / tr.PB, pb = tl - n * tr.PB;
    const auto p = transform(ring0 + s * stage_bytes, pb * kTilePx);
    if constexpr (STAGED) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&ring.empty[s]);
    }
    fence_proxy_async();
    warpgroup_sync(wg);
    wgmma_fence();
    fence_operands(acc);
#pragma unroll
    for (int k = 0; k < kTilePx / 8; ++k)
#pragma unroll
      for (int q = 0; q < p.kN; ++q) {
        if (k == 0 && q == 0) wgmma_m64n64k8_ss<false>(acc, p.a[0], p.b[0]);     // D = product: a fresh sum per tile
        else wgmma_m64n64k8_ss(acc, p.a[q] + 2 * k, p.b[q] + 2 * k);
      }
    wgmma_commit();
    wgmma_wait<0>();
    fence_operands(acc);
    if constexpr (!STAGED) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&ring.empty[s]);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) tot[i] += acc[i];
  }
}

// Epilogue (all threads, once every stage is consumed and the ring is free): both warpgroups' tot and, unless null,
// row sums are added into a zeroed [64][P] matrix + [64] row sums over the ring; returns it complete.
template <int P>
__device__ __forceinline__ const float* cta_sums(uint8_t* smem, const float (&tot)[32], const float (*rowsum)[kPer]) {
  const int tid = threadIdx.x;
  float* s = reinterpret_cast<float*>(smem);
  __syncthreads();
  for (int e = tid; e < kTileCh * P + kTileCh; e += kTcThreads) s[e] = 0.f;
  __syncthreads();
  if (tid < 32 * kProducerWarp) {
    add_fragment<8>(s, P, tot, tid >> 5, tid & 31);
    if (rowsum) add_rowsums(s + kTileCh * P, *rowsum, tid & 127);
  }
  __syncthreads();
  return s;
}

// this CTA's row of partial: [D][gridDim.y][gridDim.x][kNacc]
__device__ __forceinline__ float* partial_row(float* partial) {
  return partial + (((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * kNacc;
}

// ------------------------------------------------------------------------------------------
// backward contraction: R = sum dy xc^T and the row sums of dy, split and centred (see the file header)
// ------------------------------------------------------------------------------------------
// Per tile: xc = x - save_mean and e = dy - K (K: the pilot shift of dy's channel, the same in every CTA of a problem)
// are split hi / lo by split_transform, and  Eh Xh^T + El Xh^T + Eh Xl^T  go into a fresh accumulator (El Xl^T dropped, as
// in the Gram kernel) that is added into the warpgroup's fp32 sum after the tile.  The tensor core's own accumulation
// loses about one low bit per instruction; over the ~1,100 instructions per warpgroup of a config-2 CTA that built up
// to 6e-3 of the dx of a y-aligned gradient (measured), per tile it stays at 12.  sum_m e xc^T is R itself: sum_m xc is
// M (mean - save_mean), zero up to the rounding of save_mean, so K (sum xc)^T is not formed (it would add back the
// M K (mean - save_mean)^T that rounding costs).  The row sums need K back:  rowsum_cta = sum_cta e + n_valid K.
// PAIR (group size 128): blockIdx.y = 4 p + 2 r + c is block (r, c) of the 128 x 128 R of pair p: dy rows from
// super-block 2p + r, x columns from super-block 2p + c (R is not symmetric: all four blocks are formed).
// PILOT = false: K = 0.  With save_mean a running mean, sum xc is not zero and the centred sum is not R.
template <class T, bool NHWC, bool PAIR = false, bool PILOT = true>
__global__ void __launch_bounds__(kTcThreads, 2)
tc_contract_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_g, const T* __restrict__ dout,
                   const Geom gm, const float* __restrict__ save_mean, float* __restrict__ partial) {
  constexpr int STAGES = kStagesBwdOf<T, NHWC>, BOX = kBoxBytes<T>;
  constexpr bool STAGED = kStaged<T, NHWC>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = ring_smem(smem_raw);
  __shared__ Ring<STAGES> ring;
  __shared__ float sShift[kTileCh], sK[kTileCh];
  const int tid = threadIdx.x, sb = blockIdx.y, d = blockIdx.z;
  const int ch0 = PAIR ? (2 * (sb >> 2) + ((sb >> 1) & 1)) * kTileCh : sb * kTileCh;     // dy channels
  const int chx = PAIR ? (2 * (sb >> 2) + (sb & 1)) * kTileCh : ch0;                    // x channels
  const TileRange<kTilePx> tr(gm);

  if (tid == 0) ring.init();
  if (tid < kTileCh) sShift[tid] = chx + tid < gm.C ? save_mean[(size_t)d * gm.C + chx + tid] : 0.f;
  __syncthreads();

  float tot[32], rowsum[kPer], dummy[kPer];
#pragma unroll
  for (int i = 0; i < 32; ++i) tot[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; ++i) { rowsum[i] = 0.f; dummy[i] = 0.f; }

  if (tid >> 5 == kProducerWarp) {
    if ((tid & 31) == 0)
      produce(ring, tr, d * gm.N, 2 * BOX, [&](int s, int px0, int img, uint64_t* bar) {
        tma_tile<T, NHWC>(smem + (size_t)s * 2 * BOX, &map_x, chx, px0, img, bar);
        tma_tile<T, NHWC>(smem + (size_t)s * 2 * BOX + BOX, &map_g, ch0, px0, img, bar);
      });
  } else {
    // dy's shift: its dependent loads overlap the producer's first TMA loads (named barrier 3: the consumers only)
    if (tid < kTileCh) sK[tid] = PILOT ? pilot_shift<T, NHWC>(dout, gm, d, ch0 + tid) : 0.f;          // 0 past C
    asm volatile("bar.sync 3, %0;" ::"n"(128 * kConsumers) : "memory");
    // per warpgroup behind the ring: the lo tiles of xc and dy (fp32 NCHW: hi in place), or hi and lo of both (bf16 / NHWC)
    const int t = tid & 127;
    const uint32_t wgbuf = smem_u32(smem + (size_t)STAGES * 2 * BOX + (size_t)(tid >> 7) * (STAGED ? 4 : 2) * kTileBytes);
    const uint32_t xlo = STAGED ? wgbuf + 2 * kTileBytes : wgbuf, dlo = xlo + kTileBytes;
    consume<STAGED>(ring, tr, smem_u32(smem), 2 * BOX, tot, [&](uint32_t tile, int px0) {
      const uint32_t xhi = STAGED ? wgbuf : tile, dhi = STAGED ? wgbuf + kTileBytes : tile + kTileBytes;
      split_transform<T, NHWC>(tile, xhi, xlo, t, sShift, px0, gm.HW, chx, gm.C, dummy);          // xc
      split_transform<T, NHWC>(tile + BOX, dhi, dlo, t, sK, px0, gm.HW, ch0, gm.C, rowsum);      // dy - K
      const uint64_t xh = make_kmajor_sw128_desc(xhi), dh = make_kmajor_sw128_desc(dhi);
      const uint64_t xl = make_kmajor_sw128_desc(xlo), dl = make_kmajor_sw128_desc(dlo);
      return Products<3>{{dh, dl, dh}, {xh, xh, xl}};
    });
  }

  // both warpgroups' sums + row sums (K folded back in) -> this CTA's partial row
  const float* s = cta_sums<kTileCh>(smem, tot, &rowsum);
  // in-tensor pixels of the range: 32 per tile, less (PB * 32 - HW) for every last tile of an image in it
  const int n_valid = (tr.end - tr.begin) * kTilePx - (tr.end / tr.PB - tr.begin / tr.PB) * (tr.PB * kTilePx - gm.HW);
  float* prow = partial_row(partial);
  for (int e = tid; e < kTileCh * kTileCh; e += kTcThreads) prow[e] = s[e];
  if (tid < kTileCh) prow[kTileCh * kTileCh + tid] = fmaf((float)n_valid, sK[tid], s[kTileCh * kTileCh + tid]);
}

// ------------------------------------------------------------------------------------------
// split-precision Gram kernel (forward statistics): G = HH + LH + LH^T, see the file header
// ------------------------------------------------------------------------------------------
template <class T, bool NHWC>
__global__ void __launch_bounds__(kTcThreads, 2)
tc_gram_kernel(const __grid_constant__ CUtensorMap map_x, const T* __restrict__ x, const Geom gm,
               float* __restrict__ shift_out, float* __restrict__ partial) {
  constexpr int STAGES = kGramStagesOf<T, NHWC>, BOX = kBoxBytes<T>;
  constexpr bool STAGED = kStaged<T, NHWC>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = ring_smem(smem_raw);
  __shared__ Ring<STAGES> ring;
  __shared__ float sShift[kTileCh];
  const int tid = threadIdx.x, sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kTileCh;
  const TileRange<kTilePx> tr(gm);

  if (tid == 0) ring.init();
  if (tid < kTileCh) {
    const float sh = pilot_shift<T, NHWC>(x, gm, d, ch0 + tid);
    sShift[tid] = sh;
    if (blockIdx.x == 0) shift_out[((size_t)d * gridDim.y + sb) * kTileCh + tid] = sh;
  }
  __syncthreads();

  float tot[32], rowsum[kPer];
#pragma unroll
  for (int i = 0; i < 32; ++i) tot[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; ++i) rowsum[i] = 0.f;

  if (tid >> 5 == kProducerWarp) {
    if ((tid & 31) == 0)
      produce(ring, tr, d * gm.N, BOX, [&](int s, int px0, int img, uint64_t* bar) {
        tma_tile<T, NHWC>(smem + (size_t)s * BOX, &map_x, ch0, px0, img, bar);
      });
  } else {
    // per warpgroup behind the ring: the lo tile (fp32 NCHW), or the hi staging tile and the lo tile (bf16 / NHWC)
    const int t = tid & 127;
    const uint32_t wgbuf = smem_u32(smem + (size_t)STAGES * BOX + (size_t)(tid >> 7) * (STAGED ? 2 : 1) * kTileBytes);
    const uint32_t lo = STAGED ? wgbuf + kTileBytes : wgbuf;
    const uint64_t ldesc = make_kmajor_sw128_desc(lo);
    consume<STAGED>(ring, tr, smem_u32(smem), BOX, tot, [&](uint32_t tile, int px0) {       // hi hi^T + (2 lo) hi^T
      const uint32_t hi = STAGED ? wgbuf : tile;
      split_transform<T, NHWC, true>(tile, hi, lo, t, sShift, px0, gm.HW, ch0, gm.C, rowsum);
      const uint64_t bdesc = make_kmajor_sw128_desc(hi);
      return Products<2>{{bdesc, ldesc}, {bdesc, bdesc}};
    });
  }

  // both warpgroups' sums S = HH + 2 LH, G = (S + S^T) / 2 and the row sums -> this CTA's partial row
  constexpr int P = kTileCh + 1;                   // odd pitch: the transposed read is conflict-free
  const float* s = cta_sums<P>(smem, tot, &rowsum);
  float* prow = partial_row(partial);
  for (int e = tid; e < kTileCh * kTileCh; e += kTcThreads) {
    const int r = e >> 6, c = e & 63;
    prow[e] = 0.5f * (s[r * P + c] + s[c * P + r]);
  }
  if (tid < kTileCh) prow[kTileCh * kTileCh + tid] = s[kTileCh * P + tid];
}

// ------------------------------------------------------------------------------------------
// group size 128, off-diagonal Gram block: G10 = sum_m s1 s0^T of pair p (s1: super-block 2p + 1, s0: super-block 2p),
// split precision over the whole 128-vector:  G10 = H1 H0^T + L1 H0^T + H1 L0^T  (L1 L0^T dropped, as lo lo^T above)
// ------------------------------------------------------------------------------------------
// fp32 only.  Stage = the two [64 ch x 32 px] tiles of one image block.  The three products share ONE accumulator (no
// transpose is needed off the diagonal), so registers stay below the diagonal kernel's.  Shared memory per CTA: NCHW
// 4 stages x 16 KB + two lo tiles per warpgroup (hi in place) = 96 KB; NHWC 2 stages x 16 KB + hi and lo staging of
// both tiles per warpgroup = 96 KB; two CTAs per SM either way.  The pilot shifts are the diagonal kernel's (shift).
template <bool NHWC>
__global__ void __launch_bounds__(kTcThreads, 2)
tc_gram_pair_kernel(const __grid_constant__ CUtensorMap map_x, const Geom gm, const float* __restrict__ shift,
                    float* __restrict__ partial) {
  constexpr int STAGES = kPairStagesOf<NHWC>, BOX = kTileBytes;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = ring_smem(smem_raw);
  __shared__ Ring<STAGES> ring;
  __shared__ float sShift[2][kTileCh];             // [0] rows (super-block 2p + 1), [1] columns (super-block 2p)
  const int tid = threadIdx.x, p = blockIdx.y, d = blockIdx.z, SB = gm.C / kTileCh;
  const int chr = (2 * p + 1) * kTileCh, chc = 2 * p * kTileCh;
  const TileRange<kTilePx> tr(gm);

  if (tid == 0) ring.init();
  if (tid < 2 * kTileCh) sShift[tid >> 6][tid & 63] = shift[((size_t)d * SB + 2 * p + 1 - (tid >> 6)) * kTileCh + (tid & 63)];
  __syncthreads();

  float tot[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) tot[i] = 0.f;

  if (tid >> 5 == kProducerWarp) {
    if ((tid & 31) == 0)
      produce(ring, tr, d * gm.N, 2 * BOX, [&](int s, int px0, int img, uint64_t* bar) {
        tma_tile<float, NHWC>(smem + (size_t)s * 2 * BOX, &map_x, chr, px0, img, bar);
        tma_tile<float, NHWC>(smem + (size_t)s * 2 * BOX + BOX, &map_x, chc, px0, img, bar);
      });
  } else {
    // per warpgroup behind the ring: NCHW the lo tiles of rows and columns (hi in place); NHWC hi, lo of rows, hi, lo of columns
    const int t = tid & 127;
    const uint32_t wgbuf = smem_u32(smem + (size_t)STAGES * 2 * BOX + (size_t)(tid >> 7) * (NHWC ? 4 : 2) * kTileBytes);
    const uint32_t lo_r = NHWC ? wgbuf + kTileBytes : wgbuf, lo_c = NHWC ? wgbuf + 3 * kTileBytes : wgbuf + kTileBytes;
    float dummy[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) dummy[i] = 0.f;
    consume<NHWC>(ring, tr, smem_u32(smem), 2 * BOX, tot, [&](uint32_t tile, int px0) {      // h1 h0^T + l1 h0^T + h1 l0^T
      const uint32_t hi_r = NHWC ? wgbuf : tile, hi_c = NHWC ? wgbuf + 2 * kTileBytes : tile + BOX;
      split_transform<float, NHWC>(tile, hi_r, lo_r, t, sShift[0], px0, gm.HW, chr, gm.C, dummy);
      split_transform<float, NHWC>(tile + BOX, hi_c, lo_c, t, sShift[1], px0, gm.HW, chc, gm.C, dummy);
      const uint64_t hr = make_kmajor_sw128_desc(hi_r), lr = make_kmajor_sw128_desc(lo_r);
      const uint64_t hc = make_kmajor_sw128_desc(hi_c), lc = make_kmajor_sw128_desc(lo_c);
      return Products<3>{{hr, lr, hr}, {hc, hc, lc}};
    });
  }

  // both warpgroups' sums -> this CTA's partial row; its row-sum slots stay 0 (the diagonal kernel has them)
  const float* s = cta_sums<kTileCh>(smem, tot, nullptr);
  float* prow = partial_row(partial);
  for (int e = tid; e < kNacc; e += kTcThreads) prow[e] = s[e];
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

// The ring + per-warpgroup fp32 tiles: Gram lo (bf16 / NHWC: + hi staging); contraction lo of xc and dy (bf16 / NHWC: +
// hi staging of both).  97 KB per contraction CTA in every instantiation.
template <class T, bool NHWC>
constexpr size_t tc_smem_bytes(bool two) {
  constexpr bool staged = kStaged<T, NHWC>;
  return two ? (size_t)kStagesBwdOf<T, NHWC> * 2 * kBoxBytes<T> + (size_t)kConsumers * (staged ? 4 : 2) * kTileBytes + 1024
             : (size_t)kGramStagesOf<T, NHWC> * kBoxBytes<T> + (size_t)kConsumers * (staged ? 2 : 1) * kTileBytes + 1024;
}
// group size 128 (fp32): the off-diagonal Gram kernel
template <bool NHWC> constexpr size_t tc_pair_smem_bytes() {
  return (size_t)kPairStagesOf<NHWC> * 2 * kTileBytes + (size_t)kConsumers * (NHWC ? 4 : 2) * kTileBytes + 1024;
}

}  // namespace

int tc::make_map(CUtensorMap* map, const void* base, const Geom& gm, bool bf16, bool nhwc, bool apply_box) {
  const cuuint64_t es = bf16 ? 2 : 4;
  const cuuint32_t estr[3] = {1, 1, 1};
  const cuuint64_t dims[3] = {(cuuint64_t)(nhwc ? gm.C : gm.HW), (cuuint64_t)(nhwc ? gm.HW : gm.C), (cuuint64_t)gm.N * gm.D};
  const cuuint64_t strides[2] = {(cuuint64_t)dims[0] * es, (cuuint64_t)gm.C * gm.HW * es};
  const cuuint32_t box[3] = {nhwc ? (bf16 ? 64u : 32u) : (bf16 && apply_box ? 64u : (cuuint32_t)kTilePx),
                             nhwc ? (cuuint32_t)kTilePx : (cuuint32_t)kTileCh, 1};
  const bool swizzle = nhwc || !bf16 || apply_box;
  return (int)g_encode(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                       const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

int tc_init() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess) return e == cudaSuccess ? -1 : (int)e;
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  using bf16 = __nv_bfloat16;
  const KernelSmem kernels[] = {
      {(const void*)tc_gram_kernel<float, false>, tc_smem_bytes<float, false>(false)},
      {(const void*)tc_gram_kernel<bf16, false>, tc_smem_bytes<bf16, false>(false)},
      {(const void*)tc_gram_kernel<float, true>, tc_smem_bytes<float, true>(false)},
      {(const void*)tc_gram_kernel<bf16, true>, tc_smem_bytes<bf16, true>(false)},
      {(const void*)tc_contract_kernel<float, false>, tc_smem_bytes<float, false>(true)},
      {(const void*)tc_contract_kernel<bf16, false>, tc_smem_bytes<bf16, false>(true)},
      {(const void*)tc_contract_kernel<float, true>, tc_smem_bytes<float, true>(true)},
      {(const void*)tc_contract_kernel<bf16, true>, tc_smem_bytes<bf16, true>(true)},
      {(const void*)tc_contract_kernel<float, false, false, false>, tc_smem_bytes<float, false>(true)},
      {(const void*)tc_contract_kernel<bf16, false, false, false>, tc_smem_bytes<bf16, false>(true)},
      {(const void*)tc_contract_kernel<float, true, false, false>, tc_smem_bytes<float, true>(true)},
      {(const void*)tc_contract_kernel<bf16, true, false, false>, tc_smem_bytes<bf16, true>(true)},
      {(const void*)tc_contract_kernel<float, false, true>, tc_smem_bytes<float, false>(true)},
      {(const void*)tc_contract_kernel<float, true, true>, tc_smem_bytes<float, true>(true)},
      {(const void*)tc_gram_pair_kernel<false>, tc_pair_smem_bytes<false>()},
      {(const void*)tc_gram_pair_kernel<true>, tc_pair_smem_bytes<true>()}};
  if (int rc = opt_in(kernels)) return rc;
  if (int rc = dense_init()) return rc;
  return tc_apply_init();
}

// The TMA/wgmma contraction takes group sizes that tile a 64-channel super-block or span two of them (128), rows
// that TMA can address (16-byte strides and base) and at least one full 32-pixel box per row.
// TF32 operands are rounded to nearest, so product errors are zero-mean and shrink as 1/sqrt(M); below a
// few thousand samples per channel they do not, and the (exact fp32, FFMA) tiled kernels take the call (group sizes
// up to 64; group size 128 has no tiled kernel and is refused there).
bool tc_supports(const Geom& gm, int vec) {
  return gm.GS >= 8 && (kTileCh % gm.GS == 0 || gm.GS == 2 * kTileCh) && vec == 4 && gm.HW >= kTilePx &&
         (long long)gm.N * gm.HW >= 4096;
}

int tc_superblocks(const Geom& gm) { return (gm.C + kTileCh - 1) / kTileCh; }

// partial: [D][SB][nchunks][64*64+64] per-CTA moments;  shift: [D][SB][64] pilot shift of every channel
int tc_stats(const void* x, bool bf16, bool nhwc, const Geom& gm, int nchunks, float* shift, float* partial, cudaStream_t st) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map(&mx, x, gm, bf16, nhwc)) return rc;
  const dim3 grid(nchunks, tc_superblocks(gm), gm.D);
  dispatch(bf16, nhwc, [&](auto t, auto layout) {
    using T = decltype(t);
    constexpr bool NHWC = decltype(layout)::value;
    tc_gram_kernel<T, NHWC><<<grid, kTcThreads, tc_smem_bytes<T, NHWC>(false), st>>>(mx, static_cast<const T*>(x), gm, shift, partial);
  });
  return 0;
}

// partial: [D][SB/2][nchunks][64*64+64] off-diagonal blocks of the 128-channel groups; shift: tc_stats' pilot shifts
int tc_gram_pair(const void* x, bool nhwc, const Geom& gm, int nchunks, const float* shift, float* partial, cudaStream_t st) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map(&mx, x, gm, false, nhwc)) return rc;
  const dim3 grid(nchunks, tc_superblocks(gm) / 2, gm.D);
  if (nhwc) tc_gram_pair_kernel<true><<<grid, kTcThreads, tc_pair_smem_bytes<true>(), st>>>(mx, gm, shift, partial);
  else tc_gram_pair_kernel<false><<<grid, kTcThreads, tc_pair_smem_bytes<false>(), st>>>(mx, gm, shift, partial);
  return 0;
}

// group size 128: partial [D][2 SB][nchunks][64*64+64], block (r, c) of group p at 4 p + 2 r + c
int tc_bwd_reduce(const void* x, const void* dout, bool bf16, bool nhwc, const Geom& gm, int nchunks, const float* save_mean,
                  float* partial, cudaStream_t st, bool pilot) {
  CUtensorMap mx, mg;
  bind_context();
  if (int rc = make_map(&mx, x, gm, bf16, nhwc)) return rc;
  if (int rc = make_map(&mg, dout, gm, bf16, nhwc)) return rc;
  dispatch(bf16, nhwc, [&](auto t, auto layout) {
    using T = decltype(t);
    constexpr bool NHWC = decltype(layout)::value;
    constexpr size_t smem = tc_smem_bytes<T, NHWC>(true);
    const T* g = static_cast<const T*>(dout);
    dim3 grid(nchunks, tc_superblocks(gm), gm.D);
    if constexpr (!kBf16<T>) {
      if (gm.GS == 2 * kTileCh) {                // group size 128: the four 64 x 64 blocks of every group's R
        grid.y *= 2;
        tc_contract_kernel<T, NHWC, true><<<grid, kTcThreads, smem, st>>>(mx, mg, g, gm, save_mean, partial);
        return;
      }
    }
    if (pilot) tc_contract_kernel<T, NHWC><<<grid, kTcThreads, smem, st>>>(mx, mg, g, gm, save_mean, partial);
    else tc_contract_kernel<T, NHWC, false, false><<<grid, kTcThreads, smem, st>>>(mx, mg, g, gm, save_mean, partial);
  });
  return 0;
}

}  // namespace dwt

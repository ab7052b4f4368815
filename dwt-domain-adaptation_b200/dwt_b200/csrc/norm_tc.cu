// Tensor-core path for the two CONTRACTIONS over the flattened N*H*W axis when groups are large
// (group size 8..64, i.e. BASELINE.json config 2: C=256, group_size=64):
//
//   stats       G = sum_m (x-K)(x-K)^T        per 64-channel super-block (gs x gs diagonal blocks kept)
//   bwd_reduce  R = sum_m dy (x-mean)^T
//
// 2*gs flop per 4 bytes read puts these far below the TF32 tensor ridge: they are HBM-bound.  Both kernels are
// persistent CTAs (two per SM) over a contiguous range of [64 channels x 32 pixels] tiles, warp-specialised:
//
//   warp 8      TMA producer: cp.async.bulk.tensor.3d (box 32 px x 64 ch x 1 image, SWIZZLE_128B) into a
//               shared-memory ring, mbarrier complete_tx.
//   warps 0-7   two consumer warpgroups taking alternate tiles: each transforms its landed tile in place for the
//               tensor core, then issues wgmma.mma_async kind::tf32 (M = 64 channels, K = 8 pixels per instruction)
//               into an fp32 accumulator held in its registers, and releases the stage.  Operands are K-major straight
//               from the swizzled tile (NCHW rows ARE K-major: the reference's transposing copy, whitening.py:46,
//               disappears).
//   epilogue    the two warpgroups' accumulators are summed in shared memory -> per-CTA partial -> global.  The
//               fixed-order reduction of the partials and the dense algebra (Cholesky / inverse / EMA, or the backward
//               coefficients) run as the small follow-up launches of norm_dense.cu.
//
// stats (tc_gram_kernel) -- SPLIT precision.  The covariance feeds a Cholesky factor whose error is the Gram
// error times the condition number (the eps = 1e-3 shrinkage is absolute and stops helping once activations are
// large), so a single tf32 pass is not enough (y errors of 1e-3..5e-3 at cond >= 1e4).  Each centred sample
// s = x - K is split hi = trunc_tf32(s) and lo = s - hi (exact in fp32; the core keeps its top 11 bits), and
//       G = HH + LH + LH^T         HH = sum hi hi^T,  LH = sum lo hi^T        (lo lo^T ~ 3e-7 G is dropped)
// comes out of two M=64 N=64 K=8 MMAs per 8 pixels: A = the hi tile (written back in place) or the lo tile (a
// per-warpgroup buffer), B = the hi tile.  The row sums the mean needs are summed by the transform.
//
// bwd_reduce (tc_contract_kernel) -- single pass: R multiplies already-formed W's in the coefficient algebra and
// its tf32 product errors are zero-mean over M >= 4096 samples (round-to-nearest operands).
//
// Reference: utils/whitening.py:46-47 of the reference project and its autograd transpose.
#include <cuda.h>

#include "dwt_common.cuh"
#include "norm_launch.h"
#include "tc_ptx.cuh"

namespace dwt {
namespace {

using namespace tc;

constexpr int kConsumers = 2;                           // consumer warpgroups per CTA (warps 0-7)
constexpr int kProducerWarp = 4 * kConsumers;           // warp 8
constexpr int kTcThreads = 128 * kConsumers + 32;
constexpr int kPer = 512 / 128;                         // 16-byte chunks of a tile per consumer thread
constexpr int kTilePx = 32, kTileCh = 64;
constexpr int kTileBytes = kTileCh * kTilePx * 4;       // 8192
constexpr int kStagesBwd = 6;                           // x + dy per stage: 96 KB per CTA, two CTAs per SM
constexpr int kNacc = kTileCh * kTileCh + kTileCh;      // per-CTA partial: 64x64 moments + 64 row sums
constexpr int kGramStages = 10;                         // 80 KB ring + 2 x 8 KB lo tiles per CTA, two CTAs per SM
constexpr int kMaxStages = kGramStages > kStagesBwd ? kGramStages : kStagesBwd;
// Consumer warpgroup w takes tiles w, w + 2, ...; both ring lengths are even, so every stage (and all phases of its
// barriers) belongs to one warpgroup, and an mbarrier parity wait never meets a barrier two phases ahead.
static_assert(kGramStages % kConsumers == 0 && kStagesBwd % kConsumers == 0, "stage ownership");

struct TcBarriers {
  uint64_t full[kMaxStages];       // TMA landed the stage                  (1 arrival + tx bytes)
  uint64_t empty[kMaxStages];      // the owning warpgroup's MMAs are done  (one arrival per consumer warp)
};

// Tile range of this CTA inside its (domain, super-block) problem.
struct TileRange {
  int begin, end, PB;     // tiles [begin, end), pixel blocks per image
  __device__ TileRange(const Geom& gm) {
    PB = (gm.HW + kTilePx - 1) / kTilePx;
    const long long T = (long long)gm.N * PB;
    begin = (int)(T * blockIdx.x / gridDim.x);
    end = (int)(T * (blockIdx.x + 1) / gridDim.x);
  }
};

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float a, float b, float c, float d) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// Pilot shift of channel ch0 + r: the mean of <= 32 mid-image pixels of image 0 of domain d.
__device__ __forceinline__ float pilot_shift(const float* __restrict__ x, const Geom& gm, int d, int c) {
  if (c >= gm.C) return 0.f;
  const int np = gm.HW < 32 ? gm.HW : 32, p0 = ((gm.HW - np) / 2) & ~3;
  const float* px = x + ((size_t)d * gm.N * gm.C + c) * gm.HW + p0;
  float a = 0.f;
  for (int k = 0; k < np; ++k) a += __ldg(px + k);
  return a / (float)np;
}

// In-place transform of one landed tile by the 128 threads of a consumer warpgroup (thread t):
//   v <- RN_tf32(v - shift[row]) inside the tensor, 0 outside; returns per-thread row sums of (v - shift).
// Chunk q = t + 128*i (16-byte units): row = q >> 3, physical chunk jp = q & 7, logical chunk = jp ^ (row & 7).
__device__ __forceinline__ void transform_tile(uint32_t tile, int t, const float (&shift)[kPer], int px0, int HW, int ch0,
                                               int C, float (&rowsum)[kPer]) {
  float4 v[kPer];
#pragma unroll
  for (int i = 0; i < kPer; ++i) v[i] = lds128(tile + 16u * (t + 128 * i));
#pragma unroll
  for (int i = 0; i < kPer; ++i) {
    const int q = t + 128 * i, row = q >> 3, jp = q & 7, j = jp ^ (row & 7);
    const int px = px0 + 4 * j;
    const bool rowok = (ch0 + row) < C;
    float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool ok = rowok && (px + k) < HW;
      const float s = ok ? e[k] - shift[i] : 0.f;
      rowsum[i] += s;
      e[k] = round_tf32(s);
    }
    sts128(tile + 16u * (t + 128 * i), e[0], e[1], e[2], e[3]);
  }
}

// Split transform of one landed Gram tile: s = x - shift inside the tensor, 0 outside; hi = trunc_tf32(s) in place,
// lo = s - hi (exact) to the warpgroup's lo tile at the same swizzled position; returns per-thread row sums of s.  hi is
// written explicitly so that HH and LH see the same hi whatever rounding the tensor core applies to fp32 words.  Two
// chunks at a time: the accumulators leave few registers at two CTAs per SM.
__device__ __forceinline__ void gram_transform(uint32_t tile, uint32_t lo, int t, const float (&shift)[kPer], int px0, int HW,
                                               int ch0, int C, float (&rowsum)[kPer]) {
#pragma unroll
  for (int h = 0; h < kPer; h += 2) {
    float4 v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) v[i] = lds128(tile + 16u * (t + 128 * (h + i)));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = t + 128 * (h + i), row = q >> 3, j = (q & 7) ^ (row & 7);
      const int px = px0 + 4 * j;
      const bool rowok = (ch0 + row) < C;
      float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w}, l[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float s = (rowok && (px + k) < HW) ? e[k] - shift[h + i] : 0.f;
        rowsum[h + i] += s;
        e[k] = __uint_as_float(__float_as_uint(s) & kTf32Mask);
        l[k] = s - e[k];
      }
      sts128(tile + 16u * q, e[0], e[1], e[2], e[3]);
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

__device__ __forceinline__ void init_ring(TcBarriers& bars, int stages) {
  for (int s = 0; s < stages; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], 4); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// backward contraction: R = sum dy xc^T and the row sums of dy
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTcThreads, 2)
tc_contract_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_g, const Geom gm,
                   const float* __restrict__ save_mean, float* __restrict__ partial) {
  constexpr int STAGES = kStagesBwd;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ TcBarriers bars;
  __shared__ float sShift[kTileCh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kTileCh;
  const TileRange tr(gm);
  const int ntiles = tr.end - tr.begin;

  if (tid == 0) init_ring(bars, STAGES);
  if (tid < kTileCh) sShift[tid] = ch0 + tid < gm.C ? save_mean[(size_t)d * gm.C + ch0 + tid] : 0.f;
  __syncthreads();

  float acc[32], rowsum[kPer];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; ++i) rowsum[i] = 0.f;

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (lane == 0) {
      for (int it = 0; it < ntiles; ++it) {
        const int s = it % STAGES;
        mbar_wait_relaxed(&bars.empty[s], ((it / STAGES) & 1) ^ 1);
        const int t = tr.begin + it, n = t / tr.PB, pb = t - n * tr.PB;
        uint8_t* dst = smem + (size_t)s * 2 * kTileBytes;
        mbar_arrive_expect_tx(&bars.full[s], 2 * kTileBytes);
        tma_load_3d(dst, &map_x, pb * kTilePx, ch0, d * gm.N + n, &bars.full[s]);
        tma_load_3d(dst + kTileBytes, &map_g, pb * kTilePx, ch0, d * gm.N + n, &bars.full[s]);
      }
    }
  } else {
    // ===== consumer warpgroups: transform, then D[64 x 64] += dy_tile (A) * xc_tile^T (B) =====
    const int wg = warp >> 2, t = tid & 127;
    float shift[kPer], zero[kPer], dummy[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) { shift[i] = sShift[(t + 128 * i) >> 3]; zero[i] = 0.f; dummy[i] = 0.f; }
    for (int it = wg; it < ntiles; it += kConsumers) {
      const int s = it % STAGES;
      mbar_wait(&bars.full[s], (it / STAGES) & 1);
      const int tl = tr.begin + it, n = tl / tr.PB, pb = tl - n * tr.PB;
      const uint32_t tile = smem_u32(smem + (size_t)s * 2 * kTileBytes);
      transform_tile(tile, t, shift, pb * kTilePx, gm.HW, ch0, gm.C, dummy);                     // xc
      transform_tile(tile + kTileBytes, t, zero, pb * kTilePx, gm.HW, ch0, gm.C, rowsum);        // dy, sums
      fence_proxy_async();
      warpgroup_sync(wg);
      wgmma_fence();
      fence_operands(acc);
      const uint64_t xdesc = make_kmajor_sw128_desc(tile), adesc = make_kmajor_sw128_desc(tile + kTileBytes);
#pragma unroll
      for (int k = 0; k < kTilePx / 8; ++k) wgmma_m64n64k8_ss(acc, adesc + 2 * k, xdesc + 2 * k);
      wgmma_commit();
      wgmma_wait<0>();
      fence_operands(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.empty[s]);
    }
  }

  // ===== epilogue: both warpgroups' accumulators + row sums -> this CTA's partial row =====
  __syncthreads();                                 // every stage consumed: the ring is free
  float* sAcc = reinterpret_cast<float*>(smem);    // [64][64] + [64]
  for (int e = tid; e < kNacc; e += kTcThreads) sAcc[e] = 0.f;
  __syncthreads();
  if (warp < kProducerWarp) {
    add_fragment<8>(sAcc, kTileCh, acc, warp, lane);
    add_rowsums(sAcc + kTileCh * kTileCh, rowsum, tid & 127);
  }
  __syncthreads();
  float* prow = partial + (((size_t)d * gridDim.y + sb) * gridDim.x + blockIdx.x) * kNacc;
  for (int e = tid; e < kNacc; e += kTcThreads) prow[e] = sAcc[e];
}

// ------------------------------------------------------------------------------------------
// split-precision Gram kernel (forward statistics): G = HH + LH + LH^T, see the file header
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTcThreads, 2)
tc_gram_kernel(const __grid_constant__ CUtensorMap map_x, const float* __restrict__ x, const Geom gm,
               float* __restrict__ shift_out, float* __restrict__ partial) {
  constexpr int STAGES = kGramStages;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ TcBarriers bars;
  __shared__ float sShift[kTileCh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kTileCh;
  const TileRange tr(gm);
  const int ntiles = tr.end - tr.begin;

  if (tid == 0) init_ring(bars, STAGES);
  if (tid < kTileCh) {
    const float sh = pilot_shift(x, gm, d, ch0 + tid);
    sShift[tid] = sh;
    if (blockIdx.x == 0) shift_out[((size_t)d * gridDim.y + sb) * kTileCh + tid] = sh;
  }
  __syncthreads();

  float hh[32], lh[32], rowsum[kPer];
#pragma unroll
  for (int i = 0; i < 32; ++i) { hh[i] = 0.f; lh[i] = 0.f; }
#pragma unroll
  for (int i = 0; i < kPer; ++i) rowsum[i] = 0.f;

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (lane == 0) {
      int n = tr.begin / tr.PB, pb = tr.begin - n * tr.PB;
      for (int it = 0; it < ntiles; ++it) {
        const int s = it % STAGES;
        mbar_wait_relaxed(&bars.empty[s], ((it / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&bars.full[s], kTileBytes);
        tma_load_3d(smem + (size_t)s * kTileBytes, &map_x, pb * kTilePx, ch0, d * gm.N + n, &bars.full[s]);
        if (++pb == tr.PB) { pb = 0; ++n; }
      }
    }
  } else {
    // ===== consumer warpgroups: HH[64 x 64] += hi * hi^T,  LH[64 x 64] += lo * hi^T =====
    const int wg = warp >> 2, t = tid & 127;
    const uint32_t lo = smem_u32(smem + (size_t)STAGES * kTileBytes + (size_t)wg * kTileBytes);
    const uint64_t ldesc = make_kmajor_sw128_desc(lo);
    float shift[kPer];
#pragma unroll
    for (int i = 0; i < kPer; ++i) shift[i] = sShift[(t + 128 * i) >> 3];
    for (int it = wg; it < ntiles; it += kConsumers) {
      const int s = it % STAGES;
      mbar_wait(&bars.full[s], (it / STAGES) & 1);
      const int tl = tr.begin + it, n = tl / tr.PB, pb = tl - n * tr.PB;
      const uint32_t tile = smem_u32(smem + (size_t)s * kTileBytes);
      gram_transform(tile, lo, t, shift, pb * kTilePx, gm.HW, ch0, gm.C, rowsum);
      fence_proxy_async();
      warpgroup_sync(wg);
      wgmma_fence();
      fence_operands(hh);
      fence_operands(lh);
      const uint64_t bdesc = make_kmajor_sw128_desc(tile);
#pragma unroll
      for (int k = 0; k < kTilePx / 8; ++k) {
        wgmma_m64n64k8_ss(hh, bdesc + 2 * k, bdesc + 2 * k);
        wgmma_m64n64k8_ss(lh, ldesc + 2 * k, bdesc + 2 * k);
      }
      wgmma_commit();
      wgmma_wait<0>();                             // the lo tile is rewritten by this warpgroup's next transform
      fence_operands(hh);
      fence_operands(lh);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.empty[s]);
    }
  }

  // ===== epilogue: G = HH + LH + LH^T and the row sums -> this CTA's partial row =====
  constexpr int P = kTileCh + 1;                   // odd pitch: the transposed read of LH is conflict-free
  __syncthreads();                                 // every stage consumed: the ring is free
  float* sH = reinterpret_cast<float*>(smem);      // [64][P]
  float* sL = sH + kTileCh * P;                    // [64][P]
  float* sRS = sL + kTileCh * P;                   // [64]
  for (int e = tid; e < 2 * kTileCh * P + kTileCh; e += kTcThreads) sH[e] = 0.f;
  __syncthreads();
  if (warp < kProducerWarp) {
    add_fragment<8>(sH, P, hh, warp, lane);
    add_fragment<8>(sL, P, lh, warp, lane);
    add_rowsums(sRS, rowsum, tid & 127);
  }
  __syncthreads();
  float* prow = partial + (((size_t)d * gridDim.y + sb) * gridDim.x + blockIdx.x) * kNacc;
  for (int e = tid; e < kTileCh * kTileCh; e += kTcThreads) {
    const int r = e >> 6, c = e & 63;
    prow[e] = (sH[r * P + c] + sL[r * P + c]) + sL[c * P + r];
  }
  if (tid < kTileCh) prow[kTileCh * kTileCh + tid] = sRS[tid];
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

int make_map(CUtensorMap* map, const float* base, const Geom& gm) {
  const cuuint64_t dims[3] = {(cuuint64_t)gm.HW, (cuuint64_t)gm.C, (cuuint64_t)gm.N * gm.D};
  const cuuint64_t strides[2] = {(cuuint64_t)gm.HW * 4, (cuuint64_t)gm.C * gm.HW * 4};
  const cuuint32_t box[3] = {kTilePx, kTileCh, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return (int)g_encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

size_t tc_smem_bytes(bool two) {
  return two ? (size_t)kStagesBwd * 2 * kTileBytes + 1024
             : (size_t)kGramStages * kTileBytes + (size_t)kConsumers * kTileBytes + 1024;
}

}  // namespace

int tc_init() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess) return e == cudaSuccess ? -1 : (int)e;
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  e = cudaFuncSetAttribute(tc_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes(false));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(tc_contract_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes(true));
  // two ~90-97 KB CTAs per SM need the full shared-memory carve-out
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_gram_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_contract_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess) e = (cudaError_t)dense_init();
  if (e == cudaSuccess) return tc_apply_init();
  return (int)e;
}

// The TMA/wgmma contraction takes group sizes that tile a 64-channel super-block, rows that TMA can
// address (16-byte strides and base) and at least one full 32-pixel box per row.
// TF32 operands are rounded to nearest, so product errors are zero-mean and shrink as 1/sqrt(M); below a
// few thousand samples per channel they do not, and the (exact fp32, FFMA) tiled kernels take the call.
bool tc_supports(const Geom& gm, int vec) {
  return gm.GS >= 8 && kTileCh % gm.GS == 0 && vec == 4 && gm.HW >= kTilePx && (long long)gm.N * gm.HW >= 4096;
}

int tc_superblocks(const Geom& gm) { return (gm.C + kTileCh - 1) / kTileCh; }

// partial: [D][SB][nchunks][64*64+64] per-CTA moments;  shift: [D][SB][64] pilot shift of every channel
int tc_stats(const float* x, const Geom& gm, int nchunks, float* shift, float* partial, cudaStream_t st) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map(&mx, x, gm)) return rc;
  dim3 grid(nchunks, tc_superblocks(gm), gm.D);
  tc_gram_kernel<<<grid, kTcThreads, tc_smem_bytes(false), st>>>(mx, x, gm, shift, partial);
  return 0;
}

int tc_bwd_reduce(const float* x, const float* dout, const Geom& gm, int nchunks, const float* save_mean,
                  float* partial, cudaStream_t st) {
  CUtensorMap mx, mg;
  bind_context();
  if (int rc = make_map(&mx, x, gm)) return rc;
  if (int rc = make_map(&mg, dout, gm)) return rc;
  dim3 grid(nchunks, tc_superblocks(gm), gm.D);
  tc_contract_kernel<<<grid, kTcThreads, tc_smem_bytes(true), st>>>(mx, mg, gm, save_mean, partial);
  return 0;
}

}  // namespace dwt

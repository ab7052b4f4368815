// Tensor-core path for the two APPLY passes when groups are large (group size 8..64):
//
//   apply       y  = W (x - mean)                               one input tensor
//   bwd_apply   dx = A1 (dy - mean_M dy) + Bm (x - mean)        two input tensors
//
// Per 64-channel super-block the per-group matrices form one block-diagonal 64x64 matrix M, and a
// [64 ch x 64 px] tile of the NCHW tensor gives out = M * tile.  wgmma takes tf32 operands from shared memory only
// K-major, and the landed tile is pixel-major, so the product is computed transposed, out^T = tile^T M^T:
// A = tile^T (64 pixels x 64 channels) is loaded from the swizzled tile into the wgmma register fragment, and
// B = M (rows = output channel, K = input channel) sits K-major in shared memory for the whole kernel.
// A single-pass TF32 product is NOT accurate enough here -- each output is one length-64 dot product
// whose terms can cancel by the condition number of the covariance -- so both operands are split
// v = hi + lo and all four partial products are accumulated in fp32 (lo*lo still moves the largest output errors,
// ~1e-6 absolute, by a third -- enough to flip a ReLU mask downstream):
//   matrix  hi = RN_tf32(m), lo = RN_tf32(m - hi)
//   tile    v = x - shift (centred while it is loaded into registers), hi = trunc_tf32(v), lo = RN_tf32(v - hi)
// Centring before the product keeps the fp32 accumulation error relative to |y| rather than to |M x|; centring after
// it (M x - M shift) doubled the largest output errors on inputs with a large mean.
//
// CTA = 2 consumer warpgroups + 1 TMA producer warp, one per SM, persistent over a contiguous range of 64-pixel
// tiles of one (domain, super-block):
//   warp 8      TMA producer into a ring (per input 2 boxes of 32 px x 64 ch, SWIZZLE_128B)
//   warps 0-7   two consumer warpgroups taking alternate tiles: load the tile into registers (hi / lo split),
//               release the stage, 4 x 8 wgmma m64n64k8 per input, then store the 64 x 64 output block.
//
// bf16 activations (DWT_DTYPE_BF16): the kernel is templated on the storage type T.  A bf16 input lands as ONE box of
// 64 px x 64 ch (128-byte rows, SWIZZLE_128B: the A-fragment reads of a warp -- 8 consecutive pixels of 4 channels -- hit
// four distinct 16-byte chunks); each value is widened to fp32 as it is loaded into the fragment and the output is stored
// rounded to nearest-even, 2 bytes per element.  Everything between is the fp32 kernel on the same tiles in the same order.
//
// channels-last activations (DWT_LAYOUT_NHWC): the kernel is also templated on the layout.  A tile is the same 64 px x 64 ch
// block, landed as pixel rows of 128 bytes (SWIZZLE_128B) from a {C, HW, N*D} tensor map: per 32-pixel half, fp32 two
// boxes of 32 ch x 32 px, bf16 one box of 64 ch x 32 px.  The A fragment -- 8 pixels x 4 channels per warp -- reads 32
// distinct banks.  The output fragment is stored at NHWC addresses, two adjacent channels per store (8 bytes fp32, 4 bytes
// bf16).  Same fragments, same products, same order: y and dx are bit for bit the NCHW kernel's on x.contiguous().
//
// group size 128 (fp32, both layouts): tc_apply128_kernel, below -- the K = 128 product in two K = 64 halves into one
// accumulator.  ptxas (sm_90a): forward NCHW 152 / NHWC 144 registers, no spills; backward NCHW 168 registers with 40
// bytes of spill stores / loads, NHWC 168 with 44 (the per-input argument arrays, indexed at run time by the rolled
// half loop); dynamic shared memory 129 KB forward, 193 KB backward.
//
// Reference: the grouped 1x1 convolution at utils/whitening.py:55 of the reference project and its backward.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdlib>
#include <type_traits>

#include "dwt_common.cuh"
#include "norm_launch.h"
#include "tc_ptx.cuh"

namespace dwt {
namespace {

using namespace tc;

constexpr int kBoxPx = 32, kCh = 64;
constexpr int kBoxBytes = kCh * kBoxPx * 4;          // 8192
constexpr int kTilePx = 64, kNBox = kTilePx / kBoxPx;
constexpr int kMatBytes = kCh * kCh * 4;             // one 64x64 matrix: two K halves of [64 rows x 128 B]
constexpr int kConsumers = 2;
constexpr int kProducerWarp = 4 * kConsumers;
constexpr int kApThreads = 128 * kConsumers + 32;
constexpr int kMaxStages = 6;

template <class T> constexpr bool kBf16 = !std::is_same<T, float>::value;

//   one input:  6 stages of 16 KB + hi / lo matrix (32 KB) = 129 KB        bf16: 6 x 8 KB + 32 KB = 81 KB
//   two inputs: 4 stages of 32 KB + 2 hi / lo matrices (64 KB) = 193 KB    bf16: 4 x 16 KB + 64 KB = 129 KB
template <class T, int NIN> struct ApCfg {
  static constexpr int STAGES = NIN == 1 ? 6 : 4;
  static constexpr int SLOT = NIN * kCh * kTilePx * (int)sizeof(T);
  static constexpr size_t SMEM = (size_t)STAGES * SLOT + (size_t)2 * NIN * kMatBytes + 1024;
  static_assert(STAGES % kConsumers == 0 && STAGES <= kMaxStages, "stage ownership");
};

struct ApBarriers {
  uint64_t full[kMaxStages];       // TMA landed the stage
  uint64_t empty[kMaxStages];      // the owning warpgroup holds the tile in registers (one arrival per warp)
};

// DWT_TC_INTERLEAVE=0/1 (development): tile order of the apply kernels
inline int tile_interleave() {
  static const int v = [] { const char* e = getenv("DWT_TC_INTERLEAVE"); return (e && e[0] == '1') ? 1 : 0; }();
  return v;
}

struct ApplyArgs {
  const float* mats;      // per (domain, group) records
  int rec_stride;         // floats per record
  int off[2];             // offset of the matrix applied to input i inside a record
  const float* shift[2];  // per-channel shift of input i
  int shift_stride[2];    // floats per domain in shift[i]
  void* out;              // T
  int interleave;         // 1: CTA b takes tiles b, b + grid, b + 2 grid, ... (neighbouring CTAs on neighbouring tiles)
};

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// Byte offset of element (row, k) in a [64 rows x 64 K] K-major, 128-byte-swizzled operand: two K halves of
// [64 rows x 32 tf32] (8 KB each), 16-byte chunk (k % 32) / 4 of a row XOR-ed with row % 8.
__device__ __forceinline__ uint32_t kmajor_off(int row, int k) {
  return (uint32_t)((k >> 5) * (kCh * 128) + row * 128 + ((((k & 31) >> 2) ^ (row & 7)) << 4) + (k & 3) * 4);
}
// Byte offset of (channel ch, pixel p) in the landed tile of one input, SWIZZLE_128B.  fp32: box p / 32 is
// [64 ch x 128 B].  bf16: one box [64 ch x 128 B] of 64 pixels.  NHWC: pixel rows of 128 B; fp32 channel half ch / 32 is
// [64 px x 128 B] (two boxes of 32 px), bf16 one [64 px x 128 B] (two boxes of 32 px).
template <class T, bool NHWC>
__device__ __forceinline__ uint32_t tile_off(int ch, int p) {
  if constexpr (NHWC) {
    if constexpr (kBf16<T>) return (uint32_t)(p * 128 + (((ch >> 3) ^ (p & 7)) << 4) + (ch & 7) * 2);
    return (uint32_t)((ch >> 5) * (kTilePx * 128) + p * 128 + ((((ch & 31) >> 2) ^ (p & 7)) << 4) + (ch & 3) * 4);
  }
  if constexpr (kBf16<T>) return (uint32_t)(ch * 128 + (((p >> 3) ^ (ch & 7)) << 4) + (p & 7) * 2);
  const int pp = p & 31;
  return (uint32_t)((p >> 5) * kBoxBytes + ch * 128 + (((pp >> 2) ^ (ch & 7)) << 4) + (pp & 3) * 4);
}
// the landed value at addr, as fp32 (bf16 -> fp32 is exact: the high half of the word)
template <class T>
__device__ __forceinline__ float lds_f(uint32_t addr) {
  if constexpr (kBf16<T>) {
    unsigned short u;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(u) : "r"(addr));
    return __uint_as_float((uint32_t)u << 16);
  } else {
    return lds32(addr);
  }
}

// BIAS (one input): out = M (x - shift) + bias, bias [C] in the second input's slot (args.shift[1]); the accumulator starts
// at the bias of its channel (the colouring transform's beta)
template <class T, int NIN, bool NHWC, bool BIAS = false>
__global__ void __launch_bounds__(kApThreads, 1)
tc_apply_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Geom gm,
                const ApplyArgs args) {
  using Cfg = ApCfg<T, NIN>;
  constexpr int STAGES = Cfg::STAGES, SLOT = Cfg::SLOT;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  uint8_t* sRing = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  uint8_t* sMat = sRing + (size_t)STAGES * SLOT;     // [NIN][hi, lo][kMatBytes]
  __shared__ ApBarriers bars;
  __shared__ float sShift[2][kCh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kCh;
  const int PB = (gm.HW + kTilePx - 1) / kTilePx;
  const long long NT = (long long)gm.N * PB;
  // tile of step `it`: a contiguous range per CTA, or (interleave) the CTAs of a super-block walk the tensor side by side
  const int t_step = args.interleave ? (int)gridDim.x : 1;
  const int t_begin = args.interleave ? (int)blockIdx.x : (int)(NT * blockIdx.x / gridDim.x);
  const int ntiles = args.interleave ? (int)((NT - blockIdx.x + gridDim.x - 1) / gridDim.x)
                                     : (int)(NT * (blockIdx.x + 1) / gridDim.x) - t_begin;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < NIN * kCh) {
    const int i = tid / kCh, r = tid - i * kCh, c = ch0 + r;
    sShift[i][r] = (c < gm.C && args.shift[i] != nullptr) ? __ldg(args.shift[i] + (size_t)d * args.shift_stride[i] + c) : 0.f;
  }
  if constexpr (BIAS) {
    static_assert(NIN == 1, "the bias takes the second input's slot");
    if (tid >= kCh && tid < 2 * kCh) sShift[1][tid - kCh] = ch0 + tid - kCh < gm.C ? __ldg(args.shift[1] + ch0 + tid - kCh) : 0.f;
  }
  __syncthreads();

  // block-diagonal entry (row n, column k) of matrix m of this super-block, full fp32
  auto entry = [&](int m, int n, int k) {
    const int GS = gm.GS, gi = n / GS, g = sb * (kCh / GS) + gi;
    if (g >= gm.G || k / GS != gi) return 0.f;
    return __ldg(args.mats + ((size_t)d * gm.G + g) * args.rec_stride + args.off[m] + (n - gi * GS) * GS + (k - gi * GS));
  };
  // the split matrices as the B operand, resident for the whole kernel
  for (int e = tid; e < NIN * kCh * kCh; e += kApThreads) {
    const int m = e / (kCh * kCh), n = (e / kCh) % kCh, k = e % kCh;
    const float w = entry(m, n, k), hi = round_tf32(w);
    const uint32_t o = kmajor_off(n, k);
    *reinterpret_cast<float*>(sMat + (size_t)(2 * m) * kMatBytes + o) = hi;
    *reinterpret_cast<float*>(sMat + (size_t)(2 * m + 1) * kMatBytes + o) = round_tf32(w - hi);
  }
  fence_proxy_async();
  __syncthreads();

  if (warp == kProducerWarp) {
    // ===== TMA producer =====
    if (lane == 0) {
      for (int it = 0; it < ntiles; ++it) {
        const int t = t_begin + it * t_step, n = t / PB, pb = t - n * PB, s = it % STAGES;
        mbar_wait_relaxed(&bars.empty[s], ((it / STAGES) & 1) ^ 1);
        uint8_t* dst = sRing + (size_t)s * SLOT;
        if constexpr (NHWC) {
          // per 32-pixel half (halves entirely past the row end are not issued, as below): fp32 two boxes of 32 channels,
          // bf16 one of 64; an input's half lands at + h * 4 KB, a 32-channel half of fp32 at + 8 KB
          constexpr int HALF = SLOT / NIN / 2;
          int nh = (gm.HW - pb * kTilePx + kBoxPx - 1) / kBoxPx;
          nh = nh < kNBox ? nh : kNBox;
          mbar_arrive_expect_tx(&bars.full[s], NIN * nh * HALF);
#pragma unroll
          for (int i = 0; i < NIN; ++i)
            for (int h = 0; h < nh; ++h) {
              uint8_t* b = dst + i * (SLOT / NIN) + h * (kBoxPx * 128);
              const CUtensorMap* m = i == 0 ? &map0 : &map1;
              tma_load_3d(b, m, ch0, pb * kTilePx + h * kBoxPx, d * gm.N + n, &bars.full[s]);
              if constexpr (!kBf16<T>) tma_load_3d(b + kTilePx * 128, m, ch0 + 32, pb * kTilePx + h * kBoxPx, d * gm.N + n, &bars.full[s]);
            }
        } else if constexpr (kBf16<T>) {                  // one 64-pixel box per input
          mbar_arrive_expect_tx(&bars.full[s], SLOT);
#pragma unroll
          for (int i = 0; i < NIN; ++i)
            tma_load_3d(dst + i * (SLOT / NIN), i == 0 ? &map0 : &map1, pb * kTilePx, ch0, d * gm.N + n, &bars.full[s]);
        } else {
          // 32-pixel boxes of the tile that lie entirely past the row end are not issued (they only feed output
          // pixels that are never stored, whatever the stale shared memory holds)
          int nbox = (gm.HW - pb * kTilePx + kBoxPx - 1) / kBoxPx;
          nbox = nbox < kNBox ? nbox : kNBox;
          mbar_arrive_expect_tx(&bars.full[s], NIN * nbox * kBoxBytes);
#pragma unroll
          for (int i = 0; i < NIN; ++i)
            for (int j = 0; j < nbox; ++j)
              tma_load_3d(dst + (i * kNBox + j) * kBoxBytes, i == 0 ? &map0 : &map1, pb * kTilePx + j * kBoxPx, ch0,
                          d * gm.N + n, &bars.full[s]);
        }
      }
    }
  } else {
    // ===== consumer warpgroups: D[64 px x 64 ch] = sum_i tile_i^T M_i^T =====
    const int wg = warp >> 2;
    // A fragment (tf32 m64k8): a[r] = element (pixel 16 w + l/4 + 8 (r & 1), channel k0 + l%4 + 4 (r >> 1)) of warp w
    // D fragment: d[4 j + r] = (pixel 16 w + l/4 + 8 (r >> 1), channel 8 j + 2 (l%4) + (r & 1))
    const int prow = 16 * (warp & 3) + (lane >> 2), kq = lane & 3;
    const uint32_t mat0 = smem_u32(sMat);
    for (int it = wg; it < ntiles; it += kConsumers) {
      const int s = it % STAGES;
      mbar_wait(&bars.full[s], (it / STAGES) & 1);
      const uint32_t slot = smem_u32(sRing + (size_t)s * SLOT);
      uint32_t ahi[NIN][kCh / 8][4], alo[NIN][kCh / 8][4];
#pragma unroll
      for (int i = 0; i < NIN; ++i)
#pragma unroll
        for (int ks = 0; ks < kCh / 8; ++ks)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int k = 8 * ks + kq + 4 * (r >> 1);
            const float v = lds_f<T>(slot + i * (SLOT / NIN) + tile_off<T, NHWC>(k, prow + 8 * (r & 1))) - sShift[i][k];
            const uint32_t h = __float_as_uint(v) & kTf32Mask;
            ahi[i][ks][r] = h;
            alo[i][ks][r] = __float_as_uint(round_tf32(v - __uint_as_float(h)));
          }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.empty[s]);   // the tile is in registers: the stage can be refilled
      float acc[32];
      if constexpr (BIAS) {
        // acc[4 j + r] belongs to channel 8 j + 2 (l%4) + (r & 1) (the D fragment above)
#pragma unroll
        for (int j = 0; j < kCh / 8; ++j) {
          const float b0 = sShift[1][8 * j + 2 * kq], b1 = sShift[1][8 * j + 2 * kq + 1];
          acc[4 * j] = b0; acc[4 * j + 1] = b1; acc[4 * j + 2] = b0; acc[4 * j + 3] = b1;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0.f;
      }
      wgmma_fence();
      fence_operands(acc);
#pragma unroll
      for (int i = 0; i < NIN; ++i)
#pragma unroll
        for (int ks = 0; ks < kCh / 8; ++ks) {
          // k-step ks: K half ks / 4, 32 bytes further per step inside the 128-byte row
          const uint32_t koff = (uint32_t)((ks >> 2) * (kCh * 128) + (ks & 3) * 32);
          const uint64_t bhi = make_kmajor_sw128_desc(mat0 + (uint32_t)(2 * i) * kMatBytes + koff);
          const uint64_t blo = make_kmajor_sw128_desc(mat0 + (uint32_t)(2 * i + 1) * kMatBytes + koff);
          wgmma_m64n64k8_rs(acc, ahi[i][ks], bhi);
          wgmma_m64n64k8_rs(acc, ahi[i][ks], blo);
          wgmma_m64n64k8_rs(acc, alo[i][ks], bhi);
          wgmma_m64n64k8_rs(acc, alo[i][ks], blo);
        }
      wgmma_commit();
      wgmma_wait<0>();
      fence_operands(acc);
      const int t = t_begin + it * t_step, n = t / PB, pb = t - n * PB;
      T* obase = static_cast<T*>(args.out) + (size_t)(d * gm.N + n) * gm.C * gm.HW;
      if constexpr (NHWC) {
        // channels c, c + 1 of pixel px: adjacent, one store (C % 8 == 0: both or neither inside the tensor)
        const int px = pb * kTilePx + prow;
        T* o = obase + (size_t)px * gm.C + ch0 + 2 * kq;
#pragma unroll
        for (int j = 0; j < kCh / 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (ch0 + 8 * j + 2 * kq < gm.C && px + 8 * h < gm.HW) {
              T* oj = o + (size_t)h * 8 * gm.C + 8 * j;
              const float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
              if constexpr (kBf16<T>) *reinterpret_cast<__nv_bfloat162*>(oj) = __floats2bfloat162_rn(a0, a1);
              else *reinterpret_cast<float2*>(oj) = make_float2(a0, a1);
            }
          }
      } else {
#pragma unroll
        for (int j = 0; j < kCh / 8; ++j)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int c = 8 * j + 2 * kq + (r & 1), px = pb * kTilePx + prow + 8 * (r >> 1);
            if (ch0 + c < gm.C && px < gm.HW) {
              if constexpr (kBf16<T>) obase[(size_t)(ch0 + c) * gm.HW + px] = __float2bfloat16_rn(acc[4 * j + r]);
              else obase[(size_t)(ch0 + c) * gm.HW + px] = acc[4 * j + r];
            }
          }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// group size 128 (fp32): output block r = blockIdx.y & 1 of pair p = blockIdx.y >> 1 (channels (2p + r) * 64 ..) is
//   out_r = sum_i sum_h M_i[r][h] (in_i[h] - shift_i[h])           in_i[h] = input i at super-block 2p + h
// -- the K = 128 product in two K = 64 halves accumulated into ONE fp32 accumulator: a warpgroup takes a tile's h = 0
// stage, then its h = 1 stage.  Same split-tf32 operands, same centring on load, same fragments and store as above.
// The 2 x NIN blocks [64 x 64] of M (hi and lo) stay resident: 64 KB forward, 128 KB backward.  Each warpgroup owns
// SPW ring stages of one 64-channel half of every input (16 KB per input): forward 4 x 16 KB = 64 KB (128 KB in all),
// backward 2 x 32 KB = 64 KB (192 KB in all); one CTA per SM.  Zero blocks (W is lower-, A1 = W^T upper-triangular)
// are multiplied like any other: their products are exact zeros.
// ------------------------------------------------------------------------------------------
template <int NIN> struct Ap128Cfg {
  static constexpr int SPW = NIN == 1 ? 2 : 1;                 // ring stages per consumer warpgroup
  static constexpr int STAGES = kConsumers * SPW;
  static constexpr int SLOT = NIN * kCh * kTilePx * 4;
  static constexpr size_t SMEM = (size_t)STAGES * SLOT + (size_t)2 * 2 * NIN * kMatBytes + 1024;
  static_assert(STAGES <= kMaxStages, "stages");
};

template <int NIN, bool NHWC>
__global__ void __launch_bounds__(kApThreads, 1)
tc_apply128_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Geom gm,
                   const ApplyArgs args) {
  using Cfg = Ap128Cfg<NIN>;
  constexpr int SPW = Cfg::SPW, SLOT = Cfg::SLOT;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  uint8_t* sRing = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  uint8_t* sMat = sRing + (size_t)Cfg::STAGES * SLOT;     // [NIN][h][hi, lo][kMatBytes]
  __shared__ ApBarriers bars;
  __shared__ float sShift[NIN][2][kCh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int p = blockIdx.y >> 1, r = blockIdx.y & 1, d = blockIdx.z, ch0 = (2 * p + r) * kCh;
  const int PB = (gm.HW + kTilePx - 1) / kTilePx;
  const long long NT = (long long)gm.N * PB;
  const int t_begin = (int)(NT * blockIdx.x / gridDim.x);
  const int ntiles = (int)(NT * (blockIdx.x + 1) / gridDim.x) - t_begin;
  // j-th load of warpgroup w (tile it = 2 (j / 2) + w, half h = j % 2): stage w + 2 (j % SPW), parity (j / SPW) & 1
  auto stage_of = [](int w, int j) { return w + kConsumers * (j % SPW); };

  if (tid == 0) {
    for (int s = 0; s < Cfg::STAGES; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < NIN * 2 * kCh) {
    const int i = tid / (2 * kCh), h = (tid / kCh) & 1, k = tid % kCh;
    sShift[i][h][k] = __ldg(args.shift[i] + (size_t)d * args.shift_stride[i] + (2 * p + h) * kCh + k);
  }
  // the split matrices: block (r, h) of input i's 128 x 128 group matrix, K-major as the B operand
  for (int e = tid; e < NIN * 2 * kCh * kCh; e += kApThreads) {
    const int m = e / (2 * kCh * kCh), h = (e / (kCh * kCh)) & 1, n = (e / kCh) % kCh, k = e % kCh;
    const float w = __ldg(args.mats + ((size_t)d * gm.G + p) * args.rec_stride + args.off[m] + (size_t)(r * kCh + n) * (2 * kCh) +
                          h * kCh + k);
    const float hi = round_tf32(w);
    const uint32_t o = kmajor_off(n, k);
    *reinterpret_cast<float*>(sMat + (size_t)(4 * m + 2 * h) * kMatBytes + o) = hi;
    *reinterpret_cast<float*>(sMat + (size_t)(4 * m + 2 * h + 1) * kMatBytes + o) = round_tf32(w - hi);
  }
  fence_proxy_async();
  __syncthreads();

  if (warp == kProducerWarp) {
    // ===== TMA producer: per pair of tiles (one per warpgroup) the h = 0 halves, then the h = 1 halves =====
    if (lane == 0) {
      for (int it0 = 0; it0 < ntiles; it0 += kConsumers)
        for (int h = 0; h < 2; ++h)
          for (int w = 0; w < kConsumers && it0 + w < ntiles; ++w) {
            const int t = t_begin + it0 + w, n = t / PB, pb = t - n * PB, j = it0 + h, s = stage_of(w, j);
            const int chh = (2 * p + h) * kCh;
            mbar_wait_relaxed(&bars.empty[s], ((j / SPW) & 1) ^ 1);
            uint8_t* dst = sRing + (size_t)s * SLOT;
            int nb = (gm.HW - pb * kTilePx + kBoxPx - 1) / kBoxPx;      // 32-pixel boxes not entirely past the row end
            nb = nb < kNBox ? nb : kNBox;
            mbar_arrive_expect_tx(&bars.full[s], NIN * nb * kBoxBytes);
#pragma unroll
            for (int i = 0; i < NIN; ++i)
              for (int b = 0; b < nb; ++b) {
                const CUtensorMap* m = i == 0 ? &map0 : &map1;
                if constexpr (NHWC) {
                  uint8_t* bb = dst + i * (SLOT / NIN) + b * (kBoxPx * 128);
                  tma_load_3d(bb, m, chh, pb * kTilePx + b * kBoxPx, d * gm.N + n, &bars.full[s]);
                  tma_load_3d(bb + kTilePx * 128, m, chh + 32, pb * kTilePx + b * kBoxPx, d * gm.N + n, &bars.full[s]);
                } else {
                  tma_load_3d(dst + (i * kNBox + b) * kBoxBytes, m, pb * kTilePx + b * kBoxPx, chh, d * gm.N + n, &bars.full[s]);
                }
              }
          }
    }
  } else {
    // ===== consumer warpgroups: D[64 px x 64 ch] = sum_h sum_i tile_i[h]^T M_i[r][h]^T =====
    const int wg = warp >> 2;
    const int prow = 16 * (warp & 3) + (lane >> 2), kq = lane & 3;
    const uint32_t mat0 = smem_u32(sMat);
    for (int it = wg; it < ntiles; it += kConsumers) {
      float acc[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) acc[q] = 0.f;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int j = it - wg + h, s = stage_of(wg, j);
        mbar_wait(&bars.full[s], (j / SPW) & 1);
        const uint32_t slot = smem_u32(sRing + (size_t)s * SLOT);
        uint32_t ahi[NIN][kCh / 8][4], alo[NIN][kCh / 8][4];
#pragma unroll
        for (int i = 0; i < NIN; ++i)
#pragma unroll
          for (int ks = 0; ks < kCh / 8; ++ks)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int k = 8 * ks + kq + 4 * (q >> 1);
              const float v = lds32(slot + i * (SLOT / NIN) + tile_off<float, NHWC>(k, prow + 8 * (q & 1))) - sShift[i][h][k];
              const uint32_t hb = __float_as_uint(v) & kTf32Mask;
              ahi[i][ks][q] = hb;
              alo[i][ks][q] = __float_as_uint(round_tf32(v - __uint_as_float(hb)));
            }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars.empty[s]);   // the half is in registers: the stage can be refilled
        wgmma_fence();
        fence_operands(acc);
#pragma unroll
        for (int i = 0; i < NIN; ++i)
#pragma unroll
          for (int ks = 0; ks < kCh / 8; ++ks) {
            const uint32_t koff = (uint32_t)((ks >> 2) * (kCh * 128) + (ks & 3) * 32);
            const uint64_t bhi = make_kmajor_sw128_desc(mat0 + (uint32_t)(4 * i + 2 * h) * kMatBytes + koff);
            const uint64_t blo = make_kmajor_sw128_desc(mat0 + (uint32_t)(4 * i + 2 * h + 1) * kMatBytes + koff);
            wgmma_m64n64k8_rs(acc, ahi[i][ks], bhi);
            wgmma_m64n64k8_rs(acc, ahi[i][ks], blo);
            wgmma_m64n64k8_rs(acc, alo[i][ks], bhi);
            wgmma_m64n64k8_rs(acc, alo[i][ks], blo);
          }
        wgmma_commit();
        wgmma_wait<0>();                               // the fragments are reloaded for the next half
        fence_operands(acc);
      }
      const int t = t_begin + it, n = t / PB, pb = t - n * PB;
      float* obase = static_cast<float*>(args.out) + (size_t)(d * gm.N + n) * gm.C * gm.HW;
      if constexpr (NHWC) {
        const int px = pb * kTilePx + prow;
        float* o = obase + (size_t)px * gm.C + ch0 + 2 * kq;
#pragma unroll
        for (int jj = 0; jj < kCh / 8; ++jj)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            if (px + 8 * hh < gm.HW)
              *reinterpret_cast<float2*>(o + (size_t)hh * 8 * gm.C + 8 * jj) = make_float2(acc[4 * jj + 2 * hh], acc[4 * jj + 2 * hh + 1]);
      } else {
#pragma unroll
        for (int jj = 0; jj < kCh / 8; ++jj)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = 8 * jj + 2 * kq + (q & 1), px = pb * kTilePx + prow + 8 * (q >> 1);
            if (px < gm.HW) obase[(size_t)(ch0 + c) * gm.HW + px] = acc[4 * jj + q];
          }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode_ap = nullptr;

// a box is 128 bytes wide either way: 32 fp32 or 64 bf16 pixels of 64 channels (bf16 needs HW % 8 == 0: 16-byte strides).
// nhwc: dims {C, HW, N*D}, boxes of 32 fp32 or 64 bf16 channels x 32 pixels (C % 8 == 0: 16-byte strides).
int make_map_ap(CUtensorMap* map, const void* base, const Geom& gm, bool bf16, bool nhwc) {
  const cuuint64_t es = bf16 ? 2 : 4;
  const cuuint32_t estr[3] = {1, 1, 1};
  if (nhwc) {
    const cuuint64_t dims[3] = {(cuuint64_t)gm.C, (cuuint64_t)gm.HW, (cuuint64_t)gm.N * gm.D};
    const cuuint64_t strides[2] = {(cuuint64_t)gm.C * es, (cuuint64_t)gm.HW * gm.C * es};
    const cuuint32_t box[3] = {bf16 ? 64u : 32u, (cuuint32_t)kBoxPx, 1};
    return (int)g_encode_ap(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base),
                            dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  const cuuint64_t dims[3] = {(cuuint64_t)gm.HW, (cuuint64_t)gm.C, (cuuint64_t)gm.N * gm.D};
  const cuuint64_t strides[2] = {(cuuint64_t)gm.HW * es, (cuuint64_t)gm.C * gm.HW * es};
  const cuuint32_t box[3] = {bf16 ? (cuuint32_t)kTilePx : (cuuint32_t)kBoxPx, kCh, 1};
  return (int)g_encode_ap(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base),
                          dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

template <class T, int NIN> constexpr size_t ap_smem() { return ApCfg<T, NIN>::SMEM; }

template <class T, int NIN, bool NHWC, bool BIAS = false>
cudaError_t ap_attrs() {
  cudaError_t e = cudaFuncSetAttribute(tc_apply_kernel<T, NIN, NHWC, BIAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ap_smem<T, NIN>());
  // a 129 / 193 KB CTA needs the full shared-memory carve-out
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_apply_kernel<T, NIN, NHWC, BIAS>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  return e;
}

template <int NIN, bool NHWC>
cudaError_t ap128_attrs() {
  cudaError_t e = cudaFuncSetAttribute(tc_apply128_kernel<NIN, NHWC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Ap128Cfg<NIN>::SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_apply128_kernel<NIN, NHWC>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  return e;
}

template <int NIN, bool BIAS = false>
void launch_apply(bool bf16, bool nhwc, dim3 grid, const CUtensorMap& m0, const CUtensorMap& m1, const Geom& gm, const ApplyArgs& a,
                  cudaStream_t st) {
  if (gm.GS == 2 * kCh) {                          // group size 128 (fp32 only: the C ABI refuses bf16 there)
    if (nhwc) tc_apply128_kernel<NIN, true><<<grid, kApThreads, Ap128Cfg<NIN>::SMEM, st>>>(m0, m1, gm, a);
    else tc_apply128_kernel<NIN, false><<<grid, kApThreads, Ap128Cfg<NIN>::SMEM, st>>>(m0, m1, gm, a);
    return;
  }
  if (nhwc) {
    if (bf16) tc_apply_kernel<__nv_bfloat16, NIN, true, BIAS><<<grid, kApThreads, ap_smem<__nv_bfloat16, NIN>(), st>>>(m0, m1, gm, a);
    else tc_apply_kernel<float, NIN, true, BIAS><<<grid, kApThreads, ap_smem<float, NIN>(), st>>>(m0, m1, gm, a);
  } else {
    if (bf16) tc_apply_kernel<__nv_bfloat16, NIN, false, BIAS><<<grid, kApThreads, ap_smem<__nv_bfloat16, NIN>(), st>>>(m0, m1, gm, a);
    else tc_apply_kernel<float, NIN, false, BIAS><<<grid, kApThreads, ap_smem<float, NIN>(), st>>>(m0, m1, gm, a);
  }
}

}  // namespace

int tc_apply_init() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess) return e == cudaSuccess ? -1 : (int)e;
  g_encode_ap = reinterpret_cast<EncodeTiledFn>(fn);
  e = ap_attrs<float, 1, false>();
  if (e == cudaSuccess) e = ap_attrs<float, 2, false>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 1, false>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 2, false>();
  if (e == cudaSuccess) e = ap_attrs<float, 1, true>();
  if (e == cudaSuccess) e = ap_attrs<float, 2, true>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 1, true>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 2, true>();
  if (e == cudaSuccess) e = ap_attrs<float, 1, false, true>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 1, false, true>();
  if (e == cudaSuccess) e = ap_attrs<float, 1, true, true>();
  if (e == cudaSuccess) e = ap_attrs<__nv_bfloat16, 1, true, true>();
  if (e == cudaSuccess) e = ap128_attrs<1, false>();
  if (e == cudaSuccess) e = ap128_attrs<2, false>();
  if (e == cudaSuccess) e = ap128_attrs<1, true>();
  if (e == cudaSuccess) e = ap128_attrs<2, true>();
  return (int)e;
}

// y = W (x - mean) (+ bias): W from save_w [D][G][gs*gs], mean from save_mean [D][C], bias [C] or null (group sizes 8..64)
int tc_apply(const void* x, void* y, bool bf16, bool nhwc, const Geom& gm, int nctas, const float* save_mean, const float* save_w,
             cudaStream_t st, const float* bias) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map_ap(&mx, x, gm, bf16, nhwc)) return rc;
  ApplyArgs a{};
  a.interleave = tile_interleave();
  a.mats = save_w; a.rec_stride = gm.GS * gm.GS; a.off[0] = 0; a.off[1] = 0;
  a.shift[0] = save_mean; a.shift_stride[0] = gm.C; a.shift[1] = nullptr; a.shift_stride[1] = 0;
  a.out = y;
  a.shift[1] = bias;                               // null: no bias
  const dim3 grid(nctas, (gm.C + kCh - 1) / kCh, gm.D);
  if (bias) launch_apply<1, true>(bf16, nhwc, grid, mx, mx, gm, a, st);
  else launch_apply<1>(bf16, nhwc, grid, mx, mx, gm, a, st);
  return 0;
}

// dx = A1 (dy - dybar) + Bm (x - mean): coef [D][G][2 gs^2 + gs] = A1 | Bm | cvec, dybar [D][SB*64]
int tc_bwd_apply(const void* x, const void* dout, void* dx, bool bf16, bool nhwc, const Geom& gm, int nctas, const float* coef,
                 const float* save_mean, const float* dybar, cudaStream_t st) {
  CUtensorMap mx, mg;
  bind_context();
  if (int rc = make_map_ap(&mg, dout, gm, bf16, nhwc)) return rc;
  if (int rc = make_map_ap(&mx, x, gm, bf16, nhwc)) return rc;
  ApplyArgs a{};
  a.interleave = tile_interleave();
  a.mats = coef; a.rec_stride = coef_stride(gm.GS); a.off[0] = 0; a.off[1] = gm.GS * gm.GS;
  a.shift[0] = dybar; a.shift_stride[0] = ((gm.C + kCh - 1) / kCh) * kCh;
  a.shift[1] = save_mean; a.shift_stride[1] = gm.C;
  a.out = dx;
  launch_apply<2>(bf16, nhwc, dim3(nctas, (gm.C + kCh - 1) / kCh, gm.D), mg, mx, gm, a, st);
  return 0;
}

}  // namespace dwt

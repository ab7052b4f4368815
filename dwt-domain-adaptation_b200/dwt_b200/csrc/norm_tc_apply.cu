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
// CTA = 2 consumer warpgroups + 1 TMA producer warp (tc_ring.cuh), one per SM, persistent over a contiguous range of
// 64-pixel tiles of one (domain, super-block); both kernels are built from the same pieces:
//   warp 8      issue_stage: TMA of every input's tile into a Ring stage (per input 2 boxes of 32 px x 64 ch, SWIZZLE_128B)
//   warps 0-7   two consumer warpgroups taking alternate tiles: load_split_fragment (the tile into registers, centred,
//               hi / lo), release the stage, split_mma (4 x 8 wgmma m64n64k8 per input against the matrices that
//               split_matrices made resident), then store_tile (the 64 x 64 output block, guarded against C and HW).
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
// accumulator.  ptxas (sm_90a): forward NCHW 151 / NHWC 145 registers, no spills; backward NCHW and NHWC 168 registers
// with 40 bytes of spill stores / loads (the per-input argument arrays, indexed at run time by the rolled half loop);
// dynamic shared memory 129 KB forward, 193 KB backward.
//
// Reference: the grouped 1x1 convolution at utils/whitening.py:55 of the reference project and its backward.
#include <cuda.h>
#include <cuda_bf16.h>

#include "dwt_common.cuh"
#include "norm_launch.h"
#include "tc_ring.cuh"

namespace dwt {
namespace {

using namespace tc;

constexpr int kBoxPx = 32, kCh = 64;
constexpr int kBoxBytes = kCh * kBoxPx * 4;          // 8192
constexpr int kTilePx = 64, kNBox = kTilePx / kBoxPx;
constexpr int kMatBytes = kCh * kCh * 4;             // one 64x64 matrix: two K halves of [64 rows x 128 B]

//   one input:  6 stages of 16 KB + hi / lo matrix (32 KB) = 129 KB        bf16: 6 x 8 KB + 32 KB = 81 KB
//   two inputs: 4 stages of 32 KB + 2 hi / lo matrices (64 KB) = 193 KB    bf16: 4 x 16 KB + 64 KB = 129 KB
template <class T, int NIN> struct ApCfg {
  static constexpr int STAGES = NIN == 1 ? 6 : 4;
  static constexpr int SLOT = NIN * kCh * kTilePx * (int)sizeof(T);
  static constexpr size_t SMEM = (size_t)STAGES * SLOT + (size_t)2 * NIN * kMatBytes + 1024;
};

struct ApplyArgs {
  const float* mats;      // per (domain, group) records
  int rec_stride;         // floats per record
  int off[2];             // offset of the matrix applied to input i inside a record
  const float* shift[2];  // per-channel shift of input i
  int shift_stride[2];    // floats per domain in shift[i]
  void* out;              // T
};

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

// The split matrices as the B operand, resident for the whole kernel: entry(m, n, k) (row n, K index k) of matrix
// m = 0 .. NMAT-1 goes to hi = RN_tf32 at sMat + 2 m kMatBytes and lo = RN_tf32(rest) one matrix further, K-major.
template <int NMAT, class Entry>
__device__ __forceinline__ void split_matrices(uint8_t* sMat, Entry entry) {
  for (int e = threadIdx.x; e < NMAT * kCh * kCh; e += kTcThreads) {
    const int m = e / (kCh * kCh), n = (e / kCh) % kCh, k = e % kCh;
    const float w = entry(m, n, k), hi = round_tf32(w);
    const uint32_t o = kmajor_off(n, k);
    *reinterpret_cast<float*>(sMat + (size_t)(2 * m) * kMatBytes + o) = hi;
    *reinterpret_cast<float*>(sMat + (size_t)(2 * m + 1) * kMatBytes + o) = round_tf32(w - hi);
  }
  fence_proxy_async();
  __syncthreads();
}

// TMA of one stage: channels ch0.. and pixels px0.. of image img of every input, input i at dst + i * SLOT / NIN.  The
// 32-pixel halves that lie entirely past the row end are not issued (they only feed output pixels that are never
// stored, whatever the stale shared memory holds).  NCHW fp32: one box of 32 px per half, 8 KB apart; NCHW bf16: one
// box of 64 px; NHWC: per half (4 KB apart) fp32 two boxes of 32 channels, 8 KB apart, bf16 one box of 64.
template <class T, bool NHWC, int NIN>
__device__ __forceinline__ void issue_stage(uint8_t* dst, const CUtensorMap* map0, const CUtensorMap* map1, int ch0, int px0,
                                            int img, int HW, uint64_t* bar) {
  constexpr int IN = kCh * kTilePx * (int)sizeof(T);
  int nh = (HW - px0 + kBoxPx - 1) / kBoxPx;
  nh = (kBf16<T> && !NHWC) || nh > kNBox ? kNBox : nh;
  mbar_arrive_expect_tx(bar, NIN * nh * (IN / kNBox));
#pragma unroll
  for (int i = 0; i < NIN; ++i) {
    const CUtensorMap* m = i == 0 ? map0 : map1;
    uint8_t* b = dst + i * IN;
    if constexpr (kBf16<T> && !NHWC) {
      tma_load_3d(b, m, px0, ch0, img, bar);
    } else {
      for (int h = 0; h < nh; ++h) {
        if constexpr (NHWC) {
          tma_load_3d(b + h * (kBoxPx * 128), m, ch0, px0 + h * kBoxPx, img, bar);
          if constexpr (!kBf16<T>) tma_load_3d(b + h * (kBoxPx * 128) + kTilePx * 128, m, ch0 + 32, px0 + h * kBoxPx, img, bar);
        } else {
          tma_load_3d(b + h * kBoxBytes, m, px0 + h * kBoxPx, ch0, img, bar);
        }
      }
    }
  }
}

// The A fragment (tf32 m64k8) of one input from its landed tile: a[ks][r] = element (pixel 16 w + l/4 + 8 (r & 1),
// channel 8 ks + l%4 + 4 (r >> 1)) of warp w, lane l, centred v = x - shift and split hi = trunc_tf32(v), lo = RN(v - hi).
template <class T, bool NHWC>
__device__ __forceinline__ void load_split_fragment(uint32_t tile, const float* shift, uint32_t (&hi)[kCh / 8][4],
                                                    uint32_t (&lo)[kCh / 8][4]) {
  const int prow = 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2), kq = threadIdx.x & 3;
#pragma unroll
  for (int ks = 0; ks < kCh / 8; ++ks)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = 8 * ks + kq + 4 * (r >> 1);
      const float v = lds_f<T>(tile + tile_off<T, NHWC>(k, prow + 8 * (r & 1))) - shift[k];
      const uint32_t h = __float_as_uint(v) & kTf32Mask;
      hi[ks][r] = h;
      lo[ks][r] = __float_as_uint(round_tf32(v - __uint_as_float(h)));
    }
}

// acc += sum_i A_i M_i^T in split tf32: per k-step the four products hi hi, hi lo, lo hi, lo lo against input i's resident
// hi matrix at mat[i] and its lo one kMatBytes further.  Returns once the MMAs are done: the fragments can be reloaded.
template <int NIN>
__device__ __forceinline__ void split_mma(float (&acc)[32], const uint32_t (&ahi)[NIN][kCh / 8][4],
                                          const uint32_t (&alo)[NIN][kCh / 8][4], const uint32_t (&mat)[NIN]) {
  wgmma_fence();
  fence_operands(acc);
#pragma unroll
  for (int i = 0; i < NIN; ++i)
#pragma unroll
    for (int ks = 0; ks < kCh / 8; ++ks) {
      // k-step ks: K half ks / 4, 32 bytes further per step inside the 128-byte row
      const uint32_t koff = (uint32_t)((ks >> 2) * (kCh * 128) + (ks & 3) * 32);
      const uint64_t bhi = make_kmajor_sw128_desc(mat[i] + koff);
      const uint64_t blo = make_kmajor_sw128_desc(mat[i] + kMatBytes + koff);
      wgmma_m64n64k8_rs(acc, ahi[i][ks], bhi);
      wgmma_m64n64k8_rs(acc, ahi[i][ks], blo);
      wgmma_m64n64k8_rs(acc, alo[i][ks], bhi);
      wgmma_m64n64k8_rs(acc, alo[i][ks], blo);
    }
  wgmma_commit();
  wgmma_wait<0>();
  fence_operands(acc);
}

// The output D[64 px x 64 ch] of the tile at (image img, channels ch0.., pixels px0..): acc[4 j + r] is (pixel
// 16 w + l/4 + 8 (r >> 1), channel 8 j + 2 (l%4) + (r & 1)).  Stored inside the tensor only (past C: the last
// super-block of a C that 64 does not divide; past HW: the last tile of an image); bf16 rounded to nearest-even.
template <class T, bool NHWC>
__device__ __forceinline__ void store_tile(void* out, const Geom& gm, int img, int ch0, int px0, const float (&acc)[32]) {
  const int prow = 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2), kq = threadIdx.x & 3;
  T* obase = static_cast<T*>(out) + (size_t)img * gm.C * gm.HW;
  if constexpr (NHWC) {
    // channels c, c + 1 of pixel px: adjacent, one store (C % 8 == 0: both or neither inside the tensor)
    const int px = px0 + prow;
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
        const int c = 8 * j + 2 * kq + (r & 1), px = px0 + prow + 8 * (r >> 1);
        if (ch0 + c < gm.C && px < gm.HW) {
          if constexpr (kBf16<T>) obase[(size_t)(ch0 + c) * gm.HW + px] = __float2bfloat16_rn(acc[4 * j + r]);
          else obase[(size_t)(ch0 + c) * gm.HW + px] = acc[4 * j + r];
        }
      }
  }
}

// BIAS (one input): out = M (x - shift) + bias, bias [C] in the second input's slot (args.shift[1]); the accumulator starts
// at the bias of its channel (the colouring transform's beta)
template <class T, int NIN, bool NHWC, bool BIAS = false>
__global__ void __launch_bounds__(kTcThreads, 1)
tc_apply_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Geom gm,
                const ApplyArgs args) {
  using Cfg = ApCfg<T, NIN>;
  constexpr int STAGES = Cfg::STAGES, SLOT = Cfg::SLOT;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  uint8_t* sRing = ring_smem(smem_dyn);
  uint8_t* sMat = sRing + (size_t)STAGES * SLOT;     // [NIN][hi, lo][kMatBytes]
  __shared__ Ring<STAGES> ring;
  __shared__ float sShift[2][kCh];
  const int tid = threadIdx.x, sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kCh;
  const TileRange<kTilePx> tr(gm);
  const int ntiles = tr.end - tr.begin;

  if (tid == 0) ring.init();
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
  split_matrices<NIN>(sMat, [&](int m, int n, int k) {
    const int GS = gm.GS, gi = n / GS, g = sb * (kCh / GS) + gi;
    if (g >= gm.G || k / GS != gi) return 0.f;
    return __ldg(args.mats + ((size_t)d * gm.G + g) * args.rec_stride + args.off[m] + (n - gi * GS) * GS + (k - gi * GS));
  });

  if (tid >> 5 == kProducerWarp) {
    if ((tid & 31) == 0)
      for (int it = 0; it < ntiles; ++it) {
        const int t = tr.begin + it, n = t / tr.PB, pb = t - n * tr.PB, s = it % STAGES;
        mbar_wait_relaxed(&ring.empty[s], ((it / STAGES) & 1) ^ 1);
        issue_stage<T, NHWC, NIN>(sRing + (size_t)s * SLOT, &map0, &map1, ch0, pb * kTilePx, d * gm.N + n, gm.HW, &ring.full[s]);
      }
  } else {
    // ===== consumer warpgroups: D[64 px x 64 ch] = sum_i tile_i^T M_i^T =====
    const int kq = tid & 3;
    uint32_t mat[NIN];
#pragma unroll
    for (int i = 0; i < NIN; ++i) mat[i] = smem_u32(sMat) + (uint32_t)(2 * i) * kMatBytes;
    for (int it = tid >> 7; it < ntiles; it += kConsumers) {
      const int s = it % STAGES;
      mbar_wait(&ring.full[s], (it / STAGES) & 1);
      const uint32_t slot = smem_u32(sRing + (size_t)s * SLOT);
      uint32_t ahi[NIN][kCh / 8][4], alo[NIN][kCh / 8][4];
#pragma unroll
      for (int i = 0; i < NIN; ++i) load_split_fragment<T, NHWC>(slot + i * (SLOT / NIN), sShift[i], ahi[i], alo[i]);
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&ring.empty[s]);   // the tile is in registers: the stage can be refilled
      float acc[32];
      if constexpr (BIAS) {
        // acc[4 j + r] belongs to channel 8 j + 2 (l%4) + (r & 1) (store_tile)
#pragma unroll
        for (int j = 0; j < kCh / 8; ++j) {
          const float b0 = sShift[1][8 * j + 2 * kq], b1 = sShift[1][8 * j + 2 * kq + 1];
          acc[4 * j] = b0; acc[4 * j + 1] = b1; acc[4 * j + 2] = b0; acc[4 * j + 3] = b1;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0.f;
      }
      split_mma<NIN>(acc, ahi, alo, mat);
      const int t = tr.begin + it, n = t / tr.PB;
      store_tile<T, NHWC>(args.out, gm, d * gm.N + n, ch0, (t - n * tr.PB) * kTilePx, acc);
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
};

template <int NIN, bool NHWC>
__global__ void __launch_bounds__(kTcThreads, 1)
tc_apply128_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Geom gm,
                   const ApplyArgs args) {
  using Cfg = Ap128Cfg<NIN>;
  constexpr int SPW = Cfg::SPW, SLOT = Cfg::SLOT;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  uint8_t* sRing = ring_smem(smem_dyn);
  uint8_t* sMat = sRing + (size_t)Cfg::STAGES * SLOT;     // [NIN][h][hi, lo][kMatBytes]
  __shared__ Ring<Cfg::STAGES> ring;
  __shared__ float sShift[NIN][2][kCh];
  const int tid = threadIdx.x, p = blockIdx.y >> 1, r = blockIdx.y & 1, d = blockIdx.z, ch0 = (2 * p + r) * kCh;
  const TileRange<kTilePx> tr(gm);
  const int ntiles = tr.end - tr.begin;
  // j-th load of warpgroup w (tile it = 2 (j / 2) + w, half h = j % 2): stage w + 2 (j % SPW), parity (j / SPW) & 1
  auto stage_of = [](int w, int j) { return w + kConsumers * (j % SPW); };

  if (tid == 0) ring.init();
  if (tid < NIN * 2 * kCh) {
    const int i = tid / (2 * kCh), h = (tid / kCh) & 1, k = tid % kCh;
    sShift[i][h][k] = __ldg(args.shift[i] + (size_t)d * args.shift_stride[i] + (2 * p + h) * kCh + k);
  }
  // matrix 2 i + h: block (r, h) of input i's 128 x 128 group matrix
  split_matrices<2 * NIN>(sMat, [&](int m, int n, int k) {
    return __ldg(args.mats + ((size_t)d * gm.G + p) * args.rec_stride + args.off[m >> 1] + (size_t)(r * kCh + n) * (2 * kCh) +
                 (m & 1) * kCh + k);
  });

  if (tid >> 5 == kProducerWarp) {
    // ===== TMA producer: per pair of tiles (one per warpgroup) the h = 0 halves, then the h = 1 halves =====
    if ((tid & 31) == 0)
      for (int it0 = 0; it0 < ntiles; it0 += kConsumers)
        for (int h = 0; h < 2; ++h)
          for (int w = 0; w < kConsumers && it0 + w < ntiles; ++w) {
            const int t = tr.begin + it0 + w, n = t / tr.PB, pb = t - n * tr.PB, j = it0 + h, s = stage_of(w, j);
            mbar_wait_relaxed(&ring.empty[s], ((j / SPW) & 1) ^ 1);
            issue_stage<float, NHWC, NIN>(sRing + (size_t)s * SLOT, &map0, &map1, (2 * p + h) * kCh, pb * kTilePx, d * gm.N + n,
                                          gm.HW, &ring.full[s]);
          }
  } else {
    // ===== consumer warpgroups: D[64 px x 64 ch] = sum_h sum_i tile_i[h]^T M_i[r][h]^T =====
    const int wg = tid >> 7;
    for (int it = wg; it < ntiles; it += kConsumers) {
      float acc[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) acc[q] = 0.f;
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        const int j = it - wg + h, s = stage_of(wg, j);
        mbar_wait(&ring.full[s], (j / SPW) & 1);
        const uint32_t slot = smem_u32(sRing + (size_t)s * SLOT);
        uint32_t ahi[NIN][kCh / 8][4], alo[NIN][kCh / 8][4], mat[NIN];
#pragma unroll
        for (int i = 0; i < NIN; ++i) {
          load_split_fragment<float, NHWC>(slot + i * (SLOT / NIN), sShift[i][h], ahi[i], alo[i]);
          mat[i] = smem_u32(sMat) + (uint32_t)(4 * i + 2 * h) * kMatBytes;
        }
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&ring.empty[s]);   // the half is in registers: the stage can be refilled
        split_mma<NIN>(acc, ahi, alo, mat);
      }
      const int t = tr.begin + it, n = t / tr.PB;
      store_tile<float, NHWC>(args.out, gm, d * gm.N + n, ch0, (t - n * tr.PB) * kTilePx, acc);
    }
  }
}

template <int NIN, bool BIAS = false>
void launch_apply(bool bf16, bool nhwc, dim3 grid, const CUtensorMap& m0, const CUtensorMap& m1, const Geom& gm, const ApplyArgs& a,
                  cudaStream_t st) {
  if (gm.GS == 2 * kCh) {                          // group size 128 (fp32 only: the C ABI refuses bf16 there)
    if (nhwc) tc_apply128_kernel<NIN, true><<<grid, kTcThreads, Ap128Cfg<NIN>::SMEM, st>>>(m0, m1, gm, a);
    else tc_apply128_kernel<NIN, false><<<grid, kTcThreads, Ap128Cfg<NIN>::SMEM, st>>>(m0, m1, gm, a);
    return;
  }
  dispatch(bf16, nhwc, [&](auto t, auto layout) {
    using T = decltype(t);
    constexpr bool NHWC = decltype(layout)::value;
    tc_apply_kernel<T, NIN, NHWC, BIAS><<<grid, kTcThreads, ApCfg<T, NIN>::SMEM, st>>>(m0, m1, gm, a);
  });
}

}  // namespace

int tc_apply_init() {
  using bf16 = __nv_bfloat16;
  const KernelSmem kernels[] = {
      {(const void*)tc_apply_kernel<float, 1, false>, ApCfg<float, 1>::SMEM},
      {(const void*)tc_apply_kernel<float, 2, false>, ApCfg<float, 2>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 1, false>, ApCfg<bf16, 1>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 2, false>, ApCfg<bf16, 2>::SMEM},
      {(const void*)tc_apply_kernel<float, 1, true>, ApCfg<float, 1>::SMEM},
      {(const void*)tc_apply_kernel<float, 2, true>, ApCfg<float, 2>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 1, true>, ApCfg<bf16, 1>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 2, true>, ApCfg<bf16, 2>::SMEM},
      {(const void*)tc_apply_kernel<float, 1, false, true>, ApCfg<float, 1>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 1, false, true>, ApCfg<bf16, 1>::SMEM},
      {(const void*)tc_apply_kernel<float, 1, true, true>, ApCfg<float, 1>::SMEM},
      {(const void*)tc_apply_kernel<bf16, 1, true, true>, ApCfg<bf16, 1>::SMEM},
      {(const void*)tc_apply128_kernel<1, false>, Ap128Cfg<1>::SMEM},
      {(const void*)tc_apply128_kernel<2, false>, Ap128Cfg<2>::SMEM},
      {(const void*)tc_apply128_kernel<1, true>, Ap128Cfg<1>::SMEM},
      {(const void*)tc_apply128_kernel<2, true>, Ap128Cfg<2>::SMEM}};
  return opt_in(kernels);
}

// y = W (x - mean) (+ bias): W from save_w [D][G][gs*gs], mean from save_mean [D][C], bias [C] or null (group sizes 8..64)
int tc_apply(const void* x, void* y, bool bf16, bool nhwc, const Geom& gm, int nctas, const float* save_mean, const float* save_w,
             cudaStream_t st, const float* bias) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map(&mx, x, gm, bf16, nhwc, true)) return rc;
  ApplyArgs a{};
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
  if (int rc = make_map(&mg, dout, gm, bf16, nhwc, true)) return rc;
  if (int rc = make_map(&mx, x, gm, bf16, nhwc, true)) return rc;
  ApplyArgs a{};
  a.mats = coef; a.rec_stride = coef_stride(gm.GS); a.off[0] = 0; a.off[1] = gm.GS * gm.GS;
  a.shift[0] = dybar; a.shift_stride[0] = ((gm.C + kCh - 1) / kCh) * kCh;
  a.shift[1] = save_mean; a.shift_stride[1] = gm.C;
  a.out = dx;
  launch_apply<2>(bf16, nhwc, dim3(nctas, (gm.C + kCh - 1) / kCh, gm.D), mg, mx, gm, a, st);
  return 0;
}

}  // namespace dwt

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
// Reference: the grouped 1x1 convolution at utils/whitening.py:55 of the reference project and its backward.
#include <cuda.h>
#include <cstdlib>

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

//   one input:  6 stages of 16 KB + hi / lo matrix (32 KB) = 129 KB
//   two inputs: 4 stages of 32 KB + 2 hi / lo matrices (64 KB) = 193 KB
template <int NIN> struct ApCfg {
  static constexpr int STAGES = NIN == 1 ? 6 : 4;
  static constexpr int SLOT = NIN * kNBox * kBoxBytes;
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
  float* out;
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
// Byte offset of (channel ch, pixel p) in the landed tile of one input: box p / 32 is [64 ch x 128 B], SWIZZLE_128B.
__device__ __forceinline__ uint32_t tile_off(int ch, int p) {
  const int pp = p & 31;
  return (uint32_t)((p >> 5) * kBoxBytes + ch * 128 + (((pp >> 2) ^ (ch & 7)) << 4) + (pp & 3) * 4);
}

template <int NIN>
__global__ void __launch_bounds__(kApThreads, 1)
tc_apply_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1, const Geom gm,
                const ApplyArgs args) {
  using Cfg = ApCfg<NIN>;
  constexpr int STAGES = Cfg::STAGES, SLOT = Cfg::SLOT;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  uint8_t* sRing = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  uint8_t* sMat = sRing + (size_t)STAGES * SLOT;     // [NIN][hi, lo][kMatBytes]
  __shared__ ApBarriers bars;
  __shared__ float sShift[2][kCh];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int sb = blockIdx.y, d = blockIdx.z, ch0 = sb * kCh;
  const int PB = (gm.HW + kTilePx - 1) / kTilePx;
  const long long T = (long long)gm.N * PB;
  // tile of step `it`: a contiguous range per CTA, or (interleave) the CTAs of a super-block walk the tensor side by side
  const int t_step = args.interleave ? (int)gridDim.x : 1;
  const int t_begin = args.interleave ? (int)blockIdx.x : (int)(T * blockIdx.x / gridDim.x);
  const int ntiles = args.interleave ? (int)((T - blockIdx.x + gridDim.x - 1) / gridDim.x)
                                     : (int)(T * (blockIdx.x + 1) / gridDim.x) - t_begin;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&bars.full[s], 1); mbar_init(&bars.empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid < NIN * kCh) {
    const int i = tid / kCh, r = tid - i * kCh, c = ch0 + r;
    sShift[i][r] = (c < gm.C && args.shift[i] != nullptr) ? __ldg(args.shift[i] + (size_t)d * args.shift_stride[i] + c) : 0.f;
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
        // 32-pixel boxes of the tile that lie entirely past the row end are not issued (they only feed output
        // pixels that are never stored, whatever the stale shared memory holds)
        int nbox = (gm.HW - pb * kTilePx + kBoxPx - 1) / kBoxPx;
        nbox = nbox < kNBox ? nbox : kNBox;
        mbar_wait_relaxed(&bars.empty[s], ((it / STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&bars.full[s], NIN * nbox * kBoxBytes);
        uint8_t* dst = sRing + (size_t)s * SLOT;
#pragma unroll
        for (int i = 0; i < NIN; ++i)
          for (int j = 0; j < nbox; ++j)
            tma_load_3d(dst + (i * kNBox + j) * kBoxBytes, i == 0 ? &map0 : &map1, pb * kTilePx + j * kBoxPx, ch0,
                        d * gm.N + n, &bars.full[s]);
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
            const float v = lds32(slot + i * kNBox * kBoxBytes + tile_off(k, prow + 8 * (r & 1))) - sShift[i][k];
            const uint32_t h = __float_as_uint(v) & kTf32Mask;
            ahi[i][ks][r] = h;
            alo[i][ks][r] = __float_as_uint(round_tf32(v - __uint_as_float(h)));
          }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars.empty[s]);   // the tile is in registers: the stage can be refilled
      float acc[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = 0.f;
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
      float* obase = args.out + (size_t)(d * gm.N + n) * gm.C * gm.HW;
#pragma unroll
      for (int j = 0; j < kCh / 8; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int c = 8 * j + 2 * kq + (r & 1), px = pb * kTilePx + prow + 8 * (r >> 1);
          if (ch0 + c < gm.C && px < gm.HW) obase[(size_t)(ch0 + c) * gm.HW + px] = acc[4 * j + r];
        }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode_ap = nullptr;

int make_map_ap(CUtensorMap* map, const float* base, const Geom& gm) {
  const cuuint64_t dims[3] = {(cuuint64_t)gm.HW, (cuuint64_t)gm.C, (cuuint64_t)gm.N * gm.D};
  const cuuint64_t strides[2] = {(cuuint64_t)gm.HW * 4, (cuuint64_t)gm.C * gm.HW * 4};
  const cuuint32_t box[3] = {kBoxPx, kCh, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  return (int)g_encode_ap(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

template <int NIN> constexpr size_t ap_smem() { return ApCfg<NIN>::SMEM; }

}  // namespace

int tc_apply_init() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess) return e == cudaSuccess ? -1 : (int)e;
  g_encode_ap = reinterpret_cast<EncodeTiledFn>(fn);
  e = cudaFuncSetAttribute(tc_apply_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ap_smem<1>());
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_apply_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ap_smem<2>());
  // a 129 / 193 KB CTA needs the full shared-memory carve-out
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_apply_kernel<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_apply_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  return (int)e;
}

// y = W (x - mean): W from save_w [D][G][gs*gs], mean from save_mean [D][C]
int tc_apply(const float* x, float* y, const Geom& gm, int nctas, const float* save_mean, const float* save_w,
             cudaStream_t st) {
  CUtensorMap mx;
  bind_context();
  if (int rc = make_map_ap(&mx, x, gm)) return rc;
  ApplyArgs a{};
  a.interleave = tile_interleave();
  a.mats = save_w; a.rec_stride = gm.GS * gm.GS; a.off[0] = 0; a.off[1] = 0;
  a.shift[0] = save_mean; a.shift_stride[0] = gm.C; a.shift[1] = nullptr; a.shift_stride[1] = 0;
  a.out = y;
  dim3 grid(nctas, (gm.C + kCh - 1) / kCh, gm.D);
  tc_apply_kernel<1><<<grid, kApThreads, ap_smem<1>(), st>>>(mx, mx, gm, a);
  return 0;
}

// dx = A1 (dy - dybar) + Bm (x - mean): coef [D][G][2 gs^2 + gs] = A1 | Bm | cvec, dybar [D][SB*64]
int tc_bwd_apply(const float* x, const float* dout, float* dx, const Geom& gm, int nctas, const float* coef,
                 const float* save_mean, const float* dybar, cudaStream_t st) {
  CUtensorMap mx, mg;
  bind_context();
  if (int rc = make_map_ap(&mg, dout, gm)) return rc;
  if (int rc = make_map_ap(&mx, x, gm)) return rc;
  ApplyArgs a{};
  a.interleave = tile_interleave();
  a.mats = coef; a.rec_stride = coef_stride(gm.GS); a.off[0] = 0; a.off[1] = gm.GS * gm.GS;
  a.shift[0] = dybar; a.shift_stride[0] = ((gm.C + kCh - 1) / kCh) * kCh;
  a.shift[1] = save_mean; a.shift_stride[1] = gm.C;
  a.out = dx;
  dim3 grid(nctas, (gm.C + kCh - 1) / kCh, gm.D);
  tc_apply_kernel<2><<<grid, kApThreads, ap_smem<2>(), st>>>(mg, mx, gm, a);
  return 0;
}

}  // namespace dwt

// What the tensor-core reductions (norm_tc.cu) and applies (norm_tc_apply.cu) share: the warp roles, the mbarrier ring,
// a CTA's tile range, the shared-memory load of a landed activation, and on the host the tensor map, the shared-memory
// opt-in and the (storage type, layout) dispatch.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include <type_traits>

#include "dwt_common.cuh"
#include "tc_ptx.cuh"

namespace dwt {
namespace tc {

// warps 0-7: two consumer warpgroups taking alternate tiles; warp 8: the TMA producer
constexpr int kConsumers = 2;
constexpr int kProducerWarp = 4 * kConsumers;
constexpr int kTcThreads = 128 * kConsumers + 32;

// Activation storage T: float, or __nv_bfloat16 (DWT_DTYPE_BF16)
template <class T> constexpr bool kBf16 = !std::is_same<T, float>::value;

// Consumer warpgroup w takes tiles w, w + 2, ...; all ring lengths are even, so every stage (and all phases of its
// barriers) belongs to one warpgroup, and an mbarrier parity wait never meets a barrier two phases ahead.
template <int STAGES> struct Ring {
  static_assert(STAGES % kConsumers == 0, "stage ownership");
  uint64_t full[STAGES];       // TMA landed the stage                  (1 arrival + tx bytes)
  uint64_t empty[STAGES];      // the owning warpgroup is done with it  (one arrival per consumer warp)
  __device__ void init() {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
};

// The dynamic shared memory of a ring kernel, aligned for SWIZZLE_128B (1024-byte atoms)
__device__ __forceinline__ uint8_t* ring_smem(uint8_t* raw) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
}

// Tile range of this CTA inside its (domain, super-block) problem: tiles [begin, end) of PX pixels, PB per image.
template <int PX> struct TileRange {
  int begin, end, PB;
  __device__ TileRange(const Geom& gm) {
    PB = (gm.HW + PX - 1) / PX;
    const long long T = (long long)gm.N * PB;
    begin = (int)(T * blockIdx.x / gridDim.x);
    end = (int)(T * (blockIdx.x + 1) / gridDim.x);
  }
};

// The landed value at addr, as fp32 (bf16 -> fp32 is exact: the high half of the word)
template <class T>
__device__ __forceinline__ float lds_f(uint32_t addr) {
  if constexpr (kBf16<T>) {
    unsigned short u;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(u) : "r"(addr));
    return __uint_as_float((uint32_t)u << 16);
  } else {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
  }
}

// ---- host

// 3-D map of an activation tensor, SWIZZLE_128B unless noted.  NCHW: dims {HW, C, N*D}, box 32 px x 64 ch (128-byte
// rows); bf16 boxes are 64-byte rows without swizzle (read by ld.shared only), or with apply_box 64 px x 64 ch (128-byte
// rows, swizzled); TMA then needs HW % 8 == 0 for 16-byte strides.  NHWC: dims {C, HW, N*D}, box 32 (fp32) or 64 (bf16)
// channels x 32 px, 128-byte rows; strides of C elements (C % 8 == 0 for every group size the tensor-core path takes).
int make_map(CUtensorMap* map, const void* base, const Geom& gm, bool bf16, bool nhwc, bool apply_box = false);

// Opts each kernel into its dynamic shared memory and the full carve-out (the ring kernels' CTAs take 73-193 KB)
struct KernelSmem { const void* kernel; size_t smem; };
template <size_t N>
int opt_in(const KernelSmem (&table)[N]) {
  for (const auto& k : table) {
    cudaError_t e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}

// f(T{}, std::bool_constant<NHWC>{}) for the storage type and layout of a call
template <class F>
void dispatch(bool bf16, bool nhwc, F&& f) {
  if (bf16) {
    if (nhwc) f(__nv_bfloat16{}, std::true_type{});
    else f(__nv_bfloat16{}, std::false_type{});
  } else {
    if (nhwc) f(float{}, std::true_type{});
    else f(float{}, std::false_type{});
  }
}

}  // namespace tc
}  // namespace dwt

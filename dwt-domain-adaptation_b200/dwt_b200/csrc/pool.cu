// Channels-last max-pool, forward + backward: the op that sits between the stem whitening site and layer1
// (`x = self.maxpool(self.relu(...))`, resnet50_dwt_mec_officehome.py:337-338; nn.MaxPool2d(3, 2, 1) at :295).
//
// Why it is here: the stock ATen kernels for this op in NHWC fp32 (max_pool_forward_nhwc, max_pool_backward_nhwc
// with an int64 argmax map of 308 MB) take many times what 1.1 GB of algorithmic traffic needs.  Both passes here
// are pure gathers -- no atomics, deterministic:
//   forward   one CTA per output row, one thread per output float4 (4 channels of one output pixel): k*k coalesced
//             float4 loads (a warp covers whole pixels: C/4 consecutive float4), max with ATen's rule (strict >, NaN wins, first maximum
//             in row-major window order keeps the index), one float4 store + 4 index BYTES (window-local k*k index);
//   backward  one CTA per input row, one thread per INPUT float4: the <= ceil(k/s)^2 windows that contain the pixel
//             are visited, and a window's gradient is taken iff its saved index names this pixel; the stem geometry
//             (3 x 3 / 2 / 1, even H and W) has its own kernel: one thread per 2 x 2 input patch, all loads up front.
// Algorithmic bytes: forward 4*(in + out) + out, backward 4*(in + out) + out  (in, out = element counts); bf16 activations
// (DWT_DTYPE_BF16) 2*(in + out) + out: the same kernels on 8-byte channel quads, widened to fp32 as they load and rounded
// to nearest-even as they store -- exact for the forward (a maximum is one of its inputs), and for the backward's sums
// of at most ceil(k/s)^2 gradients it is the fp32 sum rounded once.
//
// Semantics = torch.nn.functional.max_pool2d(x, k, s, p) (dilation 1, ceil_mode False) and its autograd, bit for bit
// including the tie rule (post-ReLU windows of all zeros are common: the gradient goes to the first element).  The index
// starts at the window's first IN-IMAGE position, (max(0, -h0), max(0, -w0)) for a window whose top-left corner is
// (h0, w0): a window whose in-image elements are all -inf keeps it, and its gradient goes to that element as in ATen
// (a start at the top-left corner would name padding there, and the backward would drop the window's gradient).
#include <cuda_bf16.h>

#include "dwt_common.cuh"
#include "norm_launch.h"

namespace dwt {
namespace {

struct PoolGeom {
  int N, H, W, C4, OH, OW, k, s, p, c4shift;
};

// K > 0: the window is a compile-time constant (nn.MaxPool2d(3, 2, 1) of the ResNet stem): the loops over the window unroll
// and the divisions by the stride become shifts -- the generic version spent more time on index arithmetic than on memory
template <int K, int S, int P>
__device__ __forceinline__ PoolGeom fixed(PoolGeom g) {
  if constexpr (K > 0) { g.k = K; g.s = S; g.p = P; }
  return g;
}

__device__ __forceinline__ bool takes(float v, float best) { return (v > best) || (v != v); }

// Storage of one channel quad: a float4, or four bf16 in a uint2
template <class T> struct Quad;
template <> struct Quad<float> {
  using V = float4;
  static __device__ __forceinline__ float4 widen(const float4& v) { return v; }
  static __device__ __forceinline__ float4 narrow(const float4& v) { return v; }
};
template <> struct Quad<__nv_bfloat16> {
  using V = uint2;
  static __device__ __forceinline__ float4 widen(const uint2& u) {
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xFFFF0000u));
  }
  static __device__ __forceinline__ uint2 narrow(const float4& v) {
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    return make_uint2(*reinterpret_cast<const unsigned*>(&a), *reinterpret_cast<const unsigned*>(&b));
  }
};

// One CTA per output row (n, oh): the W*C4 float4 of up to k input rows are re-read from L1/L2 by neighbouring
// windows; threads run over (ow, c4) with 32-bit index arithmetic only.
template <class T, int K, int S, int P, bool POW2>
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                          uint8_t* __restrict__ idx, const PoolGeom g0) {
  using Q = Quad<T>;
  using V = typename Q::V;
  const PoolGeom g = fixed<K, S, P>(g0);
  const int n = blockIdx.x / g.OH, oh = blockIdx.x - n * g.OH;
  const int h0 = oh * g.s - g.p;
  const V* xn = reinterpret_cast<const V*>(x) + (size_t)n * g.H * g.W * g.C4;
  const size_t obase = ((size_t)n * g.OH + oh) * g.OW * g.C4;
  for (int t = threadIdx.x; t < g.OW * g.C4; t += blockDim.x) {
    const int ow = POW2 ? (t >> g.c4shift) : t / g.C4, c4 = t - ow * g.C4;
    const int w0 = ow * g.s - g.p;
    float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    const unsigned first = (unsigned)(max(0, -h0) * g.k + max(0, -w0));   // the first in-image position
    unsigned bi[4] = {first, first, first, first};
#pragma unroll
    for (int kh = 0; kh < g.k; ++kh) {
      const int h = h0 + kh;
      if (h < 0 || h >= g.H) continue;
      const V* xr = xn + (size_t)h * g.W * g.C4 + c4;
#pragma unroll
      for (int kw = 0; kw < g.k; ++kw) {
        const int w = w0 + kw;
        if (w < 0 || w >= g.W) continue;
        const float4 v = Q::widen(__ldg(xr + (size_t)w * g.C4));
        const float e[4] = {v.x, v.y, v.z, v.w};
        const unsigned code = (unsigned)(kh * g.k + kw);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (takes(e[c], best[c])) { best[c] = e[c]; bi[c] = code; }
      }
    }
    reinterpret_cast<V*>(y)[obase + t] = Q::narrow(make_float4(best[0], best[1], best[2], best[3]));
    reinterpret_cast<uint32_t*>(idx)[obase + t] = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
  }
}

// One CTA per input row (n, h): every input float4 gathers from the <= ceil(k/s)^2 windows that contain it.
template <class T, int K, int S, int P, bool POW2>
__global__ void __launch_bounds__(256) maxpool_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ idx,
                                                          T* __restrict__ dx, const PoolGeom g0) {
  using Q = Quad<T>;
  using V = typename Q::V;
  const PoolGeom g = fixed<K, S, P>(g0);
  const int n = blockIdx.x / g.H, h = blockIdx.x - n * g.H;
  // windows (oh, ow) with oh*s - p <= h <= oh*s - p + k - 1
  int oh0 = h + g.p - g.k + 1;
  oh0 = oh0 <= 0 ? 0 : (oh0 + g.s - 1) / g.s;
  int oh1 = (h + g.p) / g.s;
  if (oh1 > g.OH - 1) oh1 = g.OH - 1;
  const V* dyn = reinterpret_cast<const V*>(dy) + (size_t)n * g.OH * g.OW * g.C4;
  const uint32_t* ixn = reinterpret_cast<const uint32_t*>(idx) + (size_t)n * g.OH * g.OW * g.C4;
  V* dxr = reinterpret_cast<V*>(dx) + ((size_t)n * g.H + h) * g.W * g.C4;
  for (int t = threadIdx.x; t < g.W * g.C4; t += blockDim.x) {
    const int w = POW2 ? (t >> g.c4shift) : t / g.C4, c4 = t - w * g.C4;
    int ow0 = w + g.p - g.k + 1;
    ow0 = ow0 <= 0 ? 0 : (ow0 + g.s - 1) / g.s;
    int ow1 = (w + g.p) / g.s;
    if (ow1 > g.OW - 1) ow1 = g.OW - 1;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int oh = oh0; oh <= oh1; ++oh) {            // ascending (oh, ow): the same summation order for every run
      const unsigned kh = (unsigned)(h - (oh * g.s - g.p));
      for (int ow = ow0; ow <= ow1; ++ow) {
        const unsigned code = kh * g.k + (unsigned)(w - (ow * g.s - g.p));
        const size_t o = ((size_t)oh * g.OW + ow) * g.C4 + c4;
        const uint32_t m = __ldg(ixn + o);
        const bool h0 = (m & 0xFFu) == code, h1 = ((m >> 8) & 0xFFu) == code, h2 = ((m >> 16) & 0xFFu) == code, h3 = (m >> 24) == code;
        if (h0 || h1 || h2 || h3) {
          const float4 gq = Q::widen(__ldg(dyn + o));
          if (h0) acc[0] += gq.x;
          if (h1) acc[1] += gq.y;
          if (h2) acc[2] += gq.z;
          if (h3) acc[3] += gq.w;
        }
      }
    }
    dxr[t] = Q::narrow(make_float4(acc[0], acc[1], acc[2], acc[3]));
  }
}

// Forward of the ResNet stem pool (3 x 3, stride 2, pad 1, H and W multiples of 4, C/4 a power of two): one thread per
// 2 x 2 OUTPUT patch and channel quad.  The four windows share a 5 x 5 input patch: 25 loads for 4 outputs instead of
// 36 -- the generic kernel's nine reads per output made it L2-bandwidth-bound (1.39 GB of L2 reads for 0.81 GB of DRAM
// traffic, 0.69 of the HBM peak).  The patch is streamed row by row; every output sees its window in row-major order
// (rows ascending, columns ascending inside a row), so the tie rule (first maximum keeps the index, NaN wins) is the
// generic kernel's.
template <class T>
__global__ void __launch_bounds__(256) maxpool_fwd_3s2_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                              uint8_t* __restrict__ idx, const PoolGeom g) {
  using Q = Quad<T>;
  using V = typename Q::V;
  const int OH2 = g.OH >> 1, OW2 = g.OW >> 1;
  const int n = blockIdx.y / OH2, a = blockIdx.y - n * OH2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= OW2 * g.C4) return;
  const int b = i >> g.c4shift, c4 = i & (g.C4 - 1);
  const V* xn = reinterpret_cast<const V*>(x) + (size_t)n * g.H * g.W * g.C4 + c4;
  float best[2][2][4];
  unsigned bi[2][2][4];
  const int h0 = 4 * a - 1, w0 = 4 * b - 1;
#pragma unroll
  for (int oa = 0; oa < 2; ++oa)
#pragma unroll
    for (int ob = 0; ob < 2; ++ob) {
      // window (oa, ob) starts at (h0 + 2 oa, w0 + 2 ob): its first in-image position, as in the generic kernel
      const unsigned first = (unsigned)(max(0, -(h0 + 2 * oa)) * 3 + max(0, -(w0 + 2 * ob)));
#pragma unroll
      for (int c = 0; c < 4; ++c) { best[oa][ob][c] = -INFINITY; bi[oa][ob][c] = first; }
    }
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    const int h = h0 + r;
    if (h < 0 || h >= g.H) continue;                       // only r == 0 at the top edge (H % 4 == 0)
    float4 row[5];
    bool in[5];
#pragma unroll
    for (int cc = 0; cc < 5; ++cc) {
      const int w = w0 + cc;
      in[cc] = w >= 0 && w < g.W;
      row[cc] = in[cc] ? Q::widen(__ldg(xn + ((size_t)h * g.W + w) * g.C4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int oa = 0; oa < 2; ++oa) {
      const int kh = r - 2 * oa;
      if (kh < 0 || kh > 2) continue;
#pragma unroll
      for (int ob = 0; ob < 2; ++ob)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int cc = 2 * ob + kw;
          if (!in[cc]) continue;
          const float e[4] = {row[cc].x, row[cc].y, row[cc].z, row[cc].w};
          const unsigned code = (unsigned)(kh * 3 + kw);
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (takes(e[c], best[oa][ob][c])) { best[oa][ob][c] = e[c]; bi[oa][ob][c] = code; }
        }
    }
  }
#pragma unroll
  for (int oa = 0; oa < 2; ++oa)
#pragma unroll
    for (int ob = 0; ob < 2; ++ob) {
      const size_t o = (((size_t)n * g.OH + 2 * a + oa) * g.OW + 2 * b + ob) * g.C4 + c4;
      reinterpret_cast<V*>(y)[o] = Q::narrow(make_float4(best[oa][ob][0], best[oa][ob][1], best[oa][ob][2], best[oa][ob][3]));
      reinterpret_cast<uint32_t*>(idx)[o] = bi[oa][ob][0] | (bi[oa][ob][1] << 8) | (bi[oa][ob][2] << 16) | (bi[oa][ob][3] << 24);
    }
}

// Backward of the ResNet stem pool (3 x 3, stride 2, pad 1, even H and W, C/4 a power of two): one thread per 2 x 2 INPUT
// patch and channel quad.  The patch (rows 2k, 2k+1; columns 2j, 2j+1) is touched by exactly the four windows
// (k + a, j + b), a, b in {0, 1}: their 4 index words and 4 gradient float4 are loaded up front (8 independent loads in
// flight per thread instead of a dependent index -> compare -> gradient chain per input element; the gradient tensor is a
// quarter of the input and stays in L2), then the four outputs are composed with the same ascending (oh, ow) summation
// order as the generic kernel.  Window-local codes kh * 3 + kw:
//   (2k, 2j):     w00 code 4                      (2k, 2j+1):   w00 code 5, w01 code 3
//   (2k+1, 2j):   w00 code 7, w10 code 1          (2k+1, 2j+1): w00 code 8, w01 code 6, w10 code 2, w11 code 0
__device__ __forceinline__ void take(float4& acc, const float4& gq, uint32_t m, unsigned code) {
  if ((m & 0xFFu) == code) acc.x += gq.x;
  if (((m >> 8) & 0xFFu) == code) acc.y += gq.y;
  if (((m >> 16) & 0xFFu) == code) acc.z += gq.z;
  if ((m >> 24) == code) acc.w += gq.w;
}

template <class T>
__global__ void __launch_bounds__(256) maxpool_bwd_3s2_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ idx,
                                                              T* __restrict__ dx, const PoolGeom g) {
  using Q = Quad<T>;
  using V = typename Q::V;
  const int H2 = g.H >> 1, W2 = g.W >> 1;
  const int n = blockIdx.y / H2, k = blockIdx.y - n * H2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= W2 * g.C4) return;
  const int j = i >> g.c4shift, c4 = i & (g.C4 - 1);
  const V* dyn = reinterpret_cast<const V*>(dy) + (size_t)n * g.OH * g.OW * g.C4;
  const uint32_t* ixn = reinterpret_cast<const uint32_t*>(idx) + (size_t)n * g.OH * g.OW * g.C4;
  uint32_t m[2][2];
  float4 gq[2][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const bool ok = (k + a < g.OH) && (j + b < g.OW);
      const size_t o = ((size_t)(k + a) * g.OW + (j + b)) * g.C4 + c4;
      m[a][b] = ok ? __ldg(ixn + o) : 0xFFFFFFFFu;          // 0xFF matches no code
      gq[a][b] = ok ? Q::widen(__ldg(dyn + o)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  float4 o00 = make_float4(0.f, 0.f, 0.f, 0.f), o01 = o00, o10 = o00, o11 = o00;
  take(o00, gq[0][0], m[0][0], 4u);
  take(o01, gq[0][0], m[0][0], 5u); take(o01, gq[0][1], m[0][1], 3u);
  take(o10, gq[0][0], m[0][0], 7u); take(o10, gq[1][0], m[1][0], 1u);
  take(o11, gq[0][0], m[0][0], 8u); take(o11, gq[0][1], m[0][1], 6u); take(o11, gq[1][0], m[1][0], 2u); take(o11, gq[1][1], m[1][1], 0u);
  V* r0 = reinterpret_cast<V*>(dx) + (((size_t)n * g.H + 2 * k) * g.W + 2 * j) * g.C4 + c4;
  V* r1 = r0 + (size_t)g.W * g.C4;
  r0[0] = Q::narrow(o00); r0[g.C4] = Q::narrow(o01);
  r1[0] = Q::narrow(o10); r1[g.C4] = Q::narrow(o11);
}

}  // namespace

namespace {
int pow2_shift(int v) {
  int sh = 0;
  while ((1 << sh) < v) ++sh;
  return (1 << sh) == v ? sh : -1;
}

template <class T>
void maxpool_fwd(const T* x, T* y, uint8_t* idx, int N, int H, int W, int C, int OH, int OW, int k, int s, int p, cudaStream_t st) {
  const int sh = pow2_shift(C / 4);
  const PoolGeom g{N, H, W, C / 4, OH, OW, k, s, p, sh < 0 ? 0 : sh};
  if (k == 3 && s == 2 && p == 1 && sh >= 0 && H % 4 == 0 && W % 4 == 0 && (long long)N * (OH / 2) <= 65535) {
    const int items = (OW / 2) * (C / 4), threads = items >= 256 ? 256 : ((items + 31) / 32) * 32;
    maxpool_fwd_3s2_kernel<T><<<dim3((items + threads - 1) / threads, N * (OH / 2)), threads, 0, st>>>(x, y, idx, g);
  } else if (k == 3 && s == 2 && p == 1 && sh >= 0) maxpool_fwd_kernel<T, 3, 2, 1, true><<<N * OH, 256, 0, st>>>(x, y, idx, g);
  else maxpool_fwd_kernel<T, 0, 0, 0, false><<<N * OH, 256, 0, st>>>(x, y, idx, g);
}

template <class T>
void maxpool_bwd(const T* dy, const uint8_t* idx, T* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int p, cudaStream_t st) {
  const int sh = pow2_shift(C / 4);
  const PoolGeom g{N, H, W, C / 4, OH, OW, k, s, p, sh < 0 ? 0 : sh};
  if (k == 3 && s == 2 && p == 1 && sh >= 0 && H % 2 == 0 && W % 2 == 0 && (long long)N * (H / 2) <= 65535) {
    const int items = (W / 2) * (C / 4), threads = items >= 256 ? 256 : ((items + 31) / 32) * 32;
    maxpool_bwd_3s2_kernel<T><<<dim3((items + threads - 1) / threads, N * (H / 2)), threads, 0, st>>>(dy, idx, dx, g);
  } else if (k == 3 && s == 2 && p == 1 && sh >= 0) maxpool_bwd_kernel<T, 3, 2, 1, true><<<N * H, 256, 0, st>>>(dy, idx, dx, g);
  else maxpool_bwd_kernel<T, 0, 0, 0, false><<<N * H, 256, 0, st>>>(dy, idx, dx, g);
}
}  // namespace

void maxpool_fwd_launch(const void* x, void* y, bool bf16, uint8_t* idx, int N, int H, int W, int C, int OH, int OW, int k, int s, int p,
                        cudaStream_t st) {
  if (bf16) maxpool_fwd(static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), idx, N, H, W, C, OH, OW, k, s, p, st);
  else maxpool_fwd(static_cast<const float*>(x), static_cast<float*>(y), idx, N, H, W, C, OH, OW, k, s, p, st);
}

void maxpool_bwd_launch(const void* dy, const uint8_t* idx, void* dx, bool bf16, int N, int H, int W, int C, int OH, int OW, int k, int s,
                        int p, cudaStream_t st) {
  if (bf16) maxpool_bwd(static_cast<const __nv_bfloat16*>(dy), idx, static_cast<__nv_bfloat16*>(dx), N, H, W, C, OH, OW, k, s, p, st);
  else maxpool_bwd(static_cast<const float*>(dy), idx, static_cast<float*>(dx), N, H, W, C, OH, OW, k, s, p, st);
}

}  // namespace dwt

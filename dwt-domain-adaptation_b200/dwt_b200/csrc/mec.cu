// Min-Entropy-Consensus loss: both log-softmaxes, the per-row min over classes of the
// pairwise cross-entropy diagonal, the batch mean AND both logit gradients in one launch
// of one CTA (the problem is [N,K] ~ [64,65]: pure latency, so a single pass with warp
// shuffles replaces the reference's ~12 launches and its [N,K,K] eye-broadcast).
//
// Reference: utils/consensus_loss.py:11-24 (/root/reference).
//   loss = mean_n min_k  -(log_softmax(x)[n,k] + log_softmax(y)[n,k]) / 2
//   d loss / d x[n,k] = (softmax(x)[n,k] - [k == k*_n]) / (2N)       (same for y)
#include <float.h>

#include "dwt_common.cuh"
#include "norm_launch.h"

namespace dwt {
namespace {

constexpr int kMecThreads = 1024;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// log_softmax(x)[k] = (x[k] - a) - b for one row of max mx and log partition sum ls = log(sum_k exp(x[k] - mx)).
// Once |mx| is large, (a, b) = (mx, ls): subtracting the max first keeps ls's absolute precision, which rounding
// mx + ls to fp32 would cost (gradient error 2e-5 at logits ~1e3, 2e-4 at ~1e4).  Below kShiftedFrom the row keeps
// (a, b) = (mx + ls, 0), the earlier form, bit for bit: there that rounding costs at most 2^-18 absolute, and a
// training step carries a one-ulp change of this gradient to a ~1e-2 change of the logits after one update, so
// results (and the benchmark's outputs) stay reproducible across builds.
constexpr float kShiftedFrom = 64.f;

struct Lsm {
  float a, b;
};

__device__ __forceinline__ Lsm lsm_of(float mx, float ls) {
  return fabsf(mx) < kShiftedFrom ? Lsm{mx + ls, 0.f} : Lsm{mx, ls};
}

__device__ __forceinline__ float lsm(float x, Lsm l) { return (x - l.a) - l.b; }

// One warp's work on row pair (x, y) of the MEC term.  The row minimum of s_k = -(lsm(x)[k] + lsm(y)[k]) / 2 follows
// torch.min: the first minimum, and a NaN wins (the first NaN), so a non-finite row reaches the loss as NaN instead of
// leaving best at FLT_MAX.
struct MecRow {
  Lsm lx, ly;
  float best;               // min_k s_k (NaN if any s_k is NaN)
  int bk;                   // its class k*
};

__device__ __forceinline__ MecRow mec_row(const float* __restrict__ xr, const float* __restrict__ yr, int K, int lane) {
  MecRow r;
  float mx = -FLT_MAX, my = -FLT_MAX;
  for (int k = lane; k < K; k += 32) { mx = fmaxf(mx, xr[k]); my = fmaxf(my, yr[k]); }
  mx = warp_max(mx); my = warp_max(my);
  float sx = 0.f, sy = 0.f;
  for (int k = lane; k < K; k += 32) { sx += expf(xr[k] - mx); sy += expf(yr[k] - my); }
  r.lx = lsm_of(mx, logf(warp_sum(sx)));
  r.ly = lsm_of(my, logf(warp_sum(sy)));
  float best = FLT_MAX; int bk = 0x7fffffff;
  for (int k = lane; k < K; k += 32) {
    const float s = -0.5f * (lsm(xr[k], r.lx) + lsm(yr[k], r.ly));
    if (s < best || (s != s && best == best)) { best = s; bk = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
    const bool onan = ob != ob, bnan = best != best;
    if (ob < best || (onan && !bnan) || ((ob == best || (onan && bnan)) && ok < bk)) { best = ob; bk = ok; }
  }
  r.best = best; r.bk = bk;
  return r;
}

__global__ void __launch_bounds__(kMecThreads) mec_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                           int N, int K, float* __restrict__ loss,
                                                           float* __restrict__ gx, float* __restrict__ gy) {
  __shared__ float sRow[kMecThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const float scale = 0.5f / (float)N;
  float wsum = 0.f;     // this warp's sum of row minima (rows visited in increasing order)
  for (int n = warp; n < N; n += nwarps) {
    const float* xr = x + (size_t)n * K;
    const float* yr = y + (size_t)n * K;
    const MecRow r = mec_row(xr, yr, K, lane);
    wsum += r.best;
    for (int k = lane; k < K; k += 32) {
      const float hot = (k == r.bk) ? 1.f : 0.f;
      gx[(size_t)n * K + k] = scale * (expf(lsm(xr[k], r.lx)) - hot);
      gy[(size_t)n * K + k] = scale * (expf(lsm(yr[k], r.ly)) - hot);
    }
  }
  if (lane == 0) sRow[warp] = wsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < nwarps; ++w) t += sRow[w];
    *loss = t / (float)N;
  }
}

// Head loss of the training step in one launch (SURVEY.md §8f-2; resnet50_dwt_mec_officehome.py:421-428):
//   logits [3B, K] = source | target | target-aug ;  labels [B]
//   loss = mean_n NLL(log_softmax(source_n), label_n) + lambda * MEC(target, target-aug)
// losses[0..2] = total, classification, lambda*MEC ; grad [3B, K] = d total / d logits.
// Labels follow F.nll_loss (the reference's call, defaults): label -100 (ignore_index) drops the row from the
// sum AND from the mean's denominator; any other label outside [0, K) is an error there (device assert) --
// here it is never dereferenced: the row is dropped like an ignored one and bit 1 of *status is set.
__global__ void __launch_bounds__(kMecThreads) head_loss_kernel(const float* __restrict__ logits,
                                                                 const long long* __restrict__ labels, int B, int K,
                                                                 float lambda, float* __restrict__ losses,
                                                                 float* __restrict__ grad, int* __restrict__ status) {
  __shared__ float sCls[kMecThreads / 32], sMec[kMecThreads / 32];
  __shared__ int sValid;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  if (threadIdx.x == 0) sValid = 0;
  __syncthreads();
  {
    int nv = 0, bad = 0;
    for (int n = threadIdx.x; n < B; n += blockDim.x) {
      const long long y = labels[n];
      if (y >= 0 && y < K) ++nv;
      else if (y != -100) bad = 1;
    }
    if (nv) atomicAdd(&sValid, nv);
    if (bad && status != nullptr) atomicOr(status, DWT_STATUS_BAD_LABEL);
  }
  __syncthreads();
  const int valid = sValid;
  float cls = 0.f, mec = 0.f;
  for (int n = warp; n < 2 * B; n += nwarps) {
    if (n < B) {                                   // source row: softmax cross-entropy
      const float* xr = logits + (size_t)n * K;
      const long long yl = labels[n];
      const bool use = yl >= 0 && yl < K;
      const int y = use ? (int)yl : 0;
      float mx = -FLT_MAX;
      for (int k = lane; k < K; k += 32) mx = fmaxf(mx, xr[k]);
      mx = warp_max(mx);
      float sx = 0.f;
      for (int k = lane; k < K; k += 32) sx += expf(xr[k] - mx);
      const Lsm l = lsm_of(mx, logf(warp_sum(sx)));
      cls += (lane == 0 && use) ? ((l.a - xr[y]) + l.b) : 0.f;     // -lsm(x)[y]
      const float sc = use ? 1.f / (float)valid : 0.f;
      for (int k = lane; k < K; k += 32) grad[(size_t)n * K + k] = sc * (expf(lsm(xr[k], l)) - (k == y ? 1.f : 0.f));
    } else {                                       // target row n and its augmented twin n + B: MEC
      const float* xr = logits + (size_t)n * K;
      const float* yr = logits + (size_t)(n + B) * K;
      const MecRow r = mec_row(xr, yr, K, lane);
      mec += (lane == 0) ? r.best : 0.f;
      const float sc = lambda * 0.5f / (float)B;
      for (int k = lane; k < K; k += 32) {
        const float hot = (k == r.bk) ? 1.f : 0.f;
        grad[(size_t)n * K + k] = sc * (expf(lsm(xr[k], r.lx)) - hot);
        grad[(size_t)(n + B) * K + k] = sc * (expf(lsm(yr[k], r.ly)) - hot);
      }
    }
  }
  if (lane == 0) { sCls[warp] = cls; sMec[warp] = mec; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float c = 0.f, m = 0.f;
    for (int w = 0; w < nwarps; ++w) { c += sCls[w]; m += sMec[w]; }
    c /= (float)valid;                              // 0/0 = NaN when every label is ignored, like F.nll_loss
    m = lambda * m / (float)B;
    losses[0] = c + m; losses[1] = c; losses[2] = m;
  }
}

}  // namespace

void head_loss_launch(const float* logits, const long long* labels, int B, int K, float lambda, float* losses,
                      float* grad, int* status, cudaStream_t st) {
  int threads = 2 * B * 32;
  if (threads > kMecThreads) threads = kMecThreads;
  if (threads < 32) threads = 32;
  head_loss_kernel<<<1, threads, 0, st>>>(logits, labels, B, K, lambda, losses, grad, status);
}

void mec_launch(const float* x, const float* y, int N, int K, float* loss, float* gx, float* gy, cudaStream_t st) {
  int threads = N * 32;
  if (threads > kMecThreads) threads = kMecThreads;
  if (threads < 32) threads = 32;
  mec_kernel<<<1, threads, 0, st>>>(x, y, N, K, loss, gx, gy);
}

}  // namespace dwt

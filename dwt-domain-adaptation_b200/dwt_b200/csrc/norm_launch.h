// Host-side launch entry points of the kernel families (internal to libdwt_b200.so).
#pragma once
#include <stdint.h>

#include "dwt_common.cuh"

namespace dwt {

// The driver-API tensor-map encoder needs a current context and autograd worker threads arrive without one.
// cudaFree(0) binds the primary context but is illegal inside a stream capture: do it once per thread (the
// first call of a thread is a warm-up call, never a captured one).
inline void bind_context() {
  thread_local bool bound = false;
  if (!bound) { cudaFree(nullptr); bound = true; }
}

// register-resident path, GS in {1,2,4}  (norm_small.cu)
bool small_supports(int GS);
void small_stats(const float* x, const Geom& gm, int vec, const FwdFin& fin, float* partial, int* counters,
                 cudaStream_t st);
void small_eval_prep(const Geom& gm, const FwdFin& fin, cudaStream_t st);
void small_apply(const float* x, float* y, const Geom& gm, int vec, int chunks, int epi, const float* mean,
                 const float* w, const float* gamma, const float* beta, const float* residual, cudaStream_t st);
void small_bwd_reduce(const float* x, const float* dout, const Geom& gm, int vec, const BwdFin& fin,
                      const float* beta, float* partial, int* counters, cudaStream_t st);
void small_bwd_prep(const Geom& gm, const BwdFin& fin, cudaStream_t st);
void small_bwd_apply(const float* x, const float* dout, float* dx, const Geom& gm, int vec, int chunks, int epi,
                     const float* coef, const float* mean, const float* w, const float* gamma, const float* beta,
                     cudaStream_t st);

// shared-memory tiled path, any GS <= 64  (norm_tiled.cu)
int tiled_smem_bytes(int GS);
int tiled_init();   // opt in to large dynamic shared memory; returns cudaError_t as int
void tiled_stats(const float* x, const Geom& gm, int vec, const FwdFin& fin, float* partial, int* counters,
                 cudaStream_t st);
void tiled_eval_prep(const Geom& gm, const FwdFin& fin, cudaStream_t st);
void tiled_apply(const float* x, float* y, const Geom& gm, int vec, int chunks, const float* mean, const float* w,
                 cudaStream_t st);
void tiled_bwd_reduce(const float* x, const float* dout, const Geom& gm, int vec, const BwdFin& fin, float* partial,
                      int* counters, cudaStream_t st);
void tiled_bwd_prep(const Geom& gm, const BwdFin& fin, cudaStream_t st);
void tiled_bwd_apply(const float* x, const float* dout, float* dx, const Geom& gm, int vec, int chunks,
                     const float* coef, cudaStream_t st);

// TMA + wgmma contraction path, group sizes 8..64 tiling a 64-channel super-block  (norm_tc.cu)
int tc_init();      // driver entry point for cuTensorMapEncodeTiled + shared-memory opt-in; 0 on success
bool tc_supports(const Geom& gm, int vec);
int tc_superblocks(const Geom& gm);
int tc_stats(const float* x, const Geom& gm, int nchunks, float* shift, float* partial, cudaStream_t st);
int tc_bwd_reduce(const float* x, const float* dout, const Geom& gm, int nchunks, const float* save_mean,
                  float* partial, cudaStream_t st);

// dense per-group algebra behind the contraction (norm_dense.cu)
int dense_init();
void dense_partial_reduce(const float* partial, int nchunks, int problems, float* gram, cudaStream_t st);
void dense_fwd_factor(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st);
void dense_bwd_coef(const float* rgram, const Geom& gm, const BwdFin& fin, float* dybar, cudaStream_t st);

// TMA + wgmma apply path (norm_tc_apply.cu): split-TF32 GEMM of the block-diagonal group matrices
int tc_apply_init();
int tc_apply(const float* x, float* y, const Geom& gm, int nctas, const float* save_mean, const float* save_w,
             cudaStream_t st);
int tc_bwd_apply(const float* x, const float* dout, float* dx, const Geom& gm, int nctas, const float* coef,
                 const float* save_mean, const float* dybar, cudaStream_t st);

// channels-last (NHWC) register-resident path, GS in {1,2,4}, C/4 a power of two  (norm_cl.cu)
bool cl_supports(int C, int GS);
int cl_fwd_width(int C, int GS);
int cl_bwd_width(int C, int GS);
void cl_stats(const float* x, const Geom& gm, int nctas, int gz, float* partial, float* shift, cudaStream_t st);
void cl_fwd_finalize(const float* partial, int nrows, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st);
void cl_apply(const float* x, float* y, const Geom& gm, int nctas, int gz, int epi, const float* mean, const float* w,
              const float* gamma, const float* beta, const float* residual, uint8_t* mask, cudaStream_t st);
void cl_bwd_reduce(const float* x, const float* dout, const float* dout2, const Geom& gm, int nctas, int gz, int epi, const float* mean, const float* w,
                   const float* gamma, const float* beta, const uint8_t* mask, float* partial, cudaStream_t st);
void cl_bwd_finalize(const float* partial, int nrows, const Geom& gm, const BwdFin& fin, cudaStream_t st);
void cl_bwd_apply(const float* x, const float* dout, const float* dout2, float* dx, const Geom& gm, int nctas, int gz, int epi, const float* coef,
                  const float* mean, const float* w, const float* gamma, const float* beta, const uint8_t* mask, float* dres,
                  cudaStream_t st);

// channels-last max-pool (pool.cu)
void maxpool_fwd_launch(const float* x, float* y, uint8_t* idx, int N, int H, int W, int C, int OH, int OW, int k, int s, int p,
                        cudaStream_t st);
void maxpool_bwd_launch(const float* dy, const uint8_t* idx, float* dx, int N, int H, int W, int C, int OH, int OW, int k, int s,
                        int p, cudaStream_t st);

// MEC loss (mec.cu)
// paired target augmentation (augment.cu); mean / stdv are HOST arrays of 3
void augment_pair_launch(const uint8_t* images, int B, int SH, int SW, int CR, const int* crop_plain, const int* crop_aug,
                         const uint8_t* flip, const float* affine, const float* mean, const float* stdv,
                         float* out_plain, float* out_aug, int nhwc, cudaStream_t st);
void head_loss_launch(const float* logits, const long long* labels, int B, int K, float lambda, float* losses,
                      float* grad, int* status, cudaStream_t st);
void mec_launch(const float* x, const float* y, int N, int K, float* loss, float* gx, float* gy, cudaStream_t st);

}  // namespace dwt

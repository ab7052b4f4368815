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
// Activation pointers are void: fp32, or bf16 when `bf16` (vec must be 4: HW % 4 == 0, 8-byte-aligned tensors; the fp32
// plan of the shape, loads widened to fp32, stores rounded to nearest-even).  Statistics and coefficients are fp32.
void small_stats(const void* x, bool bf16, const Geom& gm, int vec, const FwdFin& fin, float* partial, int* counters,
                 cudaStream_t st);
void small_eval_prep(const Geom& gm, const FwdFin& fin, cudaStream_t st);
void small_apply(const void* x, void* y, bool bf16, const Geom& gm, int vec, int chunks, int epi, const float* mean,
                 const float* w, const float* gamma, const float* beta, const void* residual, cudaStream_t st);
void small_bwd_reduce(const void* x, const void* dout, bool bf16, const Geom& gm, int vec, const BwdFin& fin,
                      const float* beta, float* partial, int* counters, cudaStream_t st);
void small_bwd_prep(const Geom& gm, const BwdFin& fin, cudaStream_t st);
void small_bwd_apply(const void* x, const void* dout, void* dx, bool bf16, const Geom& gm, int vec, int chunks, int epi,
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

// TMA + wgmma contraction path, group sizes 8..64 tiling a 64-channel super-block, and 128 spanning two  (norm_tc.cu)
int tc_init();      // driver entry point for cuTensorMapEncodeTiled + shared-memory opt-in; 0 on success
bool tc_supports(const Geom& gm, int vec);
int tc_superblocks(const Geom& gm);
// Activation pointers are void: fp32, or bf16 when `bf16` (NCHW: HW % 8 == 0; 16-byte aligned; the same schedule, loads
// widened to fp32, stores rounded to nearest-even).  `nhwc`: dense channels-last tensors (HW % 4 == 0, 16-byte aligned;
// the same schedule and arithmetic as NCHW).  Partials, shifts, statistics and coefficients are fp32 either way.
int tc_stats(const void* x, bool bf16, bool nhwc, const Geom& gm, int nchunks, float* shift, float* partial, cudaStream_t st);
// group size 128 (fp32): the off-diagonal 64 x 64 Gram block of every 128-channel group, around tc_stats' shifts.
// tc_bwd_reduce at group size 128 forms all four blocks of every group's R.
int tc_gram_pair(const void* x, bool nhwc, const Geom& gm, int nchunks, const float* shift, float* partial, cudaStream_t st);
// pilot = false (group sizes 8..64): dy is not centred.  The centring drops K (sum xc)^T, which is zero only when save_mean
// is the batch mean (training); with running statistics R must be formed without it.
int tc_bwd_reduce(const void* x, const void* dout, bool bf16, bool nhwc, const Geom& gm, int nchunks, const float* save_mean,
                  float* partial, cudaStream_t st, bool pilot = true);

// dense per-group algebra behind the contraction (norm_dense.cu)
int dense_init();
void dense_partial_reduce(const float* partial, int nchunks, int problems, float* gram, cudaStream_t st);
void dense_fwd_factor(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st);
void dense_bwd_coef(const float* rgram, const Geom& gm, const BwdFin& fin, float* dybar, cudaStream_t st);
// ZCA basis, group sizes 8..64: W = S^-1/2 by `iters` Newton-Schulz steps.  save_p [D][G][iters][GS*GS] (S, P_1..P_{iters-1})
// is written by the forward and read by the backward; both leave what dense_fwd_factor / dense_bwd_coef leave.
void dense_fwd_zca(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, int iters, float* save_p,
                   cudaStream_t st);
void dense_bwd_zca(const float* rgram, const Geom& gm, const BwdFin& fin, int iters, const float* save_p, float* dybar,
                   cudaStream_t st);
// exact ZCA basis, group sizes 8..64: W = U diag(lambda^-1/2) U^T by a Jacobi eigensolver.  save_e [D][G][GS+1][GS]
// (U, then lambda) is written by the forward and read by the backward; both leave what dense_fwd_factor / dense_bwd_coef leave.
void dense_fwd_eigh(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, float* save_e, cudaStream_t st);
void dense_bwd_eigh(const float* rgram, const Geom& gm, const BwdFin& fin, const float* save_e, float* dybar, cudaStream_t st);
// colouring, group sizes 8..64 (dwt_whiten_color_*): fwd_factor that also writes gw [D][G][gs*gs] = color W; and the Cholesky
// backward on Gamma^T R with A1 = W^T color^T, plus dcolor [G][gs*gs] = sum_d R W^T and dbias [C] = sum_d sum dy over the
// domains in order (both or neither; rgram null: eval without them)
void dense_fwd_color(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, const float* color, float* gw,
                     cudaStream_t st);
void dense_bwd_color(const float* rgram, const Geom& gm, const BwdFin& fin, const float* color, float* dcolor, float* dbias,
                     float* dybar, cudaStream_t st);
// instance whitening, group sizes 8..64 (dwt_whiten_instance_*; gm.D = images, gm.N = 1): fwd_factor's work with one CTA
// per (image, group) and no EMA, W = NaN for a group that is not positive definite.  The backward is dense_bwd_coef.
void dense_fwd_instance(const float* gram, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st);
// switchable whitening, group sizes 8..64 (dwt_whiten_switch_*; gm.D = images, gm.N = 1).  save_stats [D + 1][G][gs*gs + gs]:
// each image's (cov, mean), then the batch's.  dense_sw_stats fills it from tc_stats' per-image moments (train: the batch
// row by the law of total covariance; eval: the running buffers); dense_sw_fwd_factor mixes, factors, writes save_mean /
// save_w and runs the EMA.  dense_sw_bwd turns tc_bwd_reduce's R (about save_mean, no pilot) into tc_bwd_apply's coef,
// dybar and mean (mu = the images' own means), and dmix when it is given.  Scratch: pd [D][G][rec], part [D][G][8],
// sums [G][rec].
struct SwFin {
  float a, b;                 // S = a cov_hat + b I (1 - eps, eps)
  float momentum;
  int train, update_running;
  const float* mix;           // [6] a_b, a_i, w_bw, w_iw, w_bn, w_in
  float* rmean;               // [C]
  float* rcov;                // [G][gs*gs]
  float* save_mean;           // [D][C]
  float* save_w;              // [D][G][gs*gs]
  float* save_stats;          // [D + 1][G][gs*gs + gs]
  int* status;
};
void dense_sw_stats(const float* gram, const float* shift, const Geom& gm, const SwFin& fin, cudaStream_t st);
void dense_sw_fwd_factor(const Geom& gm, const SwFin& fin, cudaStream_t st);
void dense_sw_bwd(const float* rgram, const Geom& gm, const SwFin& fin, float* pd, float* part, float* sums, float* dmix,
                  float* coef, float* dybar, float* mu, cudaStream_t st);
// latent-domain whitening, group sizes 8..64 (dwt_whiten_latent_*; gm.D = images, gm.N = 1), K latent domains weighted
// per image by weights [D][K].  save_stats (rec = gs*gs + gs): [D][G][rec] each image's (cov, mean), [K][G][rec] each
// domain's (Sigma_k, mu_k), [K][G][gs*gs] W_k, [K] s_k (dwt_b200.h).  dense_ld_stats fills the statistics rows from tc_stats'
// per-image moments (train: weighted by the law of total covariance; eval: the running buffers) and s_k; dense_ld_fwd
// factors every (domain, group), runs its EMA and mixes every (image, group) into save_w = A_n and save_mean = m~_n.
// dense_ld_bwd turns tc_bwd_reduce's R (about save_mean, no pilot) into tc_bwd_apply's coef, dybar and mean (mu = the
// images' own means), and dweights when it is given.  Scratch: sums, pd [K][G][rec], pc [K][G],
// part [D][G][kLdMaxDomains].
// Domain slots per (image, group): ld_bwd_coef keeps one register accumulator per slot, and part and ld_dw use it as
// their stride, so no domain count above it can be accepted.
constexpr int kLdMaxDomains = 8;
static_assert(DWT_MAX_LATENT_DOMAINS <= kLdMaxDomains, "latent-domain whitening: raise kLdMaxDomains with the header limit");
struct LdFin {
  float a, b;                 // S = a Sigma + b I (1 - eps, eps)
  float momentum;
  int train, update_running;
  int K;                      // latent domains, 1..8
  const float* weights;       // [D][K]
  float* rmean;               // [K][C]
  float* rcov;                // [K][G][gs*gs]
  float* save_mean;           // [D][C]  m~_n
  float* save_w;              // [D][G][gs*gs]  A_n
  float* save_stats;
  int* status;
};
void dense_ld_stats(const float* gram, const float* shift, const Geom& gm, const LdFin& fin, cudaStream_t st);
void dense_ld_fwd(const Geom& gm, const LdFin& fin, cudaStream_t st);
void dense_ld_bwd(const float* rgram, const Geom& gm, const LdFin& fin, float* sums, float* pd, float* pc, float* part,
                  float* dweights, float* coef, float* dybar, float* mu, cudaStream_t st);

// TMA + wgmma apply path (norm_tc_apply.cu): split-TF32 GEMM of the block-diagonal group matrices
int tc_apply_init();
// bias [C] (group sizes 8..64): y = W (x - mean) + bias, the accumulator starting at bias
int tc_apply(const void* x, void* y, bool bf16, bool nhwc, const Geom& gm, int nctas, const float* save_mean, const float* save_w,
             cudaStream_t st, const float* bias = nullptr);
int tc_bwd_apply(const void* x, const void* dout, void* dx, bool bf16, bool nhwc, const Geom& gm, int nctas, const float* coef,
                 const float* save_mean, const float* dybar, cudaStream_t st);

// channels-last (NHWC) register-resident path, GS in {1,2,4}, C a multiple of 4, C/4 <= 16384  (norm_cl.cu)
bool cl_supports(int C, int GS);
// column slabs (grid.y) of the sweeping kernels; every launch plan and workspace size of a call uses this count
int cl_slabs(int C);
// threads per row lane of a slab CW columns wide
int cl_lane(int C, int CW);
int cl_fwd_width(int C, int GS);
int cl_bwd_width(int C, int GS);
// Activation pointers are void: fp32, or bf16 when `bf16` (DWT_DTYPE_BF16; the same kernels, loads widened to fp32 and
// stores rounded to nearest-even).  Statistics, partial rows, coefficients and running buffers are fp32 either way.
// The finalize launches serve a second site (the two-site tail) when fin2 is given: its partial rows start at
// partial + pstride, its pilot shifts at shift + sstride.
void cl_stats(const void* x, bool bf16, const Geom& gm, int nctas, int gz, float* partial, float* shift, cudaStream_t st);
void cl_fwd_finalize(const float* partial, int nrows, const float* shift, const Geom& gm, const FwdFin& fin, cudaStream_t st,
                     const FwdFin* fin2 = nullptr, size_t pstride = 0, size_t sstride = 0);
void cl_apply(const void* x, void* y, bool bf16, const Geom& gm, int nctas, int gz, int epi, const float* mean, const float* w,
              const float* gamma, const float* beta, const void* residual, uint8_t* mask, cudaStream_t st);
// epi 7 (residual tail): masks dout (+ dout2) with the byte map and writes the masked gradient to dz
void cl_bwd_reduce(const void* x, const void* dout, const void* dout2, bool bf16, const Geom& gm, int nctas, int gz, int epi, const float* mean,
                   const float* w, const float* gamma, const float* beta, const uint8_t* mask, void* dz, float* partial, cudaStream_t st);
void cl_bwd_finalize(const float* partial, int nrows, const Geom& gm, const BwdFin& fin, cudaStream_t st,
                     const BwdFin* fin2 = nullptr, size_t pstride = 0);
// epi 0, 1 or 3; the residual tail runs it with epi 1 on the dz of its reduction
void cl_bwd_apply(const void* x, const void* dout, const void* dout2, void* dx, bool bf16, const Geom& gm, int nctas, int gz, int epi,
                  const float* coef, const float* mean, const float* w, const float* gamma, const float* beta, cudaStream_t st);
// two-site tail relu(site(x) + site_d(xd)): site's epilogue AFFINE|RELU|RESIDUAL, site_d's AFFINE
void cl_tail2_apply(const void* x, const void* xd, void* y, bool bf16, const Geom& gm, int nctas, int gz, const float* mean, const float* w,
                    const float* gamma, const float* beta, const float* mean_d, const float* w_d, const float* gamma_d,
                    const float* beta_d, uint8_t* mask, cudaStream_t st);
void cl_tail2_bwd_reduce(const void* x, const void* xd, const void* dout, const void* dout2, bool bf16, const Geom& gm, int nctas, int gz,
                         const float* mean, const float* mean_d, const uint8_t* mask, void* dz, float* partial, size_t pstride,
                         cudaStream_t st);
void cl_tail2_bwd_apply(const void* x, const void* xd, const void* dz, void* dx, void* dxd, bool bf16, const Geom& gm, int nctas, int gz,
                        const float* coef, const float* coef_d, cudaStream_t st);

// latent-domain batch norm (norm_ldbn.cu; dwt_bn_latent_*).  Rows of one (image, channel) split into S segments of P
// pixels; NCHW: any HW (bf16: HW % 4 == 0), channels-last: C % 4 == 0.  save (dwt_b200.h): [N][C] m_n (eval: the
// centre), v_n, a_n, b_n, then [D][C] mu_d, sigma2_d, r_d.
struct LdbnGeom {
  int N, C, HW, D;
  int nhwc, bf16;
  int S, P;       // segments per row, pixels per segment
  int qc, pr;     // channels-last: float4 columns x pixel rows of a CTA
};
struct LdbnFin {
  int N, C, D, S;
  double M;                   // HW
  float eps, momentum;
  int train, update_running;
  const float* weights;       // [N][D]
  float* rmean;               // [D][C]
  float* rvar;                // [D][C]
  const float* gamma;         // [C] or null (with beta)
  const float* beta;
  float* save;
  float* dgamma;              // backward: [C] or null (with dbeta)
  float* dbeta;
  int* status;
};
// The site epilogue of the latent-domain bandwidth passes (dwt_latent_site_*): out = relu(gamma zhat + beta [+ residual])
// with DWT_EPI_* bits; epi 0 is the layer.  A ReLU without a residual is recomputed by the backward passes from x with the forward's
// coefficients; a channels-last residual leaves the forward's byte map (one byte per float4, the four out > 0 bits), which
// the backward reduction reads to write the masked gradient dz.  An NCHW residual's backward is the AFFINE one on dz.
struct LdEpi {
  const float* gamma;         // [C]
  const float* beta;
  const float* p0;            // batch norm: save_stats' a_n [N][C]; whitening: save_mean (m~_n)
  const float* p1;            // batch norm: save_stats' b_n [N][C]; whitening: save_w (A_n)
  const void* res;            // forward RESIDUAL: x's shape, layout and dtype
  uint8_t* mask;              // channels-last RESIDUAL: forward writes, backward reduction reads
  void* dz;                   // backward reduction, channels-last RESIDUAL: dout * mask, x's dtype
};

LdbnGeom ldbn_plan(int N, int C, int HW, int D, bool nhwc, bool bf16);
int ldbn_finalize_ctas(int C);
// scratch floats of a call: two partial arrays of `part`, four [N][C] arrays of `nc` (pilot and the apply coefficients),
// dweights shares `dw`
size_t ldbn_scratch_floats(const LdbnGeom& g, size_t* part, size_t* nc, size_t* dw);
void ldbn_stats(const void* x, const LdbnGeom& g, float* pa, float* pb, float* pilot, cudaStream_t st);
void ldbn_fwd_finalize(const LdbnFin& f, const float* pa, const float* pb, const float* pilot, float* alpha, float* shift,
                       cudaStream_t st);
// the bandwidth passes below take the epilogue epi (AFFINE is in the coefficients; ep.p0 / p1 = a_n / b_n)
void ldbn_apply(const void* x, void* y, const LdbnGeom& g, const float* alpha, const float* shift, int epi,
                const LdEpi& ep, cudaStream_t st);
void ldbn_bwd_reduce(const void* x, const void* dy, const LdbnGeom& g, const float* centre, float* pa, float* pb, int epi,
                     const LdEpi& ep, cudaStream_t st);
// dweights null: no dwpart, no ldbn_dw launch
void ldbn_bwd_finalize(const LdbnFin& f, const float* pa, const float* pb, float* ca, float* cp, float* cq, float* dwpart,
                       float* dweights, cudaStream_t st);
void ldbn_bwd_apply(const void* x, const void* dy, void* dx, const LdbnGeom& g, const float* ca, const float* cp,
                    const float* cq, const float* centre, int epi, const LdEpi& ep, cudaStream_t st);

// latent-domain whitening at group sizes 1, 2, 4 (norm_ldbn.cu; dwt_whiten_latent_small_*) on latent-domain batch
// norm's segments: NCHW a warp per (image, group, segment) reads the group's gs channel rows, planned by ldbn_plan over
// N x C/gs rows; channels-last ldbn_plan's CTAs, a thread's 4 channels being 4/gs whole groups.  Partials
// [N][S][G][lds_partial_floats]: forward the gs sums and the gs(gs+1)/2 lower cross-products about the pilot (each row's
// first pixel), backward g_n = sum dy and R_n = sum dy (x - m_n)^T about the image's own mean.  save_stats and the
// save layout are dwt_whiten_latent_*'s.
struct LdsFin {
  int N, C, G, GS, K, S;
  double M;                   // HW
  float a, b;                 // S = a Sigma + b I (1 - eps, eps)
  float momentum;
  int train, update_running;
  const float* weights;       // [N][K]
  float* rmean;               // [K][C]
  float* rcov;                // [K][G][gs*gs]
  float* save_mean;           // [N][C]  m~_n
  float* save_w;              // [N][G][gs*gs]  A_n
  float* save_stats;
  int* status;
};
constexpr int kLdsMaxDomains = 8;   // dweights shares per (image, group)
static_assert(DWT_MAX_LATENT_DOMAINS <= kLdsMaxDomains, "latent-domain whitening: raise kLdsMaxDomains with the header limit");
LdbnGeom lds_plan(int N, int C, int HW, int GS, int K, bool nhwc, bool bf16);
// floats per (image, segment, group) partial: the larger of the forward's and the backward's
int lds_partial_floats(int GS);
// floats per (image, group) of the backward apply's coefficients: A_n (lower) | B_n | c_n | m_n
int lds_coef_floats(int GS);
// The bandwidth passes take the epilogue epi (ep.p0 / p1 = save_mean / save_w).  Under AFFINE diag(gamma) folds into
// A_n's rows and beta into the bias; the backward's reductions take dz, the finalize scales g_n, R_n by gamma and writes
// dgamma / dbeta (per-image shares in pgb [2][N][C], then added over the images in order), the apply maps gamma dz.
// forward: statistics -> finalize (per-image moments into save_stats and im [N][G][gs + gs(gs+1)/2] fp64, then per
// (domain, group) moments, W_k and EMA, then per (image, group) A_n, m~_n) -> apply y = A_n (x - m~_n)
void lds_stats(const void* x, const LdbnGeom& g, int GS, float* part, float* pilot, cudaStream_t st);
void lds_fwd_finalize(const LdsFin& f, const float* part, const float* pilot, double* im, cudaStream_t st);
void lds_apply(const void* x, void* y, const LdbnGeom& g, int GS, int epi, const LdEpi& ep, cudaStream_t st);
// backward: reduction about the saved image means -> finalize (red [N][G][gs + gs^2], pd [K][G][gs^2 + gs] P_k | mubar_k,
// pc [K][G] <P_k, Sigma_k>, coef [N][G][lds_coef_floats], dwpart [N][G][kLdsMaxDomains]; dweights null: no dwpart;
// gamma null: no AFFINE, pgb, dgamma and dbeta unused; dgamma null: no dgamma / dbeta) -> apply dx = A_n^T dy +
// B_n (x - m_n) + c_n
void lds_bwd_reduce(const void* x, const void* dy, const LdbnGeom& g, int GS, const float* save_stats, float* part, int epi,
                    const LdEpi& ep, cudaStream_t st);
void lds_bwd_finalize(const LdsFin& f, const float* part, float* red, float* pd, float* pc, float* coef, float* dwpart,
                      float* dweights, const float* gamma, float* pgb, float* dgamma, float* dbeta, cudaStream_t st);
void lds_bwd_apply(const void* x, const void* dy, void* dx, const LdbnGeom& g, int GS, const float* coef, int epi,
                   const LdEpi& ep, cudaStream_t st);

// channels-last max-pool (pool.cu); bf16: x, y, dy, dx are bf16 (compared and summed in fp32, stored rounded)
void maxpool_fwd_launch(const void* x, void* y, bool bf16, uint8_t* idx, int N, int H, int W, int C, int OH, int OW, int k, int s, int p,
                        cudaStream_t st);
void maxpool_bwd_launch(const void* dy, const uint8_t* idx, void* dx, bool bf16, int N, int H, int W, int C, int OH, int OW, int k, int s,
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

/*
 * dwt_b200.h -- C ABI of the H100-native DWT hot path (libdwt_b200.so).
 *
 * Plain C, no torch types: raw device pointers, sizes, scalars, a caller-owned
 * workspace and a CUDA stream.  Every entry point is stream-ordered, never
 * synchronises the host, never allocates, and returns 0 on success or a negative
 * DWT_E_* code (text through dwt_last_error()).  There is NO CPU path: the library
 * only launches sm_90a kernels.
 *
 * What each entry point replaces in the reference (paths relative to
 * /root/reference; the reference has no FFI -- its "plugin boundary" is Python
 * module lookup by bare name, utils/ on sys.path, SURVEY.md §8b -- so these are
 * the functions a ctypes shim behind the same nn.Module classes binds;
 * INTEGRATION.md shows that binding):
 *
 *   dwt_whiten_fwd   _Whitening.forward            utils/whitening.py:37-61
 *                    (+ the caller's shared gamma/beta/ReLU epilogue,
 *                     resnet50_dwt_mec_officehome.py:59-63,220-222, when asked)
 *   dwt_whiten_bwd   autograd through the above     utils/whitening.py:41-55
 *   dwt_whiten_zca_fwd/bwd  the same layer in the ZCA basis (Newton-Schulz iteration; not in the reference)
 *   dwt_whiten_eigh_fwd/bwd the same layer in the exact ZCA basis (Jacobi eigendecomposition; not in the reference)
 *   dwt_whiten_color_fwd/bwd whitening followed by a learnable per-group colouring matrix and bias (not in the reference)
 *   dwt_whiten_instance_fwd/bwd  instance whitening: each image by its own statistics (not in the reference)
 *   dwt_whiten_switch_fwd/bwd  switchable whitening: a learned mix of batch and per-image statistics (not in the reference)
 *   dwt_whiten_latent_fwd/bwd  latent-domain whitening: statistics of up to 8 domains under per-image soft weights (not in
 *                    the reference)
 *   dwt_whiten_latent_small_fwd/bwd  the same at group sizes 1, 2, 4 and any H*W (not in the reference)
 *   dwt_bn_latent_fwd/bwd  latent-domain batch norm: batch norm by the statistics of up to 8 domains under per-image soft
 *                    weights (the mDA layer; not in the reference)
 *   dwt_bn_fwd/bwd   _BatchNorm.forward             utils/batch_norm.py:54-69
 *   dwt_tail2_fwd/bwd  the residual tail of a downsampling Bottleneck: two norm sites and the ReLU in one pass
 *                    resnet50_dwt_mec_officehome.py:236-240
 *   dwt_mec_fwd_bwd  MinEntropyConsensusLoss.forward utils/consensus_loss.py:11-24
 *   dwt_head_loss_fwd_bwd  the training loop's NLL + lambda*MEC   resnet50_dwt_mec_officehome.py:421-428
 *   dwt_augment_pair the loader's two target views  resnet50_dwt_mec_officehome.py:481-492,526-542;
 *                                                   utils/folder.py:127-147
 *   dwt_maxpool_fwd/bwd  nn.MaxPool2d(3, 2, 1) behind the stem site   resnet50_dwt_mec_officehome.py:295,337-338
 *
 * Threading: calls may come from any host thread (PyTorch runs backward on its own); the error text is
 * per thread.  One process drives ONE device (the reference's and torchrun's model): kernel attributes
 * (shared-memory opt-in, carve-out) and the TMA encoder are set up once per process, on the device that is
 * current at the first call.  Every entry point may be captured into a CUDA graph.
 *
 * Tensor layout: activations are fp32 (or bf16, DWT_DTYPE_BF16), contiguous [n_domains * N, C, HW]
 * ("NCHW" with H*W flattened); domain d owns images [d*N, (d+1)*N).  The
 * reference calls one module per domain (n_domains = 1); the fused domain-triple
 * site passes n_domains = 3 in the order source | target | target-aug.
 */
#ifndef DWT_B200_H_
#define DWT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DWT_B200_ABI_VERSION 10
#define DWT_MAX_DOMAINS 4
/* latent-domain whitening (dwt_whiten_latent_*): domains weighted per image, not contiguous slices of the batch */
#define DWT_MAX_LATENT_DOMAINS 8
#define DWT_MAX_GROUP_SIZE 64
/* the one group size above DWT_MAX_GROUP_SIZE: whitening on the tensor-core kernels only, fp32 (dwt_whiten_fwd) */
#define DWT_TC_MAX_GROUP_SIZE 128

/* error codes */
#define DWT_OK 0
#define DWT_E_INVALID (-1)     /* bad argument (shape, group size, null pointer)  */
#define DWT_E_WORKSPACE (-2)   /* workspace too small / misaligned               */
#define DWT_E_LAUNCH (-3)      /* CUDA launch or driver error                    */
#define DWT_E_UNSUPPORTED (-4) /* valid in the reference, not built here         */

/* mode */
#define DWT_MODE_TRAIN 0 /* batch statistics (training, or track_running_stats=False) */
#define DWT_MODE_EVAL 1  /* running statistics                                        */

/* memory layout of the activation tensors, OR-ed into `mode`:
 * default = [n_domains*N, C, HW] (NCHW); DWT_LAYOUT_NHWC = [n_domains*N, HW, C] (torch.channels_last: the layout
 * cuDNN's tensor-core convolutions want, so a channels-last model needs no NCHW<->NHWC copies around its convolutions).
 * Built for two kernel families:
 *   - group sizes 1, 2, 4 with C a multiple of 4, C/4 <= 16384 (the channels-last kernels, every epilogue, dout2);
 *   - whitening at group sizes 8, 16, 32, 64 (fp32 or bf16) and 128 (fp32) on the tensor-core kernels: HW >= 32 and
 *     HW % 4 == 0, N*HW >= 4096 per domain, x / y / dout / dx 16-byte aligned (else DWT_E_INVALID), epilogue 0 and no
 *     dout2 (else DWT_E_UNSUPPORTED).  Same schedule and arithmetic as the NCHW call: every output, statistic, running-buffer update and
 *     status bit is bit for bit that of the NCHW call on the same values.  Profile families tc_*_nhwc[_bf16].
 * Any other channels-last geometry is DWT_E_UNSUPPORTED. */
#define DWT_LAYOUT_NHWC 0x100

/* activation storage, OR-ed into `mode` (dwt_whiten_*, dwt_bn_*), `kind` (dwt_tail2_*) or `flags` (dwt_maxpool_*):
 * default = fp32; DWT_DTYPE_BF16 = every ACTIVATION pointer of the call points at bfloat16 -- x, y, residual, dout,
 * dout2, dx, dresidual / dz, dwt_tail_site.x / .dx, and the max-pool's x, y, dy, dx.  Running buffers, gamma / beta and
 * their gradients, save_mean / save_w and the workspace stay fp32.  Built for three kernel families:
 *   - channels-last (DWT_LAYOUT_NHWC; the tail and the max-pool are channels-last anyway), group size 1, 2, 4 with C
 *     a multiple of 4, C/4 <= 16384; bf16 tensors 8-byte aligned;
 *   - NCHW whitening at group size 1, 2, 4 and NCHW batch norm (dwt_whiten_*, dwt_bn_*; every mode and epilogue) with
 *     HW % 4 == 0; x, y, residual, dout and dx 8-byte aligned; no dout2 (DWT_E_UNSUPPORTED, as in fp32 NCHW);
 *   - whitening on the tensor-core kernels: group size 8, 16, 32, 64, HW >= 32, N*HW >= 4096 per domain; NCHW with
 *     HW % 8 == 0 and x and dout 16-byte aligned (TMA), or channels-last with HW % 4 == 0 and x, y, dout, dx 16-byte
 *     aligned (see DWT_LAYOUT_NHWC).
 * Any other geometry is DWT_E_UNSUPPORTED (NCHW group sizes 1, 2, 4 and batch norm at HW % 4 != 0 included); a
 * misaligned tensor is DWT_E_INVALID.  bf16 launches report in the profile as <family>_bf16 and count 2 bytes per
 * activation element.
 * The kernels run the fp32 schedule of the same shape: loads widen to fp32, stores round to nearest-even, so statistics,
 * running-buffer updates, dgamma / dbeta and status bits are bit for bit those of the fp32 call on the widened inputs,
 * and every bf16 output is that call's fp32 output rounded.  Two things are rounded where a bf16 caller would round
 * them: the two-site tail's identity site_d(xd) before it is added, and dout + dout2 (once; both passes use that sum). */
#define DWT_DTYPE_BF16 0x200

/* epilogue flags */
#define DWT_EPI_NONE 0
#define DWT_EPI_AFFINE 1 /* out = y * gamma[c] + beta[c]        */
#define DWT_EPI_RELU 2   /* out = max(out, 0)  (needs AFFINE)   */
#define DWT_EPI_RESIDUAL 4 /* forward only: out = max(y*gamma + beta + residual, 0)  (needs AFFINE|RELU);
                              the Bottleneck tail `relu(bn3(conv3) + identity)`, resnet50_dwt_mec_officehome.py:239-240 */

typedef struct CUstream_st *dwt_stream_t; /* == cudaStream_t */

#if defined(__GNUC__)
#define DWT_API __attribute__((visibility("default")))
#else
#define DWT_API
#endif

DWT_API int dwt_abi_version(void);
DWT_API const char *dwt_last_error(void);

/* Workspace: one caller-owned device buffer, ZERO-FILLED once when allocated (the
 * kernels keep their arrival counters self-resetting), reusable by any sequence of
 * calls issued on ONE stream.  Size for the largest call the caller will make.
 * Group sizes 1..64 (returns 0 for any other, DWT_TC_MAX_GROUP_SIZE included).  A group-size-128 call on C channels
 * needs no more than the group-size-64 call on 2C channels: size it with dwt_workspace_bytes(N, 2*C, HW, 64, n_domains)
 * (a smaller workspace is refused with DWT_E_WORKSPACE, never overrun). */
DWT_API size_t dwt_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains);

/* Device status word (first int of the workspace): 0 = ok; bits below are OR-ed in by the kernels and stay
 * set until the caller clears the word.  Read it with a device->host copy when you want to know; nothing
 * syncs for it (dwt_b200.raise_on_status() in the Python layer polls it every k calls and raises). */
#define DWT_STATUS_NOT_PD 1    /* a batch (or running) covariance was not positive definite: the reference raises
                                  from torch.cholesky (whitening.py:53); here W is NaN for that group and that
                                  domain's running-statistics update is skipped                                  */
#define DWT_STATUS_BAD_LABEL 2 /* dwt_head_loss_fwd_bwd: a label outside [0, K) other than -100 (F.nll_loss would
                                  device-assert); the row is dropped like an ignored one, never dereferenced     */

/*
 * Whitening forward.
 *   x, y            [n_domains*N, C, HW]
 *   running_mean[d] [C]            (the reference's [1,C,1,1] buffer), may alias across d
 *   running_cov[d]  [C/gs, gs, gs] ("running_variance"),               may alias across d
 *   save_mean       [n_domains, C]            mean used (batch or running)
 *   save_w          [n_domains, C/gs, gs, gs] W = inverse(cholesky((1-eps) cov + eps I))
 *   gamma, beta     [C] or NULL (epilogue)
 *   residual        same shape/layout as x, or NULL (DWT_EPI_RESIDUAL)
 *   relu_mask       NULL, or (channels-last RESIDUAL epilogue) one byte per float4 of the output in memory order
 *                   [n_domains*N*HW*C/4]: bit k = (out[4i+k] > 0).  The backward needs it because the
 *                   pre-activation cannot be recomputed without the residual.
 * TRAIN: batch mean/cov; when update_running, the EMA r = (1-m) r + m stat is applied
 * domain by domain in order (so aliased buffers see s, then t, then t_aug --
 * SURVEY.md H5), on the UN-shrunk covariance (whitening.py:57-59).
 * EVAL: mean/cov come from the running buffers, nothing is written to them.
 * group_size: 1..64 dividing C, or 128 (DWT_TC_MAX_GROUP_SIZE, C a multiple of 128) on the tensor-core kernels only:
 * fp32, HW >= 32 and HW % 4 == 0, N*HW >= 4096 per domain, NCHW x / y 16-byte aligned (channels-last: x, y, dout,
 * dx 16-byte aligned, else DWT_E_INVALID), epilogue 0 and no dout2.  Group size 128 below that geometry, in bf16, with
 * an epilogue or a dout2, and every other group size above 64, is DWT_E_UNSUPPORTED.  Same modes, status and EMA
 * semantics as below 64; dwt_whiten_bwd takes the same group sizes.
 */
DWT_API int dwt_whiten_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size,
                   int n_domains, int mode, float eps, float momentum, int update_running,
                   float *const *running_mean, float *const *running_cov, const float *gamma,
                   const float *beta, const float *residual, uint8_t *relu_mask, int epilogue, float *save_mean,
                   float *save_w, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Whitening backward (closed form, SURVEY.md §8a).  dout is the gradient of the
 * forward's output (after the epilogue, if any).  dgamma/dbeta [C] are written
 * (summed over domains) when the epilogue has AFFINE; pass NULL otherwise.
 * Epilogue AFFINE|RELU|RESIDUAL (channels-last only): dout is the gradient of relu(z + residual); the ReLU mask is
 * read from the forward's relu_mask and the masked gradient dout * (out > 0) -- the gradient of the identity branch
 * -- is written to dresidual (required, tensor-sized) by the reduction pass; the apply pass reads it back instead of
 * dout and the mask (resnet50_dwt_mec_officehome.py:239-240).  Without RESIDUAL pass relu_mask = dresidual = NULL.
 */
DWT_API int dwt_whiten_bwd(const float *x, const float *dout, const float *dout2, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int n_domains, int mode, float eps, const float *save_mean,
                   const float *save_w, const float *gamma, const float *beta, const uint8_t *relu_mask,
                   float *dresidual, int epilogue, float *dgamma, float *dbeta, void *workspace,
                   size_t workspace_bytes, dwt_stream_t stream);

/*
 * Whitening in the ZCA basis (decorrelated batch norm / IterNorm): W = S^-1/2 by Newton-Schulz iteration instead of
 * the inverse Cholesky factor of dwt_whiten_fwd.  Per domain and group, with S = (1-eps) cov + eps I (the statistics,
 * pilot shift and shrinkage of dwt_whiten_fwd):
 *   t = tr S,  N = S / t,  P_0 = I,  P_k = (3 P_{k-1} - P_{k-1}^3 N) / 2  (k = 1..iterations),  W = P_T / sqrt(t),
 *   y = W (x - mean).
 * At a finite T this is IterNorm's partial whitening (W -> S^-1/2 as T grows), and dwt_whiten_zca_bwd differentiates
 * that function, not the limit.  W is not symmetrised: save_w holds P_T / sqrt(t) as computed.
 *   iterations  T, 1..DWT_ZCA_MAX_ITERATIONS (else DWT_E_INVALID)
 *   save_p      [n_domains, C/gs, iterations, gs, gs], 16-byte aligned (else DWT_E_INVALID): slot 0 holds S, slot k
 *               holds P_k (k = 1..T-1); written by fwd, read by bwd
 *   everything else as dwt_whiten_fwd / dwt_whiten_bwd with epilogue 0 and no dout2.
 * Running buffers get the EMA of the un-shrunk covariance, in domain order: after a training call they and save_mean
 * equal dwt_whiten_fwd's bit for bit, so running buffers are interchangeable between the two bases.  mode takes
 * DWT_MODE_*, DWT_LAYOUT_NHWC and DWT_DTYPE_BF16.
 * Built for the tensor-core kernels only: group size 8, 16, 32, 64, HW >= 32 and HW % 4 == 0, N*HW >= 4096 per domain,
 * NCHW bf16 also HW % 8 == 0, tensors aligned as for dwt_whiten_fwd.  Every other group size (1, 2, 4, 128), every
 * other geometry, and a call whose tensor-core kernels could not be set up is DWT_E_UNSUPPORTED.
 * Status: a non-finite or non-positive tr S, or a non-finite W, sets DWT_STATUS_NOT_PD and skips that domain's EMA.  An
 * indefinite S whose iteration stays finite is NOT detected (batch statistics cannot be indefinite; running buffers a
 * caller supplies for eval can).
 * Profile families dense_fwd_zca / dense_bwd_zca (_bf16) for the per-group algebra; the other passes keep tc_*.  The
 * workspace is sized by dwt_workspace_bytes as for dwt_whiten_fwd.
 */
#define DWT_ZCA_MAX_ITERATIONS 16
DWT_API int dwt_whiten_zca_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                       int mode, float eps, float momentum, int update_running, float *const *running_mean,
                       float *const *running_cov, int iterations, float *save_mean, float *save_w, float *save_p,
                       void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_zca_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW, int group_size,
                       int n_domains, int mode, float eps, int iterations, const float *save_mean, const float *save_w,
                       const float *save_p, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Whitening in the exact ZCA basis (decorrelated batch norm): W = S^-1/2 = U diag(lambda^-1/2) U^T from the
 * eigendecomposition S = U diag(lambda) U^T, with S = (1-eps) cov + eps I as in dwt_whiten_fwd, and y = W (x - mean).
 * Unlike dwt_whiten_zca_fwd's finite Newton-Schulz iteration this whitens fully at every condition number: the output
 * covariance is S^-1/2 cov S^-1/2, which tends to I as eps -> 0.  A cyclic Jacobi eigensolver diagonalises S in float32 per group; it stops after the
 * first sweep that rotates nothing, at most 16 sweeps, and reruns are bit-identical.  W = V V^T with
 * V = U diag(lambda^-1/4) is symmetric bit for bit.  dwt_whiten_eigh_bwd differentiates W(S) by the Daleckii-Krein
 * formula  dL/dS = U [(U^T R U) o F] U^T,  F_ij = -1 / (sqrt(l_i) sqrt(l_j) (sqrt(l_i) + sqrt(l_j))),  R = dL/dW, which
 * is finite for repeated eigenvalues.
 *   save_e      [n_domains, C/gs, gs + 1, gs], 16-byte aligned (else DWT_E_INVALID): rows 0..gs-1 hold U (column j the
 *               eigenvector of lambda_j), row gs holds lambda; written by fwd, read by bwd
 *   everything else as dwt_whiten_zca_fwd / dwt_whiten_zca_bwd without iterations: the same statistics, running-buffer
 *   EMA (bit for bit dwt_whiten_fwd's), geometry, layouts, dtypes and workspace.  Every other group size (1, 2, 4, 128)
 *   or geometry is DWT_E_UNSUPPORTED with a text naming the exact ZCA basis.
 * Status: a non-finite S, or an eigenvalue that is not finite and positive, sets DWT_STATUS_NOT_PD and skips that
 * domain's EMA; in eval mode this also catches an indefinite running buffer.
 * Profile families dense_fwd_eigh / dense_bwd_eigh (_bf16) for the per-group algebra; the other passes keep tc_*.
 */
DWT_API int dwt_whiten_eigh_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                       int mode, float eps, float momentum, int update_running, float *const *running_mean,
                       float *const *running_cov, float *save_mean, float *save_w, float *save_e,
                       void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_eigh_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW, int group_size,
                       int n_domains, int mode, float eps, const float *save_mean, const float *save_w,
                       const float *save_e, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Whitening followed by a learnable colouring (the whitening-and-colouring transform of Siarohin, Sangineto and Sebe,
 * "Whitening and Coloring Batch Transform", ICLR 2019), in the Cholesky basis of dwt_whiten_fwd:
 *     y = color_g W (x - mean) + bias
 *   color       [C/gs, gs, gs] (color_g: a full gs x gs matrix per group), bias [C]; shared by every domain of the call;
 *               float32, 16-byte aligned (a null or misaligned pointer is DWT_E_INVALID)
 *   save_w      W = L^-1 exactly as dwt_whiten_fwd writes it, bit for bit; color W lives in the workspace only
 *   everything else as dwt_whiten_fwd without epilogue: statistics, shrinkage, running-buffer EMA, eval mode from the
 *   running buffers, DWT_STATUS_NOT_PD (a not positive definite group skips its domain's EMA).
 * dwt_whiten_color_bwd, with R_d = sum_m dout (x - mean)^T per domain and group, M = N*HW:
 *   dcolor = sum_d R_d W_d^T,  dbias = sum_d sum_m dout   [C/gs, gs, gs] and [C], both or neither (NULL: not formed),
 *               summed over the domains in a fixed order (reruns are bit-identical)
 *   train: dx = W^T color^T (dout - mean_M dout) + Bm (x - mean), Bm the Cholesky backward of dwt_whiten_bwd on color^T R
 *   eval:  dx = W^T color^T dout (no reduction pass unless dcolor / dbias are asked for)
 * mode takes DWT_MODE_*, DWT_LAYOUT_NHWC and DWT_DTYPE_BF16, with dwt_whiten_zca_fwd's layout, dtype and alignment rules.
 * Built for the tensor-core kernels only: group size 8, 16, 32, 64.  Every other group size (1, 2, 4, 128), every other
 * geometry, and a call whose tensor-core kernels could not be set up is DWT_E_UNSUPPORTED with a text naming the
 * colouring transform.  Workspace: dwt_workspace_bytes as for dwt_whiten_fwd.
 * Profile families dense_fwd_color / dense_bwd_color (_bf16) for the per-group algebra; the other passes keep tc_*.
 */
DWT_API int dwt_whiten_color_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                       int mode, float eps, float momentum, int update_running, float *const *running_mean,
                       float *const *running_cov, const float *color, const float *bias, float *save_mean, float *save_w,
                       void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_color_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW, int group_size,
                       int n_domains, int mode, float eps, const float *save_mean, const float *save_w, const float *color,
                       float *dcolor, float *dbias, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Instance whitening: every image whitened by its own statistics (the per-sample whitening of Switchable Whitening,
 * Pan et al., ICCV 2019; the instance-whitening statistic of RobustNet, Choi et al., CVPR 2021; the whitening step of
 * WCT style transfer, Li et al., NeurIPS 2017).  It is to dwt_whiten_fwd what InstanceNorm is to BatchNorm.  Per image n
 * and group g, with M = HW:
 *     mean = sum_pixels x / M,  cov = (x - mean)(x - mean)^T / M (biased),  S = (1-eps) cov + eps I = L L^T,
 *     W = L^-1,  y = W (x - mean).
 * No running buffers and no modes: training and inference compute the same thing, and dwt_whiten_instance_bwd always
 * differentiates through mean and cov (the closed form of dwt_whiten_bwd per image, with R = sum_pixels dout (x-mean)^T):
 *     dx = W^T (dout - mean_M dout) + Bm (x - mean),  Bm = (2 (1-eps) / M) sym(W^T Phi(-R W^T) W).
 *   x, y, dout, dx  [N, C, HW] (or channels-last [N, HW, C] with DWT_LAYOUT_NHWC), fp32 or bf16 (DWT_DTYPE_BF16)
 *   flags           DWT_LAYOUT_NHWC | DWT_DTYPE_BF16 (any other bit: DWT_E_INVALID)
 *   save_mean       [N, C] per-image mean;  save_w [N, C/gs, gs, gs] per-image W (16-byte aligned); written by fwd,
 *                   read by bwd
 * The statistics, factorisation, apply and backward are the tensor-core whitening kernels with the images as the domains
 * (same split-TF32 arithmetic, pilot shift and fixed-order reductions: reruns are bit-identical).  bf16 loads widen to
 * fp32 and stores round to nearest-even: every bf16 output is the fp32 call's output on the widened input, rounded.
 * Channels-last outputs are bit for bit those of the NCHW call on the same values.
 * Built for group size 8, 16, 32, 64 dividing C, HW >= 256 and HW % 4 == 0 (NCHW bf16: HW % 8 == 0), N <= 65535 and
 * N*C*HW < 2^31; there is no floor on N or N*HW.  Anything else -- and a call whose tensor-core kernels could not be set
 * up -- is DWT_E_UNSUPPORTED with a text naming instance whitening.  x, y, dout, dx and save_w must be 16-byte aligned
 * (else DWT_E_INVALID).  Every n_domains rule of the other entry points (DWT_MAX_DOMAINS) is unchanged: this family has
 * no domain count.
 * Status: an (image, group) whose S is not positive definite or not finite sets DWT_STATUS_NOT_PD, and its W, and so its
 * output and its dx, are NaN; other images and groups are not affected.
 * Workspace: dwt_instance_workspace_bytes(N, C, HW, group_size) bytes, 256-byte aligned, zero-filled once (it may be the
 * same buffer as the other entry points'; the status word is shared).  It returns 0 for a geometry the entry points refuse.
 * Profile families iw_stats, iw_fwd_finalize, iw_apply, iw_bwd_reduce, iw_bwd_finalize, iw_bwd_apply (_nhwc, _bf16);
 * the geometry in the profile name reports the images as domains of one image each.
 */
DWT_API size_t dwt_instance_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size);
DWT_API int dwt_whiten_instance_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int flags,
                       float eps, float *save_mean, float *save_w, void *workspace, size_t workspace_bytes,
                       dwt_stream_t stream);
DWT_API int dwt_whiten_instance_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW,
                       int group_size, int flags, float eps, const float *save_mean, const float *save_w, void *workspace,
                       size_t workspace_bytes, dwt_stream_t stream);

/*
 * Switchable whitening (Pan et al., ICCV 2019): every image whitened by a learned mixture of the batch's and its own
 * statistics.  Per image n and group g, with M = HW, the image's own mean and biased covariance mu_n, cov_n (as
 * dwt_whiten_instance_fwd), the batch's mu_b, cov_b over all N*M pixels (DWT_MODE_EVAL: the running buffers instead) and
 * mix = (a_b, a_i, w_bw, w_iw, w_bn, w_in), six device floats:
 *     m_n = a_b mu_b + a_i mu_n,   cov_hat = w_bw cov_b + w_iw cov_n + w_bn diag(cov_b) + w_in diag(cov_n),
 *     S = (1-eps) cov_hat + eps I = L L^T,   W = L^-1,   y = W (x - m_n).
 * Each covariance is about its own mean.  mix is used as given: no softmax, normalisation or sign check (the softmax
 * belongs to the caller, SwitchableWTransform2d).
 * DWT_MODE_TRAIN with update_running: running = (1-momentum) running + momentum stat on the unshrunk (mu_b, cov_b), the
 * convention of dwt_whiten_fwd (the buffers are interchangeable with its running_mean[0] / running_cov[0]); skipped, with
 * DWT_STATUS_NOT_PD, for a group whose mu_b or cov_b is not finite.  DWT_MODE_EVAL reads the buffers and writes nothing.
 * dwt_whiten_switch_bwd is the exact gradient of the forward (in eval the batch statistics are constants):
 *     P_n = dL/dcov_hat = (1-eps) sym(W^T Phi(-R W^T) W), R = sum_pixels dout (x - m_n)^T;  dm_n = -W^T sum_pixels dout
 *     Q_n = w_iw P_n + w_in diag(P_n),  Q_b = sum_n (w_bw P_n + w_bn diag(P_n))
 *     dx = W^T dout + (a_i/M) dm_n + (2/M) Q_n (x - mu_n)  [train: + (a_b/NM) sum_k dm_k + (2/NM) Q_b (x - mu_b)]
 *     dmix = sum over images and groups of (<dm_n, mu_b>, <dm_n, mu_n>, <P_n, cov_b>, <P_n, cov_n>, <P_n, diag cov_b>,
 *            <P_n, diag cov_n>)
 *   x, y, dout, dx  [N, C, HW] (or channels-last [N, HW, C] with DWT_LAYOUT_NHWC), fp32 or bf16 (DWT_DTYPE_BF16)
 *   mode            DWT_MODE_TRAIN / DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16 (any other bit: DWT_E_INVALID)
 *   running_mean [C], running_cov [C/gs, gs, gs]: read in eval, updated in train with update_running (else unused, may be
 *                   NULL)
 *   save_mean [N, C] the mixed mean m_n;  save_w [N, C/gs, gs, gs] W;  save_stats [N + 1, C/gs, gs*gs + gs]: rows 0..N-1
 *                   each image's (cov_n, mu_n), row N the (cov_b, mu_b) the call used.  Written by fwd, read by bwd.
 *   dmix [6]        written (never accumulated) by bwd; NULL skips it
 * mix, save_w and save_stats must be 16-byte aligned, as must x, y, dout and dx (else DWT_E_INVALID).
 * The batch moments come from the per-image ones by the law of total covariance (cov_b = mean cov_n + cov(mu_n)),
 * summed in fp64 over the images in order about image 0's mean: no second pass over x.  Every reduction is in a fixed
 * order: reruns are bit-identical, dmix included.  bf16 loads widen to fp32 and stores round to nearest-even: every bf16
 * output is the fp32 call's output on the widened input, rounded.  Channels-last outputs are bit for bit those of NCHW.
 * Geometry as dwt_whiten_instance_*: group size 8, 16, 32, 64 dividing C, HW >= 256 and HW % 4 == 0 (NCHW bf16:
 * HW % 8 == 0), N <= 65535 and N*C*HW < 2^31.  Anything else -- and a call whose tensor-core kernels could not be set
 * up -- is DWT_E_UNSUPPORTED with a text naming switchable whitening.
 * Status: an (image, group) whose S is not positive definite, or whose S or m_n is not finite (a non-finite mix, say),
 * gets a NaN W, so NaN output and dx, and sets DWT_STATUS_NOT_PD; other images and groups are not affected, except that in
 * training the batch terms of the backward carry the NaN to that group's dx in every image, and dmix is NaN.
 * Workspace: dwt_switch_workspace_bytes(N, C, HW, group_size) bytes, 256-byte aligned, zero-filled once (it may be the
 * same buffer as the other entry points'; the status word is shared).  It returns 0 for a geometry the entry points refuse.
 * Profile families sw_stats, sw_fwd_finalize, sw_apply, sw_bwd_reduce, sw_bwd_finalize, sw_bwd_apply (_nhwc, _bf16).
 */
DWT_API size_t dwt_switch_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size);
DWT_API int dwt_whiten_switch_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int mode,
                   float eps, float momentum, int update_running, float *running_mean, float *running_cov,
                   const float *mix, float *save_mean, float *save_w, float *save_stats,
                   void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_switch_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int mode, float eps, const float *mix, const float *save_mean, const float *save_w,
                   const float *save_stats, float *dmix, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Latent-domain whitening (the whitening form of the mDA layer, Mancini et al., CVPR 2018): K = n_domains domains whose
 * membership is a weight per image, weights [N, K] (soft assignments inferred by the network, or one-hot labels of uneven,
 * interleaved domains).  Per group g, with M = HW, each image's own mean and biased covariance m_n, C_n (as
 * dwt_whiten_instance_fwd) and s_k = sum_n w_nk:
 *     mu_k = sum_n w_nk m_n / s_k,   Sigma_k = sum_n w_nk [C_n + (m_n - mu_k)(m_n - mu_k)^T] / s_k   (the w-weighted pixel
 *     moments; DWT_MODE_EVAL: domain k's running buffers instead),   S_k = (1-eps) Sigma_k + eps I = L_k L_k^T,  W_k = L_k^-1,
 *     y_n = sum_k w_nk W_k (x_n - mu_k) = A_n (x_n - m~_n),   A_n = sum_k w_nk W_k,   A_n m~_n = sum_k w_nk W_k mu_k.
 * weights are used as given: no softmax, normalisation or sign check (the softmax belongs to the caller).
 * Edge rules:
 *   - a domain with s_k == 0 exactly is skipped: no W_k, no share in any output, running buffers untouched, no status,
 *     dweights[:, k] = 0 (the function is not differentiable there);
 *   - a domain with s_k < 0 or NaN, non-finite statistics, or an S_k that is not positive definite gets W_k = NaN, sets
 *     DWT_STATUS_NOT_PD and skips its EMA;
 *   - every sum over images or domains skips a weight that is exactly 0 instead of multiplying by it: an image whose weight
 *     on a bad domain is 0 stays finite, and so does its dx;
 *   - an (image, group) whose A_n has a diagonal entry that is not positive and finite (negative weights, no weight at all),
 *     or whose A_n or m~_n is not finite, gets A_n = NaN (m~_n = 0), so NaN output and dx in that group, and sets
 *     DWT_STATUS_NOT_PD.  A bad domain's NaN reaches, in training, that group's dx in every image with weight on it, and
 *     dweights[:, k].
 * DWT_MODE_TRAIN with update_running: running_k = (1-momentum) running_k + momentum (mu_k, Sigma_k), unshrunk and biased,
 * the convention of dwt_whiten_fwd (with one-hot weights the buffers are those of a WTransform2d per domain).
 * DWT_MODE_EVAL reads the buffers and writes nothing; s_k still comes from the weights (the zero-mass rule).
 * dwt_whiten_latent_bwd is the exact gradient of the forward (in eval mu_k and Sigma_k are constants).  With
 * g_n = sum_pixels dout, R_n = sum_pixels dout (x - m_n)^T:
 *     Wbar_k = sum_n w_nk [R_n + g_n (m_n - mu_k)^T],  mubar_k = -W_k^T sum_n w_nk g_n,
 *     P_k = dL/dSigma_k = (1-eps) sym(W_k^T Phi(-Wbar_k W_k^T) W_k)   (dwt_whiten_bwd's Cholesky backward)
 *     dx = A_n^T dout + (1/M) sum_k (w_nk/s_k) [mubar_k + 2 P_k (x - mu_k)]         (eval: A_n^T dout)
 *     dweights_nk = sum_g <W_k, R_n + g_n (m_n - mu_k)^T>
 *                   + (1/s_k) [<mubar_k, m_n - mu_k> + <P_k, C_n + (m_n - mu_k)(m_n - mu_k)^T - Sigma_k>]   (eval: first term)
 *   x, y, dout, dx  [N, C, HW] (or channels-last [N, HW, C] with DWT_LAYOUT_NHWC), fp32 or bf16 (DWT_DTYPE_BF16)
 *   n_domains       K, 1..DWT_MAX_LATENT_DOMAINS (else DWT_E_INVALID)
 *   mode            DWT_MODE_TRAIN / DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16 (any other bit: DWT_E_INVALID)
 *   running_mean [K, C], running_cov [K, C/gs, gs, gs] (contiguous): read in eval, updated in train with update_running
 *                   (else unused, may be NULL)
 *   weights [N, K]  fp32, device
 *   save_mean [N, C] m~_n;  save_w [N, C/gs, gs, gs] A_n;  save_stats, with rec = gs*gs + gs and G = C/gs, floats:
 *                   [N][G][rec] each image's (C_n, m_n), [K][G][rec] each domain's (Sigma_k, mu_k), [K][G][gs*gs] W_k,
 *                   [K] s_k -- (N + K) G rec + K G gs^2 + K in all.  Written by fwd, read by bwd.
 *   dweights [N, K] written (never accumulated) by bwd; NULL skips it
 * weights, save_w and save_stats must be 16-byte aligned, as must x, y, dout and dx (else DWT_E_INVALID).
 * The statistics, apply and backward contraction are dwt_whiten_instance_*'s tensor-core passes; the domain moments come
 * from the per-image ones in fp64 over the images in order about image 0's mean (no second pass over x), and every other
 * reduction is in a fixed order too: reruns are bit-identical, dweights included.  bf16 loads widen to fp32 and stores round
 * to nearest-even: every bf16 output is the fp32 call's output on the widened input, rounded.  Channels-last outputs are
 * bit for bit those of NCHW.
 * Geometry as dwt_whiten_instance_*: group size 8, 16, 32, 64 dividing C, HW >= 256 and HW % 4 == 0 (NCHW bf16:
 * HW % 8 == 0), N <= 65535 and N*C*HW < 2^31.  Anything else -- and a call whose tensor-core kernels could not be set
 * up -- is DWT_E_UNSUPPORTED with a text naming latent-domain whitening.  DWT_MAX_DOMAINS and the other entry points'
 * rules are unchanged.
 * Workspace: dwt_latent_workspace_bytes(N, C, HW, group_size, n_domains) bytes, 256-byte aligned, zero-filled once (it may
 * be the same buffer as the other entry points'; the status word is shared).  It returns 0 for a call the entry points
 * refuse for its geometry or n_domains.
 * Profile families ld_stats, ld_fwd_finalize, ld_apply, ld_bwd_reduce, ld_bwd_finalize, ld_bwd_apply (_nhwc, _bf16).
 */
DWT_API size_t dwt_latent_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains);
DWT_API int dwt_whiten_latent_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size, int n_domains,
                   int mode, float eps, float momentum, int update_running, float *running_mean, float *running_cov,
                   const float *weights, float *save_mean, float *save_w, float *save_stats,
                   void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_latent_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int n_domains, int mode, float eps, const float *weights, const float *save_mean,
                   const float *save_w, const float *save_stats, float *dweights, void *workspace, size_t workspace_bytes,
                   dwt_stream_t stream);

/*
 * Latent-domain whitening at group sizes 1, 2, 4 (the whitening sites of ResNet-50-DWT and the digits LeNet): the
 * function, edge rules, EMA, backward, dweights and every argument and save layout of dwt_whiten_latent_fwd / _bwd
 * above, so a caller changes only which symbols it calls.  What differs is the geometry and the kernels:
 *   group_size 1, 2 or 4 dividing C, any HW >= 1, 1..DWT_MAX_LATENT_DOMAINS domains, N*C*HW < 2^31; channels-last needs
 *   C % 4 == 0 and NCHW bf16 HW % 4 == 0.  Anything else is DWT_E_UNSUPPORTED with a text naming latent-domain whitening
 *   at group sizes 1, 2, 4.
 *   x, y, dout, dx fp32 16-byte, bf16 8-byte aligned; weights, save_w and save_stats 16-byte, save_mean and dweights
 *   4-byte aligned (else DWT_E_INVALID).
 * The kernels are latent-domain batch norm's four bandwidth passes on its segments, a group of gs channels in place of one
 * channel: per (image, segment, group) the gs sums and gs(gs+1)/2 cross-products about each row's first pixel (forward)
 * or g_n and R_n about the image's own mean (backward), then y = A_n (x - m~_n) and dx = A_n^T dout + B_n (x - m_n) + c_n
 * with the per-image coefficients in registers.  The finalize kernels give every (image, group) a thread and every
 * (domain, group) a warp; the domain moments are taken in fp64 about image 0's mean (lane l adds images l, l + 32, ...
 * in order, then the lanes by a fixed butterfly) and every reduction runs in a fixed order (no float atomics): reruns
 * are bit-identical, dweights included.  The statistics pass also runs in eval
 * (the backward's centre is the image's own mean): 12 B per element forward, 20 B backward in fp32.  bf16 loads widen to
 * fp32 and stores round to nearest-even on the fp32 plan of the shape: every bf16 output is the fp32 call's output on the
 * widened input, rounded.  Neither call syncs the host; both may be captured into a CUDA graph.
 * Workspace: dwt_latent_small_workspace_bytes(N, C, HW, group_size, n_domains) bytes, 256-byte aligned, zero-filled once
 * (it may be the same buffer as the other entry points'; the status word is shared).  It returns 0 for a call the entry
 * points refuse for its geometry or n_domains.
 * Profile families lds_stats, lds_fwd_finalize, lds_apply, lds_bwd_reduce, lds_bwd_finalize, lds_bwd_apply (_nhwc, _bf16
 * on the bandwidth passes).
 */
DWT_API size_t dwt_latent_small_workspace_bytes(int64_t N, int64_t C, int64_t HW, int group_size, int n_domains);
DWT_API int dwt_whiten_latent_small_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size,
                   int n_domains, int mode, float eps, float momentum, int update_running, float *running_mean,
                   float *running_cov, const float *weights, float *save_mean, float *save_w, float *save_stats,
                   void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_whiten_latent_small_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int n_domains, int mode, float eps, const float *weights, const float *save_mean,
                   const float *save_w, const float *save_stats, float *dweights, void *workspace, size_t workspace_bytes,
                   dwt_stream_t stream);

/*
 * Latent-domain batch norm (the mDA layer of Mancini et al., CVPR 2018, in its batch-norm form): D = n_domains domains
 * whose membership is a weight per image, weights [N, D], as dwt_whiten_latent_*.  Per channel c, with M = HW, each
 * image's own mean and biased variance m_n, v_n and s_d = sum_n w_nd:
 *     mu_d = sum_n w_nd m_n / s_d,   sigma2_d = sum_n w_nd [v_n + (m_n - mu_d)^2] / s_d   (DWT_MODE_EVAL: domain d's
 *     running_mean / running_var instead),   r_d = (sigma2_d + eps)^-1/2,
 *     y_n = gamma sum_d w_nd r_d (x_n - mu_d) + beta = gamma (a_n x_n + b_n) + beta,  a_n = sum_d w_nd r_d,
 *     b_n = -sum_d w_nd r_d mu_d   (gamma = beta = NULL: no affine).
 * weights are used as given (no softmax, normalisation or sign check).  With one-hot weights every domain's output and
 * buffers are those of F.batch_norm on its subset of the batch.
 * Edge rules, per (domain, channel) unless said otherwise:
 *   - s_d == 0 exactly: the domain is skipped -- no share in any output, buffers untouched, no status, dweights[:, d] = 0;
 *   - s_d < 0 or NaN, mu_d or sigma2_d not finite, or sigma2_d + eps <= 0: r_d = NaN, DWT_STATUS_NOT_PD, that domain's EMA
 *     skipped for that channel;
 *   - every sum over images or domains skips a weight that is exactly 0 instead of multiplying by it: an image with
 *     weight 0 on a bad domain stays finite, and so does its dx;
 *   - an (image, channel) whose a_n is not positive and finite or whose b_n is not finite gets a_n = NaN, b_n = 0 (NaN
 *     output and dx there) and sets DWT_STATUS_NOT_PD;
 *   - 0 < M s_d <= 1 (the unbiased variance is undefined): the buffers stay untouched, no status; the output still uses
 *     the biased sigma2_d.
 * DWT_MODE_TRAIN with update_running: running_mean_d = (1-momentum) running_mean_d + momentum mu_d and running_var_d =
 * (1-momentum) running_var_d + momentum sigma2_d M s_d / (M s_d - 1), F.batch_norm's convention.  DWT_MODE_EVAL reads the
 * buffers and writes nothing; s_d still comes from the weights (the zero-mass rule).
 * dwt_bn_latent_bwd is the exact gradient of the forward (in eval mu_d and sigma2_d are constants).  With g = gamma dout,
 * G_n = sum_pixels g, H_n = sum_pixels g (x - m_n), A_d = sum_n w_nd G_n, B_d = sum_n w_nd [H_n + G_n (m_n - mu_d)]:
 *     dx = a_n g - sum_d (w_nd / (M s_d)) [r_d A_d + r_d^3 B_d (x - mu_d)]                               (eval: a_n g)
 *     dweights_nd = sum_c { r_d [H_n + G_n (m_n - mu_d)]
 *                           - (1/s_d) [r_d A_d (m_n - mu_d) + r_d^3 B_d (v_n + (m_n - mu_d)^2 - sigma2_d) / 2] }  (eval: first term)
 *     dgamma = sum dout zhat, dbeta = sum dout (from the sums of dout, so gamma = 0 is fine).
 *   x, y, dout, dx  [N, C, HW] (or channels-last [N, HW, C] with DWT_LAYOUT_NHWC), fp32 or bf16 (DWT_DTYPE_BF16);
 *                   fp32 16-byte, bf16 8-byte aligned (else DWT_E_INVALID)
 *   n_domains       D, 1..DWT_MAX_LATENT_DOMAINS (else DWT_E_INVALID)
 *   mode            DWT_MODE_TRAIN / DWT_MODE_EVAL | DWT_LAYOUT_NHWC | DWT_DTYPE_BF16 (any other bit: DWT_E_INVALID)
 *   running_mean, running_var [D, C] (contiguous): read in eval, updated in train with update_running (else unused, may be
 *                   NULL)
 *   weights [N, D]  fp32, device
 *   gamma, beta     [C] or both NULL;  dgamma, dbeta [C] or both NULL (written, never accumulated; they need gamma)
 *   save_stats      (4 N + 3 D) C floats, 16-byte aligned, written by fwd and read by bwd: [N][C] m_n (eval: the centre
 *                   -b_n / a_n, 0 for a bad image), [N][C] v_n (train), [N][C] a_n, [N][C] b_n, then [D][C] mu_d,
 *                   [D][C] sigma2_d, [D][C] r_d (0 for a skipped domain)
 *   dweights [N, D] written (never accumulated) by bwd; NULL skips it
 *   eps             bwd: unused (r_d is saved); kept so both calls take the forward's arguments
 * Statistics are per-(image, channel) sums about the row's first pixel; the domain moments are taken from them in fp64
 * about image 0's mean, and every reduction runs in a fixed order (no float atomics): reruns are bit-identical, dweights,
 * dgamma and dbeta included.  Apart from the statistics pass and the backward reduction nothing reads x again: 12 B per
 * element forward, 20 B backward in fp32 (eval forward: 8 B).  bf16 loads widen to fp32 and stores round to nearest-even
 * on the fp32 plan of the shape: every bf16 output is the fp32 call's output on the widened input, rounded.
 * Geometry: any C >= 1 and HW >= 1 with N*C*HW < 2^31; channels-last needs C % 4 == 0 and NCHW bf16 HW % 4 == 0.  Anything
 * else is DWT_E_UNSUPPORTED with a text naming latent-domain batch norm.
 * Workspace: dwt_bn_latent_workspace_bytes(N, C, HW, n_domains) bytes, 256-byte aligned, zero-filled once (it may be the
 * same buffer as the other entry points'; the status word is shared).  It returns 0 for a call the entry points refuse for
 * its geometry or n_domains.  Neither call syncs the host; both may be captured into a CUDA graph.
 * Profile families ldbn_stats, ldbn_fwd_finalize, ldbn_apply, ldbn_bwd_reduce, ldbn_bwd_finalize, ldbn_bwd_apply
 * (_nhwc, _bf16 on the bandwidth passes).
 */
DWT_API size_t dwt_bn_latent_workspace_bytes(int64_t N, int64_t C, int64_t HW, int n_domains);
DWT_API int dwt_bn_latent_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int n_domains, int mode, float eps,
                   float momentum, int update_running, float *running_mean, float *running_var, const float *weights,
                   const float *gamma, const float *beta, float *save_stats, void *workspace, size_t workspace_bytes,
                   dwt_stream_t stream);
DWT_API int dwt_bn_latent_bwd(const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW, int n_domains,
                   int mode, float eps, const float *weights, const float *gamma, const float *save_stats, float *dweights,
                   float *dgamma, float *dbeta, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Latent-domain sites: a latent-domain layer with the norm site of ResNet-50-DWT fused behind it,
 *     out = relu(gamma (.) zhat + beta [+ residual]),
 * zhat being the output of dwt_bn_latent_fwd (kind DWT_KIND_BN, group_size 1) or dwt_whiten_latent_small_fwd (kind
 * DWT_KIND_WHITEN, group sizes 1, 2, 4) without gamma / beta.  Everything but the epilogue -- the function, edge rules, EMA,
 * modes, layouts, dtypes, geometry, alignment, workspace (dwt_bn_latent_workspace_bytes / dwt_latent_small_workspace_bytes)
 * and save layouts -- is that entry point's: batch norm reads and writes save_stats only (save_mean, save_w unused, may be
 * NULL), whitening save_mean, save_w and save_stats.  running_second is batch norm's running_var or whitening's
 * running_cov.  With epilogue 0 (and gamma = beta = NULL) both calls are those entry points.
 *   epilogue    DWT_EPI_* bits as in dwt_whiten_fwd: AFFINE (gamma, beta [C] required, and only with it), RELU (needs
 *               AFFINE), RESIDUAL (needs AFFINE|RELU; forward: residual of x's shape, layout and dtype)
 *   relu_mask   channels-last RESIDUAL only (else NULL): one byte per float4 of the output in memory order [N*HW*C/4],
 *               bit k = !(pre-activation <= 0); written by fwd, read by bwd
 * The ReLU is torch.relu's and its gradient threshold_backward's: a NaN pre-activation (a bad image or domain of the edge
 * rules) stays NaN and passes its gradient, so the layer's edge rules hold under every epilogue.
 *   dresidual   bwd, channels-last RESIDUAL only (else NULL): receives dz = dout * (out > 0), the gradient of the identity
 *               branch; the backward apply reads it back instead of dout
 *   dgamma, dbeta  bwd: [C], written (never accumulated), or both NULL; need AFFINE
 * The forward folds gamma, beta into the apply's coefficients (batch norm: alpha = gamma a_n, shift = gamma b_n + beta;
 * whitening: diag(gamma) A_n and gamma (-A_n m~_n) + beta) and adds the residual and takes the ReLU in registers.  A ReLU
 * without a residual is recomputed by both backward passes from x with the forward's coefficients and FMA order, so its
 * mask is the forward's bit for bit (batch norm's backward therefore takes beta too).  An NCHW residual has no byte map: its
 * backward is the AFFINE call on dz = dout * (out > 0), which the caller forms (RESIDUAL in an NCHW backward:
 * DWT_E_INVALID).  Whitening's backward runs on gamma dz, and dgamma_i = sum_n [sum_{j<=i} (A_n)_ij Rz_n,ij + (A_n (m_n -
 * m~_n))_i gz_n,i], dbeta_i = sum_n gz_n,i from the per-(image, group) sums gz_n = sum dz, Rz_n = sum dz (x - m_n)^T the
 * backward reduction already takes (no further pass over x).  Reductions keep their fixed order: reruns are bit-identical;
 * bf16 outputs (residual widened too) are the fp32 call's on the widened inputs, rounded once.
 * Refusals: kind not DWT_KIND_BN / DWT_KIND_WHITEN, batch norm at group_size != 1, a bad epilogue combination, gamma / beta
 * / residual / dresidual / relu_mask outside the epilogue that uses them, misaligned gamma, beta (4 bytes), residual or
 * dresidual (x's rule): DWT_E_INVALID; whitening at group_size 8 and above: DWT_E_UNSUPPORTED; then every refusal of the
 * layer's own entry points, whose texts (naming the layer) the pair ends with " [latent-domain site]".
 * Profile families: those of the layer's entry points (ldbn_*, lds_*), the residual and byte map counted in the bytes.
 */
DWT_API int dwt_latent_site_fwd(int kind, const float *x, float *y, int64_t N, int64_t C, int64_t HW, int group_size,
                   int n_domains, int mode, float eps, float momentum, int update_running, float *running_mean,
                   float *running_second, const float *weights, const float *gamma, const float *beta,
                   const float *residual, uint8_t *relu_mask, int epilogue, float *save_mean, float *save_w,
                   float *save_stats, void *workspace, size_t workspace_bytes, dwt_stream_t stream);
DWT_API int dwt_latent_site_bwd(int kind, const float *x, const float *dout, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int n_domains, int mode, float eps, const float *weights, const float *gamma,
                   const float *beta, const uint8_t *relu_mask, float *dresidual, int epilogue, const float *save_mean,
                   const float *save_w, const float *save_stats, float *dweights, float *dgamma, float *dbeta,
                   void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Domain batch norm (F.batch_norm semantics): biased batch variance normalises,
 * the UNBIASED one goes into running_var with weight `factor` (momentum, or
 * 1/num_batches_tracked for the cumulative average, batch_norm.py:59-64).
 *   weight, bias [C] or NULL ; save_mean, save_invstd [n_domains, C]
 */
DWT_API int dwt_bn_fwd(const float *x, float *y, int64_t N, int64_t C, int64_t HW, int n_domains, int mode,
               float eps, float factor, int update_running, float *const *running_mean,
               float *const *running_var, const float *weight, const float *bias, const float *residual,
               uint8_t *relu_mask, int epilogue, float *save_mean, float *save_invstd, void *workspace,
               size_t workspace_bytes, dwt_stream_t stream);

DWT_API int dwt_bn_bwd(const float *x, const float *dout, const float *dout2, float *dx, int64_t N, int64_t C, int64_t HW,
               int n_domains, int mode, const float *save_mean, const float *save_invstd,
               const float *weight, const float *bias, const uint8_t *relu_mask, float *dresidual, int epilogue,
               float *dweight, float *dbias, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Two-site residual tail of a downsampling Bottleneck (block 0 of a stage, resnet50_dwt_mec_officehome.py:236-240),
 * training mode, channels-last only (the channels-last kernels: C a multiple of 4, C/4 <= 16384, else DWT_E_UNSUPPORTED):
 *   out = relu(site(x) + site_d(xd)),   site(x)    = gamma   W   (x  - mu)   + beta     (the norm site after conv3)
 *                                       site_d(xd) = gamma_d W_d (xd - mu_d) + beta_d   (the downsample branch's site)
 * sites[0] describes site, sites[1] site_d; both have the same N, C, HW, group_size and n_domains.  The identity
 * tensor site_d(xd) is never written.  Bit for bit the same as the two-call composition
 *   dwt_*_fwd(xd -> identity, AFFINE);  dwt_*_fwd(x -> out, AFFINE|RELU|RESIDUAL, residual = identity)
 * and its backward (dwt_*_bwd of both sites, the second fed the first's dresidual), including running-statistic
 * updates and, per site, the non-positive-definite handling of DWT_STATUS_NOT_PD.
 *   kind        DWT_KIND_WHITEN (as dwt_whiten_*, group_size 1, 2, 4) or DWT_KIND_BN (as dwt_bn_*, group_size 1),
 *               optionally | DWT_DTYPE_BF16
 *   relu_mask   the byte map of dwt_whiten_fwd's RESIDUAL epilogue: written by fwd, read by bwd
 *   dz          bwd: tensor-sized scratch, receives dout * (out > 0) (the gradient of both sites' outputs)
 *   dout2       NULL, or a second addend of the incoming gradient, as for dwt_whiten_bwd
 * The workspace is sized by dwt_workspace_bytes for the same geometry.
 */
#define DWT_KIND_WHITEN 0
#define DWT_KIND_BN 1
typedef struct {
  const float *x;              /* the site's input [n_domains*N, HW, C], 16-byte aligned                         */
  float eps, momentum;         /* as in dwt_whiten_fwd / dwt_bn_fwd (momentum = batch norm's factor)             */
  int update_running;          /* fwd: apply the EMA to running_mean / running_cov (batch norm: running_var)     */
  float *const *running_mean;  /* [n_domains], may alias across domains; read only when update_running         */
  float *const *running_cov;
  const float *gamma, *beta;   /* [C], required                                                                  */
  float *save_mean, *save_w;   /* [n_domains, C], [n_domains, C/gs, gs, gs]: written by fwd, read by bwd        */
  float *dx;                   /* bwd: gradient of x                                                             */
  float *dgamma, *dbeta;       /* bwd: [C] (summed over domains), or both NULL                                    */
} dwt_tail_site;

DWT_API int dwt_tail2_fwd(int kind, const dwt_tail_site *sites, float *y, uint8_t *relu_mask, int64_t N, int64_t C,
                  int64_t HW, int group_size, int n_domains, void *workspace, size_t workspace_bytes,
                  dwt_stream_t stream);
DWT_API int dwt_tail2_bwd(int kind, const dwt_tail_site *sites, const float *dout, const float *dout2,
                  const uint8_t *relu_mask, float *dz, int64_t N, int64_t C, int64_t HW, int group_size,
                  int n_domains, void *workspace, size_t workspace_bytes, dwt_stream_t stream);

/*
 * Min-Entropy-Consensus loss, forward and both gradients in one launch.
 *   x, y [N, K] logits;  loss [1];  gx, gy [N, K] = d loss / d x, d loss / d y.
 * loss = mean_n min_k -(log_softmax(x) + log_softmax(y))[n,k] / 2
 */
DWT_API int dwt_mec_fwd_bwd(const float *x, const float *y, int64_t N, int64_t K, float *loss, float *gx,
                    float *gy, dwt_stream_t stream);

/*
 * The whole head loss of one training step in one launch (resnet50_dwt_mec_officehome.py:421-428):
 *   logits [3B, K] = source | target | target-aug, labels [B] (int64)
 *   total = mean_n NLL(log_softmax(source_n), label_n) + lambda * MEC(target, target-aug)
 * losses [3] = total, classification, lambda*MEC ;  grad [3B, K] = d total / d logits.
 * Labels as in F.nll_loss: -100 rows are ignored (dropped from the sum and the mean's denominator); any other label
 * outside [0, K) sets DWT_STATUS_BAD_LABEL in *status (device int, may be NULL: e.g. the workspace's status word)
 * and is dropped too -- never dereferenced.
 */
DWT_API int dwt_head_loss_fwd_bwd(const float *logits, const int64_t *labels, int64_t B, int64_t K, float lambda,
                          float *losses, float *grad, int *status, dwt_stream_t stream);

/*
 * Paired target augmentation (SURVEY.md §8f-4): both views the reference's loader derives from one image
 * (utils/folder.py:127-147 applying the two pipelines of resnet50_dwt_mec_officehome.py:526-542), in one launch.
 *   images      [B, src_h, src_w, 3] uint8, already resized (device)
 *   crop_plain  [B, 2] int32 (top, left) of the plain view's RandomCrop;  crop_aug  [B, 2] of the augmented view's
 *   flip        [B] uint8, RandomHorizontalFlip outcome;  affine [B, 6] float32, the 2x3 matrix that
 *               _random_affine_augmentation (:481-487) hands to cv2.warpAffine     (all device pointers)
 *   mean, stdv  HOST arrays of 3 (Normalize, :530)
 *   out_plain / out_aug  [B, 3, crop, crop] float32 (NCHW, layout 0) or [B, crop, crop, 3] (DWT_LAYOUT_NHWC); either
 *               may be NULL (the source domain has no augmented view).
 * The affine warp reproduces cv2.warpAffine (INTER_LINEAR, constant border 0) bit for bit; the reference's
 * GaussianBlur has kernel size 1 (sigma 0.1, :489-491) and is the identity.  Crop corners are clamped into the image.
 */
DWT_API int dwt_augment_pair(const uint8_t *images, int64_t B, int src_h, int src_w, int crop, const int32_t *crop_plain,
                     const int32_t *crop_aug, const uint8_t *flip, const float *affine, const float *mean,
                     const float *stdv, float *out_plain, float *out_aug, int layout, dwt_stream_t stream);

/*
 * Channels-last max-pool and its backward: the op between the stem whitening site and layer1
 * (nn.MaxPool2d(3, 2, 1), resnet50_dwt_mec_officehome.py:295,337-338).  Semantics = torch max_pool2d (dilation 1,
 * ceil_mode False) and its autograd, bit for bit including ties (first maximum in row-major window order) and NaN.
 *   flags  0 (fp32) or DWT_DTYPE_BF16 (x, y, dy, dx in bf16, 8-byte aligned; gradients summed in fp32, rounded once)
 *   x  [N, H, W, C] fp32 (torch.channels_last), C % 4 == 0;  y [N, OH, OW, C], OH = (H + 2*padding - kernel)/stride + 1
 *   argmax [N, OH, OW, C] uint8: window-local index kh*kernel + kw of the maximum (written by fwd, read by bwd)
 *   dy [N, OH, OW, C] -> dx [N, H, W, C] (every element written; no atomics, deterministic)
 */
DWT_API int dwt_maxpool_fwd(const float *x, float *y, uint8_t *argmax, int64_t N, int64_t H, int64_t W, int64_t C,
                    int kernel, int stride, int padding, int flags, dwt_stream_t stream);
DWT_API int dwt_maxpool_bwd(const float *dy, const uint8_t *argmax, float *dx, int64_t N, int64_t H, int64_t W, int64_t C,
                    int kernel, int stride, int padding, int flags, dwt_stream_t stream);

/*
 * Measurement hooks (used by bench.py; not part of the reference's surface).
 * dwt_launch_count: kernels launched by this library since it was loaded.
 * dwt_profile_begin/end: while enabled, every kernel launch is bracketed by CUDA events on
 * its own stream; dwt_profile_end waits for them and returns one entry per kernel family with
 * the launch count, the summed device time and the summed ALGORITHMIC bytes (DESIGN.md §4).
 */
typedef struct {
  char name[48];
  int64_t launches;
  double ms;
  double bytes;
} dwt_profile_entry;

DWT_API int64_t dwt_launch_count(void);
DWT_API void dwt_profile_begin(void);
DWT_API int dwt_profile_end(dwt_profile_entry *out, int max_entries);

#ifdef __cplusplus
}
#endif
#endif /* DWT_B200_H_ */

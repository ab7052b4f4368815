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
 *   dwt_bn_fwd/bwd   _BatchNorm.forward             utils/batch_norm.py:54-69
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
 * Tensor layout: activations are fp32, contiguous [n_domains * N, C, HW]
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

#define DWT_B200_ABI_VERSION 5
#define DWT_MAX_DOMAINS 4
#define DWT_MAX_GROUP_SIZE 64

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
 * default = [n_domains*N, C, HW] (NCHW); DWT_LAYOUT_NHWC = [n_domains*N, HW, C] (torch.channels_last), built for
 * group sizes 1, 2, 4 with C/4 a power of two (the layout cuDNN's tensor-core convolutions want: a
 * channels-last model needs no NCHW<->NHWC copies around its convolutions). */
#define DWT_LAYOUT_NHWC 0x100

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
 * calls issued on ONE stream.  Size for the largest call the caller will make. */
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
 * read from the forward's relu_mask and, when dresidual is not NULL, the masked gradient dout * (out > 0) -- the
 * gradient of the identity branch -- is written there in the same pass (resnet50_dwt_mec_officehome.py:239-240).
 * Without RESIDUAL pass relu_mask = dresidual = NULL.
 */
DWT_API int dwt_whiten_bwd(const float *x, const float *dout, const float *dout2, float *dx, int64_t N, int64_t C, int64_t HW,
                   int group_size, int n_domains, int mode, float eps, const float *save_mean,
                   const float *save_w, const float *gamma, const float *beta, const uint8_t *relu_mask,
                   float *dresidual, int epilogue, float *dgamma, float *dbeta, void *workspace,
                   size_t workspace_bytes, dwt_stream_t stream);

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
 *   x  [N, H, W, C] fp32 (torch.channels_last), C % 4 == 0;  y [N, OH, OW, C], OH = (H + 2*padding - kernel)/stride + 1
 *   argmax [N, OH, OW, C] uint8: window-local index kh*kernel + kw of the maximum (written by fwd, read by bwd)
 *   dy [N, OH, OW, C] -> dx [N, H, W, C] (every element written; no atomics, deterministic)
 */
DWT_API int dwt_maxpool_fwd(const float *x, float *y, uint8_t *argmax, int64_t N, int64_t H, int64_t W, int64_t C,
                    int kernel, int stride, int padding, dwt_stream_t stream);
DWT_API int dwt_maxpool_bwd(const float *dy, const uint8_t *argmax, float *dx, int64_t N, int64_t H, int64_t W, int64_t C,
                    int kernel, int stride, int padding, dwt_stream_t stream);

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

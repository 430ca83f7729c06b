/* pconv_b200.h -- C ABI of libpconv_b200.so: the H100 (sm_90a) partial-convolution hot path.
 *
 * The reference (yu45020/Text_Segmentation_Image_Inpainting) has NO native boundary: its hot
 * path is Python nn.Modules calling ATen (SURVEY 8b).  The drop-in boundary is therefore the
 * nn.Module surface mirrored in text_segmentation_image_inpainting_b200/models/, and THIS
 * header is the C ABI those modules' autograd Functions bind with ctypes.  Each entry point
 * cites the reference statement(s) it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless named h_*; no torch types cross this boundary;
 *  - activations are NHWC ("channels_last") contiguous, dtype PCB_F32 or PCB_BF16;
 *  - hole masks are uint8 planes [n, h, w] (1 = valid, 0 = hole), one plane per channel range;
 *  - every call enqueues on `stream` and returns immediately; nothing synchronises;
 *  - return value: 0 = ok, nonzero = error; pcb_last_error() gives the message (thread-local).
 */
#ifndef PCONV_B200_H_
#define PCONV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void *pcb_stream_t;          /* cudaStream_t */

enum { PCB_F32 = 0, PCB_BF16 = 1 };
enum { PCB_ACT_NONE = 0, PCB_ACT_RELU = 1, PCB_ACT_LEAKY = 2, PCB_ACT_RELU6 = 3 };
enum { PCB_MAX_PARTS = 8 };

/* One channel range of the (virtually concatenated, virtually nearest-upsampled) conv input.
 * Replaces: torch.cat of features and of masks (models/image_inpainting.py:183-185) and
 * DoubleUpSample (models/partial_convolution.py:229-231) as index math in the consumer. */
typedef struct {
    const void    *x;          /* first channel of this range inside an NHWC tensor, or NULL (backward-only calls) */
    const uint8_t *mask;       /* hole plane [n, h>>mask_up, w>>mask_up]; NULL = all valid            */
    int32_t c;                 /* channels in this range                                               */
    int32_t x_cstride;         /* channel count (pixel stride, in elements) of the tensor x lives in   */
    int32_t x_up;              /* log2 nearest-upsample factor of x      (0 or 1)                      */
    int32_t mask_up;           /* log2 nearest-upsample factor of mask   (0 or 1)                      */
} pcb_part;

typedef struct {
    int32_t n, h, w, cin;      /* logical conv input (after virtual upsample / concat)                 */
    int32_t cout, kh, kw;
    int32_t stride, pad_h, pad_w, dil;
    int32_t groups;
    int32_t ho, wo;            /* output size (caller computes; checked)                               */
    int32_t dtype;             /* PCB_F32 | PCB_BF16 : storage type of x, y, dy, dx and of w/wt         */
    int32_t same_holes;        /* PartialConv(same_holes=True): msum = cin * box(mask of part 0)        */
    int32_t no_guard;          /* PartialConvNoHoles: no zero guard, new mask all ones (may emit NaN)   */
    int32_t plain;             /* ordinary convolution (PartialConv1x1 / nn.Conv2d): renormaliser == 1   */
    int32_t force_generic;     /* never take the tensor-core path for this problem                      */
    int32_t nparts;
    pcb_part parts[PCB_MAX_PARTS];
} pcb_conv;

/* ---- library / device ------------------------------------------------------------------ */
const char *pcb_last_error(void);
int pcb_version(void);
/* Number of kernels this library has launched since load (for bench.py's gpu_launches). */
unsigned long long pcb_launch_count(void);
/* 1 if the wgmma tensor-core path would be used for this forward problem, else 0. */
int pcb_conv_uses_tensor_cores(const pcb_conv *c);

/* ---- partial convolution --------------------------------------------------------------- */

/* Scratch (bytes) the tensor-core path needs for forward / backward_weight (per-pixel tap-validity
 * bit masks); 0 when the generic path is taken.  Contents are not preserved between calls. */
size_t pcb_pconv_workspace(const pcb_conv *c);

/* Compute-dtype weight operands.  The tensor-core path wants the K axis padded to its 64-element block
 * structure (and a transposed copy for the data gradient); the generic path wants a plain KRSC cast.
 * pcb_conv_weight_layout gives the element counts (of c->dtype) of the two buffers (dgrad_elems may be 0);
 * pcb_conv_weight_prepare fills them from the fp32 master weight, physically [cout][kh][kw][cin/groups]
 * (= an OIHW nn.Conv2d weight in torch.channels_last memory format).                              */
void pcb_conv_weight_layout(const pcb_conv *c, size_t *fwd_elems, size_t *dgrad_elems);
int pcb_conv_weight_prepare(const pcb_conv *c, const float *w_master_krsc, void *w_fwd, void *w_dgrad, pcb_stream_t stream);
/* The same for buffers that pcb_conv_weight_prepare already filled for this very problem description: only the weight
 * entries are rewritten, the zero padding is left alone (no memsets).  For training loops that update the fp32 masters
 * every step (the reference's optimiser step, train loop of SURVEY 8d).                                          */
int pcb_conv_weight_refresh(const pcb_conv *c, const float *w_master_krsc, void *w_fwd, void *w_dgrad, pcb_stream_t stream);

/* PartialConv.forward / PartialConvNoHoles.forward (models/partial_convolution.py:49-80, :121-137):
 *   y = where(s==0, 0, conv(x*m; W)/s + b),  s = box-sum of the mask (all-ones mask_conv, :41-47,59-66),
 *   new_mask = (s != 0).
 * w_fwd  : from pcb_conv_weight_prepare
 * bias   : fp32 [cout] or NULL
 * y      : NHWC [n,ho,wo,y_cstride], y_cstride >= cout (channels [cout, y_cstride) are written as zeros)
 * msum   : fp32 [mg][n,ho,wo]  mask sums s (0 at holes); mg = 1, or groups when groups>1 && !same_holes
 * newmask: u8   [mg][n,ho,wo]
 * workspace : pcb_pconv_workspace(c) bytes (may be NULL when that is 0)                        */
int pcb_pconv_forward(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                      uint8_t *newmask, void *workspace, pcb_stream_t stream);
/* The same in two calls, for callers that run a network's mask chain ahead of its feature path on another stream
 * (mask updates never depend on features, partial_convolution.py:59-77): pcb_pconv_mask_pass computes what depends only
 * on the masks (msum, newmask and, in `workspace`, the tap-validity words the chosen kernel wants);
 * pcb_pconv_forward_premasked is the rest and must be ordered after it (same arguments as pcb_pconv_forward). */
int pcb_pconv_mask_pass(const pcb_conv *c, float *msum, uint8_t *newmask, void *workspace, pcb_stream_t stream);
int pcb_pconv_forward_premasked(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                      uint8_t *newmask, void *workspace, pcb_stream_t stream);
/* Forward with the STATISTICS PASS of the BatchNorm that follows the convolution (partial_convolution.py:193-197,
 * BaseModels.py:95-99) fused into the convolution epilogue: bn_sums[co] += sum over pixels of y[.., co], bn_sums[cout + co] +=
 * sum of y^2 (of the values as stored, holes contribute their zeros).  bn_sums = [2][cout] doubles, ZERO on entry; only for
 * problems with pcb_conv_fuses_bn_stats(c) == 1 (the tensor-core kernels); bn_sums NULL = plain forward.
 * mask_pass_done != 0: pcb_pconv_mask_pass already ran (see pcb_pconv_forward_premasked).                                    */
int pcb_conv_fuses_bn_stats(const pcb_conv *c);
int pcb_pconv_forward_bn(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                         uint8_t *newmask, void *workspace, int mask_pass_done, double *bn_sums, pcb_stream_t stream);

/* Backward of the renormalisation (autograd of partial_convolution.py:71-72):
 *   dc = dy * [s>0] / s          (NHWC [n,ho,wo,dc_cstride]; channels [cout, dc_cstride) zeroed)
 *   dbias[co] = sum dy*[s>0]     (fp32, optional, overwritten)                                 */
int pcb_pconv_renorm_backward(const pcb_conv *c, const void *dy, int dy_cstride, const float *msum, void *dc, int dc_cstride,
                              float *dbias, pcb_stream_t stream);

/* dx_p = (conv_transpose(dc; W) * m)[channels of part p]   (autograd of partial_convolution.py:51).
 * dx[p] : NHWC [n,h,w,dx_cstride[p]] at the conv-input resolution (a 2x-upsampled part still gets a full
 *         resolution gradient; reduce it with pcb_upsample2x_backward), or NULL when part p needs none.
 * parts[].mask are the INPUT masks (dx is zeroed at input holes); parts[].x is not read.      */
int pcb_pconv_backward_data(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_fwd, const void *w_dgrad,
                            void *const *dx, const int32_t *dx_cstride, pcb_stream_t stream);
/* 1 when pcb_pconv_backward_data computes the gradient of a 2x-UPSAMPLED source part (x_up == 1) directly at that source's own
 * (half) resolution -- dx[p] is then a [n, h/2, w/2, dx_cstride] buffer and no 2x2 reduction pass follows (sub-pixel path of the
 * tensor-core kernels and the kernel-to-row path of the RGB tails: image_inpainting.py:183-185 + partial_convolution.py:229-231
 * folded into the convolution).  0: dx[p] of
 * every part is a full-resolution [n, h, w, dx_cstride] buffer and the caller reduces 2x2 blocks itself. */
int pcb_conv_dgrad_at_source_resolution(const pcb_conv *c);

/* dw[co][r][s][ci] = sum_pixels dc[p][co] * (x*m)[p@tap][ci]   (fp32 KRSC, logical/unpadded, overwritten).
 * workspace: pcb_pconv_workspace(c) bytes (may be NULL when that is 0).                         */
int pcb_pconv_backward_weight(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream);
/* same, ACCUMULATING into dw (dw is not zeroed first): for a gradient buffer the caller already zeroed -- e.g. a flat gradient arena
 * cleared once per step -- or for gradient accumulation over micro-batches. */
int pcb_pconv_backward_weight_acc(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream);

/* Debug aid: after a device synchronise, returns the (sticky) pipeline-timeout code set by a tensor-core
 * kernel whose mbarrier wait expired (0 = none) and clears it. */
int pcb_debug_pipeline_status(int *code);

/* ---- masks ----------------------------------------------------------------------------- */
/* dense fp32 NCHW mask (the reference API, partial_convolution.py:50) -> c u8 planes [c][n,h,w]. */
int pcb_mask_planes_from_dense(const float *mask_nchw, int n, int c, int h, int w, uint8_t *planes, pcb_stream_t stream);
/* plane (optionally 2x nearest upsampled) -> dense fp32 NCHW channels [c0, c0+c) of an [n,ctot,h,w] tensor. */
int pcb_mask_plane_to_dense(const uint8_t *plane, int n, int h, int w, int up, float *dst_nchw, int ctot, int c0, int c,
                            pcb_stream_t stream);

/* ---- BatchNorm2d (+activation) --------------------------------------------------------- */
/* nn.BatchNorm2d + act as built by PartialActivatedBN (partial_convolution.py:193-201) and
 * Conv_block (BaseModels.py:95-99).  x/y NHWC [count, c].                                     */
int pcb_bn_stats(const void *x, int dtype, long long count, int c, double *sum, double *sqsum, pcb_stream_t stream);
/* accumulate-only statistics: sums = [2][c] doubles (sum | sum of squares) that the CALLER zeroed -- e.g. a slice of a per-step
 * zero arena, so a training step issues one memset instead of one per BatchNorm.                                              */
int pcb_bn_stats_acc(const void *x, int dtype, long long count, int c, double *sums, pcb_stream_t stream);
/* Training-mode forward of nn.BatchNorm2d (+act, +residual) from COMPLETE sums in one launch: mean / biased var / invstd,
 * running-statistics + num_batches_tracked update (unbiased var, momentum), y = act(x*scale+shift) [+ residual].
 * The sums come from pcb_bn_stats_acc or from the producing convolution's epilogue (pcb_pconv_forward_bn).
 * coef: [4][c] floats written for the backward: scale | shift | mean | invstd.  c % 8 == 0, c <= 2048.                      */
int pcb_bn_forward_fused(const void *x, int dtype, long long count, int c, const double *sums, const float *gamma,
                         const float *beta, float *running_mean, float *running_var, long long *num_batches_tracked,
                         float momentum, float eps, int act, float slope, const void *residual, void *y, float *coef,
                         pcb_stream_t stream);
/* training: mean/var from (sum,sqsum); updates running stats (unbiased var, momentum) and
 * num_batches_tracked; writes scale = gamma*invstd, shift = beta - mean*scale, save_mean, save_invstd.
 * eval (training==0): scale/shift from the running stats; sum/sqsum ignored.                  */
int pcb_bn_finalize(const double *sum, const double *sqsum, long long count, int c, const float *gamma,
                    const float *beta, float *running_mean, float *running_var, long long *num_batches_tracked,
                    float momentum, float eps, int training, float *scale, float *shift, float *save_mean,
                    float *save_invstd, pcb_stream_t stream);
/* y = act(x*scale + shift) (scale/shift NULL = identity => plain activation, PartialActivation :204-211);
 * residual (optional, same shape) is added AFTER the activation (DoublePartialResidual x2 + x1,
 * image_inpainting.py:216; PartialInvertedResidual x + out, MobileNetV2.py:186-187).          */
int pcb_bn_act_forward(const void *x, int dtype, long long count, int c, const float *scale, const float *shift,
                       int act, float slope, const void *residual, void *y, pcb_stream_t stream);
/* reductions for the BN backward: sum_g[c] += sum gz, sum_gx[c] += sum gz * xhat, with
 * gz = gy * act'(x*scale+shift), xhat = (x - mean) * invstd.                                   */
int pcb_bn_act_backward_reduce(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                               const float *shift, const float *mean, const float *invstd, int act, float slope,
                               double *sum_g, double *sum_gx, pcb_stream_t stream);
/* same without the memset: sums = [2][c] doubles (sum gz | sum gz*xhat) zeroed by the caller; c % 8 == 0, c <= 2048 */
int pcb_bn_act_backward_reduce_acc(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                   const float *shift, const float *mean, const float *invstd, int act, float slope,
                                   double *sums, pcb_stream_t stream);
/* Whole training-mode backward of a SMALL tensor (count <= ~16 K rows) in ONE launch: reduction + apply + dgamma/dbeta
 * [+ division by the producing partial convolution's mask sums when msum != NULL].  coef = the [4][c] block of
 * pcb_bn_forward_fused (scale | shift | mean | invstd).  c % 8 == 0. */
int pcb_bn_act_backward_small(const void *gy, const void *x, int dtype, long long count, int c, const float *coef, int act,
                              float slope, const float *msum, void *dx, float *dgamma, float *dbeta, pcb_stream_t stream);
/* dx = scale * (gz - sum_g/count - xhat * sum_gx/count)  (training) or scale * gz (eval / no BN: scale NULL => gz).
 * dgamma = sum_gx, dbeta = sum_g (fp32, optional).                                             */
int pcb_bn_act_backward_apply(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                              const float *shift, const float *mean, const float *invstd, int act, float slope,
                              const double *sum_g, const double *sum_gx, int training, void *dx, float *dgamma,
                              float *dbeta, pcb_stream_t stream);
/* The same with the renormalisation backward of the partial convolution that produced x fused in
 * (partial_convolution.py:71-77 under autograd): dc = dx / msum, 0 where msum == 0 -- one pass instead of
 * pcb_bn_act_backward_apply + pcb_pconv_renorm_backward.  Only valid when that convolution has no bias, one mask
 * group, the zero guard (not PartialConvNoHoles) and c % 8 == 0; msum is the [count] fp32 plane pcb_pconv_forward wrote. */
int pcb_bn_act_backward_apply_renorm(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                     const float *shift, const float *mean, const float *invstd, int act, float slope,
                                     const double *sum_g, const double *sum_gx, int training, const float *msum, void *dc,
                                     float *dgamma, float *dbeta, pcb_stream_t stream);

/* ---- resampling / glue ------------------------------------------------------------------ */
/* nn.Upsample(scale_factor=2, mode='nearest') on NHWC (DoubleUpSample, partial_convolution.py:224-231). */
int pcb_upsample2x_forward(const void *x, int dtype, int n, int h, int w, int c, void *y, pcb_stream_t stream);
int pcb_upsample2x_backward(const void *gy, int dtype, int n, int h, int w, int c, void *gx, pcb_stream_t stream);
/* channel concat of up to PCB_MAX_PARTS NHWC tensors (each optionally 2x nearest-upsampled) into y[n,h,w,sum c]:
 * torch.cat([x_up, skip], 1) of image_inpainting.py:184 fused with the upsample before it.     */
int pcb_concat_forward(const pcb_part *parts, int nparts, int dtype, int n, int h, int w, void *y, pcb_stream_t stream);
/* backward: splits gy[n,h,w,ctot] into per-part gradients (2x2-summed for upsampled parts).
 * gx[i] : NHWC [n, h>>up_i, w>>up_i, c_i] dense.                                               */
int pcb_concat_backward(const void *gy, const int32_t *c, const int32_t *up, int nparts, int dtype, int n, int h,
                        int w, void *const *gx, pcb_stream_t stream);

/* ---- segmentation-network glue (models/text_segmentation.py, models/common.py) ------------------- */
/* nn.AvgPool2d(k, stride, pad) with count_include_pad=True on NHWC (text_segmentation.py:33,66-67; ASP, common.py:62-68). */
int pcb_avgpool_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, int k, int stride, int pad, pcb_stream_t stream);
int pcb_avgpool_backward(const void *gy, void *gx, int dtype, int n, int h, int w, int c, int k, int stride, int pad, pcb_stream_t stream);
/* F.interpolate(mode='bilinear', align_corners=False, scale_factor=scale) on NHWC (text_segmentation.py:54,76,109,113);
 * h, w are the INPUT (low-resolution) sizes. */
int pcb_bilinear_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, int scale, pcb_stream_t stream);
int pcb_bilinear_backward(const void *gy, void *gx, int dtype, int n, int h, int w, int c, int scale, pcb_stream_t stream);
/* nn.AdaptiveAvgPool2d(1) -> fp32 [n][c] (scSE squeeze, common.py:19,35) and its backward (broadcast of g/hw). */
int pcb_gap_forward(const void *x, int dtype, int n, long long hw, int c, float *out, pcb_stream_t stream);
int pcb_gap_backward(const float *g, void *dx, int dtype, int n, long long hw, int c, int accumulate, pcb_stream_t stream);
/* scSE gate (common.py:37-43): sse = sigmoid(<x[p,:], ws>), y = x*cse[n,:] + x*sse; sse_out fp32 [n*hw] is saved for backward.
 * backward: dx, dcse fp32 [n][c], dws fp32 [c] (both overwritten). */
int pcb_scse_forward(const void *x, const float *cse, const float *ws, void *y, float *sse_out, int dtype, int n, long long hw, int c,
                     pcb_stream_t stream);
int pcb_scse_backward(const void *gy, const void *x, const float *cse, const float *ws, const float *sse, void *dx, float *dcse,
                      float *dws, int dtype, int n, long long hw, int c, pcb_stream_t stream);

/* ---- loss / optimiser used by the benchmark step (SURVEY 8d: loss = out.abs().mean()) ------ */
int pcb_l1_mean_forward(const void *x, int dtype, long long numel, float *loss /* device scalar, overwritten */,
                        double *scratch /* device, 1 double */, pcb_stream_t stream);
int pcb_l1_mean_backward(const void *x, int dtype, long long numel, float gscale, void *gx, pcb_stream_t stream);
/* fused SGD + momentum + Nesterov + weight decay over one flat fp32 tensor (checkpoints/ReadME.md:4 recipe). */
int pcb_sgd_step(float *param, const float *grad, float *momentum_buf, long long numel, float lr, float momentum,
                 float weight_decay, int nesterov, int first_step, pcb_stream_t stream);
/* same, with the gradient multiplied by `grad_scale` first: data-parallel training all-reduces the SUM of the per-rank gradient
   arenas and folds the 1/world of the mean in here instead of a separate pass over the arena. */
int pcb_sgd_step_scaled(float *param, const float *grad, float *momentum_buf, long long numel, float lr, float momentum,
                        float weight_decay, int nesterov, int first_step, float grad_scale, pcb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PCONV_B200_H_ */

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
 * y      : NHWC [n,ho,wo,y_cstride], y_cstride >= cout (channels [cout, rup(cout, 8)) are written as zeros; channels past
 *          that are not outputs and may be left untouched)
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
/* Inference forward with the EVAL-MODE BatchNorm and the activation that follow the convolution applied in its epilogue
 * (partial_convolution.py:193-201 and BaseModels.py:95-99 with the BatchNorm in eval mode): with v = the value
 * pcb_pconv_forward would store (0 at holes),
 *   y = act(v * scale[co] + shift[co])      rounded to the storage type once,
 * so hole pixels hold act(shift[co]) -- the reference's BatchNorm runs over the zeros the partial convolution wrote.
 * Channels [cout, rup(cout, 8)) are zeros.  scale / shift: fp32 [cout] from pcb_bn_finalize(training = 0), or both NULL for an
 * activation alone ([PartialConv, PartialActivation] blocks).  act: PCB_ACT_*, slope: LeakyReLU's negative slope.
 * Only for problems with pcb_conv_fuses_affine_act(c) == 1 (the tensor-core kernels other than the small-Cout ones, and the
 * depthwise 3x3 kernels -- the problems pcb_conv_fuses_bn_stats accepts); others are rejected.  mask_pass_done: see pcb_pconv_forward_premasked.                                                                */
int pcb_conv_fuses_affine_act(const pcb_conv *c);
int pcb_pconv_forward_affine_act(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                                 uint8_t *newmask, void *workspace, int mask_pass_done, const float *scale, const float *shift,
                                 int act, float slope, pcb_stream_t stream);

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

/* The data gradient of a layer whose input came out of an in-place ReLU (the VGG16 blocks of loss.py:244-260), with that
 * ReLU's backward applied in the kernel's epilogue: dx = 0 where relu_x <= 0 (torch's threshold_backward), otherwise what
 * pcb_pconv_backward_data stores.  relu_x: the layer's input (bf16 NHWC, channel stride relu_cstride, 16-byte aligned); one part,
 * dx[n,h,w,dx_cstride].  Only for problems with pcb_conv_dgrad_fuses_relu(c) == 1 (bf16, stride 1, the TMA-fed kernel). */
int pcb_conv_dgrad_fuses_relu(const pcb_conv *c);
int pcb_pconv_backward_data_relu(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_dgrad, void *dx, int dx_cstride,
                                 const void *relu_x, int relu_cstride, pcb_stream_t stream);

/* dw[co][r][s][ci] = sum_pixels dc[p][co] * (x*m)[p@tap][ci]   (fp32 KRSC, logical/unpadded, overwritten).
 * workspace: pcb_pconv_workspace(c) bytes (may be NULL when that is 0).                         */
int pcb_pconv_backward_weight(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream);
/* same, ACCUMULATING into dw (dw is not zeroed first): for a gradient buffer the caller already zeroed -- e.g. a flat gradient arena
 * cleared once per step -- or for gradient accumulation over micro-batches. */
int pcb_pconv_backward_weight_acc(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream);

/* Debug aid: after a device synchronise, returns the (sticky) pipeline-timeout code set by a tensor-core
 * kernel whose mbarrier wait expired (0 = none) and clears it. */
int pcb_debug_pipeline_status(int *code);
/* Debug aid (host only, nothing is launched): the kernel family each direction of this problem runs on, as PCB_ROUTE_* codes in
 * routes[0..2] = forward, data gradient, weight gradient.  GENERIC: conv_generic.cu; DEPTHWISE: dwconv.cu; the tensor-core routes:
 * STEM (space-to-depth 4x4 problem, conv_stem.cu), K2R (kernel-to-row RGB tail, conv_k2r.cu), SMALLCO (mma.sync, cout <= 8,
 * conv_smallco.cu), TMA (TMA-fed wgmma), TMA_S2 (the stride-2 data gradient as four stride-1 parity classes), GATHER (cp.async-fed
 * wgmma); NONE: the direction is refused (the data gradient of a row-packed layer, which its callers run with force_generic). */
enum { PCB_ROUTE_NONE = 0, PCB_ROUTE_GENERIC = 1, PCB_ROUTE_DEPTHWISE = 2, PCB_ROUTE_STEM = 3, PCB_ROUTE_K2R = 4,
       PCB_ROUTE_SMALLCO = 5, PCB_ROUTE_TMA = 6, PCB_ROUTE_TMA_S2 = 7, PCB_ROUTE_GATHER = 8 };
int pcb_debug_conv_routes(const pcb_conv *c, int32_t routes[3]);

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
/* Post-processing of the text-segmentation logits in one launch (Examples/demo_segmentation.py:33-36, Dataloader.py:308-316):
 *   b   = MaxPool2d(3, stride 1, pad 1)(sigmoid(x) > 0.5)            over the whole [h, w] map (x: channel 0 of an NHWC tensor
 *                                                                      with pixel stride `cstride`, PCB_F32 or PCB_BF16),
 *   out = upsample_bilinear2d(b[:h_valid, :w_valid], (oh, ow), align_corners=False) > 0     (the unpad, then the resize).
 * out: uint8 [n, oh, ow], 1 / 0.  Exact: the resize sums {0, 1} values with non-negative weights, so the kernel tests the taps
 * with positive weight; the threshold is 1 / (1 + expf(-x)) > 0.5 in fp32.                                                     */
int pcb_seg_mask_postprocess(const void *logits, int dtype, int n, int h, int w, int cstride, int h_valid, int w_valid, int oh,
                             int ow, uint8_t *out, pcb_stream_t stream);

/* ---- text removal (engine.TextRemovalStep): the glue between segmentation, mask and inpainting ---------------------------
 * `page`: fp32 NCHW [n, 3, h, w], contiguous, device memory.
 *
 * EvaluateSet's page resize (Dataloader.py:290-291): out fp32 NCHW [n, 3, rh, rw] =
 * to_tensor(to_pil_image(page[i]).resize((rw, rh), Image.BICUBIC)) per image.  Each byte is mul(255) in fp32, clamped to
 * [0, 255] (NaN to 0) and truncated, as to_pil_image makes it; then Pillow's two integer passes (horizontal first, clipped
 * uint8 between them, 22-bit weights) and / 255.  At most a 16x reduction per axis (h <= 16 rh, w <= 16 rw).  `workspace`:
 * device memory of pcb_page_resize_workspace(n, h, w, rh, rw) bytes (0 for out-of-range sizes), 256-byte aligned; three
 * launches, no host synchronisation. */
size_t pcb_page_resize_workspace(int n, int h, int w, int rh, int rw);
int pcb_page_resize_bicubic(const float *page, int n, int h, int w, int rh, int rw, void *workspace, float *out, pcb_stream_t stream);
/* The segmentation input (EvaluateSet, Dataloader.py:271-273, 296-303): per pixel of the [hs, ws] grid (hs >= h, ws >= w),
 * (page - mean) / std in fp32 (sub, then div, each rounded; `norm`: HOST pointer to mean[3], std[3], or NULL to skip it),
 * rounded once to `dtype`, zero outside the page.  out: [n, hs, ws, 8] NHWC (channels 3..7 zero), every element written. */
int pcb_removal_seg_input(const float *page, int n, int h, int w, const float *norm, int hs, int ws, void *out, int dtype,
                          pcb_stream_t stream);
/* The U-Net's input from the demo's text mask (uint8 [n, h, w], nonzero = text): the mask as a {0, 255} image, > 0.4 * 255,
 * cv2.dilate with a 10x10 kernel (anchor 5: rows and columns -5 .. +4, pixels outside the page ignored) (Dataloader.py:120-121),
 * then on the [hu, wu] grid (hu >= h, wu >= w): valid uint8 [n, hu, wu] = 1 - hole and corrupted [n, hu, wu, 8] NHWC in
 * `dtype` = page * valid in fp32 rounded once (:128-131; channels 3..7 zero).  Outside the page: valid 0, corrupted 0. */
int pcb_removal_holes(const uint8_t *text_mask, const float *page, int n, int h, int w, int hu, int wu, uint8_t *valid,
                      void *corrupted, int dtype, pcb_stream_t stream);
/* The composite (loss.py:196, comp_img) cropped to the page: out fp32 NCHW [n, 3, h, w] = valid ? page : fill, where `fill` is
 * the U-Net output on the [hu, wu] grid, NHWC with pixel stride `cstride` (channels 0..2 read) in `dtype`, and `valid` the
 * plane pcb_removal_holes wrote. */
int pcb_removal_composite(const void *fill, int dtype, int cstride, const float *page, const uint8_t *valid, int n, int h, int w,
                          int hu, int wu, float *out, pcb_stream_t stream);
/* The segmentation demo's region image (Examples/demo_segmentation.py:17-25, 40-45, draw_bounding_box(page, mask, threshold)):
 * out uint8 [n, h, w, 3] = np.array(to_pil_image(page[i])) with the convex hull of every outer contour of the text mask (uint8
 * [n, 1, h, w], nonzero = text) whose cv2.contourArea exceeds `area_threshold` filled as cv2.drawContours(..., -1) fills it,
 * in RGB (50, 128, 30).  Computed from the regions of the mask (DESIGN 4.14): union-find labelling, windowed areas, hulls of
 * the row extents, fillPoly's LINE_8 spans.  `workspace`: device memory of pcb_text_regions_workspace(n, h, w) bytes (0 for
 * out-of-range sizes: (h + 1) * (w + 1) < 2^31, n <= 65535), 256-byte aligned; eleven launches whose grids depend on (n, h, w)
 * only, no host synchronisation (capturable).  Every output byte is written. */
size_t pcb_text_regions_workspace(int n, int h, int w);
int pcb_text_region_hulls(const uint8_t *text_mask, const float *page, int n, int h, int w, double area_threshold, void *workspace,
                          uint8_t *out, pcb_stream_t stream);

/* ---- inpainting training data (ImageInpaintingData.process_images, Dataloader.py:110-162) -------------------------------
 * One decoded source per image: RGB uint8 [h][rgb_stride] (3 bytes per pixel) and the text mask uint8 [h][mask_stride]. */
typedef struct {
    const uint8_t *rgb;
    const uint8_t *mask;
    int32_t h, w, rgb_stride, mask_stride;
} pcb_inpaint_src;
/* What one image draws: the crop box (RandomResizedCrop.get_params: top i, left j, height h, width w), the RandomGrayscale flag
 * and random_masks' strokes in output pixels (lines x0, y0, x1, y1, width; ellipses x0, y0, x1, y1 with inclusive corners). */
typedef struct {
    int32_t top, left, height, width;
    int32_t gray;
    int32_t nlines, nellipses;
    int32_t lines[5][5];
    int32_t ellipses[5][4];
} pcb_inpaint_params;
/* Host-side check of a staged batch (h_srcs, h_params: HOST copies; h_params may be NULL): 1..cap_n images, each within the
 * cap_h x cap_w capacity, row strides large enough, crop boxes inside their sources, stroke counts 0..5.  The capacity may be
 * at most 8x the output size `out`. */
int pcb_inpaint_validate(const pcb_inpaint_src *h_srcs, const pcb_inpaint_params *h_params, int n, int cap_n, int cap_h, int cap_w,
                         int out);
/* Draw the parameters of n <= 1024 images on the device (Philox4x32-10, key = rng[0], counter = (slot, image, rng[1])) and
 * advance rng[1]: RandomResizedCrop.get_params(scale=(0.5, 2), ratio=(3/4, 4/3)), RandomGrayscale(0.4) and, if `strokes`,
 * random_masks(size=out, offset=10).  srcs, rng, params: device memory. */
int pcb_inpaint_sample(const pcb_inpaint_src *srcs, int n, int out, int strokes, uint64_t *rng, pcb_inpaint_params *params,
                       pcb_stream_t stream);
/* process_images for a batch from device-resident sources and parameters, two launches: Pillow-exact bicubic crop + resize of
 * image and text mask, the strokes (if `strokes`), mask > 0.4 * 255, cv2.dilate(10x10), the grayscale flag, ToTensor and
 * clean * (1 - mask).  tmp: uint8 [n][cap_h][out][4] scratch.  Outputs: corrupted [n][out][out][8] NHWC in `dtype` (channels
 * 3..7 zero), mask_plane uint8 [n][out][out] (1 = valid), clean fp32 [n][3][out][out].  Grids depend on n, cap_h and out only. */
int pcb_inpaint_prepare(const pcb_inpaint_src *srcs, const pcb_inpaint_params *params, int n, int cap_h, int cap_w, int out,
                        int strokes, uint8_t *tmp, void *corrupted, int dtype, uint8_t *mask_plane, float *clean, pcb_stream_t stream);

/* ---- inpainting data from raw/clean page pairs (TestDataset.process_images + get_mask, Dataloader.py:201-222) -------------
 * One decoded pair per image: the raw page and its text-cleaned copy, RGB uint8 [h][stride] each (3 bytes per pixel), the same
 * size (the crop box is drawn on raw and applied to both).  32 bytes with the layout of pcb_inpaint_src. */
typedef struct {
    const uint8_t *raw;
    const uint8_t *clean;
    int32_t h, w, raw_stride, clean_stride;
} pcb_inpaint_pair_src;
/* pcb_inpaint_validate for a staged pair batch; explicit parameters must also have gray == 0 (no RandomGrayscale). */
int pcb_inpaint_pair_validate(const pcb_inpaint_pair_src *h_srcs, const pcb_inpaint_params *h_params, int n, int cap_n, int cap_h,
                              int cap_w, int out);
/* pcb_inpaint_sample's draws for pair sources: the same Philox slots, so the same crop boxes and strokes for the same seed,
 * counter and sizes, with the grayscale flag always 0. */
int pcb_inpaint_pair_sample(const pcb_inpaint_pair_src *srcs, int n, int out, int strokes, uint64_t *rng, pcb_inpaint_params *params,
                            pcb_stream_t stream);
/* TestDataset.process_images for a batch, two launches: Pillow-exact bicubic crop + resize of raw and clean, Image.convert("L")
 * of both, |L_raw - L_clean| (ImageChops.difference), the strokes drawn at 255 on the difference (if `strokes`), > 0.4 * 255,
 * cv2.dilate(10x10), ToTensor and clean * (1 - mask).  tmp: uint8 [n][cap_h][out][8] scratch (raw RGB0 | clean RGB0: twice
 * pcb_inpaint_prepare's, 134 MB at n = 8, cap_h = 4096, out = 512).  Outputs as pcb_inpaint_prepare's; grids depend on n,
 * cap_h and out only. */
int pcb_inpaint_pair_prepare(const pcb_inpaint_pair_src *srcs, const pcb_inpaint_params *params, int n, int cap_h, int cap_w, int out,
                             int strokes, uint8_t *tmp, void *corrupted, int dtype, uint8_t *mask_plane, float *clean, pcb_stream_t stream);

/* ---- segmentation training data (TextSegmentationData.process_images, Dataloader.py:66-74) -------------------------------
 * One decoded source per image: the gray (`L`) page uint8 [h][page_stride] and its text mask uint8 [h][mask_stride]. */
typedef struct {
    const uint8_t *page;
    const uint8_t *mask;
    int32_t h, w, page_stride, mask_stride;
} pcb_seg_src;
/* What one image draws: the crop box (RandomResizedCrop.get_params(scale=(0.1, 2)): top i, left j, height h, width w), whether
 * ColorJitter applies brightness before contrast, and the two factors (float32, as Pillow's blend uses them). */
typedef struct {
    int32_t top, left, height, width;
    int32_t brightness_first;
    float brightness, contrast;
    int32_t reserved;
} pcb_seg_params;
/* Host-side check of a staged batch (h_srcs, h_params: HOST copies; h_params may be NULL): 1..cap_n images, each within the
 * cap_h x cap_w capacity, row strides large enough, crop boxes inside their sources and at most 8x the output size `out`,
 * order flag 0 / 1, finite non-negative factors. */
int pcb_seg_validate(const pcb_seg_src *h_srcs, const pcb_seg_params *h_params, int n, int cap_n, int cap_h, int cap_w, int out);
/* Draw the parameters of n <= 1024 images on the device (Philox4x32-10, key = rng[0], counter = (slot, image, rng[1])) and
 * advance rng[1]: RandomResizedCrop.get_params(scale=(0.1, 2), ratio=(3/4, 4/3)), the brightness / contrast order of
 * ColorJitter's randperm(4) and both factors on [0.8, 1.2].  srcs, rng, params: device memory. */
int pcb_seg_sample(const pcb_seg_src *srcs, int n, uint64_t *rng, pcb_seg_params *params, pcb_stream_t stream);
/* process_images for a batch, three launches: Pillow-exact bicubic crop + resize of page and mask, the page histogram,
 * ColorJitter's brightness and contrast blends in the drawn order (contrast about int(mean + 0.5) of the image it is applied
 * to), ToTensor and, if h_norm (host [6]: mean[3], std[3]) is given, Normalize.  tmp: uint8 [n][cap_h][out][2], planes: uint8
 * [2][n][out][out], hist: int32 [n][256] (scratch).  Outputs: x [n][out][out][8] NHWC in `dtype`, the page in channels 0..2,
 * channels 3..7 zero; target fp32 [n][out][out] (the mask's ToTensor).  Grids depend on n, cap_h and out only. */
int pcb_seg_prepare(const pcb_seg_src *srcs, const pcb_seg_params *params, int n, int cap_h, int cap_w, int out, uint8_t *tmp,
                    uint8_t *planes, int *hist, const float *h_norm, void *x, int dtype, float *target, pcb_stream_t stream);

/* ---- inpainting loss (InpaintingLoss, loss.py:185-307) ---------------------------------------------------------------
 * The VGG16 convolutions and the Gram products run on the convolution entry points above; these are the rest.  Reductions
 * ADD into caller-zeroed fp64 sums; nothing synchronises.  Image strides are in elements (n, c, h, w order), so fp32 NCHW and
 * NHWC (padded) views are both accepted.
 *
 * Pixel terms + VGG input batch, one thread per pixel: comp = m ? raw : output for the {0,1} plane m (= mask*raw +
 * (1-mask)*output, loss.py:196); sums[0] += |output-origin| where valid, sums[1] += |output-origin| in holes, sums[2] / sums[3]
 * += |horizontal| / |vertical| differences of comp (loss.py:303-307); vgg_in = [3n][h][w][8] in `dtype`: comp | output | origin,
 * channels 3..7 zero.  raw, origin: fp32 NCHW [n,3,h,w]; output: `out_dtype`, 3 channels through out_strides (host [4]). */
int pcb_inpaint_loss_pixel_forward(const float *raw, const float *origin, const void *output, int out_dtype, const long long *out_strides,
                                   const uint8_t *plane, int n, int h, int w, void *vgg_in, int dtype, double *sums, pcb_stream_t stream);
/* d loss / d output = gs * (coef[0] * m + coef[1] * (1-m)) * sign(output - origin) + (1-m) * (gs * d tv / d comp + dvgg_in[comp])
 * + dvgg_in[output], gs = *gscale (device).  coef (host [4]): valid, hole, horizontal-TV and vertical-TV weights over their element
 * counts.  dvgg_in: [2n][h][w][8] in `dtype` (comp | output) or NULL.  grad: `out_dtype`, through grad_strides (host [4]). */
int pcb_inpaint_loss_pixel_backward(const float *raw, const float *origin, const void *output, int out_dtype, const long long *out_strides,
                                    const uint8_t *plane, int n, int h, int w, const void *dvgg_in, int dtype, const float *coef,
                                    const float *gscale, void *grad, const long long *grad_strides, pcb_stream_t stream);
/* nn.MaxPool2d(2, 2) on NHWC [n,h,w,c] (h, w even, c % 8 == 0), torch's rule: a tap replaces the running maximum when it is
 * greater or NaN (row-major order), so ties go to the first maximum and NaN propagates.  The backward recomputes the window
 * maximum from x and writes every element of gx: gy at the maximum, 0 elsewhere; relu_mask != 0 also applies the backward of the
 * in-place ReLU that produced x (0 where x <= 0). */
int pcb_maxpool2x2_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, pcb_stream_t stream);
int pcb_maxpool2x2_backward(const void *gy, const void *x, void *gx, int dtype, int n, int h, int w, int c, int relu_mask, pcb_stream_t stream);
/* f: NHWC features of 3n images (comp | output | origin), hw pixels x c channels each (c % 8 == 0):
 * sums[0] += sum |f_comp - f_origin|, sums[1] += sum |f_output - f_origin|   (the perceptual L1 sums, loss.py:211-212). */
int pcb_feature_l1_forward(const void *f, int dtype, int n, long long hw, int c, double *sums, pcb_stream_t stream);
/* df (2n images comp | output) = gs * (l1_coef * sign(f - f_origin) + gram_coef * g_gram) + g_next; g_gram, g_next: [2n][hw][c]
 * or NULL. */
int pcb_feature_loss_backward(const void *f, int dtype, int n, long long hw, int c, const void *g_next, const void *g_gram, float l1_coef,
                              float gram_coef, const float *gscale, void *df, pcb_stream_t stream);
/* gram: fp32 [3n][c][c] unnormalised products F F^T (comp | output | origin); G = gram / norm (loss.py:294-300):
 * sums[0] += sum |G_comp - G_origin|, sums[1] += sum |G_output - G_origin|. */
int pcb_gram_l1_forward(const float *gram, int n, int c, float norm, double *sums, pcb_stream_t stream);
/* t: fp32 [2n][c][c] = S + S^T, S = sign(G_i - G_origin) for the images comp | output: the weight of the Gram backward
 * dF = F (S + S^T) k (a 1x1 convolution; integer-valued, so exact in bf16). */
int pcb_gram_sign_sym(const float *gram, int n, int c, float norm, float *t, pcb_stream_t stream);
/* Data gradient of a 3x3 / pad 1 / stride 1 convolution with 3 input channels (VGG16 conv1_1) in kernel-to-row form:
 * pcb_k2r_image_weight writes the fp32 [32][cout] weight of the 1x1 problem Z[p][tap*3 + ci] = sum_co dc[p][co] W[co][ci][tap]
 * (W: fp32 OIHW [cout][3][3][3]; rows 27..31 zero), which the caller lays out with pcb_conv_weight_prepare and runs with
 * pcb_pconv_forward (1x1, cout -> 32, plain) into z [n][h][w][32];  pcb_k2r_image_dgrad then sums the taps:
 * dx[q][ci] = sum_tap z[q - tap + 1][tap*3 + ci], dx: [n][h][w][8] in `dtype` (channels 3..7 zero). */
int pcb_k2r_image_weight(const float *w_oihw, int cout, float *wz, pcb_stream_t stream);
int pcb_k2r_image_dgrad(const void *z, int dtype, int n, int h, int w, void *dx, pcb_stream_t stream);
/* sums: the 16 fp64 sums [valid, hole, tv_h, tv_v, perceptual comp|output per stage (3x2), style comp|output per stage (3x2)];
 * h_inv (host [16]): their normalisers.  terms (fp32 [5], unweighted): valid, hole, tv, perceptual, style;
 * loss = 1 valid + 6 hole + 0.1 tv + 0.05 perceptual + 120 style (loss.py:223-224). */
int pcb_inpaint_loss_finalize(const double *sums, const double *h_inv, float *loss, float *terms, pcb_stream_t stream);

/* ---- segmentation losses (BinaryFocalLoss, SoftBootstrapCrossEntropy, loss.py:58-121) ------------------------------------
 * x: [n, 1, h, w] logits in `dtype` through x_strides (host [4], elements, n c h w order): NCHW or a channel-padded NHWC view.
 * target: fp32 [n][h][w].  loss PCB_SEG_FOCAL (p0 = gamma, reduction PCB_SEG_MEAN only) or PCB_SEG_BOOTSTRAP (p0 = beta,
 * one_minus_beta = 1 - beta).  Forward: out = the fp32 loss (a scalar, or [n*h*w] for PCB_SEG_NONE), reduced deterministically
 * through `partials` (device, pcb_seg_loss_partials(n*h*w) doubles) and `counter` (device, one zero-initialised uint32 per
 * concurrent call; the kernel leaves it zero).  Backward: dx = gout * d loss / d x in `dtype` through dx_strides; gout (device):
 * the upstream gradient, a scalar or [n*h*w] for PCB_SEG_NONE. */
enum { PCB_SEG_FOCAL = 0, PCB_SEG_BOOTSTRAP = 1 };
enum { PCB_SEG_NONE = 0, PCB_SEG_MEAN = 1, PCB_SEG_SUM = 2 };
int pcb_seg_loss_partials(long long count);
int pcb_seg_loss_forward(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w, int loss,
                         int reduction, float p0, float one_minus_beta, float background_weight, float words_weight, double *partials,
                         unsigned int *counter, float *out, pcb_stream_t stream);
int pcb_seg_loss_backward(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w, int loss,
                          int reduction, float p0, float one_minus_beta, float background_weight, float words_weight, const float *gout,
                          void *dx, const long long *dx_strides, pcb_stream_t stream);

/* ---- pixel average precision of segmentation logits (metrics.PixelAveragePrecision) ---------------------------------------
 * update: x, x_strides, target, n, h, w as for the losses above.  Each pixel's score is its logit rounded to bf16 (fp32 to
 * nearest-even, -0 as +0); hist (device int64 [2][65536]: pixels, positives) gains one count per pixel at the score's
 * order-preserving key (negative bf16 bits b: ~b & 0xffff, others: b | 0x8000), in row 1 when target > 0.5.  counts (device
 * int64 [5]) gains tp, fp, fn, tn at the threshold sigmoid(x) > 0.5 of the unrounded logit, and nan: NaN logits, which count
 * nowhere else.  Integer sums only: the result is independent of the launch grid and the order of its atomics.  No host
 * synchronisation, no workspace (capturable).  At most 2^40 pixels per call.
 * finalize: out (device fp64 [1]) = sklearn's average_precision_score over the histogram, 0 without positives, NaN when
 * counts[4] > 0; one CTA in a fixed order, so repeated calls agree bit for bit. */
int pcb_seg_score_update(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w,
                         long long *hist, long long *counts, pcb_stream_t stream);
int pcb_seg_score_finalize(const long long *hist, const long long *counts, double *out, pcb_stream_t stream);

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
/* the same update with the learning rate read from device memory (`lr`: one fp32, e.g. written by pcb_lr_cyclic earlier in the
   stream), so a captured graph follows a schedule.  No first-step flag: the momentum buffer is always read (zero-initialise it;
   momentum * 0 + d == d), so a buffer restored from a checkpoint is never discarded. */
int pcb_sgd_step_dev(float *param, const float *grad, float *momentum_buf, long long numel, const float *lr, float momentum,
                     float weight_decay, int nesterov, float grad_scale, pcb_stream_t stream);
/* cyclical learning rate (the reference's CyclicLR, models/utils/cls.py): one thread reads the iteration counter (device int64),
   writes that iteration's rate to `lr` (device fp32, for pcb_sgd_step_dev) and `lr64` (device fp64) and increments the counter.
   Evaluated in fp64 in the reference's operation order, each operation rounded once: triangular and triangular2 rates are
   bit-identical to the reference's; exp_range uses CUDA's pow for gamma^iteration.  step_size > 0 (iterations per half
   cycle). */
enum { PCB_CLR_TRIANGULAR = 0, PCB_CLR_TRIANGULAR2 = 1, PCB_CLR_EXP_RANGE = 2 };
int pcb_lr_cyclic(long long *iteration, double base_lr, double max_lr, double step_size, int mode, double gamma, float *lr,
                  double *lr64, pcb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PCONV_B200_H_ */

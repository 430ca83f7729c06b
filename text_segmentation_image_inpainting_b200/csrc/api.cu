// api.cu -- C-ABI entry points of libpconv_b200.so for the convolution itself (validation + dispatch between
// the wgmma tensor-core kernels and the shape-general kernels), error string, launch counter.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "pcb_common.cuh"

static thread_local char g_err[1024] = "";
static std::atomic<unsigned long long> g_launches{0};

int pcb_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return 1;
}
void pcb_count_launch(int n) { g_launches.fetch_add(static_cast<unsigned long long>(n)); }

extern "C" __attribute__((visibility("default"))) const char *pcb_last_error(void) { return g_err; }
extern "C" __attribute__((visibility("default"))) int pcb_version(void) { return 1; }
extern "C" __attribute__((visibility("default"))) unsigned long long pcb_launch_count(void) { return g_launches.load(); }

static int validate(const pcb_conv *c, bool need_x) {
    PCB_CHECK(c != nullptr, "null pcb_conv");
    PCB_CHECK(c->dtype == PCB_F32 || c->dtype == PCB_BF16, "bad dtype %d", c->dtype);
    PCB_CHECK(c->n > 0 && c->h > 0 && c->w > 0 && c->cin > 0 && c->cout > 0 && c->kh > 0 && c->kw > 0, "non-positive dimension");
    PCB_CHECK(c->stride > 0 && c->dil > 0 && c->pad_h >= 0 && c->pad_w >= 0, "bad stride/dilation/padding");
    PCB_CHECK(c->groups > 0 && c->cin % c->groups == 0 && c->cout % c->groups == 0, "groups must divide cin and cout");
    const int ho = (c->h + 2 * c->pad_h - c->dil * (c->kh - 1) - 1) / c->stride + 1;
    const int wo = (c->w + 2 * c->pad_w - c->dil * (c->kw - 1) - 1) / c->stride + 1;
    PCB_CHECK(ho == c->ho && wo == c->wo && ho > 0 && wo > 0, "output size mismatch: expected %dx%d, got %dx%d", ho, wo, c->ho, c->wo);
    PCB_CHECK(c->nparts >= 1 && c->nparts <= PCB_MAX_PARTS, "nparts out of range");
    int tot = 0;
    for (int p = 0; p < c->nparts; ++p) {
        const pcb_part &pt = c->parts[p];
        PCB_CHECK(pt.c > 0 && pt.x_cstride >= pt.c, "part %d: bad channel counts", p);
        PCB_CHECK((pt.x_up == 0 || pt.x_up == 1) && (pt.mask_up == 0 || pt.mask_up == 1), "part %d: bad upsample factor", p);
        PCB_CHECK(!(pt.x_up || pt.mask_up) || (c->h % 2 == 0 && c->w % 2 == 0), "part %d: upsampled source needs even h, w", p);
        PCB_CHECK(!need_x || pt.x != nullptr, "part %d: null x", p);
        tot += pt.c;
    }
    PCB_CHECK(tot == c->cin, "parts cover %d channels, cin is %d", tot, c->cin);
    PCB_CHECK(!(c->no_guard && c->groups != 1), "PartialConvNoHoles requires groups == 1");
    return 0;
}

// the kernel family a problem dispatches to: the depthwise kernels, the tensor-core kernels or the shape-general ones
// (force_generic: always the latter)
enum Family { FAMILY_GENERIC, FAMILY_DW, FAMILY_TC };

static Family family_of(const pcb_conv *c) {
    if (c->force_generic) return FAMILY_GENERIC;
    if (pcb_dw_eligible(c)) return FAMILY_DW;
    return pcb_tc_eligible(c) ? FAMILY_TC : FAMILY_GENERIC;
}

#define PCB_API extern "C" __attribute__((visibility("default")))

PCB_API int pcb_conv_uses_tensor_cores(const pcb_conv *c) { return (c && family_of(c) == FAMILY_TC) ? 1 : 0; }

// 1 when pcb_pconv_backward_data writes the gradient of a 2x-UPSAMPLED source directly at that source's own (half) resolution:
// dx[p] of such a part is then a [n, h/2, w/2, dx_cstride] buffer and no 2x2 reduction pass follows (the tensor-core sub-pixel path)
PCB_API int pcb_conv_dgrad_at_source_resolution(const pcb_conv *c) { return (c && family_of(c) == FAMILY_TC && pcb_tc_subpixel(c)) ? 1 : 0; }

PCB_API size_t pcb_pconv_workspace(const pcb_conv *c) { return (c && family_of(c) == FAMILY_TC) ? pcb_tc_workspace(c) : 0; }

PCB_API void pcb_conv_weight_layout(const pcb_conv *c, size_t *fwd_elems, size_t *dgrad_elems) {
    const Family f = family_of(c);
    if (f == FAMILY_DW) { *fwd_elems = static_cast<size_t>(c->cin) * c->kh * c->kw; *dgrad_elems = 0; return; }   // [taps][c]
    if (f == FAMILY_TC) { pcb_tc_weight_layout(c, fwd_elems, dgrad_elems); return; }
    *fwd_elems = static_cast<size_t>(c->cout) * c->kh * c->kw * (c->cin / c->groups);
    *dgrad_elems = 0;
}

int pcb_cast_weights(const float *src, void *dst, long long n, int dtype, cudaStream_t st);   // elementwise.cu

static int weight_prepare(const pcb_conv *c, const float *w_master_krsc, void *w_fwd, void *w_dgrad, bool zero_padding, pcb_stream_t stream) {
    PCB_CHECK(c && w_master_krsc && w_fwd, "pcb_conv_weight_prepare: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Family f = family_of(c);
    if (f == FAMILY_DW) return pcb_dw_weight_prepare(c, w_master_krsc, w_fwd, st);
    if (f == FAMILY_TC) return pcb_tc_weight_prepare(c, w_master_krsc, w_fwd, w_dgrad, zero_padding, st);
    return pcb_cast_weights(w_master_krsc, w_fwd, static_cast<long long>(c->cout) * c->kh * c->kw * (c->cin / c->groups), c->dtype, st);
}

PCB_API int pcb_conv_weight_prepare(const pcb_conv *c, const float *w_master_krsc, void *w_fwd, void *w_dgrad, pcb_stream_t stream) {
    return weight_prepare(c, w_master_krsc, w_fwd, w_dgrad, true, stream);
}

PCB_API int pcb_conv_weight_refresh(const pcb_conv *c, const float *w_master_krsc, void *w_fwd, void *w_dgrad, pcb_stream_t stream) {
    return weight_prepare(c, w_master_krsc, w_fwd, w_dgrad, false, stream);
}

static bool fuses_epilogue(const pcb_conv *c) {
    if (!c) return false;
    const Family f = family_of(c);
    return f == FAMILY_DW || (f == FAMILY_TC && pcb_tc_fuses_epilogue(c));
}

// 1 when the forward kernel this problem dispatches to can accumulate the per-channel BatchNorm statistics of its output itself
PCB_API int pcb_conv_fuses_bn_stats(const pcb_conv *c) { return fuses_epilogue(c) ? 1 : 0; }

// 1 when the forward kernel this problem dispatches to can apply an eval-mode BatchNorm + activation in its epilogue: the same
// problems as pcb_conv_fuses_bn_stats
PCB_API int pcb_conv_fuses_affine_act(const pcb_conv *c) { return fuses_epilogue(c) ? 1 : 0; }

static int pconv_forward_impl(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                              uint8_t *newmask, void *workspace, bool mask_pass_done, double *bn_sums, const pcb_ep *ep,
                              pcb_stream_t stream) {
    if (int rc = validate(c, true)) return rc;
    PCB_CHECK(w_fwd && y && msum && newmask && y_cstride >= c->cout, "pcb_pconv_forward: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (c->plain) msum = nullptr;                         // ordinary convolution: no mask pass, renormaliser 1 (msum / newmask untouched)
    else if (!mask_pass_done)
        if (int rc = pcb_mask_sums(c, msum, newmask, st)) return rc;
    PCB_CHECK(bn_sums == nullptr || pcb_conv_fuses_bn_stats(c), "pcb_pconv_forward_bn: this problem's kernel does not fuse the BatchNorm statistics (ask pcb_conv_fuses_bn_stats first)");
    PCB_CHECK(ep == nullptr || pcb_conv_fuses_affine_act(c), "pcb_pconv_forward_affine_act: this problem's kernel does not apply a fused BatchNorm + activation (ask pcb_conv_fuses_affine_act first)");
    const Family f = family_of(c);
    if (f == FAMILY_DW) {
        PCB_CHECK(y_cstride % 8 == 0, "depthwise forward: y channel stride must be a multiple of 8");
        return pcb_dw_forward(c, w_fwd, bias, y, y_cstride, msum, bn_sums, ep, st);
    }
    if (f == FAMILY_TC) {
        PCB_CHECK(workspace != nullptr, "pcb_pconv_forward: workspace required for the tensor-core path");
        PCB_CHECK((reinterpret_cast<uintptr_t>(w_fwd) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "w / y must be 16-byte aligned");
        return pcb_tc_forward_ws(c, w_fwd, bias, y, y_cstride, msum, static_cast<uint64_t *>(workspace), mask_pass_done, bn_sums, ep, st);
    }
    return pcb_generic_forward(c, w_fwd, bias, y, y_cstride, msum, st);
}

PCB_API int pcb_pconv_forward(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                              uint8_t *newmask, void *workspace, pcb_stream_t stream) {
    return pconv_forward_impl(c, w_fwd, bias, y, y_cstride, msum, newmask, workspace, false, nullptr, nullptr, stream);
}

// Forward with the statistics pass of the BatchNorm that follows (partial_convolution.py:193-197, BaseModels.py:95-99) fused into
// the convolution epilogue: bn_sums[0..cout) += sum over pixels of y, bn_sums[cout..2cout) += sum of y^2 (of the values as stored).
// `bn_sums` must be zero on entry and the problem must satisfy pcb_conv_fuses_bn_stats.  mask_pass_done: see pcb_pconv_forward_premasked.
PCB_API int pcb_pconv_forward_bn(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                                 uint8_t *newmask, void *workspace, int mask_pass_done, double *bn_sums, pcb_stream_t stream) {
    return pconv_forward_impl(c, w_fwd, bias, y, y_cstride, msum, newmask, workspace, mask_pass_done != 0, bn_sums, nullptr, stream);
}

// Inference forward with the eval-mode BatchNorm + activation behind the convolution applied in its epilogue (see the header)
PCB_API int pcb_pconv_forward_affine_act(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                                         uint8_t *newmask, void *workspace, int mask_pass_done, const float *scale, const float *shift,
                                         int act, float slope, pcb_stream_t stream) {
    PCB_CHECK(act >= PCB_ACT_NONE && act <= PCB_ACT_RELU6, "pcb_pconv_forward_affine_act: bad activation %d", act);
    PCB_CHECK((scale == nullptr) == (shift == nullptr), "pcb_pconv_forward_affine_act: scale and shift must both be given or both be NULL");
    const pcb_ep ep{scale, shift, act, slope};
    return pconv_forward_impl(c, w_fwd, bias, y, y_cstride, msum, newmask, workspace, mask_pass_done != 0, nullptr, &ep, stream);
}

// The forward in two calls, for callers that run the mask chain of a network ahead of the feature path on another stream:
// pcb_pconv_mask_pass computes everything that depends only on the masks (msum, newmask, the tap-validity words in
// `workspace`); pcb_pconv_forward_premasked is the rest and must be ordered after it.
PCB_API int pcb_pconv_mask_pass(const pcb_conv *c, float *msum, uint8_t *newmask, void *workspace, pcb_stream_t stream) {
    if (int rc = validate(c, false)) return rc;
    PCB_CHECK(msum && newmask, "pcb_pconv_mask_pass: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (int rc = pcb_mask_sums(c, msum, newmask, st)) return rc;
    if (family_of(c) == FAMILY_TC) {
        PCB_CHECK(workspace != nullptr, "pcb_pconv_mask_pass: workspace required for the tensor-core path");
        return pcb_tc_forward_mask_pass(c, static_cast<uint64_t *>(workspace), st);
    }
    return 0;
}

PCB_API int pcb_pconv_forward_premasked(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, float *msum,
                                        uint8_t *newmask, void *workspace, pcb_stream_t stream) {
    return pconv_forward_impl(c, w_fwd, bias, y, y_cstride, msum, newmask, workspace, true, nullptr, nullptr, stream);
}

PCB_API int pcb_pconv_backward_data(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_fwd, const void *w_dgrad,
                                    void *const *dx, const int32_t *dx_cstride, pcb_stream_t stream) {
    if (int rc = validate(c, false)) return rc;
    PCB_CHECK(dc && w_fwd && dx && dx_cstride && dc_cstride >= c->cout, "pcb_pconv_backward_data: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Family f = family_of(c);
    if (f == FAMILY_DW) {
        if (!dx[0]) return 0;
        PCB_CHECK(dc_cstride % 8 == 0 && dx_cstride[0] % 8 == 0, "depthwise dgrad: channel strides must be multiples of 8");
        return pcb_dw_dgrad(c, dc, dc_cstride, w_fwd, dx[0], dx_cstride[0], st);
    }
    if (f == FAMILY_TC) return pcb_tc_dgrad(c, dc, dc_cstride, w_dgrad, dx, dx_cstride, st);
    return pcb_generic_dgrad(c, dc, dc_cstride, w_fwd, dx, dx_cstride, st);
}

PCB_API int pcb_conv_dgrad_fuses_relu(const pcb_conv *c) {
    if (!c || validate(c, false) || family_of(c) != FAMILY_TC) return 0;
    return pcb_tc_dgrad_fuses_relu(c) ? 1 : 0;
}

PCB_API int pcb_pconv_backward_data_relu(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_dgrad, void *dx, int dx_cstride,
                                         const void *relu_x, int relu_cstride, pcb_stream_t stream) {
    PCB_CHECK(dc && w_dgrad && dx && relu_x && dc_cstride >= c->cout, "pcb_pconv_backward_data_relu: bad arguments");
    PCB_CHECK(pcb_conv_dgrad_fuses_relu(c), "pcb_pconv_backward_data_relu: this problem's kernel does not fuse the ReLU backward "
                                            "(ask pcb_conv_dgrad_fuses_relu first)");
    PCB_CHECK((reinterpret_cast<uintptr_t>(dc) & 15) == 0, "pcb_pconv_backward_data_relu: dc misaligned");
    void *dxs[1] = {dx};
    const int cs[1] = {dx_cstride};
    return pcb_tc_dgrad(c, dc, dc_cstride, w_dgrad, dxs, cs, static_cast<cudaStream_t>(stream), relu_x, relu_cstride);
}

static int backward_weight_impl(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, pcb_stream_t stream) {
    if (int rc = validate(c, true)) return rc;
    PCB_CHECK(dc && dw && dc_cstride >= c->cout, "pcb_pconv_backward_weight: bad arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Family f = family_of(c);
    if (f == FAMILY_DW) {
        PCB_CHECK(dc_cstride % 8 == 0, "depthwise wgrad: dc channel stride must be a multiple of 8");
        return pcb_dw_wgrad(c, dc, dc_cstride, dw, zero_dw, st);
    }
    if (f == FAMILY_TC) {
        PCB_CHECK(workspace != nullptr && (reinterpret_cast<uintptr_t>(dc) & 15) == 0, "pcb_pconv_backward_weight: workspace required / dc misaligned");
        return pcb_tc_wgrad(c, dc, dc_cstride, dw, workspace, zero_dw, st);
    }
    return pcb_generic_wgrad(c, dc, dc_cstride, dw, zero_dw, st);
}

PCB_API int pcb_pconv_backward_weight(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream) {
    return backward_weight_impl(c, dc, dc_cstride, dw, workspace, true, stream);
}

// same, ACCUMULATING into dw (no memset): for callers whose gradient buffer is already zero -- a training engine that zeroes its
// flat gradient arena once per step (one memset instead of one per layer), or genuine gradient accumulation
PCB_API int pcb_pconv_backward_weight_acc(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, pcb_stream_t stream) {
    return backward_weight_impl(c, dc, dc_cstride, dw, workspace, false, stream);
}

PCB_API int pcb_debug_pipeline_status(int *code) {
    PCB_CHECK(code != nullptr, "null code");
    return pcb_tc_read_abort_flag(code);
}

PCB_API int pcb_debug_conv_routes(const pcb_conv *c, int32_t routes[3]) {
    PCB_CHECK(routes != nullptr, "null routes");
    if (int rc = validate(c, false)) return rc;
    const Family f = family_of(c);
    if (f == FAMILY_TC) {
        pcb_tc_routes(c, routes);
        return 0;
    }
    routes[0] = routes[1] = routes[2] = (f == FAMILY_DW) ? PCB_ROUTE_DEPTHWISE : PCB_ROUTE_GENERIC;
    return 0;
}

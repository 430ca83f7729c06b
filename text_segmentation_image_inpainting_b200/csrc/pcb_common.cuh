// pcb_common.cuh -- shared host/device helpers for libpconv_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pconv_b200.h"

// ---------------------------------------------------------------------------------------------
// error plumbing (api.cu owns the storage)
// ---------------------------------------------------------------------------------------------
int pcb_set_error(const char *fmt, ...);
void pcb_count_launch(int n = 1);

#define PCB_CHECK(cond, ...)                       \
    do {                                           \
        if (!(cond)) return pcb_set_error(__VA_ARGS__); \
    } while (0)

#define PCB_CUDA(expr)                                                                           \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess)                                                                   \
            return pcb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    } while (0)

#define PCB_LAUNCH_CHECK()                                                                        \
    do {                                                                                         \
        cudaError_t _e = cudaGetLastError();                                                     \
        if (_e != cudaSuccess)                                                                   \
            return pcb_set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
        pcb_count_launch();                                                                      \
    } while (0)

// Per-device host state.  One process may drive several GPUs (a second device in the same process, or host threads each
// bound to their own device): everything cached on the host side -- SM counts, the >48 KB dynamic shared-memory opt-in of
// each kernel instantiation, abort flags, scratch buffers, internal streams -- is keyed by the CURRENT device.
constexpr int PCB_MAX_DEVICES = 64;

static inline int pcb_cur_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < PCB_MAX_DEVICES) ? dev : 0;
}

static inline int pcb_num_sms() {
    static int sms[PCB_MAX_DEVICES] = {0};
    const int dev = pcb_cur_device();
    if (!sms[dev]) {
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        sms[dev] = v > 0 ? v : 132;
    }
    return sms[dev];
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel instantiation, device): function attributes live in the
// device's context, so a flag per process would leave every device but the first without the opt-in.
#define PCB_SMEM_OPT_IN(kern, bytes)                                                                          \
    do {                                                                                                      \
        static bool pcb_done_[PCB_MAX_DEVICES] = {};                                                          \
        const int pcb_dev_ = pcb_cur_device();                                                                \
        if (!pcb_done_[pcb_dev_]) {                                                                           \
            PCB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            pcb_done_[pcb_dev_] = true;                                                                       \
        }                                                                                                     \
    } while (0)

static inline size_t pcb_dtype_size(int dtype) { return dtype == PCB_BF16 ? 2 : 4; }

// ---------------------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------------------
typedef __nv_bfloat16 bf16;

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<bf16>(bf16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float apply_act(float z, int act, float slope) {
    if (act == PCB_ACT_RELU) return z > 0.f ? z : 0.f;
    if (act == PCB_ACT_LEAKY) return z > 0.f ? z : z * slope;
    if (act == PCB_ACT_RELU6) return fminf(fmaxf(z, 0.f), 6.f);
    return z;
}
// derivative of the activation w.r.t. its pre-activation input z (torch conventions at the kinks:
// relu/leaky: grad 0 / slope at z<=0 ; relu6 (hardtanh): grad 1 only for 0 < z < 6).
__device__ __forceinline__ float act_grad(float z, int act, float slope) {
    if (act == PCB_ACT_RELU) return z > 0.f ? 1.f : 0.f;
    if (act == PCB_ACT_LEAKY) return z > 0.f ? 1.f : slope;
    if (act == PCB_ACT_RELU6) return (z > 0.f && z < 6.f) ? 1.f : 0.f;
    return 1.f;
}

// 8-element vector of T (16 B for bf16, 32 B for f32) held as floats
template <typename T> struct Vec8;
template <> struct Vec8<bf16> {
    static __device__ __forceinline__ void load(const bf16 *p, float (&v)[8]) {
        uint4 r = *reinterpret_cast<const uint4 *>(p);
        const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float2 f = __bfloat1622float2(h[i]);
            v[2 * i] = f.x;
            v[2 * i + 1] = f.y;
        }
    }
    static __device__ __forceinline__ void store(bf16 *p, const float (&v)[8]) {
        uint4 r;
        __nv_bfloat162 *h = reinterpret_cast<__nv_bfloat162 *>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        *reinterpret_cast<uint4 *>(p) = r;
    }
};
template <> struct Vec8<float> {
    static __device__ __forceinline__ void load(const float *p, float (&v)[8]) {
        float4 a = reinterpret_cast<const float4 *>(p)[0], b = reinterpret_cast<const float4 *>(p)[1];
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    static __device__ __forceinline__ void store(float *p, const float (&v)[8]) {
        reinterpret_cast<float4 *>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4 *>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// internal cross-file entry points -------------------------------------------------------------
int pcb_generic_forward(const pcb_conv *c, const void *w, const float *bias, void *y, int y_cstride, const float *msum, cudaStream_t st);
int pcb_generic_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_krsc, void *const *dx, const int *dx_cstride,
                      cudaStream_t st);
int pcb_generic_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, bool zero_dw, cudaStream_t st);
// mask box sums (all paths): msum fp32 [mg][n,ho,wo] (0 at holes), newmask u8 [mg][n,ho,wo]
int pcb_mask_sums(const pcb_conv *c, float *msum, uint8_t *newmask, cudaStream_t st);
bool pcb_tc_eligible(const pcb_conv *c);
bool pcb_tc_dgrad_supported(const pcb_conv *c);
size_t pcb_tc_workspace(const pcb_conv *c);
void pcb_tc_weight_layout(const pcb_conv *c, size_t *fwd_elems, size_t *dgrad_elems);
int pcb_tc_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd, void *w_dgrad, bool zero_padding, cudaStream_t st);
int pcb_tc_forward_mask_pass(const pcb_conv *c, uint64_t *tapmask, cudaStream_t st);
int pcb_tc_forward_ws(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, const float *msum,
                      uint64_t *tapmask, bool mask_pass_done, double *bn_sums, cudaStream_t st);
bool pcb_tc_fuses_bn_stats(const pcb_conv *c);
bool pcb_tc_subpixel(const pcb_conv *c);
int pcb_tc_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_dgrad, void *const *dx, const int *dx_cstride,
                 cudaStream_t st);
int pcb_tc_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st);
int pcb_tc_read_abort_flag(int *value);
// layers with <= 8 output channels (conv_smallco.cu); weights are read from the tensor-core operand layouts
struct pcb_smallco_layout { int ktap, koff[2], cout64; long long kf, kd; };
bool pcb_smallco_eligible(const pcb_conv *c);
int pcb_smallco_forward(const pcb_conv *c, const pcb_smallco_layout &L, const void *w_fwd, const float *bias, void *y, int y_cstride, const float *msum,
                        cudaStream_t st);
int pcb_smallco_dgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, const void *w_dgrad, void *const *dx, const int *dx_cstride,
                      cudaStream_t st);
int pcb_smallco_wgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, float *dw, bool zero_dw, cudaStream_t st);
// RGB tails as a 1x1 GEMM at source resolution (conv_k2r.cu); the *_extra operands follow the layer's regular ones
bool pcb_k2r_ok(const pcb_conv *c);
void pcb_k2r_weight_layout(const pcb_conv *c, size_t *fwd_extra, size_t *dg_extra);
size_t pcb_k2r_workspace(const pcb_conv *c);
int pcb_k2r_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd_extra, void *w_dg_extra, bool zero_padding, cudaStream_t st);
int pcb_k2r_forward(const pcb_conv *c, const pcb_smallco_layout &L, const void *w_fwd, const void *w_fwd_extra, const float *bias, void *y, int y_cstride,
                    const float *msum, void *workspace, cudaStream_t st);
int pcb_k2r_dgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, const void *w_dgrad, const void *w_dg_extra,
                  void *const *dx, const int *dx_cstride, cudaStream_t st);
int pcb_k2r_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st);
// 7x7 stride-2 image stems as a 4x4 convolution over the space-to-depth image (conv_stem.cu)
bool pcb_stem_ok(const pcb_conv *c);
size_t pcb_stem_weight_extra(const pcb_conv *c);
size_t pcb_stem_workspace(const pcb_conv *c);
int pcb_stem_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd_extra, bool zero_padding, cudaStream_t st);
int pcb_stem_forward(const pcb_conv *c, const void *w_fwd_extra, const float *bias, void *y, int y_cstride, const float *msum, void *workspace,
                     double *bn_sums, cudaStream_t st);
int pcb_stem_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st);
// depthwise fast path (dwconv.cu)
bool pcb_dw_eligible(const pcb_conv *c);
int pcb_dw_weight_prepare(const pcb_conv *c, const float *w_master, void *w_t, cudaStream_t st);
int pcb_dw_forward(const pcb_conv *c, const void *w_t, const float *bias, void *y, int y_cstride, const float *msum, double *bn_sums,
                   cudaStream_t st);
bool pcb_dw_fuses_bn_stats(const pcb_conv *c);
int pcb_dw_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_t, void *dx, int dx_cstride, cudaStream_t st);
int pcb_dw_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, bool zero_dw, cudaStream_t st);

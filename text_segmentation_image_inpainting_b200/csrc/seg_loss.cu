// seg_loss.cu -- the segmentation losses of the reference (loss.py:58-121) on [n, 1, h, w] logits: BinaryFocalLoss and
// SoftBootstrapCrossEntropy, one forward and one backward launch each.
//
// Per element, in fp32, with x the logit, t the target, s = 2t - 1, w = words_weight if t > 0 else background_weight and the
// stable bce(x, y) = max(x, 0) - x y + log1p(exp(-|x|)):
//   focal:     exp(gamma * logsigmoid(-x s)) * w * bce(x, t)                           (reduced by mean)
//   bootstrap: w * bce(x, beta t + (1 - beta) [sigmoid(x) > 0.5])                      (mean, sum or none)
// The forward reduction is deterministic: every thread sums a fixed set of elements in fp64, blocks reduce in a fixed tree
// into one partial each, and the last block to finish adds the partials in index order.  The grid depends on the element
// count only, so two calls give bit-identical results.  The backward reads the upstream gradient from device memory.
#include "pcb_common.cuh"

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int TPB = 256;
constexpr int EPT = 8;                   // elements per thread and block pass
constexpr int MAX_BLOCKS = 1024;

struct Args {
    const void *x;
    long long sn, sh, sw;
    const float *t;
    int h, w;
    long long count;
    int loss, reduction;
    float p0, omb, bg, words;            // gamma (focal) or beta (bootstrap); 1 - beta; the two weights
};

__device__ __forceinline__ long long x_offset(long long e, int h, int w, long long sn, long long sh, long long sw) {
    const long long hw = static_cast<long long>(h) * w;
    const long long b = e / hw, r = e - b * hw;
    const long long i = r / w, j = r - i * w;
    return b * sn + i * sh + j * sw;
}

template <int DT>
__device__ __forceinline__ float load_x(const Args &a, long long e) {
    const long long off = x_offset(e, a.h, a.w, a.sn, a.sh, a.sw);
    return DT == PCB_BF16 ? __bfloat162float(static_cast<const bf16 *>(a.x)[off]) : static_cast<const float *>(a.x)[off];
}

__device__ __forceinline__ float sigmoidf_stable(float x) {
    if (x >= 0.f) return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
    const float e = expf(x);
    return __fdiv_rn(e, __fadd_rn(1.f, e));
}

// max(x, 0) - x y as x (1 - y) or -x y: for y in [0, 1] both parts are non-negative, so nothing cancels
__device__ __forceinline__ float bce(float x, float y) {
    return (x >= 0.f ? x * (1.f - y) : -x * y) + log1pf(expf(-fabsf(x)));
}

__device__ __forceinline__ float log_sigmoid(float z) {
    return z < 0.f ? z - log1pf(expf(z)) : -log1pf(expf(-z));
}

// the element's loss, and (when g != nullptr) its derivative d loss_e / d x
__device__ __forceinline__ float element(const Args &a, float x, float t, float *g) {
    const float w = t > 0.f ? a.words : a.bg;
    if (a.loss == PCB_SEG_FOCAL) {
        const float s = 2.f * t - 1.f;
        const float b = bce(x, t);
        const float f = expf(a.p0 * log_sigmoid(-x * s));
        if (g) *g = w * f * (-a.p0 * s * sigmoidf_stable(x * s) * b + sigmoidf_stable(x) - t);
        return f * w * b;
    }
    const float tb = a.p0 * t + (sigmoid_above_half(x) ? a.omb : 0.f);
    if (g) *g = w * (sigmoidf_stable(x) - tb);
    return w * bce(x, tb);
}

__device__ __forceinline__ double block_sum(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x < 32) {
        s = threadIdx.x < TPB / 32 ? red[threadIdx.x] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    return s;          // valid in thread 0
}

template <int DT>
__global__ void __launch_bounds__(TPB) seg_loss_forward_kernel(Args a, double *__restrict__ partials, unsigned int *__restrict__ counter,
                                                               float *__restrict__ out) {
    __shared__ double red[TPB / 32];
    __shared__ bool last;
    const long long stride = static_cast<long long>(gridDim.x) * TPB;
    double acc = 0.0;
    for (long long e = static_cast<long long>(blockIdx.x) * TPB + threadIdx.x; e < a.count; e += stride) {
        const float v = element(a, load_x<DT>(a, e), a.t[e], nullptr);
        if (a.reduction == PCB_SEG_NONE) out[e] = v;
        else acc += static_cast<double>(v);
    }
    if (a.reduction == PCB_SEG_NONE) return;
    const double s = block_sum(acc, red);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last block: the partials in index order, each thread a fixed strided subset, then the fixed tree
    double t = 0.0;
    for (int b = threadIdx.x; b < static_cast<int>(gridDim.x); b += TPB) t += __ldcg(partials + b);
    __syncthreads();
    const double total = block_sum(t, red);
    if (threadIdx.x == 0) {
        out[0] = static_cast<float>(a.reduction == PCB_SEG_MEAN ? total / static_cast<double>(a.count) : total);
        *counter = 0u;                   // ready for the next call (graph replays included)
    }
}

template <int DT>
__global__ void __launch_bounds__(TPB) seg_loss_backward_kernel(Args a, const float *__restrict__ gout, void *__restrict__ dx,
                                                                long long dn, long long dh, long long dw) {
    const long long stride = static_cast<long long>(gridDim.x) * TPB;
    const float gs = a.reduction == PCB_SEG_NONE ? 0.f
                                                 : (a.reduction == PCB_SEG_MEAN ? static_cast<float>(static_cast<double>(gout[0]) / a.count)
                                                                                : gout[0]);
    for (long long e = static_cast<long long>(blockIdx.x) * TPB + threadIdx.x; e < a.count; e += stride) {
        float g;
        element(a, load_x<DT>(a, e), a.t[e], &g);
        g *= a.reduction == PCB_SEG_NONE ? gout[e] : gs;
        const long long off = x_offset(e, a.h, a.w, dn, dh, dw);
        if (DT == PCB_BF16) static_cast<bf16 *>(dx)[off] = __float2bfloat16_rn(g);
        else static_cast<float *>(dx)[off] = g;
    }
}

int blocks_for(long long count) {
    const long long b = (count + static_cast<long long>(TPB) * EPT - 1) / (static_cast<long long>(TPB) * EPT);
    return static_cast<int>(b < 1 ? 1 : (b > MAX_BLOCKS ? MAX_BLOCKS : b));
}

int make_args(Args &a, const void *x, int dtype, const long long *xs, const float *target, int n, int h, int w, int loss, int reduction,
              float p0, float omb, float bg, float words) {
    PCB_CHECK(x && xs && target && (dtype == PCB_F32 || dtype == PCB_BF16), "pcb_seg_loss: bad arguments");
    PCB_CHECK(n >= 1 && h >= 1 && w >= 1, "pcb_seg_loss: empty input %dx1x%dx%d", n, h, w);
    PCB_CHECK(loss == PCB_SEG_FOCAL || loss == PCB_SEG_BOOTSTRAP, "pcb_seg_loss: unknown loss %d", loss);
    PCB_CHECK(reduction == PCB_SEG_NONE || reduction == PCB_SEG_MEAN || reduction == PCB_SEG_SUM, "pcb_seg_loss: unknown reduction %d",
              reduction);
    PCB_CHECK(loss == PCB_SEG_BOOTSTRAP || reduction == PCB_SEG_MEAN, "pcb_seg_loss: the focal loss is reduced by its mean");
    a = Args{x, xs[0], xs[2], xs[3], target, h, w, static_cast<long long>(n) * h * w, loss, reduction, p0, omb, bg, words};
    return 0;
}

}  // namespace

PCB_API int pcb_seg_loss_partials(long long count) { return blocks_for(count); }

PCB_API int pcb_seg_loss_forward(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w, int loss,
                                 int reduction, float p0, float one_minus_beta, float background_weight, float words_weight,
                                 double *partials, unsigned int *counter, float *out, pcb_stream_t stream) {
    Args a;
    if (make_args(a, x, dtype, x_strides, target, n, h, w, loss, reduction, p0, one_minus_beta, background_weight, words_weight))
        return 1;
    PCB_CHECK(out && (reduction == PCB_SEG_NONE || (partials && counter)), "pcb_seg_loss_forward: missing output or partials");
    const int blocks = blocks_for(a.count);
    if (dtype == PCB_BF16) seg_loss_forward_kernel<PCB_BF16><<<blocks, TPB, 0, ST>>>(a, partials, counter, out);
    else seg_loss_forward_kernel<PCB_F32><<<blocks, TPB, 0, ST>>>(a, partials, counter, out);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_seg_loss_backward(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w, int loss,
                                  int reduction, float p0, float one_minus_beta, float background_weight, float words_weight,
                                  const float *gout, void *dx, const long long *dx_strides, pcb_stream_t stream) {
    Args a;
    if (make_args(a, x, dtype, x_strides, target, n, h, w, loss, reduction, p0, one_minus_beta, background_weight, words_weight))
        return 1;
    PCB_CHECK(gout && dx && dx_strides, "pcb_seg_loss_backward: bad arguments");
    const int blocks = blocks_for(a.count);
    if (dtype == PCB_BF16)
        seg_loss_backward_kernel<PCB_BF16><<<blocks, TPB, 0, ST>>>(a, gout, dx, dx_strides[0], dx_strides[2], dx_strides[3]);
    else
        seg_loss_backward_kernel<PCB_F32><<<blocks, TPB, 0, ST>>>(a, gout, dx, dx_strides[0], dx_strides[2], dx_strides[3]);
    PCB_LAUNCH_CHECK();
    return 0;
}

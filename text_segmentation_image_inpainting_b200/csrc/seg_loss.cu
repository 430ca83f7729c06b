// seg_loss.cu -- the segmentation losses of the reference (loss.py:58-121) on [n, 1, h, w] logits: BinaryFocalLoss and
// SoftBootstrapCrossEntropy, one forward and one backward launch each; and the pixel average precision of such logits against
// their targets (pcb_seg_score_update / pcb_seg_score_finalize, below the losses, reading the logits through the same view).
//
// Per element, in fp32, with x the logit, t the target, s = 2t - 1, w = words_weight if t > 0 else background_weight and the
// stable bce(x, y) = max(x, 0) - x y + log1p(exp(-|x|)):
//   focal:     exp(gamma * logsigmoid(-x s)) * w * bce(x, t)                           (reduced by mean)
//   bootstrap: w * bce(x, beta t + (1 - beta) [sigmoid(x) > 0.5])                      (mean, sum or none)
// The forward reduction is deterministic: every thread sums a fixed set of elements in fp64, blocks reduce in a fixed tree
// into one partial each, and the last block to finish adds the partials in index order.  The grid depends on the element
// count only, so two calls give bit-identical results.  The backward reads the upstream gradient from device memory.
#include <algorithm>

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

// ------------------------------------------------------------------------------------------------------------------------------
// Pixel average precision (metrics.PixelAveragePrecision): integer counts per bf16 score, then one fixed-order AP pass.
//
// Key: the logit rounded to bf16 (fp32 logits round to nearest-even, as torch's .to(torch.bfloat16)), -0 folded onto +0, then
// the order-preserving 16-bit map (negatives: ~bits, non-negatives: bits | 0x8000), so ascending keys are ascending scores and
// +-inf sit at the ends.  NaN logits have no key; they are counted on their own.
//
// Update grid: (SCORE_SLICES, chunks).  A CTA counts the pixels of its chunk whose key falls in its slice of the key space,
// privately in shared memory (2 x SCORE_SLICE_KEYS uint32: pixels, positives), then adds its non-zero bins to the int64
// histogram with 64-bit atomics.  The slice is the fastest grid index, so the SCORE_SLICES CTAs of a chunk run together and
// the chunk comes from DRAM once and from L2 for the others.  The CTAs of slice 0 also count tp / fp / fn / tn / nan.
// Everything is an integer sum, so the result depends neither on the grid nor on the order in which the atomics land.
// ------------------------------------------------------------------------------------------------------------------------------
namespace {

constexpr int SCORE_TPB = 512;
constexpr int SCORE_KEYS = 65536;
constexpr int SCORE_SLICES = 8;
constexpr int SCORE_SLICE_KEYS = SCORE_KEYS / SCORE_SLICES;
constexpr int SCORE_SMEM = 2 * SCORE_SLICE_KEYS * static_cast<int>(sizeof(unsigned int));
constexpr int SCORE_EPT = 16;                          // pixels per thread and chunk until the chunk count saturates
constexpr int SCORE_MAX_CHUNKS = 512;
constexpr long long SCORE_MAX_PIXELS = 1ll << 40;      // keeps a CTA's private counters below 2^32 (2^40 / 512 chunks)
constexpr int FIN_TPB = 512;
constexpr int FIN_KEYS = SCORE_KEYS / FIN_TPB;

// the order-preserving key of bf16 bits b (not NaN); -0 counts as +0
__device__ __forceinline__ unsigned int score_key(unsigned int b) {
    if (b == 0x8000u) b = 0u;
    return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}

// the unrounded logit (for the threshold counts) and its bf16 bits (the score)
template <int DT>
__device__ __forceinline__ void load_score(const Args &a, long long e, float &x, unsigned int &bits) {
    const long long off = x_offset(e, a.h, a.w, a.sn, a.sh, a.sw);
    if (DT == PCB_BF16) {
        bits = static_cast<const unsigned short *>(a.x)[off];
        x = __uint_as_float(bits << 16);
    } else {
        x = static_cast<const float *>(a.x)[off];
        bits = __bfloat16_as_ushort(__float2bfloat16_rn(x));
    }
}

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                                   // red is reused across calls
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    unsigned long long s = 0;
    if (threadIdx.x < 32) {
        s = threadIdx.x < SCORE_TPB / 32 ? red[threadIdx.x] : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    return s;          // valid in thread 0
}

template <int DT>
__global__ void __launch_bounds__(SCORE_TPB) seg_score_update_kernel(Args a, unsigned long long *__restrict__ hist,
                                                                       unsigned long long *__restrict__ counts) {
    extern __shared__ unsigned int s_bins[];           // [pixels | positives][SCORE_SLICE_KEYS]
    __shared__ unsigned long long red[SCORE_TPB / 32];
    unsigned int *s_pix = s_bins, *s_pos = s_bins + SCORE_SLICE_KEYS;
    for (int i = threadIdx.x; i < 2 * SCORE_SLICE_KEYS; i += SCORE_TPB) s_bins[i] = 0u;
    __syncthreads();
    const unsigned int base = blockIdx.x * SCORE_SLICE_KEYS;
    const bool tally = blockIdx.x == 0;
    unsigned int tp = 0, fp = 0, fn = 0, tn = 0, nan = 0;
    const long long stride = static_cast<long long>(gridDim.y) * SCORE_TPB;
    for (long long e = static_cast<long long>(blockIdx.y) * SCORE_TPB + threadIdx.x; e < a.count; e += stride) {
        float x;
        unsigned int bits;
        load_score<DT>(a, e, x, bits);
        if (x != x) {
            nan += tally;
            continue;
        }
        const bool label = a.t[e] > 0.5f;
        if (tally) {
            const bool pred = sigmoid_above_half(x);
            tp += pred & label;
            fp += pred & !label;
            fn += !pred & label;
            tn += !pred & !label;
        }
        const unsigned int k = score_key(bits) - base;  // wraps above the slice for keys below it
        if (k < SCORE_SLICE_KEYS) {
            atomicAdd(s_pix + k, 1u);
            if (label) atomicAdd(s_pos + k, 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SCORE_SLICE_KEYS; i += SCORE_TPB) {
        const unsigned int p = s_pix[i];
        if (p) {
            atomicAdd(hist + base + i, static_cast<unsigned long long>(p));
            const unsigned int q = s_pos[i];
            if (q) atomicAdd(hist + SCORE_KEYS + base + i, static_cast<unsigned long long>(q));
        }
    }
    if (!tally) return;
    const unsigned int v[5] = {tp, fp, fn, tn, nan};
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        const unsigned long long s = block_sum_u64(v[c], red);
        if (threadIdx.x == 0 && s) atomicAdd(counts + c, s);
    }
}

// One CTA.  Thread t owns the FIN_KEYS keys from 65535 - t * FIN_KEYS downwards (descending scores).  A block scan of the
// threads' pixel and positive totals (uint64, fixed order) gives each thread the counts at higher scores; each thread adds its
// terms pos_k * TP_k / N_k in fp64 in key order, and the block adds the FIN_TPB partial sums in a fixed tree.
__global__ void __launch_bounds__(FIN_TPB) seg_score_finalize_kernel(const unsigned long long *__restrict__ hist,
                                                                     const unsigned long long *__restrict__ counts, double *__restrict__ out) {
    __shared__ unsigned long long s_n[FIN_TPB], s_p[FIN_TPB];
    __shared__ double red[FIN_TPB / 32];
    const int t = threadIdx.x;
    const int hi = SCORE_KEYS - 1 - t * FIN_KEYS;
    unsigned long long n = 0, p = 0;
    for (int j = 0; j < FIN_KEYS; ++j) {
        n += hist[hi - j];
        p += hist[SCORE_KEYS + hi - j];
    }
    s_n[t] = n;
    s_p[t] = p;
    __syncthreads();
    for (int o = 1; o < FIN_TPB; o <<= 1) {            // Hillis-Steele inclusive scan
        const unsigned long long an = t >= o ? s_n[t - o] : 0ull, ap = t >= o ? s_p[t - o] : 0ull;
        __syncthreads();
        s_n[t] += an;
        s_p[t] += ap;
        __syncthreads();
    }
    const unsigned long long total_p = s_p[FIN_TPB - 1];
    unsigned long long cn = s_n[t] - n, cp = s_p[t] - p;
    double acc = 0.0;
    for (int j = 0; j < FIN_KEYS; ++j) {
        const unsigned long long nk = hist[hi - j], pk = hist[SCORE_KEYS + hi - j];
        cn += nk;
        cp += pk;
        if (pk) acc += static_cast<double>(pk) * (static_cast<double>(cp) / static_cast<double>(cn));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((t & 31) == 0) red[t >> 5] = acc;
    __syncthreads();
    if (t < 32) {
        double s = t < FIN_TPB / 32 ? red[t] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (t == 0) out[0] = counts[4] ? __longlong_as_double(0x7ff8000000000000ll) : (total_p ? s / static_cast<double>(total_p) : 0.0);
    }
}

}  // namespace

PCB_API int pcb_seg_score_update(const void *x, int dtype, const long long *x_strides, const float *target, int n, int h, int w,
                                 long long *hist, long long *counts, pcb_stream_t stream) {
    PCB_CHECK(x && x_strides && target && hist && counts && (dtype == PCB_F32 || dtype == PCB_BF16),
              "pcb_seg_score_update: bad arguments");
    PCB_CHECK(n >= 1 && h >= 1 && w >= 1, "pcb_seg_score_update: empty input %dx1x%dx%d", n, h, w);
    const long long count = static_cast<long long>(n) * h * w;
    PCB_CHECK(count <= SCORE_MAX_PIXELS, "pcb_seg_score_update: %lld pixels in one call (at most 2^40)", count);
    Args a{};
    a.x = x;
    a.sn = x_strides[0];
    a.sh = x_strides[2];
    a.sw = x_strides[3];
    a.t = target;
    a.h = h;
    a.w = w;
    a.count = count;
    const long long per_chunk = static_cast<long long>(SCORE_TPB) * SCORE_EPT;
    const long long chunks = std::min<long long>(std::max<long long>((count + per_chunk - 1) / per_chunk, 1), SCORE_MAX_CHUNKS);
    const dim3 grid(SCORE_SLICES, static_cast<unsigned int>(chunks));
    auto *hs = reinterpret_cast<unsigned long long *>(hist);
    auto *cs = reinterpret_cast<unsigned long long *>(counts);
    if (dtype == PCB_BF16) {
        PCB_SMEM_OPT_IN(seg_score_update_kernel<PCB_BF16>, SCORE_SMEM);
        seg_score_update_kernel<PCB_BF16><<<grid, SCORE_TPB, SCORE_SMEM, ST>>>(a, hs, cs);
    } else {
        PCB_SMEM_OPT_IN(seg_score_update_kernel<PCB_F32>, SCORE_SMEM);
        seg_score_update_kernel<PCB_F32><<<grid, SCORE_TPB, SCORE_SMEM, ST>>>(a, hs, cs);
    }
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_seg_score_finalize(const long long *hist, const long long *counts, double *out, pcb_stream_t stream) {
    PCB_CHECK(hist && counts && out, "pcb_seg_score_finalize: bad arguments");
    seg_score_finalize_kernel<<<1, FIN_TPB, 0, ST>>>(reinterpret_cast<const unsigned long long *>(hist),
                                                     reinterpret_cast<const unsigned long long *>(counts), out);
    PCB_LAUNCH_CHECK();
    return 0;
}

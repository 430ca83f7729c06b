// seg_ops.cu -- HBM-bound glue of the segmentation encoder-decoders (models/text_segmentation.py): average pooling
// (nn.AvgPool2d, count_include_pad=True: :33,66-67; ASP's AvgPool(k,1,(k-1)//2) models/common.py:62-68), bilinear
// upsampling with align_corners=False (:54,76,109,113), and the scSE gate (models/common.py:13-43):
//   y = x * cSE[n,c] + x * sSE[n,p],  cSE = sigmoid(MLP(GAP(x))),  sSE = sigmoid(<x[p,:], w_s>).
// NHWC, 8-channel vectors, fp32 math.
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"

namespace {

inline int sg_grid(long long items, int per_block = 256) {
    long long b = (items + per_block - 1) / per_block;
    const long long cap = 32ll * pcb_num_sms();
    return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

// ------------------------------------------------------------------------------------------------ avg pool
template <typename T, bool BWD>
__global__ void avgpool_kernel(const T *__restrict__ src, T *__restrict__ dst, int n, int h, int w, int c, int k, int stride, int pad, int ho, int wo) {
    // FWD: dst[n,ho,wo,c] = sum_{window} src[n,hi,wi,c] / k^2   (padding counted: count_include_pad=True)
    // BWD: dst[n,h,w,c]   = sum_{outputs covering (h,w)} src[n,oh,ow,c] / k^2
    const int cv = c >> 3;
    const int H = BWD ? h : ho, W = BWD ? w : wo;
    const long long nvec = static_cast<long long>(n) * H * W * cv;
    const float inv = 1.0f / static_cast<float>(k * k);
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long m = i / cv;
        const int ch = static_cast<int>(i - m * cv) * 8;
        const int x0 = static_cast<int>(m % W);
        const long long t = m / W;
        const int y0 = static_cast<int>(t % H), nn = static_cast<int>(t / H);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        for (int a = 0; a < k; ++a)
            for (int b = 0; b < k; ++b) {
                int sy, sx;
                if (!BWD) {
                    sy = y0 * stride - pad + a; sx = x0 * stride - pad + b;
                    if (sy < 0 || sy >= h || sx < 0 || sx >= w) continue;
                } else {
                    const int ty = y0 + pad - a, tx = x0 + pad - b;
                    if (ty < 0 || tx < 0) continue;
                    sy = ty / stride; sx = tx / stride;
                    if (sy * stride != ty || sx * stride != tx || sy >= ho || sx >= wo) continue;
                }
                float v[8];
                const int SH = BWD ? ho : h, SW = BWD ? wo : w;
                Vec8<T>::load(src + (static_cast<long long>(nn * SH + sy) * SW + sx) * c + ch, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[j];
            }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] *= inv;
        Vec8<T>::store(dst + i * 8, acc);
    }
}

// ------------------------------------------------------------------------------------------------ bilinear
// align_corners=False, integer scale s: src coordinate = (dst + 0.5)/s - 0.5, clamped at 0 (PyTorch semantics)
__device__ __forceinline__ void bil_coeffs(int d, int s, int in_size, int &i0, int &i1, float &l1) {
    float src = (static_cast<float>(d) + 0.5f) / static_cast<float>(s) - 0.5f;
    if (src < 0.f) src = 0.f;
    i0 = static_cast<int>(src);
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l1 = src - static_cast<float>(i0);
}

template <typename T>
__global__ void bilinear_fwd_kernel(const T *__restrict__ x, T *__restrict__ y, int n, int h, int w, int c, int s) {
    const int cv = c >> 3, H = h * s, W = w * s;
    const long long nvec = static_cast<long long>(n) * H * W * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long m = i / cv;
        const int ch = static_cast<int>(i - m * cv) * 8;
        const int ox = static_cast<int>(m % W);
        const long long t = m / W;
        const int oy = static_cast<int>(t % H), nn = static_cast<int>(t / H);
        int y0, y1, x0, x1; float ly, lx;
        bil_coeffs(oy, s, h, y0, y1, ly); bil_coeffs(ox, s, w, x0, x1, lx);
        float a[8], b[8], cc[8], d[8], o[8];
        const T *base = x + static_cast<long long>(nn) * h * w * c + ch;
        Vec8<T>::load(base + (static_cast<long long>(y0) * w + x0) * c, a);
        Vec8<T>::load(base + (static_cast<long long>(y0) * w + x1) * c, b);
        Vec8<T>::load(base + (static_cast<long long>(y1) * w + x0) * c, cc);
        Vec8<T>::load(base + (static_cast<long long>(y1) * w + x1) * c, d);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            o[j] = (1.f - ly) * ((1.f - lx) * a[j] + lx * b[j]) + ly * ((1.f - lx) * cc[j] + lx * d[j]);
        Vec8<T>::store(y + i * 8, o);
    }
}

// backward by gathering: each input pixel collects from the output pixels whose stencil touches it
template <typename T>
__global__ void bilinear_bwd_kernel(const T *__restrict__ gy, T *__restrict__ gx, int n, int h, int w, int c, int s) {
    const int cv = c >> 3, H = h * s, W = w * s;
    const long long nvec = static_cast<long long>(n) * h * w * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long m = i / cv;
        const int ch = static_cast<int>(i - m * cv) * 8;
        const int ix = static_cast<int>(m % w);
        const long long t = m / w;
        const int iy = static_cast<int>(t % h), nn = static_cast<int>(t / h);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        const int oy_lo = max(0, (iy - 1) * s), oy_hi = min(H - 1, (iy + 2) * s);
        const int ox_lo = max(0, (ix - 1) * s), ox_hi = min(W - 1, (ix + 2) * s);
        for (int oy = oy_lo; oy <= oy_hi; ++oy) {
            int y0, y1; float ly;
            bil_coeffs(oy, s, h, y0, y1, ly);
            const float wy = (y0 == iy ? (1.f - ly) : 0.f) + (y1 == iy ? ly : 0.f);
            if (wy == 0.f) continue;
            for (int ox = ox_lo; ox <= ox_hi; ++ox) {
                int x0, x1; float lx;
                bil_coeffs(ox, s, w, x0, x1, lx);
                const float wx = (x0 == ix ? (1.f - lx) : 0.f) + (x1 == ix ? lx : 0.f);
                if (wx == 0.f) continue;
                float g[8];
                Vec8<T>::load(gy + (static_cast<long long>(nn * H + oy) * W + ox) * c + ch, g);
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += wy * wx * g[j];
            }
        }
        Vec8<T>::store(gx + i * 8, acc);
    }
}

// ------------------------------------------------------------------------------------------------ GAP
// out[n][c] (fp32) = mean over hw of x[n,:,c]
template <typename T>
__global__ void __launch_bounds__(256) gap_kernel(const T *__restrict__ x, long long hw, int c, float *__restrict__ out, int chunks) {
    __shared__ float s_red[256][8];
    const int cv = c >> 3, rpb = 256 / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    const int nn = blockIdx.y;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (r < rpb) {
        const T *base = x + static_cast<long long>(nn) * hw * c;
        for (long long p = static_cast<long long>(blockIdx.x) * rpb + r; p < hw; p += static_cast<long long>(chunks) * rpb) {
            float f[8];
            Vec8<T>::load(base + p * c + v * 8, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s_red[threadIdx.x][j] = acc[j];
    }
    __syncthreads();
    if (r == 0 && v < cv) {
        const float inv = 1.0f / static_cast<float>(hw);
        for (int j = 0; j < 8; ++j) {
            float tot = 0.f;
            for (int rr = 0; rr < rpb; ++rr) tot += s_red[rr * cv + v][j];
            atomicAdd(out + static_cast<long long>(nn) * c + v * 8 + j, tot * inv);
        }
    }
}

// ------------------------------------------------------------------------------------------------ scSE gate
// sse = sigmoid(<x[p,:], ws>) ; y = x * (cse[n,:] + sse).  A pixel is handled by a GROUP of gw lanes (gw = the power of two >=
// min(c/8, 32)), lane vl of the group owning channel vectors vl, vl + gw, ...: a 24-channel tensor keeps 8 pixels per warp in
// flight instead of 3 busy lanes out of 32 (the MobileNetV2 blocks that carry the gate have 16..320 channels).
__device__ __forceinline__ float group_sum(float v, int gw) {
    for (int o = gw >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
inline int scse_group_width(int c) {
    const int cv = c >> 3;
    int gw = 1;
    while (gw < cv && gw < 32) gw <<= 1;
    return gw;
}

template <typename T>
__global__ void __launch_bounds__(256) scse_fwd_kernel(const T *__restrict__ x, const float *__restrict__ cse, const float *__restrict__ ws,
                                                       T *__restrict__ y, float *__restrict__ sse_out, long long npix, long long hw, int c, int gw) {
    const int lane = threadIdx.x & 31, sub = lane / gw, vl = lane - sub * gw, ppw = 32 / gw;
    const long long warp = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
    const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    const int cv = c >> 3;
    for (long long p0 = warp * ppw; p0 < npix; p0 += nwarps * ppw) {
        const long long p = p0 + sub;
        const bool act = p < npix;
        const long long nn = act ? p / hw : 0;
        float dot = 0.f;
        if (act)
            for (int v = vl; v < cv; v += gw) {
                float f[8];
                Vec8<T>::load(x + p * c + v * 8, f);
#pragma unroll
                for (int j = 0; j < 8; ++j) dot += f[j] * ws[v * 8 + j];
            }
        dot = group_sum(dot, gw);
        const float sse = 1.0f / (1.0f + __expf(-dot));
        if (act && vl == 0) sse_out[p] = sse;
        if (act)
            for (int v = vl; v < cv; v += gw) {
                float f[8];
                Vec8<T>::load(x + p * c + v * 8, f);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] *= (cse[nn * c + v * 8 + j] + sse);
                Vec8<T>::store(y + p * c + v * 8, f);
            }
    }
}

// dx = g*(cse+sse) + ws * [sse(1-sse) * sum_c g x] ; dcse[n,c] += sum_p g x ; dws[c] += sum_p x * sse(1-sse) * sum_c' g x
// Same lane groups; a block works inside ONE sample (blockIdx = sample * bps + slice) and a lane owns the SAME channel vectors for
// every pixel it sees, so both per-channel reductions are accumulated in registers over the lane's pixels, combined across the
// block in shared memory and reach global memory as one atomic per channel per block.  (v1 issued two shared-memory atomics
// per element; v2 one global atomic per lane and channel: with 8 lane groups per warp that was 2k same-address atomics per block.)
constexpr int SCSE_VM_MAX = 4;                      // channel vectors per lane held in registers: c <= 1024
template <typename T, int SCSE_VM>
__global__ void __launch_bounds__(256) scse_bwd_kernel(const T *__restrict__ gy, const T *__restrict__ x, const float *__restrict__ cse,
                                                       const float *__restrict__ ws, const float *__restrict__ sse_in, T *__restrict__ dx,
                                                       float *__restrict__ dcse, float *__restrict__ dws, long long hw, int c, int gw, int bps) {
    extern __shared__ float s_acc[];            // [2][c] : dcse partial, dws partial of the block
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int sub = lane / gw, vl = lane - sub * gw, ppw = 32 / gw;
    const int cv = c >> 3;
    const long long nn = blockIdx.x / bps;
    const int slice = blockIdx.x - static_cast<int>(nn) * bps;
    const long long per_block = (hw + bps - 1) / bps;
    const long long p_begin = nn * hw + slice * per_block, p_end = min((nn + 1) * hw, p_begin + per_block);
    for (int i = threadIdx.x; i < 2 * c; i += blockDim.x) s_acc[i] = 0.f;
    __syncthreads();
    float a_cse[SCSE_VM][8], a_ws[SCSE_VM][8], wsv[SCSE_VM][8], cs[SCSE_VM][8];
#pragma unroll
    for (int k = 0; k < SCSE_VM; ++k) {
        const int v = vl + gw * k;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            a_cse[k][j] = 0.f; a_ws[k][j] = 0.f;
            wsv[k][j] = v < cv ? ws[v * 8 + j] : 0.f;
            cs[k][j] = v < cv ? cse[nn * c + v * 8 + j] : 0.f;
        }
    }
    for (long long p0 = p_begin + static_cast<long long>(wib) * ppw; p0 < p_end; p0 += static_cast<long long>(wpb) * ppw) {
        const long long p = p0 + sub;
        const bool act = p < p_end;
        const float sse = act ? sse_in[p] : 0.f;
        float g[SCSE_VM][8], f[SCSE_VM][8];
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < SCSE_VM; ++k) {
            const int v = vl + gw * k;
            if (act && v < cv) {
                Vec8<T>::load(gy + p * c + v * 8, g[k]);
                Vec8<T>::load(x + p * c + v * 8, f[k]);
#pragma unroll
                for (int j = 0; j < 8; ++j) dot = fmaf(g[k][j], f[k][j], dot);
            }
        }
        dot = group_sum(dot, gw);
        const float dpre = dot * sse * (1.f - sse);
#pragma unroll
        for (int k = 0; k < SCSE_VM; ++k) {
            const int v = vl + gw * k;
            if (act && v < cv) {
                float o[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    o[j] = fmaf(g[k][j], cs[k][j] + sse, wsv[k][j] * dpre);
                    a_cse[k][j] = fmaf(g[k][j], f[k][j], a_cse[k][j]);
                    a_ws[k][j] = fmaf(f[k][j], dpre, a_ws[k][j]);
                }
                Vec8<T>::store(dx + p * c + v * 8, o);
            }
        }
    }
    // lanes of a warp that own the same vectors (different pixel sub-groups) combine first, then one shared atomic per channel and warp
#pragma unroll
    for (int k = 0; k < SCSE_VM; ++k) {
        const int v = vl + gw * k;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float a = a_cse[k][j], b = a_ws[k][j];
            for (int o = gw; o < 32; o <<= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
            if (sub == 0 && v < cv) { atomicAdd(&s_acc[v * 8 + j], a); atomicAdd(&s_acc[c + v * 8 + j], b); }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        atomicAdd(dcse + nn * c + i, s_acc[i]);
        atomicAdd(dws + i, s_acc[c + i]);
    }
}

// broadcast add: dx[n,p,c] += g[n,c] / hw   (backward of the global average pool)
template <typename T>
__global__ void gap_bwd_kernel(const float *__restrict__ g, T *__restrict__ dx, long long npix, long long hw, int c, int accumulate) {
    const int cv = c >> 3;
    const long long nvec = npix * cv;
    const float inv = 1.0f / static_cast<float>(hw);
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long p = i / cv;
        const int ch = static_cast<int>(i - p * cv) * 8;
        const long long nn = p / hw;
        float o[8];
        if (accumulate) Vec8<T>::load(dx + i * 8, o);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (accumulate ? o[j] : 0.f) + g[nn * c + ch + j] * inv;
        Vec8<T>::store(dx + i * 8, o);
    }
}

// ------------------------------------------------------------------------------------------------ text-mask post-processing
// The demo's post-processing of the segmentation logits (Examples/demo_segmentation.py:33-36, Dataloader.py:308-316):
//   b = maxpool3x3(sigmoid(x) > 0.5) over the full padded map,  crop to [h_valid, w_valid],
//   out = upsample_bilinear2d(crop, (oh, ow), align_corners=False) > 0.
// The inputs of the resize are {0, 1} and its weights are non-negative, so "sum > 0" is "some tap with a positive weight is 1":
// each output pixel tests the (at most four) taps with positive weight, which makes the result exact.  Source indices and
// lambdas follow ATen's UpSample.h (area_pixel_compute_scale / compute_source_index_and_lambda) in fp32.
__device__ __forceinline__ void post_taps(int d, int in_size, int out_size, int &i0, int &i1, bool &w0, bool &w1) {
    if (in_size == out_size) { i0 = i1 = d; w0 = true; w1 = false; return; }
    const float scale = static_cast<float>(in_size) / static_cast<float>(out_size);
    float src = scale * (static_cast<float>(d) + 0.5f) - 0.5f;
    if (src < 0.f) src = 0.f;
    i0 = min(static_cast<int>(floorf(src)), in_size - 1);
    const float l1 = fminf(fmaxf(src - static_cast<float>(i0), 0.f), 1.f);
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    w0 = (1.f - l1) > 0.f; w1 = l1 > 0.f;
}

template <typename T>
__device__ __forceinline__ bool post_pooled(const T *__restrict__ x, int cstride, int nn, int h, int w, int iy, int ix) {
    for (int dy = -1; dy <= 1; ++dy) {
        const int yy = iy + dy;
        if (yy < 0 || yy >= h) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int xx = ix + dx;
            if (xx < 0 || xx >= w) continue;
            const float v = to_f32(x[(static_cast<long long>(nn * h + yy) * w + xx) * cstride]);
            if (sigmoid_above_half(v)) return true;                 // the demo's sigmoid(x) > 0.5, exactly as torch's CPU float32
        }
    }
    return false;
}

template <typename T>
__global__ void seg_mask_post_kernel(const T *__restrict__ x, int cstride, int n, int h, int w, int hv, int wv, int oh, int ow,
                                     uint8_t *__restrict__ out) {
    const long long total = static_cast<long long>(n) * oh * ow;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ox = static_cast<int>(i % ow);
        const long long t = i / ow;
        const int oy = static_cast<int>(t % oh), nn = static_cast<int>(t / oh);
        int y0, y1, x0, x1;
        bool wy0, wy1, wx0, wx1;
        post_taps(oy, hv, oh, y0, y1, wy0, wy1);
        post_taps(ox, wv, ow, x0, x1, wx0, wx1);
        const bool v = (wy0 && wx0 && post_pooled(x, cstride, nn, h, w, y0, x0)) || (wy0 && wx1 && post_pooled(x, cstride, nn, h, w, y0, x1)) ||
                       (wy1 && wx0 && post_pooled(x, cstride, nn, h, w, y1, x0)) || (wy1 && wx1 && post_pooled(x, cstride, nn, h, w, y1, x1));
        out[i] = v ? 1 : 0;
    }
}

}  // namespace

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))
PCB_API int pcb_avgpool_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, int k, int stride, int pad, pcb_stream_t stream) {
    PCB_CHECK(x && y && c % 8 == 0 && k > 0 && stride > 0, "pcb_avgpool_forward: bad arguments (channels must be a multiple of 8)");
    const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
    const long long nvec = static_cast<long long>(n) * ho * wo * (c / 8);
    if (dtype == PCB_BF16) avgpool_kernel<bf16, false><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const bf16 *>(x), static_cast<bf16 *>(y), n, h, w, c, k, stride, pad, ho, wo);
    else avgpool_kernel<float, false><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const float *>(x), static_cast<float *>(y), n, h, w, c, k, stride, pad, ho, wo);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_avgpool_backward(const void *gy, void *gx, int dtype, int n, int h, int w, int c, int k, int stride, int pad, pcb_stream_t stream) {
    PCB_CHECK(gy && gx && c % 8 == 0 && k > 0 && stride > 0, "pcb_avgpool_backward: bad arguments");
    const int ho = (h + 2 * pad - k) / stride + 1, wo = (w + 2 * pad - k) / stride + 1;
    const long long nvec = static_cast<long long>(n) * h * w * (c / 8);
    if (dtype == PCB_BF16) avgpool_kernel<bf16, true><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<bf16 *>(gx), n, h, w, c, k, stride, pad, ho, wo);
    else avgpool_kernel<float, true><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const float *>(gy), static_cast<float *>(gx), n, h, w, c, k, stride, pad, ho, wo);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_bilinear_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, int scale, pcb_stream_t stream) {
    PCB_CHECK(x && y && c % 8 == 0 && scale >= 1, "pcb_bilinear_forward: bad arguments (channels must be a multiple of 8)");
    const long long nvec = static_cast<long long>(n) * h * scale * w * scale * (c / 8);
    if (dtype == PCB_BF16) bilinear_fwd_kernel<bf16><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const bf16 *>(x), static_cast<bf16 *>(y), n, h, w, c, scale);
    else bilinear_fwd_kernel<float><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const float *>(x), static_cast<float *>(y), n, h, w, c, scale);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_bilinear_backward(const void *gy, void *gx, int dtype, int n, int h, int w, int c, int scale, pcb_stream_t stream) {
    PCB_CHECK(gy && gx && c % 8 == 0 && scale >= 1, "pcb_bilinear_backward: bad arguments");
    const long long nvec = static_cast<long long>(n) * h * w * (c / 8);
    if (dtype == PCB_BF16) bilinear_bwd_kernel<bf16><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<bf16 *>(gx), n, h, w, c, scale);
    else bilinear_bwd_kernel<float><<<sg_grid(nvec), 256, 0, ST>>>(static_cast<const float *>(gy), static_cast<float *>(gx), n, h, w, c, scale);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_gap_forward(const void *x, int dtype, int n, long long hw, int c, float *out, pcb_stream_t stream) {
    PCB_CHECK(x && out && c % 8 == 0 && c <= 2048 && hw > 0, "pcb_gap_forward: bad arguments (channels % 8 == 0, <= 2048)");
    PCB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * n * c, ST));
    const int rpb = 256 / (c / 8);
    int chunks = static_cast<int>(std::min<long long>((hw + rpb * 8 - 1) / (rpb * 8), std::max(1, 4 * pcb_num_sms() / std::max(1, n))));
    chunks = std::max(1, chunks);
    if (dtype == PCB_BF16) gap_kernel<bf16><<<dim3(chunks, n), 256, 0, ST>>>(static_cast<const bf16 *>(x), hw, c, out, chunks);
    else gap_kernel<float><<<dim3(chunks, n), 256, 0, ST>>>(static_cast<const float *>(x), hw, c, out, chunks);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_gap_backward(const float *g, void *dx, int dtype, int n, long long hw, int c, int accumulate, pcb_stream_t stream) {
    PCB_CHECK(g && dx && c % 8 == 0, "pcb_gap_backward: bad arguments");
    const long long npix = static_cast<long long>(n) * hw;
    if (dtype == PCB_BF16) gap_bwd_kernel<bf16><<<sg_grid(npix * (c / 8)), 256, 0, ST>>>(g, static_cast<bf16 *>(dx), npix, hw, c, accumulate);
    else gap_bwd_kernel<float><<<sg_grid(npix * (c / 8)), 256, 0, ST>>>(g, static_cast<float *>(dx), npix, hw, c, accumulate);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_scse_forward(const void *x, const float *cse, const float *ws, void *y, float *sse_out, int dtype, int n, long long hw, int c,
                             pcb_stream_t stream) {
    PCB_CHECK(x && cse && ws && y && sse_out && c % 8 == 0, "pcb_scse_forward: bad arguments (channels must be a multiple of 8)");
    const long long npix = static_cast<long long>(n) * hw;
    const int gw = scse_group_width(c);
    const int grid = sg_grid(npix * gw);
    if (dtype == PCB_BF16) scse_fwd_kernel<bf16><<<grid, 256, 0, ST>>>(static_cast<const bf16 *>(x), cse, ws, static_cast<bf16 *>(y), sse_out, npix, hw, c, gw);
    else scse_fwd_kernel<float><<<grid, 256, 0, ST>>>(static_cast<const float *>(x), cse, ws, static_cast<float *>(y), sse_out, npix, hw, c, gw);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_scse_backward(const void *gy, const void *x, const float *cse, const float *ws, const float *sse, void *dx, float *dcse,
                              float *dws, int dtype, int n, long long hw, int c, pcb_stream_t stream) {
    // checked before the memsets: a refused call leaves dcse and dws untouched
    PCB_CHECK(gy && x && cse && ws && sse && dx && dcse && dws && c % 8 == 0 && c <= 8 * 32 * SCSE_VM_MAX,
              "pcb_scse_backward: bad arguments (channels a multiple of 8, at most %d)", 8 * 32 * SCSE_VM_MAX);
    const long long npix = static_cast<long long>(n) * hw;
    PCB_CUDA(cudaMemsetAsync(dcse, 0, sizeof(float) * n * c, ST));
    PCB_CUDA(cudaMemsetAsync(dws, 0, sizeof(float) * c, ST));
    const int gw = scse_group_width(c);
    // blocks per sample: ~2048 lane-slots of work per block, at most ~4 blocks per SM in total
    const long long want = std::max<long long>(1, (hw * gw + 2047) / 2048), cap = std::max<long long>(1, 4ll * pcb_num_sms() / n);
    const int bps = static_cast<int>(std::min(want, cap));
    const int grid = n * bps;
    const size_t smem = sizeof(float) * 2 * c;
#define PCB_SCSE_BWD(T, VM) scse_bwd_kernel<T, VM><<<grid, 256, smem, ST>>>(static_cast<const T *>(gy), static_cast<const T *>(x), cse, ws, sse, static_cast<T *>(dx), dcse, dws, hw, c, gw, bps)
    if (dtype == PCB_BF16) {
        if (c <= 256) PCB_SCSE_BWD(bf16, 1); else if (c <= 512) PCB_SCSE_BWD(bf16, 2); else PCB_SCSE_BWD(bf16, 4);
    } else {
        if (c <= 256) PCB_SCSE_BWD(float, 1); else if (c <= 512) PCB_SCSE_BWD(float, 2); else PCB_SCSE_BWD(float, 4);
    }
#undef PCB_SCSE_BWD
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_seg_mask_postprocess(const void *logits, int dtype, int n, int h, int w, int cstride, int h_valid, int w_valid, int oh,
                                     int ow, uint8_t *out, pcb_stream_t stream) {
    PCB_CHECK(logits && out && (dtype == PCB_F32 || dtype == PCB_BF16), "pcb_seg_mask_postprocess: bad arguments");
    PCB_CHECK(n > 0 && h > 0 && w > 0 && cstride > 0 && oh > 0 && ow > 0, "pcb_seg_mask_postprocess: non-positive size");
    PCB_CHECK(h_valid > 0 && h_valid <= h && w_valid > 0 && w_valid <= w, "pcb_seg_mask_postprocess: crop %dx%d outside the %dx%d map",
              h_valid, w_valid, h, w);
    const int grid = sg_grid(static_cast<long long>(n) * oh * ow);
    if (dtype == PCB_BF16) seg_mask_post_kernel<bf16><<<grid, 256, 0, ST>>>(static_cast<const bf16 *>(logits), cstride, n, h, w, h_valid, w_valid, oh, ow, out);
    else seg_mask_post_kernel<float><<<grid, 256, 0, ST>>>(static_cast<const float *>(logits), cstride, n, h, w, h_valid, w_valid, oh, ow, out);
    PCB_LAUNCH_CHECK();
    return 0;
}

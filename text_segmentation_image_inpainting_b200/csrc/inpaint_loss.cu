// inpaint_loss.cu -- the element-wise, pooling and reduction kernels of the inpainting loss (loss.py:185-307): the pixel terms
// fused with the composite and the VGG input batch, the 2x2/2 max-pool of VGG16 forward and backward, the perceptual L1 sums
// and their gradient, the Gram-matrix L1 sums and the sign operand of its backward.  The VGG convolutions and the Gram
// products run on the convolution kernels of this library (text_segmentation_image_inpainting_b200/loss.py).
#include <math.h>

#include "pcb_common.cuh"

namespace {

constexpr int LT = 256;               // threads per block of every kernel here

#define ST static_cast<cudaStream_t>(stream)

int grid_for(long long work) {
    long long b = (work + LT - 1) / LT;
    long long cap = 8LL * pcb_num_sms();
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Q per-thread partial sums -> one double atomic per quantity per block
template <int Q> __device__ __forceinline__ void block_sum_atomic(double (&v)[Q], double *dst) {
    __shared__ double sh[Q][LT / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        v[q] = warp_sum_d(v[q]);
        if (lane == 0) sh[q][wid] = v[q];
    }
    __syncthreads();
    if (wid == 0) {
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            double t = lane < LT / 32 ? sh[q][lane] : 0.0;
            t = warp_sum_d(t);
            if (lane == 0) atomicAdd(dst + q, t);
        }
    }
}

// torch.sign / the L1 and abs backward: sign(0) = 0, NaN stays NaN
__device__ __forceinline__ float sgnf(float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : d); }

struct Img {                            // an image tensor read or written through element strides (NCHW fp32, NHWC views)
    long long sn, sc, sh, sw;
};

// comp = mask*raw + (1-mask)*output for a {0,1} mask: raw where valid, output in holes
template <typename TO>
__device__ __forceinline__ float comp_at(const float *raw, const TO *out, Img so, const uint8_t *plane, int h, int w, int b, int c, int y,
                                         int x) {
    const long long p = ((long long)b * h + y) * w + x;
    return plane[p] ? raw[(((long long)b * 3 + c) * h + y) * w + x] : to_f32(out[b * so.sn + c * so.sc + y * so.sh + x * so.sw]);
}

// One thread per pixel: the composite, the valid / hole L1 sums, both total-variation sums, and the VGG input batch
// [3n][h][w][8] (comp | output | origin, channels 3..7 zero) in the compute dtype.
template <typename TO, typename TX>
__global__ void __launch_bounds__(LT) pixel_fwd_kernel(const float *__restrict__ raw, const float *__restrict__ orig, const TO *__restrict__ out,
                                                       Img so, const uint8_t *__restrict__ plane, int n, int h, int w, TX *__restrict__ X,
                                                       double *__restrict__ sums) {
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const long long npix = (long long)n * h * w, hw = (long long)h * w;
    for (long long p = blockIdx.x * (long long)LT + threadIdx.x; p < npix; p += (long long)gridDim.x * LT) {
        const int b = (int)(p / hw), y = (int)((p / w) % h), x = (int)(p % w);
        const bool m = plane[p] != 0;
        float vc[8], vo[8], vr[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) vc[k] = vo[k] = vr[k] = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const long long q = (((long long)b * 3 + c) * h + y) * w + x;
            const float r = raw[q], o = orig[q], v = to_f32(out[b * so.sn + c * so.sc + y * so.sh + x * so.sw]);
            const float cp = m ? r : v;
            const float d = fabsf(v - o);
            if (m) acc[0] += d; else acc[1] += d;
            if (x + 1 < w) acc[2] += fabsf(cp - comp_at(raw, out, so, plane, h, w, b, c, y, x + 1));
            if (y + 1 < h) acc[3] += fabsf(cp - comp_at(raw, out, so, plane, h, w, b, c, y + 1, x));
            vc[c] = cp; vo[c] = v; vr[c] = o;
        }
        Vec8<TX>::store(X + (((long long)b) * hw + (p % hw)) * 8, vc);
        Vec8<TX>::store(X + (((long long)n + b) * hw + (p % hw)) * 8, vo);
        Vec8<TX>::store(X + (((long long)2 * n + b) * hw + (p % hw)) * 8, vr);
    }
    block_sum_atomic<4>(acc, sums);
}

// d loss / d output per element: the valid / hole L1 terms, (1 - mask) * (TV gradient of comp + VGG gradient of comp), plus
// the VGG gradient of output.  dX: [2n][h][w][8] (comp | output) or null.  co: {valid, hole, tv_h, tv_v} coefficients.
template <typename TO, typename TX>
__global__ void __launch_bounds__(LT) pixel_bwd_kernel(const float *__restrict__ raw, const float *__restrict__ orig, const TO *__restrict__ out,
                                                       Img so, const uint8_t *__restrict__ plane, int n, int h, int w, const TX *__restrict__ dX,
                                                       float4 co, const float *__restrict__ gscale, TO *__restrict__ grad, Img sg) {
    const long long npix = (long long)n * h * w, hw = (long long)h * w;
    const float gs = *gscale;
    for (long long p = blockIdx.x * (long long)LT + threadIdx.x; p < npix; p += (long long)gridDim.x * LT) {
        const int b = (int)(p / hw), y = (int)((p / w) % h), x = (int)(p % w);
        const bool m = plane[p] != 0;
        float dxc[8], dxo[8];
        if (dX) {
            Vec8<TX>::load(dX + ((long long)b * hw + (p % hw)) * 8, dxc);
            Vec8<TX>::load(dX + (((long long)n + b) * hw + (p % hw)) * 8, dxo);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) dxc[k] = dxo[k] = 0.f;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const long long q = (((long long)b * 3 + c) * h + y) * w + x;
            const float o = orig[q], v = to_f32(out[b * so.sn + c * so.sc + y * so.sh + x * so.sw]);
            float g = gs * (m ? co.x : co.y) * sgnf(v - o);
            if (!m) {
                const float cp = v;
                float tv = 0.f;
                if (x + 1 < w) tv += co.z * sgnf(cp - comp_at(raw, out, so, plane, h, w, b, c, y, x + 1));
                if (x > 0) tv -= co.z * sgnf(comp_at(raw, out, so, plane, h, w, b, c, y, x - 1) - cp);
                if (y + 1 < h) tv += co.w * sgnf(cp - comp_at(raw, out, so, plane, h, w, b, c, y + 1, x));
                if (y > 0) tv -= co.w * sgnf(comp_at(raw, out, so, plane, h, w, b, c, y - 1, x) - cp);
                g += gs * tv + dxc[c];
            }
            g += dxo[c];
            grad[b * sg.sn + c * sg.sc + y * sg.sh + x * sg.sw] = from_f32<TO>(g);
        }
    }
}

// 2x2 / stride-2 max-pool, NHWC, 8 channels per thread.  torch's rule: a tap replaces the running maximum when it is greater
// or NaN (row-major window order), so ties go to the FIRST maximum and NaN propagates.
template <typename T>
__device__ __forceinline__ void pool_window(const T *x, long long base, long long rowstride, int c, float (&mx)[8], int (&idx)[8]) {
#pragma unroll
    for (int k = 0; k < 8; ++k) { mx[k] = -INFINITY; idx[k] = 0; }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        float v[8];
        Vec8<T>::load(x + base + (t >> 1) * rowstride + (t & 1) * c, v);
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (v[k] > mx[k] || isnan(v[k])) { mx[k] = v[k]; idx[k] = t; }
    }
}

template <typename T>
__global__ void __launch_bounds__(LT) maxpool_fwd_kernel(const T *__restrict__ x, T *__restrict__ y, int n, int h, int w, int c) {
    const int ho = h >> 1, wo = w >> 1, cv = c >> 3;
    const long long total = (long long)n * ho * wo * cv;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < total; i += (long long)gridDim.x * LT) {
        const int g = (int)(i % cv);
        const long long o = i / cv;
        const int xo = (int)(o % wo), yo = (int)((o / wo) % ho), b = (int)(o / ((long long)wo * ho));
        float mx[8];
        int idx[8];
        pool_window(x, (((long long)b * h + 2 * yo) * w + 2 * xo) * c + 8 * g, (long long)w * c, c, mx, idx);
        Vec8<T>::store(y + o * c + 8 * g, mx);
    }
}

// gradient to the window's maximum, 0 elsewhere; relu_mask: also the in-place ReLU backward of the pooled input (torch's
// threshold_backward: 0 where the ReLU output is <= 0)
template <typename T>
__global__ void __launch_bounds__(LT) maxpool_bwd_kernel(const T *__restrict__ gy, const T *__restrict__ x, T *__restrict__ gx, int n, int h,
                                                         int w, int c, int relu_mask) {
    const int ho = h >> 1, wo = w >> 1, cv = c >> 3;
    const long long total = (long long)n * ho * wo * cv;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < total; i += (long long)gridDim.x * LT) {
        const int g = (int)(i % cv);
        const long long o = i / cv;
        const int xo = (int)(o % wo), yo = (int)((o / wo) % ho), b = (int)(o / ((long long)wo * ho));
        const long long base = (((long long)b * h + 2 * yo) * w + 2 * xo) * c + 8 * g;
        float mx[8], gv[8];
        int idx[8];
        pool_window(x, base, (long long)w * c, c, mx, idx);
        Vec8<T>::load(gy + o * c + 8 * g, gv);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            float r[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) r[k] = (idx[k] == t && !(relu_mask && mx[k] <= 0.f)) ? gv[k] : 0.f;
            Vec8<T>::store(gx + base + (t >> 1) * (long long)w * c + (t & 1) * c, r);
        }
    }
}

// f: [3n][hw][c] (comp | output | origin): sums[0] += sum |f_comp - f_origin|, sums[1] += sum |f_output - f_origin|
template <typename T>
__global__ void __launch_bounds__(LT) feature_l1_kernel(const T *__restrict__ f, int n, long long img, double *__restrict__ sums) {
    double acc[2] = {0.0, 0.0};
    const long long nv = (long long)n * img / 8;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < nv; i += (long long)gridDim.x * LT) {
        const long long e = i * 8;
        float a[8], b[8], o[8];
        Vec8<T>::load(f + e, a);
        Vec8<T>::load(f + (long long)n * img + e, b);
        Vec8<T>::load(f + 2LL * n * img + e, o);
#pragma unroll
        for (int k = 0; k < 8; ++k) { acc[0] += fabsf(a[k] - o[k]); acc[1] += fabsf(b[k] - o[k]); }
    }
    block_sum_atomic<2>(acc, sums);
}

// df[i] = gs * (l1 * sign(f[i] - f_origin) + gram * g_gram[i]) + g_next[i] for the 2n images comp | output
template <typename T>
__global__ void __launch_bounds__(LT) feature_bwd_kernel(const T *__restrict__ f, int n, long long img, const T *__restrict__ gnext,
                                                         const T *__restrict__ ggram, float l1, float gram, const float *__restrict__ gscale,
                                                         T *__restrict__ df) {
    const float gs = *gscale;
    const long long nv = 2LL * n * img / 8;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < nv; i += (long long)gridDim.x * LT) {
        const long long e = i * 8;
        const long long im = e / img, eo = (2LL * n + im % n) * img + e % img;
        float a[8], o[8], r[8], gg[8], gn[8];
        Vec8<T>::load(f + e, a);
        Vec8<T>::load(f + eo, o);
        if (ggram) Vec8<T>::load(ggram + e, gg);
        if (gnext) Vec8<T>::load(gnext + e, gn);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float v = l1 * sgnf(a[k] - o[k]);
            if (ggram) v += gram * gg[k];
            v *= gs;
            r[k] = gnext ? v + gn[k] : v;
        }
        Vec8<T>::store(df + e, r);
    }
}

// g: [3n][c][c] unnormalised Gram products (F F^T); sums[0] += sum |G_comp/norm - G_origin/norm|, sums[1] the same for output
__global__ void __launch_bounds__(LT) gram_l1_kernel(const float *__restrict__ g, int n, int c, float norm, double *__restrict__ sums) {
    double acc[2] = {0.0, 0.0};
    const long long cc = (long long)c * c, total = (long long)n * cc;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < total; i += (long long)gridDim.x * LT) {
        const float o = g[2LL * n * cc + i] / norm;
        acc[0] += fabsf(g[i] / norm - o);
        acc[1] += fabsf(g[(long long)n * cc + i] / norm - o);
    }
    block_sum_atomic<2>(acc, sums);
}

// t[i][a][b] = S[a][b] + S[b][a], S = sign(G_i / norm - G_origin / norm), for the 2n images comp | output: the (symmetric,
// integer-valued, so bf16-exact) operand of the Gram backward dF = F (S + S^T) * k
__global__ void __launch_bounds__(LT) gram_sign_kernel(const float *__restrict__ g, int n, int c, float norm, float *__restrict__ t) {
    const long long cc = (long long)c * c, total = 2LL * n * cc;
    for (long long i = blockIdx.x * (long long)LT + threadIdx.x; i < total; i += (long long)gridDim.x * LT) {
        const long long im = i / cc, e = i % cc;
        const int a = (int)(e / c), b = (int)(e % c);
        const float *go = g + (2LL * n + im % n) * cc, *gi = g + im * cc;
        t[i] = sgnf(gi[e] / norm - go[e] / norm) + sgnf(gi[(long long)b * c + a] / norm - go[(long long)b * c + a] / norm);
    }
}

// Data gradient of a 3x3 / pad 1 convolution with 3 input channels (VGG16 conv1_1), kernel-to-row form (DESIGN 4.4): the 1x1
// problem Z[p][tap*3 + ci] = sum_co dc[p][co] W[co][ci][tap] runs on the tensor-core forward kernel with this [32][cout] weight
// (rows 27..31 zero) ...
__global__ void __launch_bounds__(LT) k2r_image_weight_kernel(const float *__restrict__ w_oihw, int cout, float *__restrict__ wz) {
    const int i = blockIdx.x * LT + threadIdx.x;
    if (i >= 32 * cout) return;
    const int j = i / cout, co = i % cout;
    const int tap = j / 3, ci = j % 3;
    wz[i] = j < 27 ? w_oihw[(co * 3 + ci) * 9 + tap] : 0.f;
}

// ... and this streaming pass sums the taps: dx[q][ci] = sum_tap Z[q - (tap_r - 1, tap_c - 1)][tap*3 + ci] (pixels outside the
// image contribute nothing), one thread per pixel; dx: [n][h][w][8], channels 3..7 zero
template <typename T>
__global__ void __launch_bounds__(LT) k2r_image_dgrad_kernel(const T *__restrict__ z, int n, int h, int w, T *__restrict__ dx) {
    const long long npix = (long long)n * h * w;
    for (long long p = blockIdx.x * (long long)LT + threadIdx.x; p < npix; p += (long long)gridDim.x * LT) {
        const int x = (int)(p % w), y = (int)((p / w) % h);
        const long long img = p - (long long)y * w - x;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int tr = 0; tr < 3; ++tr) {
            const int yy = y - tr + 1;
            if (yy < 0 || yy >= h) continue;
#pragma unroll
            for (int tc = 0; tc < 3; ++tc) {
                const int xx = x - tc + 1;
                if (xx < 0 || xx >= w) continue;
                const T *zr = z + (img + (long long)yy * w + xx) * 32 + (tr * 3 + tc) * 3;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) acc[ci] += to_f32(zr[ci]);
            }
        }
        Vec8<T>::store(dx + p * 8, acc);
    }
}

struct LossInv { double v[16]; };

// terms = {valid, hole, tv, perceptual, style} (unweighted), loss = 1 valid + 6 hole + 0.1 tv + 0.05 perceptual + 120 style
__global__ void loss_finalize_kernel(const double *__restrict__ s, LossInv inv, float *__restrict__ loss, float *__restrict__ terms) {
    const double valid = s[0] * inv.v[0], hole = s[1] * inv.v[1], tv = s[2] * inv.v[2] + s[3] * inv.v[3];
    double perc = 0.0, style = 0.0;
    for (int k = 0; k < 3; ++k) {
        perc += (s[4 + 2 * k] + s[5 + 2 * k]) * inv.v[4 + 2 * k];
        style += (s[10 + 2 * k] + s[11 + 2 * k]) * inv.v[10 + 2 * k];
    }
    terms[0] = (float)valid; terms[1] = (float)hole; terms[2] = (float)tv; terms[3] = (float)perc; terms[4] = (float)style;
    *loss = (float)(1.0 * valid + 6.0 * hole + 0.1 * tv + 0.05 * perc + 120.0 * style);
}

Img img_of(const long long *s) { return Img{s[0], s[1], s[2], s[3]}; }

}  // namespace

#define PCB_API extern "C" __attribute__((visibility("default")))

PCB_API int pcb_inpaint_loss_pixel_forward(const float *raw, const float *origin, const void *output, int out_dtype, const long long *out_strides,
                                           const uint8_t *plane, int n, int h, int w, void *vgg_in, int dtype, double *sums,
                                           pcb_stream_t stream) {
    PCB_CHECK(raw && origin && output && out_strides && plane && vgg_in && sums && n > 0 && h > 1 && w > 1,
              "pcb_inpaint_loss_pixel_forward: bad arguments");
    PCB_CHECK((reinterpret_cast<uintptr_t>(vgg_in) & 15) == 0, "pcb_inpaint_loss_pixel_forward: vgg_in must be 16-byte aligned");
    const Img so = img_of(out_strides);
    const int grid = grid_for((long long)n * h * w);
#define PIX_FWD(TO, TX) pixel_fwd_kernel<TO, TX><<<grid, LT, 0, ST>>>(raw, origin, static_cast<const TO *>(output), so, plane, n, h, w, \
                                                                      static_cast<TX *>(vgg_in), sums)
    if (out_dtype == PCB_BF16) { if (dtype == PCB_BF16) PIX_FWD(bf16, bf16); else PIX_FWD(bf16, float); }
    else { if (dtype == PCB_BF16) PIX_FWD(float, bf16); else PIX_FWD(float, float); }
#undef PIX_FWD
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_inpaint_loss_pixel_backward(const float *raw, const float *origin, const void *output, int out_dtype,
                                            const long long *out_strides, const uint8_t *plane, int n, int h, int w, const void *dvgg_in,
                                            int dtype, const float *coef, const float *gscale, void *grad, const long long *grad_strides,
                                            pcb_stream_t stream) {
    PCB_CHECK(raw && origin && output && out_strides && plane && coef && gscale && grad && grad_strides && n > 0 && h > 1 && w > 1,
              "pcb_inpaint_loss_pixel_backward: bad arguments");
    const Img so = img_of(out_strides), sg = img_of(grad_strides);
    const float4 co = make_float4(coef[0], coef[1], coef[2], coef[3]);
    const int grid = grid_for((long long)n * h * w);
#define PIX_BWD(TO, TX) pixel_bwd_kernel<TO, TX><<<grid, LT, 0, ST>>>(raw, origin, static_cast<const TO *>(output), so, plane, n, h, w, \
                                                                      static_cast<const TX *>(dvgg_in), co, gscale, static_cast<TO *>(grad), sg)
    if (out_dtype == PCB_BF16) { if (dtype == PCB_BF16) PIX_BWD(bf16, bf16); else PIX_BWD(bf16, float); }
    else { if (dtype == PCB_BF16) PIX_BWD(float, bf16); else PIX_BWD(float, float); }
#undef PIX_BWD
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_maxpool2x2_forward(const void *x, void *y, int dtype, int n, int h, int w, int c, pcb_stream_t stream) {
    PCB_CHECK(x && y && n > 0 && h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && c > 0 && c % 8 == 0,
              "pcb_maxpool2x2_forward: needs even h, w and c %% 8 == 0");
    const int grid = grid_for((long long)n * (h / 2) * (w / 2) * (c / 8));
    if (dtype == PCB_BF16) maxpool_fwd_kernel<bf16><<<grid, LT, 0, ST>>>(static_cast<const bf16 *>(x), static_cast<bf16 *>(y), n, h, w, c);
    else maxpool_fwd_kernel<float><<<grid, LT, 0, ST>>>(static_cast<const float *>(x), static_cast<float *>(y), n, h, w, c);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_maxpool2x2_backward(const void *gy, const void *x, void *gx, int dtype, int n, int h, int w, int c, int relu_mask,
                                    pcb_stream_t stream) {
    PCB_CHECK(gy && x && gx && n > 0 && h >= 2 && w >= 2 && h % 2 == 0 && w % 2 == 0 && c > 0 && c % 8 == 0,
              "pcb_maxpool2x2_backward: needs even h, w and c %% 8 == 0");
    const int grid = grid_for((long long)n * (h / 2) * (w / 2) * (c / 8));
    if (dtype == PCB_BF16)
        maxpool_bwd_kernel<bf16><<<grid, LT, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), static_cast<bf16 *>(gx), n, h, w, c,
                                                      relu_mask);
    else
        maxpool_bwd_kernel<float><<<grid, LT, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), static_cast<float *>(gx), n, h, w,
                                                       c, relu_mask);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_feature_l1_forward(const void *f, int dtype, int n, long long hw, int c, double *sums, pcb_stream_t stream) {
    PCB_CHECK(f && sums && n > 0 && hw > 0 && c % 8 == 0, "pcb_feature_l1_forward: bad arguments");
    const long long img = hw * c;
    const int grid = grid_for((long long)n * img / 8);
    if (dtype == PCB_BF16) feature_l1_kernel<bf16><<<grid, LT, 0, ST>>>(static_cast<const bf16 *>(f), n, img, sums);
    else feature_l1_kernel<float><<<grid, LT, 0, ST>>>(static_cast<const float *>(f), n, img, sums);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_feature_loss_backward(const void *f, int dtype, int n, long long hw, int c, const void *g_next, const void *g_gram, float l1_coef,
                                      float gram_coef, const float *gscale, void *df, pcb_stream_t stream) {
    PCB_CHECK(f && gscale && df && n > 0 && hw > 0 && c % 8 == 0, "pcb_feature_loss_backward: bad arguments");
    const long long img = hw * c;
    const int grid = grid_for(2LL * n * img / 8);
    if (dtype == PCB_BF16)
        feature_bwd_kernel<bf16><<<grid, LT, 0, ST>>>(static_cast<const bf16 *>(f), n, img, static_cast<const bf16 *>(g_next),
                                                      static_cast<const bf16 *>(g_gram), l1_coef, gram_coef, gscale, static_cast<bf16 *>(df));
    else
        feature_bwd_kernel<float><<<grid, LT, 0, ST>>>(static_cast<const float *>(f), n, img, static_cast<const float *>(g_next),
                                                       static_cast<const float *>(g_gram), l1_coef, gram_coef, gscale, static_cast<float *>(df));
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_gram_l1_forward(const float *gram, int n, int c, float norm, double *sums, pcb_stream_t stream) {
    PCB_CHECK(gram && sums && n > 0 && c > 0 && norm > 0.f, "pcb_gram_l1_forward: bad arguments");
    gram_l1_kernel<<<grid_for((long long)n * c * c), LT, 0, ST>>>(gram, n, c, norm, sums);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_gram_sign_sym(const float *gram, int n, int c, float norm, float *t, pcb_stream_t stream) {
    PCB_CHECK(gram && t && n > 0 && c > 0 && norm > 0.f, "pcb_gram_sign_sym: bad arguments");
    gram_sign_kernel<<<grid_for(2LL * n * c * c), LT, 0, ST>>>(gram, n, c, norm, t);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_k2r_image_weight(const float *w_oihw, int cout, float *wz, pcb_stream_t stream) {
    PCB_CHECK(w_oihw && wz && cout > 0, "pcb_k2r_image_weight: bad arguments");
    k2r_image_weight_kernel<<<(32 * cout + LT - 1) / LT, LT, 0, ST>>>(w_oihw, cout, wz);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_k2r_image_dgrad(const void *z, int dtype, int n, int h, int w, void *dx, pcb_stream_t stream) {
    PCB_CHECK(z && dx && n > 0 && h > 0 && w > 0, "pcb_k2r_image_dgrad: bad arguments");
    const int grid = grid_for((long long)n * h * w);
    if (dtype == PCB_BF16) k2r_image_dgrad_kernel<bf16><<<grid, LT, 0, ST>>>(static_cast<const bf16 *>(z), n, h, w, static_cast<bf16 *>(dx));
    else k2r_image_dgrad_kernel<float><<<grid, LT, 0, ST>>>(static_cast<const float *>(z), n, h, w, static_cast<float *>(dx));
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_inpaint_loss_finalize(const double *sums, const double *h_inv, float *loss, float *terms, pcb_stream_t stream) {
    PCB_CHECK(sums && h_inv && loss && terms, "pcb_inpaint_loss_finalize: bad arguments");
    LossInv inv;
    for (int k = 0; k < 16; ++k) inv.v[k] = h_inv[k];
    loss_finalize_kernel<<<1, 1, 0, ST>>>(sums, inv, loss, terms);
    PCB_LAUNCH_CHECK();
    return 0;
}

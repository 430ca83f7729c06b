// dwconv.cu -- depthwise 3x3 convolution (groups == channels) at a power-of-two stride, the HBM-bound half of the depthwise-separable
// blocks: DSConvBlock (models/BaseModels.py:105-127), InvertedResidual / RFB branches (models/MobileNetV2.py:136-138,
// models/common.py:136-143: dilation up to 29), and the depthwise PARTIAL convolutions of PartialInvertedResidual
// (models/MobileNetV2.py:174-176).  NHWC, 8 channels (16 B of bf16 / 32 B of fp32) per thread, fp32 accumulation;
// one read of x and one write of y per element is the roofline (weights are k*k*C, negligible).
// It is an internal fast path of pcb_pconv_forward / backward_* (same semantics: optional hole mask with zero-fill,
// mask-sum renormalisation, `plain` mode for ordinary convolutions); every other depthwise shape runs on the shape-general
// kernels of conv_generic.cu.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"

namespace {

// eval-mode BatchNorm + activation in the forward epilogue of the 3x3 kernels (see pcb_ep); on == 0: off
struct DwEp { const float *scale, *shift; int on, act; float slope; };

inline DwEp dw_ep(const pcb_ep *e) {
    DwEp d;
    memset(&d, 0, sizeof(d));
    if (e != nullptr) { d.on = 1; d.scale = e->scale; d.shift = e->shift; d.act = e->act; d.slope = e->slope; }
    return d;
}

struct DwParams {
    int n, h, w, c, stride, pad_h, pad_w, dil, ho, wo;
    int x_cstride, y_cstride;
    const uint8_t *mask;     // input hole plane [n, h>>mup, w>>mup] or null
    int mup;
    const float *msum;       // [mg][n*ho*wo] or null (plain): renormaliser
    int mg;                  // 1, or c (per-channel sums: groups > 1 && !same_holes)
    int no_guard;
    DwEp ep;
};

__device__ __forceinline__ bool dw_mask(const DwParams &P, int nn, int hi, int wi) {
    if (!P.mask) return true;
    return P.mask[(static_cast<long long>(nn) * (P.h >> P.mup) + (hi >> P.mup)) * (P.w >> P.mup) + (wi >> P.mup)] != 0;
}

// =================================================================================================================
// 3x3 depthwise kernels, second generation (any power-of-two stride / dilation).  A thread per output element spends most of
// its instructions on 64-bit index divisions and reloads the nine weight vectors for every output: it is issue-bound, not
// bandwidth-bound.  Here
//   * a block owns a chunk of `cvb` channel vectors (8 channels each) x PL pixel lanes; a thread keeps ONE channel vector for
//     its whole life, so the nine weight vectors (fwd / dgrad) or the nine gradient accumulators (wgrad) live in registers,
//   * rows are walked by blockIdx.y in groups, pixels of a row by the PL lanes: all index math is 32-bit adds,
//   * consecutive threads read consecutive 16-byte vectors of the same pixel (coalesced 16 * cvb byte segments), the 3x3
//     neighbourhood re-reads hit L1 / L2,
//   * the weight-gradient partials of the PL lanes are summed through shared memory in parallel and leave the block as one
//     atomic per (channel, tap).
// =================================================================================================================
struct Dw3Geom { int cvb, pl, chunks; };

inline Dw3Geom dw3_geom(int c) {
    const int cv = c >> 3;
    Dw3Geom g;
    g.cvb = 1;
    for (int d = 1; d <= 32 && d <= cv; ++d)
        if (cv % d == 0) g.cvb = d;                 // largest divisor of cv that is <= 32
    if (g.cvb < 8 && cv > 32) g.cvb = 32;           // awkward channel counts: 32-wide chunks, the last one partly idle
    g.pl = 256 / g.cvb;
    g.chunks = (cv + g.cvb - 1) / g.cvb;
    return g;
}

template <typename T> __device__ __forceinline__ void dw3_load_weights(const T *__restrict__ w_t, int c, int ch, float (&wt)[9][8]) {
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) Vec8<T>::load(w_t + static_cast<long long>(tap) * c + ch, wt[tap]);
}

constexpr int DW3_ROWS = 8;                         // output rows per block (forward / dgrad)

// EP: eval-mode BatchNorm + activation before the store (inference: never together with the statistics)
template <typename T, bool PLAIN, bool EP>
__global__ void __launch_bounds__(256) dw3_fwd_kernel(const DwParams P, const T *__restrict__ x, const T *__restrict__ w_t,
                                                      const float *__restrict__ bias, T *__restrict__ y, int cvb, int pl,
                                                      double *__restrict__ bn_sums) {
    __shared__ float s_stat[256][2];
    const int vl = static_cast<int>(threadIdx.x) % cvb;
    const int v = blockIdx.x * cvb + vl, lane_px = static_cast<int>(threadIdx.x) / cvb;
    const bool active = lane_px < pl && v < (P.c >> 3);
    if (!active && (EP || bn_sums == nullptr)) return;
    const int ch = v * 8;
    float wt[9][8], bs[8], st_s[8], st_q[8], es[8], eh[8];
    if (active) dw3_load_weights(w_t, P.c, ch, wt);
#pragma unroll
    for (int j = 0; j < 8; ++j) { bs[j] = (active && bias) ? bias[ch + j] : 0.f; st_s[j] = 0.f; st_q[j] = 0.f; es[j] = 1.f; eh[j] = 0.f; }
    if (EP && active && P.ep.scale) { Vec8<float>::load(P.ep.scale + ch, es); Vec8<float>::load(P.ep.shift + ch, eh); }
    const int rows_total = P.n * P.ho;
    const long long total = static_cast<long long>(rows_total) * P.wo;
    for (int rr = 0; rr < DW3_ROWS; ++rr) {
        const int row = blockIdx.y * DW3_ROWS + rr;
        if (row >= rows_total || !active) break;
        const int nn = row / P.ho, oh = row - nn * P.ho;
        const int hi0 = oh * P.stride - P.pad_h;
        for (int ow = lane_px; ow < P.wo; ow += pl) {
            const int wi0 = ow * P.stride - P.pad_w;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
            for (int tr = 0; tr < 3; ++tr) {
                const int hi = hi0 + tr * P.dil;
                if (hi < 0 || hi >= P.h) continue;
                const T *xrow = x + static_cast<long long>(nn * P.h + hi) * P.w * P.x_cstride + ch;
#pragma unroll
                for (int tc = 0; tc < 3; ++tc) {
                    const int wi = wi0 + tc * P.dil;
                    if (wi < 0 || wi >= P.w) continue;
                    if (!PLAIN && !dw_mask(P, nn, hi, wi)) continue;
                    float xv[8];
                    Vec8<T>::load(xrow + static_cast<long long>(wi) * P.x_cstride, xv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv[j], wt[tr * 3 + tc][j], acc[j]);
                }
            }
            const long long m = static_cast<long long>(row) * P.wo + ow;
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (PLAIN) { o[j] = acc[j] + bs[j]; continue; }
                const float s = P.msum[(P.mg == 1 ? 0 : static_cast<long long>(ch + j) * total) + m];
                if (P.no_guard) o[j] = acc[j] / s + bs[j];
                else o[j] = (s == 0.f) ? 0.f : acc[j] / s + bs[j];
            }
            if (EP) {                                   // eval-mode BatchNorm + activation: holes become apply_act(shift)
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = apply_act(fmaf(o[j], es[j], eh[j]), P.ep.act, P.ep.slope);
            }
            Vec8<T>::store(y + m * P.y_cstride + ch, o);
            if (!EP && bn_sums != nullptr) {            // BatchNorm statistics of what was stored (bf16-rounded in bf16 mode)
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float r = to_f32(from_f32<T>(o[j])); st_s[j] += r; st_q[j] = fmaf(r, r, st_q[j]); }
            }
        }
    }
    if (!EP && bn_sums != nullptr) {
        // fused statistics pass of the BatchNorm that follows the depthwise convolution (BaseModels.py:95-99): per channel,
        // the PL pixel lanes' partial sums are added through shared memory; one fp64 atomic per channel and block
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            __syncthreads();
            s_stat[threadIdx.x][0] = active ? st_s[j] : 0.f;
            s_stat[threadIdx.x][1] = active ? st_q[j] : 0.f;
            __syncthreads();
            for (int col = threadIdx.x; col < cvb * 2; col += 256) {
                const int cvl = col >> 1, q = col & 1;
                const int vv = blockIdx.x * cvb + cvl;
                if (vv >= (P.c >> 3)) continue;
                float tot = 0.f;
                for (int l = 0; l < pl; ++l) tot += s_stat[l * cvb + cvl][q];
                atomicAdd(bn_sums + static_cast<long long>(q) * P.c + vv * 8 + j, static_cast<double>(tot));
            }
        }
    }
}

// dx[p][c] = mask(p) * sum_taps dc[(p + pad - tap*dil) / stride][c] * w[tap][c]   (stride is a power of two)
template <typename T, bool PLAIN>
__global__ void __launch_bounds__(256) dw3_dgrad_kernel(const DwParams P, const T *__restrict__ dc, int dc_cstride, const T *__restrict__ w_t,
                                                        T *__restrict__ dx, int dx_cstride, int cvb, int pl, int sshift) {
    const int v = blockIdx.x * cvb + static_cast<int>(threadIdx.x) % cvb, lane_px = static_cast<int>(threadIdx.x) / cvb;
    if (lane_px >= pl || v >= (P.c >> 3)) return;
    const int ch = v * 8;
    float wt[9][8];
    dw3_load_weights(w_t, P.c, ch, wt);
    const int rows_total = P.n * P.h, smask = P.stride - 1;
    for (int rr = 0; rr < DW3_ROWS; ++rr) {
        const int row = blockIdx.y * DW3_ROWS + rr;
        if (row >= rows_total) break;
        const int nn = row / P.h, ih = row - nn * P.h;
        for (int iw = lane_px; iw < P.w; iw += pl) {
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = 0.f;
            if (PLAIN || dw_mask(P, nn, ih, iw)) {
#pragma unroll
                for (int tr = 0; tr < 3; ++tr) {
                    const int th = ih + P.pad_h - tr * P.dil;
                    if (th < 0 || (th & smask)) continue;
                    const int oh = th >> sshift;
                    if (oh >= P.ho) continue;
                    const T *drow = dc + static_cast<long long>(nn * P.ho + oh) * P.wo * dc_cstride + ch;
#pragma unroll
                    for (int tc = 0; tc < 3; ++tc) {
                        const int tw = iw + P.pad_w - tc * P.dil;
                        if (tw < 0 || (tw & smask)) continue;
                        const int ow = tw >> sshift;
                        if (ow >= P.wo) continue;
                        float dv[8];
                        Vec8<T>::load(drow + static_cast<long long>(ow) * dc_cstride, dv);
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[j] = fmaf(dv[j], wt[tr * 3 + tc][j], acc[j]);
                    }
                }
            }
            Vec8<T>::store(dx + (static_cast<long long>(row) * P.w + iw) * dx_cstride + ch, acc);
        }
    }
}

// dw[c][tap] += sum over output pixels of dc[p][c] * (x*m)[p @ tap][c]
template <typename T, bool PLAIN>
__global__ void __launch_bounds__(256) dw3_wgrad_kernel(const DwParams P, const T *__restrict__ dc, int dc_cstride, const T *__restrict__ x,
                                                        float *__restrict__ dw, int cvb, int pl, int rows_per_block) {
    __shared__ float s_red[256][9];
    const int vl = static_cast<int>(threadIdx.x) % cvb, lane_px = static_cast<int>(threadIdx.x) / cvb;
    const int v = blockIdx.x * cvb + vl;
    const bool active = lane_px < pl && v < (P.c >> 3);
    const int ch = v * 8;
    float acc[9][8];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[tap][j] = 0.f;
    const int rows_total = P.n * P.ho;
    if (active) {
        for (int rr = 0; rr < rows_per_block; ++rr) {
            const int row = blockIdx.y * rows_per_block + rr;
            if (row >= rows_total) break;
            const int nn = row / P.ho, oh = row - nn * P.ho;
            const int hi0 = oh * P.stride - P.pad_h;
            const T *dcrow = dc + static_cast<long long>(row) * P.wo * dc_cstride + ch;
            for (int ow = lane_px; ow < P.wo; ow += pl) {
                float dv[8];
                Vec8<T>::load(dcrow + static_cast<long long>(ow) * dc_cstride, dv);
                const int wi0 = ow * P.stride - P.pad_w;
#pragma unroll
                for (int tr = 0; tr < 3; ++tr) {
                    const int hi = hi0 + tr * P.dil;
                    if (hi < 0 || hi >= P.h) continue;
                    const T *xrow = x + static_cast<long long>(nn * P.h + hi) * P.w * P.x_cstride + ch;
#pragma unroll
                    for (int tc = 0; tc < 3; ++tc) {
                        const int wi = wi0 + tc * P.dil;
                        if (wi < 0 || wi >= P.w) continue;
                        if (!PLAIN && !dw_mask(P, nn, hi, wi)) continue;
                        float xv[8];
                        Vec8<T>::load(xrow + static_cast<long long>(wi) * P.x_cstride, xv);
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[tr * 3 + tc][j] = fmaf(dv[j], xv[j], acc[tr * 3 + tc][j]);
                    }
                }
            }
        }
    }
    // per channel j of the vector: stage the 9 tap partials of every thread, then cvb * 9 threads each sum one (vector, tap) column
    // over the PL pixel lanes and leave with ONE atomic
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        __syncthreads();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) s_red[threadIdx.x][tap] = active ? acc[tap][j] : 0.f;
        __syncthreads();
        for (int col = threadIdx.x; col < cvb * 9; col += 256) {
            const int cvl = col / 9, tap = col - cvl * 9;
            const int vv = blockIdx.x * cvb + cvl;
            if (vv >= (P.c >> 3)) continue;
            float tot = 0.f;
            for (int l = 0; l < pl; ++l) tot += s_red[l * cvb + cvl][tap];
            atomicAdd(dw + static_cast<long long>(vv * 8 + j) * 9 + tap, tot);
        }
    }
}


// =================================================================================================================
// 3x3 depthwise, stride 1, padding == dilation (every depthwise layer of the reference's segmentation networks), ordinary
// (mask-free) convolution: third generation.  The second generation issues nine 16-byte loads per output vector whose vertical
// re-use distance (dilation x row x channels) exceeds L1 at large dilations, i.e. up to 9x the algorithmic bytes out of L2.  Here
//   * a thread owns one output COLUMN x one channel QUAD (4 channels, 8-byte accesses) and walks down the rows of ONE
//     dilation phase (rows a, a+d, a+2d, ...): a dilated 3x3 convolution is a plain 3x3 convolution inside each phase, so
//     every input row is loaded once per thread (its three horizontal taps x-d, x, x+d) and scattered into the three output
//     rows it contributes to, which live in registers (a sliding window of accumulators) -- 3 loads per output instead of 9,
//     two of them L1 hits (the row segment is shared with the neighbouring columns of the block);
//   * weights (9 x 4 floats) and, for the weight gradient, the 9 x 4 partial sums stay in registers;
//   * the same kernel computes the data gradient (taps flipped, dc in the role of x);
//   * the forward can accumulate the BatchNorm statistics of its output (see dw3_fwd_kernel).
// =================================================================================================================
template <typename T> struct Vec4;
template <> struct Vec4<bf16> {
    static __device__ __forceinline__ void load(const bf16 *p, float (&v)[4]) {
        const uint2 r = *reinterpret_cast<const uint2 *>(p);
        v[0] = __uint_as_float(r.x << 16); v[1] = __uint_as_float(r.x & 0xffff0000u);
        v[2] = __uint_as_float(r.y << 16); v[3] = __uint_as_float(r.y & 0xffff0000u);
    }
    static __device__ __forceinline__ void store(bf16 *p, const float (&v)[4]) {
        __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
        uint2 r;
        r.x = *reinterpret_cast<uint32_t *>(&a); r.y = *reinterpret_cast<uint32_t *>(&b);
        *reinterpret_cast<uint2 *>(p) = r;
    }
};
template <> struct Vec4<float> {
    static __device__ __forceinline__ void load(const float *p, float (&v)[4]) {
        const float4 a = *reinterpret_cast<const float4 *>(p);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    }
    static __device__ __forceinline__ void store(float *p, const float (&v)[4]) { *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]); }
};

// raw (still packed) 4-channel vector: loaded early, unpacked at use -- a queue of these keeps several rows of loads in flight
template <typename T> struct Raw4;
template <> struct Raw4<bf16> {
    uint2 r;
    __device__ __forceinline__ void zero() { r = make_uint2(0u, 0u); }
    __device__ __forceinline__ void load(const bf16 *p) { r = __ldg(reinterpret_cast<const uint2 *>(p)); }
    __device__ __forceinline__ void unpack(float (&v)[4]) const {
        v[0] = __uint_as_float(r.x << 16); v[1] = __uint_as_float(r.x & 0xffff0000u);
        v[2] = __uint_as_float(r.y << 16); v[3] = __uint_as_float(r.y & 0xffff0000u);
    }
};
template <> struct Raw4<float> {
    float4 r;
    __device__ __forceinline__ void zero() { r = make_float4(0.f, 0.f, 0.f, 0.f); }
    __device__ __forceinline__ void load(const float *p) { r = __ldg(reinterpret_cast<const float4 *>(p)); }
    __device__ __forceinline__ void unpack(float (&v)[4]) const { v[0] = r.x; v[1] = r.y; v[2] = r.z; v[3] = r.w; }
};

struct Dw4Geom { int cq, xt, chunks, xtiles, nseg, rseg, pgroups, ppb; };

inline Dw4Geom dw4_geom(int c, int w, int h, int dil) {
    Dw4Geom g;
    const int quads = c >> 2;
    g.cq = 1;
    for (int d = 1; d <= 32 && d <= quads; ++d)
        if (quads % d == 0) g.cq = d;               // largest divisor of the quad count that is <= 32 (64-byte .. 256-byte pixel segments)
    g.xt = 256 / g.cq;
    if (g.xt > w) g.xt = w;
    g.chunks = quads / g.cq;
    g.xtiles = (w + g.xt - 1) / g.xt;
    const int nj = (h + dil - 1) / dil;              // rows of one phase
    g.rseg = 32;
    g.nseg = (nj + g.rseg - 1) / g.rseg;
    // a block walks `ppb` dilation phases one after the other (short phases -- large dilation -- would otherwise make blocks
    // of a few rows whose weight loads and statistics flush dominate): about 32 rows of work per thread
    g.ppb = 1;
    while (g.ppb * 2 <= dil && g.ppb * 2 * nj <= 32 && dil % (g.ppb * 2) == 0) g.ppb *= 2;
    g.pgroups = dil / g.ppb;
    return g;
}

// y[oy][ox][c] = b[c] + sum_{tr,tc} w[tr][tc][c] * x[oy + (tr-1) d][ox + (tc-1) d][c]      (FLIP: w[2-tr][2-tc], no bias: data gradient)
// The arithmetic works on four channels at a time through pointers that are walked, not re-derived: these kernels are
// ISSUE-bound, not bandwidth-bound (~100 instructions per 16 bytes moved in a scalar version with 64-bit address arithmetic).
struct F4 { float2 lo, hi; };
__device__ __forceinline__ F4 f4_zero() { F4 r; r.lo = make_float2(0.f, 0.f); r.hi = make_float2(0.f, 0.f); return r; }
__device__ __forceinline__ F4 f4_fma(const F4 &a, const F4 &b, const F4 &c) {
    F4 r;
    r.lo = make_float2(fmaf(a.lo.x, b.lo.x, c.lo.x), fmaf(a.lo.y, b.lo.y, c.lo.y));
    r.hi = make_float2(fmaf(a.hi.x, b.hi.x, c.hi.x), fmaf(a.hi.y, b.hi.y, c.hi.y));
    return r;
}
__device__ __forceinline__ F4 f4_mul(const F4 &a, const F4 &b) {
    F4 r; r.lo = make_float2(__fmul_rn(a.lo.x, b.lo.x), __fmul_rn(a.lo.y, b.lo.y)); r.hi = make_float2(__fmul_rn(a.hi.x, b.hi.x), __fmul_rn(a.hi.y, b.hi.y)); return r;
}
__device__ __forceinline__ F4 f4_add(const F4 &a, const F4 &b) {
    F4 r; r.lo = make_float2(__fadd_rn(a.lo.x, b.lo.x), __fadd_rn(a.lo.y, b.lo.y)); r.hi = make_float2(__fadd_rn(a.hi.x, b.hi.x), __fadd_rn(a.hi.y, b.hi.y)); return r;
}
template <typename T> __device__ __forceinline__ F4 f4_of(const Raw4<T> &q) {
    float v[4];
    q.unpack(v);
    F4 r; r.lo = make_float2(v[0], v[1]); r.hi = make_float2(v[2], v[3]);
    return r;
}
template <typename T> __device__ __forceinline__ F4 f4_load(const T *p) { Raw4<T> q; q.load(p); return f4_of(q); }
template <typename T> __device__ __forceinline__ void f4_store(T *p, const F4 &v) {
    const float o[4] = {v.lo.x, v.lo.y, v.hi.x, v.hi.y};
    Vec4<T>::store(p, o);
}
// the value as it will be read back from memory (bf16 mode: rounded), for the fused BatchNorm statistics
template <typename T> __device__ __forceinline__ F4 f4_as_stored(const F4 &v) {
    F4 r;
    r.lo = make_float2(to_f32(from_f32<T>(v.lo.x)), to_f32(from_f32<T>(v.lo.y)));
    r.hi = make_float2(to_f32(from_f32<T>(v.hi.x)), to_f32(from_f32<T>(v.hi.y)));
    return r;
}

constexpr int DW4_QF = 6;                           // forward / data gradient: rows of loads in flight per thread (a multiple of 3)
constexpr int DW4_Q = 3;                            // rows of loads in flight per thread = the period of the accumulator rotation
// EP: eval-mode BatchNorm + activation before the store (forward only; never together with the statistics)
template <typename T, bool FLIP, bool EP>
__global__ void __launch_bounds__(256, 2) dw4_s1_kernel(const T *__restrict__ x, int x_cstride, const T *__restrict__ w_t, const float *__restrict__ bias,
                                                        T *__restrict__ y, int y_cstride, double *__restrict__ bn_sums, const DwEp ep,
                                                        int n, int h, int w, int c, int dil, int cq, int xt, int nseg, int rseg, int ppb) {
    __shared__ float s_stat[256][2];
    const int ql = static_cast<int>(threadIdx.x) % cq, xl = static_cast<int>(threadIdx.x) / cq;
    const int ch = (blockIdx.x * cq + ql) * 4, ox = blockIdx.y * xt + xl;
    const bool active = xl < xt && ox < w;
    int z = blockIdx.z;
    const int seg = z % nseg; z /= nseg;
    const int pgroups = dil / ppb;
    const int pg = z % pgroups, nn = z / pgroups;
    // weights stay PACKED (bf16: 2 registers per tap instead of 4) and are unpacked at use: the 18 registers this frees pay for a
    // six-row load queue -- these kernels are bound by bytes in flight per SM, not by issue slots
    constexpr int QF = sizeof(T) == 2 ? DW4_QF : DW4_Q;          // fp32 storage (exact mode): raw rows are twice as wide
    Raw4<T> wt[3][3];
    F4 bs = f4_zero(), st_s = f4_zero(), st_q = f4_zero(), es, eh = f4_zero();
    es.lo = es.hi = make_float2(1.f, 1.f);
    if (EP && ep.scale) {
        const float4 a = *reinterpret_cast<const float4 *>(ep.scale + ch), b = *reinterpret_cast<const float4 *>(ep.shift + ch);
        es.lo = make_float2(a.x, a.y); es.hi = make_float2(a.z, a.w); eh.lo = make_float2(b.x, b.y); eh.hi = make_float2(b.z, b.w);
    }
#pragma unroll
    for (int tr = 0; tr < 3; ++tr)
#pragma unroll
        for (int tc = 0; tc < 3; ++tc) {
            const int tap = FLIP ? (2 - tr) * 3 + (2 - tc) : tr * 3 + tc;
            wt[tr][tc].load(w_t + static_cast<long long>(tap) * c + ch);
        }
    if (bias && !FLIP) { bs.lo = make_float2(bias[ch], bias[ch + 1]); bs.hi = make_float2(bias[ch + 2], bias[ch + 3]); }
    if (active) {
        const bool cl = ox - dil >= 0, cr = ox + dil < w;
        const long long xoff_l = -static_cast<long long>(dil) * x_cstride, xoff_r = static_cast<long long>(dil) * x_cstride;
        const long long xrow = static_cast<long long>(dil) * w * x_cstride, yrow = static_cast<long long>(dil) * w * y_cstride;
        for (int a = pg * ppb; a < (pg + 1) * ppb; ++a) {
            const int nj = (h - a + dil - 1) / dil;                    // rows of this phase: iy = a + dil * i, i in [0, nj)
            const int j0 = seg * rseg, j1 = min(nj, j0 + rseg);        // output sub-rows of this segment
            if (j0 >= nj) continue;
            const int i_lo = max(j0 - 1, 0), i_hi = min(j1 + 1, nj);   // input sub-rows [i_lo, i_hi)
            // running pointers: next row to fetch, next row to store
            const T *pf = x + ((static_cast<long long>(nn) * h + a + static_cast<long long>(dil) * i_lo) * w + ox) * x_cstride + ch;
            T *ps = y + ((static_cast<long long>(nn) * h + a + static_cast<long long>(dil) * j0) * w + ox) * y_cstride + ch;
            int fetched = i_lo;
            Raw4<T> q[QF][3];
            auto fetch = [&](Raw4<T> (&dst)[3]) {
                dst[0].zero(); dst[1].zero(); dst[2].zero();
                if (fetched < i_hi) {
                    dst[1].load(pf);
                    if (cl) dst[0].load(pf + xoff_l);
                    if (cr) dst[2].load(pf + xoff_r);
                }
                ++fetched; pf += xrow;
            };
#pragma unroll
            for (int k = 0; k < QF; ++k) fetch(q[k]);
            auto emit = [&](const F4 &accv) {
                F4 o = f4_add(accv, bs);
                if (EP) {                                      // eval-mode BatchNorm + activation
                    o = f4_fma(o, es, eh);
                    o.lo = make_float2(apply_act(o.lo.x, ep.act, ep.slope), apply_act(o.lo.y, ep.act, ep.slope));
                    o.hi = make_float2(apply_act(o.hi.x, ep.act, ep.slope), apply_act(o.hi.y, ep.act, ep.slope));
                }
                f4_store<T>(ps, o);
                ps += yrow;
                if (!EP && bn_sums != nullptr) { const F4 r = f4_as_stored<T>(o); st_s = f4_add(st_s, r); st_q = f4_fma(r, r, st_q); }
            };
            // three accumulators in rotating roles (period 3; QF is a multiple of it): while input sub-row i is processed, `top` belongs to
            // output row i-1 (receives tap row 2 and is complete), `mid` to output i (tap row 1), `bot` to output i+1 (tap row 0)
            F4 acc[3] = {f4_zero(), f4_zero(), f4_zero()};
            for (int i0 = i_lo; i0 < i_hi; i0 += QF) {
#pragma unroll
                for (int k = 0; k < QF; ++k) {
                    const int i = i0 + k;
                    if (i < i_hi) {
                        const F4 x0 = f4_of(q[k][0]), x1 = f4_of(q[k][1]), x2 = f4_of(q[k][2]);
                        fetch(q[k]);                                   // refill the slot: QF rows of loads stay in flight
                        F4 &top = acc[k % 3], &mid = acc[(k + 1) % 3], &bot = acc[(k + 2) % 3];
                        top = f4_fma(f4_of(wt[2][0]), x0, f4_fma(f4_of(wt[2][1]), x1, f4_fma(f4_of(wt[2][2]), x2, top)));
                        mid = f4_fma(f4_of(wt[1][0]), x0, f4_fma(f4_of(wt[1][1]), x1, f4_fma(f4_of(wt[1][2]), x2, mid)));
                        bot = f4_fma(f4_of(wt[0][0]), x0, f4_fma(f4_of(wt[0][1]), x1, f4_mul(f4_of(wt[0][2]), x2)));
                        if (i - 1 >= j0) emit(top);                    // complete: it just received its bottom tap row
                    }
                }
            }
            // the last input row of the PHASE has no row below it: its own output is complete as well.  It sits in the
            // accumulator that was `mid` at the last processed row i_hi - 1, i.e. role index (i_hi - 1 - i_lo + 1) % 3.
            if (j1 == nj && j1 - 1 >= j0) {
                const int role = (i_hi - i_lo) % 3;                    // (selected without dynamic register indexing)
                emit(role == 0 ? acc[0] : (role == 1 ? acc[1] : acc[2]));
            }
        }
    }
    if (!EP && bn_sums != nullptr) {
        const float ss[4] = {st_s.lo.x, st_s.lo.y, st_s.hi.x, st_s.hi.y}, sq[4] = {st_q.lo.x, st_q.lo.y, st_q.hi.x, st_q.hi.y};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            __syncthreads();
            s_stat[threadIdx.x][0] = active ? ss[j] : 0.f;
            s_stat[threadIdx.x][1] = active ? sq[j] : 0.f;
            __syncthreads();
            for (int col = threadIdx.x; col < cq * 2; col += 256) {
                const int cql = col >> 1, qq = col & 1;
                float tot = 0.f;
                for (int l = 0; l < xt; ++l) tot += s_stat[l * cq + cql][qq];
                atomicAdd(bn_sums + static_cast<long long>(qq) * c + (blockIdx.x * cq + cql) * 4 + j, static_cast<double>(tot));
            }
        }
    }
}

// dw[c][tr][tc] += sum_{oy,ox} dc[oy][ox][c] * x[oy + (tr-1) d][ox + (tc-1) d][c]
template <typename T>
__global__ void __launch_bounds__(256, 2) dw4_s1_wgrad_kernel(const T *__restrict__ x, int x_cstride, const T *__restrict__ dc, int dc_cstride,
                                                              float *__restrict__ dw, int n, int h, int w, int c, int dil, int cq, int xt, int nseg, int rseg,
                                                              int ppb) {
    __shared__ float s_red[256][9];
    const int ql = static_cast<int>(threadIdx.x) % cq, xl = static_cast<int>(threadIdx.x) / cq;
    const int ch = (blockIdx.x * cq + ql) * 4, ox = blockIdx.y * xt + xl;
    const bool active = xl < xt && ox < w;
    int z = blockIdx.z;
    const int seg = z % nseg; z /= nseg;
    const int pgroups = dil / ppb;
    const int pg = z % pgroups, nn = z / pgroups;
    F4 acc[3][3];
#pragma unroll
    for (int tr = 0; tr < 3; ++tr)
#pragma unroll
        for (int tc = 0; tc < 3; ++tc) acc[tr][tc] = f4_zero();
    if (active) {
        const bool cl = ox - dil >= 0, cr = ox + dil < w;
        const long long xoff_l = -static_cast<long long>(dil) * x_cstride, xoff_r = static_cast<long long>(dil) * x_cstride;
        const long long xrow = static_cast<long long>(dil) * w * x_cstride, drow = static_cast<long long>(dil) * w * dc_cstride;
        for (int a = pg * ppb; a < (pg + 1) * ppb; ++a) {
            const int nj = (h - a + dil - 1) / dil;
            const int j0 = seg * rseg, j1 = min(nj, j0 + rseg);
            if (j0 >= nj) continue;
            const T *xbase = x + ((static_cast<long long>(nn) * h + a) * w + ox) * x_cstride + ch;       // phase row 0
            // x rows j0-1 and j0 of the phase: the first two rows of the sliding window
            F4 xw[3][3];                                               // rows in rotating roles: role (k + r) % 3 = window row r at step k
            auto load3 = [&](int i, F4 (&dst)[3]) {
                dst[0] = dst[1] = dst[2] = f4_zero();
                if (i < 0 || i >= nj) return;
                const T *xr = xbase + static_cast<long long>(i) * xrow;
                dst[1] = f4_load<T>(xr);
                if (cl) dst[0] = f4_load<T>(xr + xoff_l);
                if (cr) dst[2] = f4_load<T>(xr + xoff_r);
            };
            load3(j0 - 1, xw[0]);
            load3(j0, xw[1]);
            // queue slot k: raw x row (i + 1) and raw dc row i of the step that will consume it
            const T *pfx = xbase + static_cast<long long>(j0 + 1) * xrow;
            const T *pfd = dc + ((static_cast<long long>(nn) * h + a + static_cast<long long>(dil) * j0) * w + ox) * dc_cstride + ch;
            int fetched = j0;
            Raw4<T> qx[DW4_Q][3], qd[DW4_Q];
            auto fetch = [&](Raw4<T> (&dx3)[3], Raw4<T> &dd) {
                dx3[0].zero(); dx3[1].zero(); dx3[2].zero(); dd.zero();
                if (fetched < j1) {
                    dd.load(pfd);
                    if (fetched + 1 < nj) {
                        dx3[1].load(pfx);
                        if (cl) dx3[0].load(pfx + xoff_l);
                        if (cr) dx3[2].load(pfx + xoff_r);
                    }
                }
                ++fetched; pfx += xrow; pfd += drow;
            };
#pragma unroll
            for (int k = 0; k < DW4_Q; ++k) fetch(qx[k], qd[k]);
            for (int i0 = j0; i0 < j1; i0 += DW4_Q) {
#pragma unroll
                for (int k = 0; k < DW4_Q; ++k) {
                    if (i0 + k < j1) {
                        F4 (&r0)[3] = xw[k % 3], (&r1)[3] = xw[(k + 1) % 3], (&r2)[3] = xw[(k + 2) % 3];
                        r2[0] = f4_of(qx[k][0]); r2[1] = f4_of(qx[k][1]); r2[2] = f4_of(qx[k][2]);
                        const F4 dv = f4_of(qd[k]);
                        fetch(qx[k], qd[k]);
#pragma unroll
                        for (int tc = 0; tc < 3; ++tc) {
                            acc[0][tc] = f4_fma(dv, r0[tc], acc[0][tc]);
                            acc[1][tc] = f4_fma(dv, r1[tc], acc[1][tc]);
                            acc[2][tc] = f4_fma(dv, r2[tc], acc[2][tc]);
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        __syncthreads();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const F4 &v = acc[tap / 3][tap % 3];
            const float e = (j == 0) ? v.lo.x : (j == 1) ? v.lo.y : (j == 2) ? v.hi.x : v.hi.y;
            s_red[threadIdx.x][tap] = active ? e : 0.f;
        }
        __syncthreads();
        for (int col = threadIdx.x; col < cq * 9; col += 256) {
            const int cql = col / 9, tap = col - cql * 9;
            float tot = 0.f;
            for (int l = 0; l < xt; ++l) tot += s_red[l * cq + cql][tap];
            atomicAdd(dw + static_cast<long long>((blockIdx.x * cq + cql) * 4 + j) * 9 + tap, tot);
        }
    }
}

// the kernel generation a problem takes in all three directions: dw4 (plain stride 1, pad == dil; the data gradient is the
// same convolution with flipped taps) or dw3 (every other 3x3 at a power-of-two stride: pcb_dw_eligible)
enum DwRoute { DW3, DW4 };

DwRoute dw_route(const pcb_conv *c) {
    if (c->stride == 1 && c->pad_h == c->dil && c->pad_w == c->dil && c->plain && c->parts[0].mask == nullptr && c->cin % 4 == 0) return DW4;
    return DW3;
}

template <typename T>
__global__ void dw_weight_transpose_kernel(const float *__restrict__ wm, int c, int taps, T *__restrict__ w_t) {
    const long long total = static_cast<long long>(c) * taps;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int tap = static_cast<int>(i % taps), ch = static_cast<int>(i / taps);
        w_t[static_cast<long long>(tap) * c + ch] = from_f32<T>(wm[i]);
    }
}

void fill(DwParams &P, const pcb_conv *c) {
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.c = c->cin; P.stride = c->stride; P.pad_h = c->pad_h;
    P.pad_w = c->pad_w; P.dil = c->dil; P.ho = c->ho; P.wo = c->wo; P.x_cstride = c->parts[0].x_cstride;
    P.mask = c->parts[0].mask; P.mup = c->parts[0].mask_up; P.no_guard = c->no_guard;
    P.mg = (c->groups > 1 && !c->same_holes) ? c->groups : 1;
}

inline int dw_grid(long long items) {
    long long b = (items + 255) / 256;
    const long long cap = 32ll * pcb_num_sms();
    return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

bool pcb_dw_eligible(const pcb_conv *c) {
    if (!(c->groups == c->cin && c->cin == c->cout && c->groups > 1 && c->nparts == 1)) return false;
    if (c->kh != 3 || c->kw != 3 || (c->stride & (c->stride - 1))) return false;
    const pcb_part &pt = c->parts[0];
    if (c->cin % 8 != 0 || c->cin > 2048 || pt.x_cstride % 8 != 0 || pt.x_up != 0) return false;
    const uintptr_t align = (c->dtype == PCB_BF16) ? 15 : 31;
    if (pt.x && (reinterpret_cast<uintptr_t>(pt.x) & align)) return false;
    return true;
}

int pcb_dw_weight_prepare(const pcb_conv *c, const float *w_master, void *w_t, cudaStream_t st) {
    const int taps = c->kh * c->kw;
    const int grid = dw_grid(static_cast<long long>(c->cin) * taps);
    if (c->dtype == PCB_BF16) dw_weight_transpose_kernel<bf16><<<grid, 256, 0, st>>>(w_master, c->cin, taps, static_cast<bf16 *>(w_t));
    else dw_weight_transpose_kernel<float><<<grid, 256, 0, st>>>(w_master, c->cin, taps, static_cast<float *>(w_t));
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_dw_forward(const pcb_conv *c, const void *w_t, const float *bias, void *y, int y_cstride, const float *msum, double *bn_sums,
                   const pcb_ep *ep, cudaStream_t st) {
    DwParams P;
    fill(P, c);
    P.ep = dw_ep(ep);
    P.y_cstride = y_cstride;
    P.msum = msum;       // plain mode: mask_sums wrote 1.0 everywhere, so the same epilogue applies
    if (dw_route(c) == DW4) {
        const Dw4Geom g = dw4_geom(c->cin, c->w, c->h, c->dil);
        const dim3 grid(g.chunks, g.xtiles, c->n * g.pgroups * g.nseg);
#define PCB_DW4_FWD(TT, EP_) dw4_s1_kernel<TT, false, EP_><<<grid, 256, 0, st>>>(static_cast<const TT *>(c->parts[0].x), c->parts[0].x_cstride, static_cast<const TT *>(w_t), bias, static_cast<TT *>(y), y_cstride, bn_sums, P.ep, c->n, c->h, c->w, c->cin, c->dil, g.cq, g.xt, g.nseg, g.rseg, g.ppb)
        if (c->dtype == PCB_BF16) { if (ep) PCB_DW4_FWD(bf16, true); else PCB_DW4_FWD(bf16, false); }
        else { if (ep) PCB_DW4_FWD(float, true); else PCB_DW4_FWD(float, false); }
#undef PCB_DW4_FWD
        PCB_LAUNCH_CHECK();
        return 0;
    }
    const Dw3Geom g = dw3_geom(c->cin);
    const dim3 grid(g.chunks, (c->n * c->ho + DW3_ROWS - 1) / DW3_ROWS);
    const bool plain = c->plain && c->parts[0].mask == nullptr;
#define PCB_DW3_FWD(TT, PL_, EP_) dw3_fwd_kernel<TT, PL_, EP_><<<grid, 256, 0, st>>>(P, static_cast<const TT *>(c->parts[0].x), static_cast<const TT *>(w_t), bias, static_cast<TT *>(y), g.cvb, g.pl, bn_sums)
    if (ep) {
        if (c->dtype == PCB_BF16) { if (plain) PCB_DW3_FWD(bf16, true, true); else PCB_DW3_FWD(bf16, false, true); }
        else { if (plain) PCB_DW3_FWD(float, true, true); else PCB_DW3_FWD(float, false, true); }
    } else {
        if (c->dtype == PCB_BF16) { if (plain) PCB_DW3_FWD(bf16, true, false); else PCB_DW3_FWD(bf16, false, false); }
        else { if (plain) PCB_DW3_FWD(float, true, false); else PCB_DW3_FWD(float, false, false); }
    }
#undef PCB_DW3_FWD
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_dw_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_t, void *dx, int dx_cstride, cudaStream_t st) {
    DwParams P;
    fill(P, c);
    if (dw_route(c) == DW4) {
        const Dw4Geom g = dw4_geom(c->cin, c->w, c->h, c->dil);
        const dim3 grid(g.chunks, g.xtiles, c->n * g.pgroups * g.nseg);
        if (c->dtype == PCB_BF16) dw4_s1_kernel<bf16, true, false><<<grid, 256, 0, st>>>(static_cast<const bf16 *>(dc), dc_cstride, static_cast<const bf16 *>(w_t), nullptr, static_cast<bf16 *>(dx), dx_cstride, nullptr, P.ep, c->n, c->h, c->w, c->cin, c->dil, g.cq, g.xt, g.nseg, g.rseg, g.ppb);
        else dw4_s1_kernel<float, true, false><<<grid, 256, 0, st>>>(static_cast<const float *>(dc), dc_cstride, static_cast<const float *>(w_t), nullptr, static_cast<float *>(dx), dx_cstride, nullptr, P.ep, c->n, c->h, c->w, c->cin, c->dil, g.cq, g.xt, g.nseg, g.rseg, g.ppb);
        PCB_LAUNCH_CHECK();
        return 0;
    }
    const Dw3Geom g = dw3_geom(c->cin);
    const dim3 grid(g.chunks, (c->n * c->h + DW3_ROWS - 1) / DW3_ROWS);
    const bool plain = c->plain && c->parts[0].mask == nullptr;
    int sshift = 0;
    while ((1 << sshift) < c->stride) ++sshift;
#define PCB_DW3_DG(TT, PL_) dw3_dgrad_kernel<TT, PL_><<<grid, 256, 0, st>>>(P, static_cast<const TT *>(dc), dc_cstride, static_cast<const TT *>(w_t), static_cast<TT *>(dx), dx_cstride, g.cvb, g.pl, sshift)
    if (c->dtype == PCB_BF16) { if (plain) PCB_DW3_DG(bf16, true); else PCB_DW3_DG(bf16, false); }
    else { if (plain) PCB_DW3_DG(float, true); else PCB_DW3_DG(float, false); }
#undef PCB_DW3_DG
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_dw_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, bool zero_dw, cudaStream_t st) {
    DwParams P;
    fill(P, c);
    const int taps = c->kh * c->kw;
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * c->cin * taps, st));
    if (dw_route(c) == DW4) {
        const Dw4Geom g = dw4_geom(c->cin, c->w, c->h, c->dil);
        const dim3 grid(g.chunks, g.xtiles, c->n * g.pgroups * g.nseg);
        if (c->dtype == PCB_BF16) dw4_s1_wgrad_kernel<bf16><<<grid, 256, 0, st>>>(static_cast<const bf16 *>(c->parts[0].x), c->parts[0].x_cstride, static_cast<const bf16 *>(dc), dc_cstride, dw, c->n, c->h, c->w, c->cin, c->dil, g.cq, g.xt, g.nseg, g.rseg, g.ppb);
        else dw4_s1_wgrad_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(c->parts[0].x), c->parts[0].x_cstride, static_cast<const float *>(dc), dc_cstride, dw, c->n, c->h, c->w, c->cin, c->dil, g.cq, g.xt, g.nseg, g.rseg, g.ppb);
        PCB_LAUNCH_CHECK();
        return 0;
    }
    const Dw3Geom g = dw3_geom(c->cin);
    // about two resident waves of blocks; every block ends with cvb * 72 atomics
    const int rows_total = c->n * c->ho;
    int row_groups = std::max(1, std::min(rows_total, (4 * pcb_num_sms() + g.chunks - 1) / g.chunks));
    const int rpbk = (rows_total + row_groups - 1) / row_groups;
    row_groups = (rows_total + rpbk - 1) / rpbk;
    const dim3 grid(g.chunks, row_groups);
    const bool plain = c->plain && c->parts[0].mask == nullptr;
#define PCB_DW3_WG(TT, PL_) dw3_wgrad_kernel<TT, PL_><<<grid, 256, 0, st>>>(P, static_cast<const TT *>(dc), dc_cstride, static_cast<const TT *>(c->parts[0].x), dw, g.cvb, g.pl, rpbk)
    if (c->dtype == PCB_BF16) { if (plain) PCB_DW3_WG(bf16, true); else PCB_DW3_WG(bf16, false); }
    else { if (plain) PCB_DW3_WG(float, true); else PCB_DW3_WG(float, false); }
#undef PCB_DW3_WG
    PCB_LAUNCH_CHECK();
    return 0;
}

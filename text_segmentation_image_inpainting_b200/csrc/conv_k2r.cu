// conv_k2r.cu -- the RGB tails of the inpainting U-Nets as a 1x1 GEMM at SOURCE resolution ("kernel-to-row"):
//     y = PartialConv(cat([nearest2x(u), v])) ,  u: >= 32 channels at half resolution, v: <= 4 channels (the image),  3x3, pad 1,
//     <= 3 output channels                         (models/image_inpainting.py:63 / :102 / :126 of the reference)
//
// A 3x3 kernel with 3 outputs has only 27 (tap, cout) columns.  Because nearest-2x upsampling repeats pixels, the contribution of
// the upsampled source to every (tap, cout) column can be computed ONCE PER SOURCE PIXEL:
//     Z[s][tap, co] = sum_c (u[s][c] * m_u[s]) * W[co][tap][c]              one 1x1 convolution  C_u -> 32  at half resolution
//     y[p][co]      = ( sum_tap Z[(p + tap - 1) >> 1][tap, co]  +  direct 3x3 over v )  / msum[p] + b[co]   (0 at holes)
// i.e. 4x fewer pixels and no im2col for the wide part; the 1x1 problem runs on the TMA-fed wgmma kernels of conv_tc.cu (its
// operand stream is the source tensor, read once), the combine pass is a streaming kernel.  The backward pass has the same shape:
//     D[s][tap, co] = sum over the four children p of s of dc[p - tap + 1][co]     (dc = renormalised output gradient)
//     du[s][c] = m_u[s] * sum_k D[s][k] W'[k][c]         1x1 data gradient, delivered at SOURCE resolution (no 2x2 reduction pass)
//     dW'[k][c] = sum_s D[s][k] u[s][c] m_u[s]           1x1 weight gradient, scattered back into the [co][tap][c] master layout
// and the 81 weight gradients of the image part are reduced on CUDA cores inside the D pass.
// The mma.sync kernels of conv_smallco.cu stay as the general path (other kernel sizes, wider second parts, PCB_DISABLE_K2R=1).
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"

namespace {

constexpr int K2R_N = 32;          // columns of the 1x1 problem: (tap, co) = tap * 3 + co, 27 used
constexpr int K2R_CO = 3;
constexpr int K2R_TAPS = 9;

struct K2rPlan {
    bool ok;
    int pu, ps;                    // upsampled (wide) part, full-resolution (narrow) part
    int cu, cs, choff_u, choff_s;
    pcb_conv sub;                  // the 1x1 problem at source resolution
    size_t sub_fe, sub_de;         // its operand sizes (bf16 elements)
    size_t fwd_extra, dg_extra;    // elements appended to the layer's operand buffers (sub operands + fp32 staging of W')
};

K2rPlan plan_of(const pcb_conv *c) {
    K2rPlan K;
    memset(&K, 0, sizeof(K));
    if (getenv("PCB_DISABLE_K2R") || !pcb_smallco_eligible(c)) return K;
    if (c->kh != 3 || c->kw != 3 || c->pad_h != 1 || c->pad_w != 1 || c->cout > K2R_CO || c->nparts != 2) return K;
    if (c->ho != c->h || c->wo != c->w || ((c->h | c->w) & 1)) return K;
    K.pu = c->parts[0].x_up ? 0 : 1;
    K.ps = 1 - K.pu;
    const pcb_part &u = c->parts[K.pu], &v = c->parts[K.ps];
    if (!u.x_up || v.x_up || u.c < 32 || (u.c & 7) || v.c > 4) return K;
    if ((u.mask && u.mask_up != 1) || (v.mask && v.mask_up != 0)) return K;
    K.cu = u.c; K.cs = v.c;
    K.choff_u = K.pu == 0 ? 0 : c->parts[0].c;
    K.choff_s = K.ps == 0 ? 0 : c->parts[0].c;
    pcb_conv &S = K.sub;
    S.n = c->n; S.h = c->h >> 1; S.w = c->w >> 1; S.cin = u.c; S.cout = K2R_N; S.kh = S.kw = 1; S.stride = 1; S.pad_h = S.pad_w = 0; S.dil = 1;
    S.groups = 1; S.ho = S.h; S.wo = S.w; S.dtype = PCB_BF16; S.nparts = 1;
    S.parts[0] = u; S.parts[0].x_up = 0; S.parts[0].mask_up = 0;
    if (!pcb_tc_eligible(&S)) return K;
    pcb_tc_weight_layout(&S, &K.sub_fe, &K.sub_de);
    K.sub_fe = (K.sub_fe + 63) / 64 * 64;
    K.sub_de = (K.sub_de + 63) / 64 * 64;
    K.fwd_extra = K.sub_fe + 2 * static_cast<size_t>(K2R_N) * K.cu;      // + fp32 W' [32][cu]
    K.dg_extra = K.sub_de;
    K.ok = true;
    return K;
}

size_t rup256(size_t v) { return (v + 255) / 256 * 256; }
size_t zbytes(const pcb_conv *c) { return rup256(static_cast<size_t>(c->n) * (c->h >> 1) * (c->w >> 1) * K2R_N * sizeof(bf16)); }

// W'[k = tap*3 + co][c] (fp32, the KRSC master of the 1x1 problem) from the layer's master weights [co][tap][cin]
__global__ void k2r_weight_kernel(const float *__restrict__ w, float *__restrict__ wsub, int cout, int cin, int choff_u, int cu) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= K2R_N * cu) return;
    const int k = i / cu, ch = i - k * cu;
    const int tap = k / K2R_CO, co = k - tap * K2R_CO;
    wsub[i] = (tap < K2R_TAPS && co < cout) ? w[(static_cast<long long>(co) * K2R_TAPS + tap) * cin + choff_u + ch] : 0.f;
}

// dw[co][tap][choff_u + c] += dW'[tap*3 + co][c]
__global__ void k2r_dw_scatter_kernel(const float *__restrict__ dwsub, float *__restrict__ dw, int cout, int cin, int choff_u, int cu) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= K2R_TAPS * K2R_CO * cu) return;
    const int k = i / cu, ch = i - k * cu;
    const int tap = k / K2R_CO, co = k - tap * K2R_CO;
    if (co < cout) dw[(static_cast<long long>(co) * K2R_TAPS + tap) * cin + choff_u + ch] += dwsub[i];
}

struct K2rParams {
    int n, h, w, hs, ws, cout, cin, no_guard;
    const bf16 *z;                 // [n][hs][ws][32]
    const bf16 *v; int v_cstride;  // narrow part, full resolution
    const uint8_t *mv;             // its hole plane or null
    const bf16 *w_fwd; long long kf; int ktap, koff_s;      // layer operand [co][tap*ktap + koff_s + c]
    const float *bias, *msum;
    bf16 *y; int y_cstride;
    // backward
    const bf16 *dc; int dc_cstride;
    bf16 *d;                       // [n][hs][ws][32]
    float *dw; int choff_s;
};

__device__ __forceinline__ void bf4_to_float(const uint2 r, float (&f)[4]) {
    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&r);
    const float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}

// ------------------------------------------------------------------------------------------------- forward: combine
// one thread per SOURCE pixel = one 2x2 block of outputs: nine Z rows of the 3x3 source neighbourhood, a 4x4 window of the image part
template <int CS>
__global__ void __launch_bounds__(256) k2r_combine_kernel(const K2rParams P) {
    __shared__ float4 s_w[K2R_TAPS * K2R_CO];            // image-part weights [tap][co] x (c0..c3)
    for (int i = threadIdx.x; i < K2R_TAPS * K2R_CO; i += blockDim.x) {
        const int tap = i / K2R_CO, co = i - tap * K2R_CO;
        float wv[4] = {0.f, 0.f, 0.f, 0.f};
        if (co < P.cout)
            for (int ch = 0; ch < CS; ++ch) wv[ch] = __bfloat162float(P.w_fwd[static_cast<long long>(co) * P.kf + static_cast<long long>(tap) * P.ktap + P.koff_s + ch]);
        s_w[i] = make_float4(wv[0], wv[1], wv[2], wv[3]);
    }
    __syncthreads();
    const long long total = static_cast<long long>(P.n) * P.hs * P.ws;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int sx = static_cast<int>(idx % P.ws);
        const long long t = idx / P.ws;
        const int sy = static_cast<int>(t % P.hs), img = static_cast<int>(t / P.hs);
        float acc[4][K2R_CO];
#pragma unroll
        for (int ch = 0; ch < 4; ++ch)
#pragma unroll
            for (int co = 0; co < K2R_CO; ++co) acc[ch][co] = 0.f;
        // wide part: Z rows of the 3x3 source neighbourhood; child (a, b) takes tap (tr, tc) from neighbour ((a+tr-1)>>1, (b+tc-1)>>1)
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            const int yy = sy + dy;
            if (yy < 0 || yy >= P.hs) continue;
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int xx = sx + dx;
                if (xx < 0 || xx >= P.ws) continue;
                const uint4 *row = reinterpret_cast<const uint4 *>(P.z + ((static_cast<long long>(img) * P.hs + yy) * P.ws + xx) * K2R_N);
                float zf[K2R_N];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint4 r = __ldg(row + q);
                    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&r);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __bfloat1622float2(h[e]);
                        zf[q * 8 + 2 * e] = f.x; zf[q * 8 + 2 * e + 1] = f.y;
                    }
                }
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int b = 0; b < 2; ++b)
#pragma unroll
                        for (int tr = 0; tr < 3; ++tr)
#pragma unroll
                            for (int tc = 0; tc < 3; ++tc) {
                                const int ny = (a + tr + 1) / 2 - 1, nx = (b + tc + 1) / 2 - 1;       // floor((a + tr - 1) / 2)
                                if (ny == dy && nx == dx) {
#pragma unroll
                                    for (int co = 0; co < K2R_CO; ++co) acc[a * 2 + b][co] += zf[(tr * 3 + tc) * K2R_CO + co];
                                }
                            }
            }
        }
        // image part: 4x4 window of v * mask around the block (zero outside the image and at holes)
        float xv[4][4][CS];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int y = 2 * sy - 1 + i;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int x = 2 * sx - 1 + j;
                bool ok = y >= 0 && y < P.h && x >= 0 && x < P.w;
                const long long q = (static_cast<long long>(img) * P.h + (ok ? y : 0)) * P.w + (ok ? x : 0);
                if (ok && P.mv) ok = P.mv[q] != 0;
                float f[4] = {0.f, 0.f, 0.f, 0.f};
                if (ok) bf4_to_float(__ldg(reinterpret_cast<const uint2 *>(P.v + q * P.v_cstride)), f);
#pragma unroll
                for (int ch = 0; ch < CS; ++ch) xv[i][j][ch] = f[ch];
            }
        }
#pragma unroll
        for (int tr = 0; tr < 3; ++tr)
#pragma unroll
            for (int tc = 0; tc < 3; ++tc)
#pragma unroll
                for (int co = 0; co < K2R_CO; ++co) {
                    const float4 wv = s_w[(tr * 3 + tc) * K2R_CO + co];
                    const float wq[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int a = 0; a < 2; ++a)
#pragma unroll
                        for (int b = 0; b < 2; ++b)
#pragma unroll
                            for (int ch = 0; ch < CS; ++ch) acc[a * 2 + b][co] = fmaf(wq[ch], xv[a + tr][b + tc][ch], acc[a * 2 + b][co]);
                }
        // y = hole ? 0 : acc / s + b  (8 channel slots per pixel; slots >= cout are zeros, like the mma.sync kernel writes them)
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b) {
                const long long q = (static_cast<long long>(img) * P.h + 2 * sy + a) * P.w + 2 * sx + b;
                const float s = P.msum ? P.msum[q] : 1.f;
                const bool hole = (s == 0.f) && !P.no_guard;
                const float inv = hole ? 0.f : 1.0f / s;
                float o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int co = 0; co < K2R_CO; ++co)
                    if (co < P.cout && !hole) o[co] = acc[a * 2 + b][co] * inv + (P.bias ? P.bias[co] : 0.f);
                Vec8<bf16>::store(P.y + q * P.y_cstride, o);
            }
    }
}

// ------------------------------------------------------------------------------------------------- backward: D rows (+ image-part wgrad)
// one thread per source pixel: the 4x4 window of dc around its children gives the 27 sums; WG adds the 27 x CS weight gradients
// of the image part (register accumulators over the thread's pixels, one warp reduction + shared/global atomics per block)
template <bool WG, int CS>
__global__ void __launch_bounds__(256) k2r_dbuild_kernel(const K2rParams P) {
    __shared__ float s_dw[WG ? K2R_TAPS * K2R_CO * 4 : 1];
    if (WG) {
        for (int i = threadIdx.x; i < K2R_TAPS * K2R_CO * 4; i += blockDim.x) s_dw[i] = 0.f;
        __syncthreads();
    }
    float gw[WG ? K2R_TAPS * K2R_CO : 1][WG ? CS : 1];
    if (WG) {
#pragma unroll
        for (int k = 0; k < K2R_TAPS * K2R_CO; ++k)
#pragma unroll
            for (int ch = 0; ch < CS; ++ch) gw[k][ch] = 0.f;
    }
    const long long total = static_cast<long long>(P.n) * P.hs * P.ws;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int sx = static_cast<int>(idx % P.ws);
        const long long t = idx / P.ws;
        const int sy = static_cast<int>(t % P.hs), img = static_cast<int>(t / P.hs);
        float win[4][4][K2R_CO];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int y = 2 * sy - 1 + i;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int x = 2 * sx - 1 + j;
                const bool ok = y >= 0 && y < P.h && x >= 0 && x < P.w;
                float f[4] = {0.f, 0.f, 0.f, 0.f};
                if (ok) bf4_to_float(__ldg(reinterpret_cast<const uint2 *>(P.dc + ((static_cast<long long>(img) * P.h + y) * P.w + x) * P.dc_cstride)), f);
#pragma unroll
                for (int co = 0; co < K2R_CO; ++co) win[i][j][co] = f[co];
            }
        }
        if (P.d) {
            float dv[K2R_N];
#pragma unroll
            for (int k = K2R_TAPS * K2R_CO; k < K2R_N; ++k) dv[k] = 0.f;
            // child p = 2s + (a, b) contributes dc[p - tap + 1] = win[a - tr + 2][b - tc + 2]
#pragma unroll
            for (int tr = 0; tr < 3; ++tr)
#pragma unroll
                for (int tc = 0; tc < 3; ++tc)
#pragma unroll
                    for (int co = 0; co < K2R_CO; ++co)
                        dv[(tr * 3 + tc) * K2R_CO + co] = (win[2 - tr][2 - tc][co] + win[2 - tr][3 - tc][co]) + (win[3 - tr][2 - tc][co] + win[3 - tr][3 - tc][co]);
            bf16 *row = P.d + idx * K2R_N;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float o[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] = dv[q * 8 + e];
                Vec8<bf16>::store(row + q * 8, o);
            }
        }
        if (WG) {
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int b = 0; b < 2; ++b) {
                    const long long q = (static_cast<long long>(img) * P.h + 2 * sy + a) * P.w + 2 * sx + b;
                    float f[4] = {0.f, 0.f, 0.f, 0.f};
                    if (!P.mv || P.mv[q] != 0) bf4_to_float(__ldg(reinterpret_cast<const uint2 *>(P.v + q * P.v_cstride)), f);
#pragma unroll
                    for (int tr = 0; tr < 3; ++tr)
#pragma unroll
                        for (int tc = 0; tc < 3; ++tc)
#pragma unroll
                            for (int co = 0; co < K2R_CO; ++co)
#pragma unroll
                                for (int ch = 0; ch < CS; ++ch)
                                    gw[(tr * 3 + tc) * K2R_CO + co][ch] = fmaf(win[a - tr + 2][b - tc + 2][co], f[ch], gw[(tr * 3 + tc) * K2R_CO + co][ch]);
                }
        }
    }
    if (WG) {
        const int lane = threadIdx.x & 31;
#pragma unroll
        for (int k = 0; k < K2R_TAPS * K2R_CO; ++k)
#pragma unroll
            for (int ch = 0; ch < CS; ++ch) {
                const float v = warp_sum(gw[k][ch]);
                if (lane == 0) atomicAdd(&s_dw[k * 4 + ch], v);
            }
        __syncthreads();
        for (int i = threadIdx.x; i < K2R_TAPS * K2R_CO * 4; i += blockDim.x) {
            const int k = i >> 2, ch = i & 3;
            const int tap = k / K2R_CO, co = k - tap * K2R_CO;
            if (co < P.cout && ch < CS) atomicAdd(P.dw + (static_cast<long long>(co) * K2R_TAPS + tap) * P.cin + P.choff_s + ch, s_dw[i]);
        }
    }
}

void base(K2rParams &P, const pcb_conv *c, const K2rPlan &K) {
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.hs = c->h >> 1; P.ws = c->w >> 1; P.cout = c->cout; P.cin = c->cin; P.no_guard = c->no_guard;
    const pcb_part &v = c->parts[K.ps];
    P.v = static_cast<const bf16 *>(v.x); P.v_cstride = v.x_cstride; P.mv = v.mask; P.choff_s = K.choff_s;
}

int grid_for(const pcb_conv *c, int per_sm) {
    const long long total = static_cast<long long>(c->n) * (c->h >> 1) * (c->w >> 1);
    return static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, static_cast<long long>(per_sm) * pcb_num_sms())));
}

// grow-only per-device scratch for the D rows of the data-gradient call (which has no workspace argument)
bf16 *dgrad_scratch(size_t bytes) {
    static void *buf[PCB_MAX_DEVICES] = {};
    static size_t cap[PCB_MAX_DEVICES] = {};
    const int dev = pcb_cur_device();
    if (cap[dev] < bytes) {
        // a smaller buffer handed out earlier is NOT freed: a captured CUDA graph may still replay launches that point into it
        // (growth happens a handful of times per process, at most one buffer per distinct problem size)
        void *fresh = nullptr;
        if (cudaMalloc(&fresh, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        buf[dev] = fresh;
        cap[dev] = bytes;
    }
    return static_cast<bf16 *>(buf[dev]);
}

}  // namespace

bool pcb_k2r_ok(const pcb_conv *c) { return plan_of(c).ok; }

void pcb_k2r_weight_layout(const pcb_conv *c, size_t *fwd_extra, size_t *dg_extra) {
    const K2rPlan K = plan_of(c);
    *fwd_extra = K.ok ? K.fwd_extra : 0;
    *dg_extra = K.ok ? K.dg_extra : 0;
}

size_t pcb_k2r_workspace(const pcb_conv *c) {
    const K2rPlan K = plan_of(c);
    if (!K.ok) return 0;
    return zbytes(c) + rup256(sizeof(float) * K2R_N * K.cu) + pcb_tc_workspace(&K.sub);
}

int pcb_k2r_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd_extra, void *w_dg_extra, bool zero_padding, cudaStream_t st) {
    const K2rPlan K = plan_of(c);
    PCB_CHECK(K.ok && w_fwd_extra && w_dg_extra, "k2r weight prepare: not a kernel-to-row layer / missing operand buffers");
    float *wsub = reinterpret_cast<float *>(static_cast<bf16 *>(w_fwd_extra) + K.sub_fe);
    k2r_weight_kernel<<<(K2R_N * K.cu + 255) / 256, 256, 0, st>>>(w_master, wsub, c->cout, c->cin, K.choff_u, K.cu);
    PCB_LAUNCH_CHECK();
    return pcb_tc_weight_prepare(&K.sub, wsub, w_fwd_extra, w_dg_extra, zero_padding, st);
}

int pcb_k2r_forward(const pcb_conv *c, const pcb_smallco_layout &L, const void *w_fwd, const void *w_fwd_extra, const float *bias, void *y, int y_cstride,
                    const float *msum, void *workspace, cudaStream_t st) {
    const K2rPlan K = plan_of(c);
    PCB_CHECK(K.ok && workspace, "k2r forward: not a kernel-to-row layer / no workspace");
    PCB_CHECK(y_cstride % 8 == 0 && y_cstride >= 8 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "small-cout forward: y must be 16-byte aligned with a channel stride that is a multiple of 8");
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    bf16 *z = reinterpret_cast<bf16 *>(ws);
    uint64_t *sub_ws = reinterpret_cast<uint64_t *>(ws + zbytes(c) + rup256(sizeof(float) * K2R_N * K.cu));
    // Z = (u * m_u) W'^T : raw accumulators (no renormaliser, no bias) of the 1x1 problem
    if (int rc = pcb_tc_forward_ws(&K.sub, w_fwd_extra, nullptr, z, K2R_N, nullptr, sub_ws, false, nullptr, st)) return rc;
    K2rParams P;
    base(P, c, K);
    P.z = z; P.w_fwd = static_cast<const bf16 *>(w_fwd); P.kf = L.kf; P.ktap = L.ktap; P.koff_s = L.koff[K.ps];
    P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride;
    if (K.cs <= 3) k2r_combine_kernel<3><<<grid_for(c, 8), 256, 0, st>>>(P);
    else k2r_combine_kernel<4><<<grid_for(c, 8), 256, 0, st>>>(P);
    PCB_LAUNCH_CHECK();
    return 0;
}

// dx[pu] is a SOURCE-resolution buffer (pcb_conv_dgrad_at_source_resolution); dx[ps], when wanted, comes from the mma.sync kernel
int pcb_k2r_dgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, const void *w_dgrad, const void *w_dg_extra,
                  void *const *dx, const int *dx_cstride, cudaStream_t st) {
    const K2rPlan K = plan_of(c);
    PCB_CHECK(K.ok, "k2r dgrad: not a kernel-to-row layer");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= 8, "small-cout dgrad: dc channel stride must be a multiple of 8");
    if (dx[K.pu]) {
        bf16 *d = dgrad_scratch(zbytes(c));
        PCB_CHECK(d != nullptr, "k2r dgrad: scratch allocation failed");
        K2rParams P;
        base(P, c, K);
        P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.d = d;
        k2r_dbuild_kernel<false, 3><<<grid_for(c, 8), 256, 0, st>>>(P);
        PCB_LAUNCH_CHECK();
        void *dxs[1] = {dx[K.pu]};
        const int cs[1] = {dx_cstride[K.pu]};
        if (int rc = pcb_tc_dgrad(&K.sub, d, K2R_N, w_dg_extra, dxs, cs, st)) return rc;
    }
    if (dx[K.ps]) {
        void *dxl[2] = {nullptr, nullptr};
        dxl[K.ps] = dx[K.ps];
        return pcb_smallco_dgrad(c, L, dc, dc_cstride, w_dgrad, dxl, dx_cstride, st);
    }
    return 0;
}

int pcb_k2r_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st) {
    const K2rPlan K = plan_of(c);
    PCB_CHECK(K.ok && workspace, "k2r wgrad: not a kernel-to-row layer / no workspace");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= 8, "small-cout wgrad: dc channel stride must be a multiple of 8");
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * c->cout * K2R_TAPS * c->cin, st));
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    bf16 *d = reinterpret_cast<bf16 *>(ws);
    float *dwsub = reinterpret_cast<float *>(ws + zbytes(c));
    void *sub_ws = ws + zbytes(c) + rup256(sizeof(float) * K2R_N * K.cu);
    K2rParams P;
    base(P, c, K);
    P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.d = d; P.dw = dw;
    // a register-heavy kernel: 128-thread blocks let more of them be resident per SM than 256-thread blocks
    if (K.cs <= 3) k2r_dbuild_kernel<true, 3><<<grid_for(c, 3), 128, 0, st>>>(P);
    else k2r_dbuild_kernel<true, 4><<<grid_for(c, 2), 128, 0, st>>>(P);
    PCB_LAUNCH_CHECK();
    if (int rc = pcb_tc_wgrad(&K.sub, d, K2R_N, dwsub, sub_ws, true, st)) return rc;
    k2r_dw_scatter_kernel<<<(K2R_TAPS * K2R_CO * K.cu + 255) / 256, 256, 0, st>>>(dwsub, dw, c->cout, c->cin, K.choff_u, K.cu);
    PCB_LAUNCH_CHECK();
    return 0;
}

// conv_stem.cu -- the 7x7 / stride-2 / pad-3 stems over an image (<= 8 channels; models/image_inpainting.py:118 of the reference,
// BaseModels / MobileNetV2 / Xception entry convolutions have other shapes and keep their paths) as a 4x4 / stride-1 convolution over
// the SPACE-TO-DEPTH image:
//     xs[n][sy][sx][(a, b, ch)] = x[n][2 sy + a][2 sx + b][ch] * mask[...]          32 channels per half-resolution cell
//     y[o] = sum_t w[t] x[2 o + t - 3]  =  sum_{j=0..3} sum_{a=0,1} w[2 j + a - 1] xs[o + j - 2][a]      (w[-1] = w[7] = 0)
// i.e. kernel 4, padding 2 in front (the "extra" output row/column a symmetric padding would give is simply not computed).  The
// stride-2 gather of 7 x 7 x 8-channel windows -- which bounds the row-packed cp.async kernel by its 16-byte gathers --
// becomes the TMA-fed implicit GEMM of conv_tc.cu with row-halo tiles: one 131-cell tile per kernel row serves the four taps, the
// K steps of the zero half of each 64-channel block are not issued.  x * mask happens in the space-to-depth pass (sub-pixels of a
// cell have different mask values, so the GEMM itself runs without hole rows); renormalisation, hole zeroing, bias and the
// BatchNorm statistics are the regular epilogue with the layer's own mask sums.  The weight gradient is the same 4x4 problem,
// gathered back into the [co][7][7][c] master layout.
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"

namespace {

constexpr int S2D_C = 32;          // (a, b, ch8)
constexpr int SK = 4;              // sub-kernel size

struct StemPlan {
    bool ok;
    pcb_conv sub;
    size_t sub_fe;                 // bf16 elements of the sub-problem's forward operand (rounded to 64)
    size_t fwd_extra;              // + fp32 staging of the re-indexed master weights
};

StemPlan plan_of(const pcb_conv *c) {
    StemPlan K;
    memset(&K, 0, sizeof(K));
    if (getenv("PCB_DISABLE_S2D_STEM")) return K;
    if (c->dtype != PCB_BF16 || c->groups != 1 || c->nparts != 1 || c->kh != 7 || c->kw != 7 || c->stride != 2 || c->pad_h != 3 || c->pad_w != 3 ||
        c->dil != 1) return K;
    const pcb_part &p = c->parts[0];
    if (p.x_up || p.c > 8 || p.x_cstride != 8 || (p.mask && p.mask_up != 0) || ((c->h | c->w) & 1)) return K;
    if (p.x && (reinterpret_cast<uintptr_t>(p.x) & 15)) return K;
    if (c->ho != c->h / 2 || c->wo != c->w / 2 || c->cout < 32 || (c->cout & 7)) return K;
    pcb_conv &S = K.sub;
    S.n = c->n; S.h = c->h / 2; S.w = c->w / 2; S.cin = S2D_C; S.cout = c->cout; S.kh = S.kw = SK; S.stride = 1; S.pad_h = S.pad_w = 2; S.dil = 1;
    S.groups = 1; S.ho = S.h; S.wo = S.w; S.dtype = PCB_BF16; S.no_guard = c->no_guard; S.nparts = 1;
    S.parts[0].x = nullptr; S.parts[0].mask = nullptr; S.parts[0].c = S2D_C; S.parts[0].x_cstride = S2D_C;
    if (!pcb_tc_eligible(&S)) return K;
    size_t de;
    pcb_tc_weight_layout(&S, &K.sub_fe, &de);
    K.sub_fe = (K.sub_fe + 63) / 64 * 64;
    K.fwd_extra = K.sub_fe + 2 * static_cast<size_t>(c->cout) * SK * SK * S2D_C;
    K.ok = true;
    return K;
}

size_t rup256(size_t v) { return (v + 255) / 256 * 256; }
size_t s2d_bytes(const pcb_conv *c) { return rup256(static_cast<size_t>(c->n) * (c->h / 2) * (c->w / 2) * S2D_C * sizeof(bf16)); }
size_t dwsub_bytes(const pcb_conv *c) { return rup256(sizeof(float) * c->cout * SK * SK * S2D_C); }

// one thread per (cell, a): two horizontally adjacent pixels (32 contiguous bytes) -> 16 channels of the cell, times the hole mask
__global__ void s2d_kernel(const bf16 *__restrict__ x, const uint8_t *__restrict__ mask, bf16 *__restrict__ xs, int n, int h, int w) {
    const int hs = h >> 1, ws = w >> 1;
    const long long total = static_cast<long long>(n) * hs * ws * 2;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int a = static_cast<int>(i & 1);
        const long long cell = i >> 1;
        const int sx = static_cast<int>(cell % ws);
        const long long t = cell / ws;
        const int sy = static_cast<int>(t % hs), img = static_cast<int>(t / hs);
        const long long q = (static_cast<long long>(img) * h + 2 * sy + a) * w + 2 * sx;
        uint4 v0 = __ldg(reinterpret_cast<const uint4 *>(x + q * 8)), v1 = __ldg(reinterpret_cast<const uint4 *>(x + q * 8 + 8));
        if (mask) {
            if (mask[q] == 0) v0 = make_uint4(0u, 0u, 0u, 0u);
            if (mask[q + 1] == 0) v1 = make_uint4(0u, 0u, 0u, 0u);
        }
        uint4 *dst = reinterpret_cast<uint4 *>(xs + cell * S2D_C + a * 16);
        dst[0] = v0; dst[1] = v1;
    }
}

// wsub[co][ja][jb][(a, b, ch)] = w[co][2 ja + a - 1][2 jb + b - 1][ch]   (fp32, the KRSC master of the 4x4 problem)
__global__ void stem_weight_kernel(const float *__restrict__ w, float *__restrict__ wsub, int cout, int cin) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cout * SK * SK * S2D_C) return;
    const int k = i % S2D_C, jb = (i / S2D_C) % SK, ja = (i / (S2D_C * SK)) % SK, co = i / (S2D_C * SK * SK);
    const int ch = k & 7, b = (k >> 3) & 1, a = k >> 4;
    const int ty = 2 * ja + a - 1, tx = 2 * jb + b - 1;
    wsub[i] = (ty >= 0 && ty < 7 && tx >= 0 && tx < 7 && ch < cin) ? w[((static_cast<long long>(co) * 7 + ty) * 7 + tx) * cin + ch] : 0.f;
}

// dw[co][ty][tx][ch] += dwsub[co][(ty+1)>>1][(tx+1)>>1][((ty+1)&1, (tx+1)&1, ch)]
__global__ void stem_dw_gather_kernel(const float *__restrict__ dwsub, float *__restrict__ dw, int cout, int cin) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cout * 49 * cin) return;
    const int ch = i % cin, tx = (i / cin) % 7, ty = (i / (cin * 7)) % 7, co = i / (cin * 49);
    const int ja = (ty + 1) >> 1, a = (ty + 1) & 1, jb = (tx + 1) >> 1, b = (tx + 1) & 1;
    dw[i] += dwsub[((static_cast<long long>(co) * SK + ja) * SK + jb) * S2D_C + (a * 2 + b) * 8 + ch];
}

int run_s2d(const pcb_conv *c, bf16 *xs, cudaStream_t st) {
    const pcb_part &p = c->parts[0];
    PCB_CHECK(p.x != nullptr, "space-to-depth stem: null x");
    const long long total = static_cast<long long>(c->n) * (c->h / 2) * (c->w / 2) * 2;
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, 16ll * pcb_num_sms())));
    s2d_kernel<<<grid, 256, 0, st>>>(static_cast<const bf16 *>(p.x), p.mask, xs, c->n, c->h, c->w);
    PCB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

bool pcb_stem_ok(const pcb_conv *c) { return plan_of(c).ok; }

size_t pcb_stem_weight_extra(const pcb_conv *c) {
    const StemPlan K = plan_of(c);
    return K.ok ? K.fwd_extra : 0;
}

size_t pcb_stem_workspace(const pcb_conv *c) {
    StemPlan K = plan_of(c);
    if (!K.ok) return 0;
    return s2d_bytes(c) + dwsub_bytes(c) + pcb_tc_workspace(&K.sub);
}

int pcb_stem_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd_extra, bool zero_padding, cudaStream_t st) {
    const StemPlan K = plan_of(c);
    PCB_CHECK(K.ok && w_fwd_extra, "space-to-depth stem: weight prepare on a layer that does not take this path");
    float *wsub = reinterpret_cast<float *>(static_cast<bf16 *>(w_fwd_extra) + K.sub_fe);
    const int total = c->cout * SK * SK * S2D_C;
    stem_weight_kernel<<<(total + 255) / 256, 256, 0, st>>>(w_master, wsub, c->cout, c->cin);
    PCB_LAUNCH_CHECK();
    return pcb_tc_weight_prepare(&K.sub, wsub, w_fwd_extra, nullptr, zero_padding, st);
}

int pcb_stem_forward(const pcb_conv *c, const void *w_fwd_extra, const float *bias, void *y, int y_cstride, const float *msum, void *workspace,
                     double *bn_sums, cudaStream_t st) {
    StemPlan K = plan_of(c);
    PCB_CHECK(K.ok && workspace, "space-to-depth stem forward: wrong layer / no workspace");
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    bf16 *xs = reinterpret_cast<bf16 *>(ws);
    if (int rc = run_s2d(c, xs, st)) return rc;
    K.sub.parts[0].x = xs;
    uint64_t *sub_ws = reinterpret_cast<uint64_t *>(ws + s2d_bytes(c) + dwsub_bytes(c));
    // tap-validity words of the 4x4 problem (in-bounds bits only: no holes) where its kernel wants them (the gather kernels of
    // non-power-of-two grids; the TMA-fed kernels zero-fill out-of-range coordinates themselves)
    if (int rc = pcb_tc_forward_mask_pass(&K.sub, sub_ws, st)) return rc;
    // the layer's own mask sums drive the epilogue (renormalise, zero at holes, bias, BatchNorm statistics); no hole rows in the GEMM
    return pcb_tc_forward_ws(&K.sub, w_fwd_extra, bias, y, y_cstride, msum, sub_ws, true, bn_sums, st);
}

int pcb_stem_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st) {
    StemPlan K = plan_of(c);
    PCB_CHECK(K.ok && workspace, "space-to-depth stem wgrad: wrong layer / no workspace");
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * c->cout * 49 * c->cin, st));
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    bf16 *xs = reinterpret_cast<bf16 *>(ws);
    float *dwsub = reinterpret_cast<float *>(ws + s2d_bytes(c));
    void *sub_ws = ws + s2d_bytes(c) + dwsub_bytes(c);
    if (int rc = run_s2d(c, xs, st)) return rc;
    K.sub.parts[0].x = xs;
    if (int rc = pcb_tc_wgrad(&K.sub, dc, dc_cstride, dwsub, sub_ws, true, st)) return rc;
    const int total = c->cout * 49 * c->cin;
    stem_dw_gather_kernel<<<(total + 255) / 256, 256, 0, st>>>(dwsub, dw, c->cout, c->cin);
    PCB_LAUNCH_CHECK();
    return 0;
}

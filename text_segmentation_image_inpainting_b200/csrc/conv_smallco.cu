// conv_smallco.cu -- partial convolution layers with at most 8 OUTPUT channels (the RGB tails of the inpainting U-Nets:
// cat(up2x(64 ch), image 3 ch) -> 3, 3x3, stride 1;  models/image_inpainting.py:63 / :102 / :126).
//
// On the wgmma path such a layer pads N = 3 to a 32..64-wide tile and its data gradient pads K = 3 to 64 per tap: >90 % of the
// tensor work multiplies zeros and the kernels end up bound by operand staging, not by math.  Here the three GEMMs are shaped around the 8-wide dimension instead, with warp-level mma.sync
// (m16n8k16, bf16 x bf16 -> fp32) whose N (or K per tap) is exactly 8:
//   forward   M = 16 pixels, N = 8 cout,          K = tap x packed channels      A: ldmatrix from a haloed, hole-masked x tile
//   dgrad     M = 16 pixels, N = 8 input chans,   K = (tap, 8 cout) pairs        A: ldmatrix rows gathered from a haloed dc tile
//   wgrad     M = 16 input chans, N = 8 cout,     K = 16 pixels                  A/B: ldmatrix.trans from the same tiles
// The input of the layer is the lazy cat([nearest-2x-upsampled source, full-resolution source]) exactly as on the other
// paths: the tile loader reads the half-resolution tensor at (y>>1, x>>1), multiplies by the hole mask (zero fill) and packs
// the parts' channels back to back in shared memory.  x * mask, the renormalisation by the mask box sum and the
// per-part input-mask multiply of the gradient are fused as everywhere else (models/partial_convolution.py:49-80).
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"

namespace {

constexpr int TH = 8, TW = 32;              // output tile: 8 rows x 32 columns, one warp per row
constexpr int SC_THREADS = 256;
constexpr int SC_MAX_KS = 5;                // <= 80 packed input channels
constexpr int SC_MAX_TAPS = 9;              // kh, kw <= 3
constexpr int SC_MAX_NT = 10;

struct ScPart {
    const bf16 *x;            // source tensor (half resolution when xup)
    const uint8_t *mask;      // hole plane or null
    bf16 *dx;                 // dgrad output (full resolution) or null
    int c, c8, cstride, xup, mup, koff, choff, dx_cstride, cc0;   // cc0: first packed channel of the part in the smem tile
};

struct ScParams {
    int n, h, w, cin, cout, kh, kw, pad_h, pad_w, ho, wo;
    int nparts;
    ScPart parts[2];
    int cp, ks, ps;           // packed channels, 16-channel K steps, shared-memory pixel stride in bytes (odd multiple of 16)
    int tiles_x, tiles_y, num_tiles;
    const bf16 *w_fwd; long long kf; int ktap;        // [co][tap*ktap + koff_p + local]
    const bf16 *w_dg; long long kd; int cout64;       // [koff_p + local][tap*cout64 + co]
    const float *bias; const float *msum; bf16 *y; int y_cstride, no_guard;
    const bf16 *dc; int dc_cstride;
    float *dw;
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t (&r)[2]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_t(uint32_t addr, uint32_t (&r)[2]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// packed channel -> K slot of the tensor-core weight layouts (parts are padded to 64 there)
__device__ __forceinline__ int slot_of(const ScParams &P, int cc) {
    return (P.nparts > 1 && cc >= P.parts[1].cc0) ? P.parts[1].koff + cc - P.parts[1].cc0 : P.parts[0].koff + cc;
}

__device__ __forceinline__ void tile_origin(const ScParams &P, int tile, int &img, int &ty0, int &tx0) {
    const int per_img = P.tiles_x * P.tiles_y;
    img = tile / per_img;
    const int r = tile - img * per_img;
    ty0 = (r / P.tiles_x) * TH;
    tx0 = (r - (r / P.tiles_x) * P.tiles_x) * TW;
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid) {
    const uint32_t sz = valid ? 16u : 0u;     // src-size 0: sixteen zero bytes
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// validity bytes of a [rows][cols] window of the input grid for each part: 1 = inside the image and not a hole
__device__ __forceinline__ void load_valid(const ScParams &P, uint8_t *sv, int img, int y0, int x0, int rows, int cols) {
    const int npix = rows * cols;
    for (int i = threadIdx.x; i < npix * P.nparts; i += SC_THREADS) {
        const int p = i >= npix ? 1 : 0, pix = i - p * npix;
        const int ty = pix / cols, tx = pix - ty * cols;
        const int y = y0 + ty, x = x0 + tx;
        const ScPart &pt = P.parts[p];
        uint8_t v = 0;
        if (y >= 0 && y < P.h && x >= 0 && x < P.w)
            v = pt.mask ? (pt.mask[(static_cast<long long>(img) * (P.h >> pt.mup) + (y >> pt.mup)) * (P.w >> pt.mup) + (x >> pt.mup)] != 0) : 1;
        sv[i] = v;
    }
}

// [rows][cols] pixels x ps bytes: cat(up?(x_p)) * mask, zero outside the image and in the padding chunks.  Sixteen lanes
// per pixel issue independent 16-byte cp.async copies (zero-filled where the validity byte is 0): everything is in flight
// at once and no index division sits in the loop.
__device__ __forceinline__ void load_x_tile(const ScParams &P, uint8_t *sx, const uint8_t *sv, int img, int y0, int x0, int rows, int cols) {
    const int cpp = P.ps >> 4;                       // 16-byte chunks per pixel (<= 11)
    const int npix = rows * cols;
    const int j = threadIdx.x & 15;
    if (j < cpp) {
        const bool data = j * 8 < P.cp;
        const int p = (P.nparts > 1 && j * 8 >= P.parts[1].cc0) ? 1 : 0;
        const ScPart &pt = P.parts[p];
        const bf16 *src = pt.x + static_cast<long long>(img) * (P.h >> pt.xup) * (P.w >> pt.xup) * pt.cstride + (j * 8 - pt.cc0);
        const int wsrc = P.w >> pt.xup;
        const uint8_t *svp = sv + p * npix;
        int ty = 0, tx = threadIdx.x >> 4;           // 16 pixels per pass; cols >= 16
        for (int pix = threadIdx.x >> 4; pix < npix; pix += 16) {
            const uint32_t dst = smem_addr(sx + static_cast<size_t>(pix) * P.ps + j * 16);
            if (data) {
                const bool v = svp[pix] != 0;
                const int y = v ? (y0 + ty) >> pt.xup : 0, x = v ? (x0 + tx) >> pt.xup : 0;
                cp_async16(dst, src + (static_cast<long long>(y) * wsrc + x) * pt.cstride, v);
            } else {
                *reinterpret_cast<uint4 *>(sx + static_cast<size_t>(pix) * P.ps + j * 16) = make_uint4(0u, 0u, 0u, 0u);
            }
            tx += 16;
            if (tx >= cols) { tx -= cols; ++ty; }
        }
    }
    cp_async_wait_all();
}

// ------------------------------------------------------------------------------------------------- forward
// KK > 0: 3x3 kernel with KK K steps known at compile time (the loops unroll: the ldmatrix -> mma chains of one warp overlap)
template <int KK>
__global__ void __launch_bounds__(SC_THREADS, 3) smallco_fwd_kernel(const ScParams P) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int kh = KK ? 3 : P.kh, kw = KK ? 3 : P.kw, nks = KK ? KK : P.ks;
    const int taps = kh * kw;
    const int rows = TH + kh - 1, cols = TW + kw - 1, npix = rows * cols;
    uint8_t *sx = smem;
    uint8_t *sw = sx + static_cast<size_t>(npix) * P.ps;          // weights [8 cout][taps * ks*16 packed channels], row pitch wp
    const int wp = (taps * nks * 32 + 16) | 16;                        // odd multiple of 16 bytes: conflict-free ldmatrix rows
    uint8_t *sv = sw + 8 * wp;                                          // validity bytes [nparts][npix]
    for (int i = threadIdx.x; i < 8 * taps * nks * 16; i += SC_THREADS) {
        const int co = i / (taps * nks * 16), k = i - co * (taps * nks * 16);
        const int tap = k / (nks * 16), cc = k - tap * (nks * 16);
        bf16 v = __float2bfloat16(0.f);
        if (cc < P.cp) v = P.w_fwd[static_cast<long long>(co) * P.kf + static_cast<long long>(tap) * P.ktap + slot_of(P, cc)];
        reinterpret_cast<bf16 *>(sw + co * wp)[k] = v;
    }
    const uint32_t sx_a = smem_addr(sx), sw_a = smem_addr(sw);
    const int j = lane >> 3, r8 = lane & 7;
    for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
        int img, ty0, tx0;
        tile_origin(P, tile, img, ty0, tx0);
        __syncthreads();
        load_valid(P, sv, img, ty0 - P.pad_h, tx0 - P.pad_w, rows, cols);
        __syncthreads();
        load_x_tile(P, sx, sv, img, ty0 - P.pad_h, tx0 - P.pad_w, rows, cols);
        __syncthreads();
        float acc[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][i] = 0.f;
#pragma unroll
        for (int tap = 0; tap < (KK ? 9 : SC_MAX_TAPS); ++tap) {
            if (!KK && tap >= taps) break;
            const int tr = tap / kw, tc = tap - tr * kw;
#pragma unroll
            for (int ks = 0; ks < (KK ? KK : SC_MAX_KS); ++ks) {
                if (!KK && ks >= nks) break;
                uint32_t b[2];
                ldsm_x2(sw_a + static_cast<uint32_t>((lane & 7) * wp + (tap * nks + ks) * 32 + ((lane >> 3) & 1) * 16), b);
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    const int col = mt * 16 + (j & 1) * 8 + r8 + tc;
                    uint32_t a[4];
                    ldsm_x4(sx_a + static_cast<uint32_t>(((warp + tr) * cols + col) * P.ps + ks * 32 + (j >> 1) * 16), a);
                    mma_16816(acc[mt], a, b);
                }
            }
        }
        // y = hole ? 0 : acc / s + b   (8 channel slots per pixel; slots >= cout are written as zeros)
        const int oy = ty0 + warp;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int ox = tx0 + mt * 16 + g + 8 * half;
                if (oy >= P.ho || ox >= P.wo) continue;
                const long long q = (static_cast<long long>(img) * P.ho + oy) * P.wo + ox;
                const float s = P.msum ? P.msum[q] : 1.f;               // null: plain convolution
                const bool hole = (s == 0.f) && !P.no_guard;
                const float inv = hole ? 0.f : 1.0f / s;
                const int co = 2 * t;
                float a = acc[mt][2 * half], b = acc[mt][2 * half + 1];
                const float b0 = (P.bias && co < P.cout) ? P.bias[co] : 0.f, b1 = (P.bias && co + 1 < P.cout) ? P.bias[co + 1] : 0.f;
                a = (hole || co >= P.cout) ? 0.f : a * inv + b0;
                b = (hole || co + 1 >= P.cout) ? 0.f : b * inv + b1;
                *reinterpret_cast<__nv_bfloat162 *>(P.y + q * P.y_cstride + co) = __floats2bfloat162_rn(a, b);
            }
    }
}

// ------------------------------------------------------------------------------------------------- data gradient
// NT > 0: 3x3 kernel with NT 8-channel output tiles known at compile time
template <int NT>
__global__ void __launch_bounds__(SC_THREADS, 2) smallco_dgrad_kernel(const ScParams P) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int kh = NT ? 3 : P.kh, kw = NT ? 3 : P.kw;
    const int taps = kh * kw;
    const int rows = TH + kh - 1, cols = TW + kw - 1;
    const int kst = (taps + 1) >> 1;                      // K steps: two taps x 8 cout each
    const int nt_count = NT ? NT : (P.cp >> 3);
    uint8_t *sdc = smem;                                  // [rows][cols] pixels x 16 B, then one zero chunk
    uint8_t *szero = sdc + static_cast<size_t>(rows) * cols * 16;
    uint8_t *sout = szero + 16;                           // [TH*TW] pixels x cp*2 bytes
    uint8_t *sw = sout + static_cast<size_t>(TH) * TW * P.cp * 2;      // weights [packed input channel][kst*16 (tap, cout)], row pitch wp
    const int wp = (kst * 32 + 16) | 16;
    uint8_t *sv = sw + static_cast<size_t>(P.cp) * wp;   // validity of the tile's own pixels [nparts][TH*TW]
    for (int i = threadIdx.x; i < P.cp * kst * 16; i += SC_THREADS) {
        const int cc = i / (kst * 16), k = i - cc * (kst * 16);
        const int tap = k >> 3, co = k & 7;
        bf16 v = __float2bfloat16(0.f);
        if (tap < taps) v = P.w_dg[static_cast<long long>(slot_of(P, cc)) * P.kd + static_cast<long long>(tap) * P.cout64 + co];
        reinterpret_cast<bf16 *>(sw + cc * wp)[k] = v;
    }
    if (threadIdx.x < 4) reinterpret_cast<uint32_t *>(szero)[threadIdx.x] = 0u;
    const uint32_t sdc_a = smem_addr(sdc), szero_a = smem_addr(szero), sw_a = smem_addr(sw);
    const int j = lane >> 3, r8 = lane & 7;
    for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
        int img, ty0, tx0;
        tile_origin(P, tile, img, ty0, tx0);
        __syncthreads();
        // dc tile: input pixel (y, x) and tap (tr, tc) read dc[y + pad - tr][x + pad - tc]
        const int y0 = ty0 + P.pad_h - (kh - 1), x0 = tx0 + P.pad_w - (kw - 1);
        for (int i = threadIdx.x; i < rows * cols; i += SC_THREADS) {
            const int ty = i / cols, tx = i - ty * cols;
            const int y = y0 + ty, x = x0 + tx;
            const bool v = y >= 0 && y < P.ho && x >= 0 && x < P.wo;
            cp_async16(sdc_a + i * 16, P.dc + ((static_cast<long long>(img) * P.ho + (v ? y : 0)) * P.wo + (v ? x : 0)) * P.dc_cstride, v);
        }
        load_valid(P, sv, img, ty0, tx0, TH, TW);
        cp_async_wait_all();
        __syncthreads();
#pragma unroll 1
        for (int mt = 0; mt < 2; ++mt) {
            float acc[SC_MAX_NT][4];
#pragma unroll
            for (int nt = 0; nt < SC_MAX_NT; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[nt][i] = 0.f;
#pragma unroll
            for (int ks = 0; ks < SC_MAX_KS; ++ks) {
                if (ks >= kst) break;
                const int tap = 2 * ks + (j >> 1);
                uint32_t addr = szero_a;
                if (tap < taps) {
                    const int tr = tap / kw, tc = tap - tr * kw;
                    addr = sdc_a + static_cast<uint32_t>(((warp + (kh - 1) - tr) * cols + mt * 16 + (j & 1) * 8 + r8 + (kw - 1) - tc) * 16);
                }
                uint32_t a[4];
                ldsm_x4(addr, a);
#pragma unroll
                for (int nt = 0; nt < (NT ? NT : SC_MAX_NT); ++nt) {
                    if (NT || nt < nt_count) {
                        uint32_t b[2];
                        ldsm_x2(sw_a + static_cast<uint32_t>((nt * 8 + (lane & 7)) * wp + ks * 32 + ((lane >> 3) & 1) * 16), b);
                        mma_16816(acc[nt], a, b);
                    }
                }
            }
#pragma unroll
            for (int nt = 0; nt < SC_MAX_NT; ++nt) {
                if (nt >= nt_count) break;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int pi = warp * TW + mt * 16 + g + 8 * half;
                    *reinterpret_cast<__nv_bfloat162 *>(sout + static_cast<size_t>(pi) * (P.cp * 2) + (nt * 8 + 2 * t) * 2) =
                        __floats2bfloat162_rn(acc[nt][2 * half], acc[nt][2 * half + 1]);
                }
            }
        }
        __syncthreads();
        // dx_part = acc * input mask of the part, 16-byte stores: sixteen lanes per pixel
        const int cpp = P.cp >> 3;
        const int jc = threadIdx.x & 15;
        if (jc < cpp) {
            const int p = (P.nparts > 1 && jc * 8 >= P.parts[1].cc0) ? 1 : 0;
            const ScPart &pt = P.parts[p];
            if (pt.dx != nullptr) {
                for (int pi = threadIdx.x >> 4; pi < TH * TW; pi += 16) {
                    const int y = ty0 + (pi >> 5), x = tx0 + (pi & 31);
                    if (y >= P.h || x >= P.w) continue;
                    uint4 v = *reinterpret_cast<const uint4 *>(sout + static_cast<size_t>(pi) * (P.cp * 2) + jc * 16);
                    if (sv[p * TH * TW + pi] == 0) v = make_uint4(0u, 0u, 0u, 0u);
                    *reinterpret_cast<uint4 *>(pt.dx + ((static_cast<long long>(img) * P.h + y) * P.w + x) * pt.dx_cstride + (jc * 8 - pt.cc0)) = v;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------- weight gradient
__global__ void __launch_bounds__(SC_THREADS, 3) smallco_wgrad_kernel(const ScParams P) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int taps = P.kh * P.kw;
    const int rows = TH + P.kh - 1, cols = TW + P.kw - 1;
    uint8_t *sx = smem;
    uint8_t *sdc = sx + static_cast<size_t>(rows) * cols * P.ps;       // [TH*TW] pixels x 16 B
    uint8_t *sv = sdc + static_cast<size_t>(TH) * TW * 16;              // validity bytes [nparts][rows*cols]
    const uint32_t sx_a = smem_addr(sx), sdc_a = smem_addr(sdc);
    // (tap, 16-channel block) units are dealt round-robin to the 8 warps; each keeps its units' 16x8 accumulators
    constexpr int UPW = (SC_MAX_TAPS * SC_MAX_KS + 7) / 8;
    const int units = taps * P.ks;
    float acc[UPW][4];
#pragma unroll
    for (int u = 0; u < UPW; ++u)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[u][i] = 0.f;
    const int j = lane >> 3, r8 = lane & 7;
    int aoff[UPW];                                        // byte offset of the unit's (tap, channel block) inside the x tile
#pragma unroll
    for (int u = 0; u < UPW; ++u) {
        const int unit = warp + 8 * u;
        aoff[u] = -1;
        if (unit < units) {
            const int tap = unit / P.ks, mt = unit - tap * P.ks;
            const int tr = tap / P.kw, tc = tap - tr * P.kw;
            aoff[u] = (tr * cols + tc) * P.ps + mt * 32;
        }
    }
    const int lane_off = ((j >> 1) * 8 + r8) * P.ps + (j & 1) * 16;
    for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
        int img, ty0, tx0;
        tile_origin(P, tile, img, ty0, tx0);
        __syncthreads();
        load_valid(P, sv, img, ty0 - P.pad_h, tx0 - P.pad_w, rows, cols);
        for (int i = threadIdx.x; i < TH * TW; i += SC_THREADS) {
            const int y = ty0 + (i >> 5), x = tx0 + (i & 31);
            const bool v = y < P.ho && x < P.wo;
            cp_async16(sdc_a + i * 16, P.dc + ((static_cast<long long>(img) * P.ho + (v ? y : 0)) * P.wo + (v ? x : 0)) * P.dc_cstride, v);
        }
        __syncthreads();
        load_x_tile(P, sx, sv, img, ty0 - P.pad_h, tx0 - P.pad_w, rows, cols);
        __syncthreads();
#pragma unroll 4
        for (int kstep = 0; kstep < TH * TW / 16; ++kstep) {
            const int prow = kstep >> 1, pcol0 = (kstep & 1) * 16;
            uint32_t b[2];
            ldsm_x2_t(sdc_a + static_cast<uint32_t>((prow * TW + pcol0 + (lane & 15)) * 16), b);
            const uint32_t base = sx_a + static_cast<uint32_t>((prow * cols + pcol0) * P.ps + lane_off);
#pragma unroll
            for (int u = 0; u < UPW; ++u) {
                if (aoff[u] < 0) break;
                uint32_t a[4];
                ldsm_x4_t(base + aoff[u], a);
                mma_16816(acc[u], a, b);
            }
        }
    }
    // D[ci][co] fragments -> fp32 KRSC gradient [cout][taps][cin]
#pragma unroll
    for (int u = 0; u < UPW; ++u) {
        const int unit = warp + 8 * u;
        if (unit >= units) break;
        const int tap = unit / P.ks, mt = unit - tap * P.ks;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int cc = mt * 16 + g + 8 * (i >> 1), co = 2 * t + (i & 1);
            if (cc >= P.cp || co >= P.cout) continue;
            const int p = (P.nparts > 1 && cc >= P.parts[1].cc0) ? 1 : 0;
            const int local = cc - P.parts[p].cc0;
            if (local >= P.parts[p].c) continue;
            atomicAdd(P.dw + (static_cast<long long>(co) * taps + tap) * P.cin + P.parts[p].choff + local, acc[u][i]);
        }
    }
}

bool fill(ScParams &P, const pcb_conv *c, const pcb_smallco_layout &L, bool grid_is_input) {
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.cin = c->cin; P.cout = c->cout; P.kh = c->kh; P.kw = c->kw; P.pad_h = c->pad_h; P.pad_w = c->pad_w;
    P.ho = c->ho; P.wo = c->wo; P.nparts = c->nparts; P.no_guard = c->no_guard;
    int cc = 0, choff = 0;
    for (int p = 0; p < c->nparts; ++p) {
        ScPart &pt = P.parts[p];
        pt.x = static_cast<const bf16 *>(c->parts[p].x); pt.mask = c->parts[p].mask;
        pt.c = c->parts[p].c; pt.c8 = (pt.c + 7) / 8 * 8; pt.cstride = c->parts[p].x_cstride; pt.xup = c->parts[p].x_up; pt.mup = c->parts[p].mask_up;
        pt.koff = L.koff[p]; pt.choff = choff; pt.cc0 = cc;
        cc += pt.c8; choff += pt.c;
    }
    P.cp = cc; P.ks = (cc + 15) / 16; P.ps = P.ks * 32 + 16;
    const int gh = grid_is_input ? c->h : c->ho, gw = grid_is_input ? c->w : c->wo;
    P.tiles_x = (gw + TW - 1) / TW; P.tiles_y = (gh + TH - 1) / TH;
    P.num_tiles = c->n * P.tiles_x * P.tiles_y;
    P.ktap = L.ktap; P.kf = L.kf; P.kd = L.kd; P.cout64 = L.cout64;
    return true;
}

// `attr_done`: one flag per device for this kernel instantiation (function attributes are per device context)
int launch(void (*kern)(const ScParams), bool (&attr_done)[PCB_MAX_DEVICES], const ScParams &P, size_t smem, int ctas_per_sm, cudaStream_t st) {
    const int dev = pcb_cur_device();
    if (!attr_done[dev]) {
        PCB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        attr_done[dev] = true;
    }
    const int grid = std::min(P.num_tiles, ctas_per_sm * pcb_num_sms());
    kern<<<grid, SC_THREADS, smem, st>>>(P);
    PCB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

bool pcb_smallco_eligible(const pcb_conv *c) {
    if (getenv("PCB_DISABLE_SMALLCO")) return false;
    if (c->dtype != PCB_BF16 || c->groups != 1 || c->stride != 1 || c->dil != 1 || c->kh > 3 || c->kw > 3 || c->cout > 8) return false;
    if (c->nparts < 1 || c->nparts > 2 || c->cin < 16) return false;
    int cp = 0;
    for (int p = 0; p < c->nparts; ++p) {
        const pcb_part &pt = c->parts[p];
        cp += (pt.c + 7) / 8 * 8;
        if (pt.x_cstride % 8 != 0 || pt.x_cstride < (pt.c + 7) / 8 * 8) return false;
        if (pt.x && (reinterpret_cast<uintptr_t>(pt.x) & 15)) return false;
        if (pt.x_up && ((c->h | c->w) & 1)) return false;
    }
    return cp <= 16 * SC_MAX_KS;
}

int pcb_smallco_forward(const pcb_conv *c, const pcb_smallco_layout &L, const void *w_fwd, const float *bias, void *y, int y_cstride, const float *msum,
                        cudaStream_t st) {
    PCB_CHECK(y_cstride % 8 == 0 && y_cstride >= 8 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "small-cout forward: y must be 16-byte aligned with a channel stride that is a multiple of 8");
    ScParams P;
    fill(P, c, L, false);
    P.w_fwd = static_cast<const bf16 *>(w_fwd); P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride;
    const int taps = c->kh * c->kw, npix = (TH + c->kh - 1) * (TW + c->kw - 1);
    const size_t smem = static_cast<size_t>(npix) * P.ps + 8 * static_cast<size_t>((taps * P.ks * 32 + 16) | 16) + 2 * npix + 16;
    static bool attr[3][PCB_MAX_DEVICES] = {};
    if (c->kh == 3 && c->kw == 3 && P.ks == 5) return launch(smallco_fwd_kernel<5>, attr[0], P, smem, 3, st);
    if (c->kh == 3 && c->kw == 3 && P.ks == 3) return launch(smallco_fwd_kernel<3>, attr[1], P, smem, 3, st);
    return launch(smallco_fwd_kernel<0>, attr[2], P, smem, 3, st);
}

int pcb_smallco_dgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, const void *w_dgrad, void *const *dx, const int *dx_cstride,
                      cudaStream_t st) {
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= 8, "small-cout dgrad: dc channel stride must be a multiple of 8");
    ScParams P;
    fill(P, c, L, true);
    P.w_dg = static_cast<const bf16 *>(w_dgrad); P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride;
    for (int p = 0; p < c->nparts; ++p) {
        P.parts[p].dx = static_cast<bf16 *>(dx[p]); P.parts[p].dx_cstride = dx_cstride[p];
        PCB_CHECK(!dx[p] || (dx_cstride[p] % 8 == 0 && dx_cstride[p] >= P.parts[p].c8 && (reinterpret_cast<uintptr_t>(dx[p]) & 15) == 0),
                  "small-cout dgrad: dx[%d] must be 16-byte aligned with a channel stride that is a multiple of 8", p);
    }
    const int kst = (c->kh * c->kw + 1) / 2;
    const size_t smem = static_cast<size_t>(TH + c->kh - 1) * (TW + c->kw - 1) * 16 + 16 + static_cast<size_t>(TH) * TW * P.cp * 2 +
                        static_cast<size_t>(P.cp) * ((kst * 32 + 16) | 16) + 2 * TH * TW + 16;
    static bool attr[3][PCB_MAX_DEVICES] = {};
    if (c->kh == 3 && c->kw == 3 && P.cp == 72) return launch(smallco_dgrad_kernel<9>, attr[0], P, smem, 2, st);
    if (c->kh == 3 && c->kw == 3 && P.cp == 40) return launch(smallco_dgrad_kernel<5>, attr[1], P, smem, 2, st);
    return launch(smallco_dgrad_kernel<0>, attr[2], P, smem, 2, st);
}

int pcb_smallco_wgrad(const pcb_conv *c, const pcb_smallco_layout &L, const void *dc, int dc_cstride, float *dw, bool zero_dw, cudaStream_t st) {
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= 8, "small-cout wgrad: dc channel stride must be a multiple of 8");
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * c->cout * c->kh * c->kw * c->cin, st));
    ScParams P;
    fill(P, c, L, false);
    P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.dw = dw;
    const int npix = (TH + c->kh - 1) * (TW + c->kw - 1);
    const size_t smem = static_cast<size_t>(npix) * P.ps + static_cast<size_t>(TH) * TW * 16 + 2 * npix + 16;
    static bool attr[PCB_MAX_DEVICES] = {};
    return launch(smallco_wgrad_kernel, attr, P, smem, 3, st);
}

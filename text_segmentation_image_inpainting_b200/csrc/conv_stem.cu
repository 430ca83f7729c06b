// conv_stem.cu -- the 7x7 / stride-2 / pad-3 stems over an image (<= 8 channels; models/image_inpainting.py:118 of the reference,
// BaseModels / MobileNetV2 / Xception entry convolutions have other shapes and keep their paths) as a 4x4 / stride-1 convolution over
// the SPACE-TO-DEPTH image:
//     xs[n][sy][sx][(a, b, ch)] = x[n][2 sy + a][2 sx + b][ch] * mask[...]          SC = 4 CC channels per half-resolution cell
//     y[o] = sum_t w[t] x[2 o + t - 3]  =  sum_{j=0..3} sum_{a=0,1} w[2 j + a - 1] xs[o + j - 2][a]      (w[-1] = w[7] = 0)
// i.e. kernel 4, padding 2 in front (the "extra" output row/column a symmetric padding would give is simply not computed).
// CC = 4 sub-pixel channels for images of up to 4 channels (SC = 16: a 3-channel image fills 12 of them), CC = 8 for 5-8.
// x * mask happens in the space-to-depth pass (sub-pixels of a cell have different mask values, so the GEMMs run without hole
// rows).  The GEMM K index of tap (ja, jb) and cell channel k is (ja * 4 + jb) * SC + k, so one kernel row ja is 4 SC
// consecutive K elements: one (SC = 16) or two (SC = 32) 64-element K blocks.
//
// Both directions have kernels of their own here.  Their A operands are im2row tiles of one kernel row -- [pixel][jb][SC],
// 128-byte rows in the 128B-swizzled layout wgmma reads -- gathered from xs by cp.async through L1 (each cell is read for four
// jb, so L2 sees it about once per kernel row).  A row-halo TMA tile with row-shifted descriptors cannot serve them: a cell is
// only 32 or 64 bytes wide.
//   forward   stem_fwd_kernel: persistent CTAs with the layer's weights (one 64-column N tile) resident in shared memory, so
//             only activations stream; the epilogue is the TMA-fed kernels' (pcb_tc_epi.cuh: renormalisation, bias, eval-mode
//             BatchNorm + activation and the BatchNorm statistics, staged in bf16 and drained by dedicated epilogue warps).
//   wgrad     stem_wgrad_kernel: D[(ja, jb, k)][co] = sum_p xs[p + (ja, jb) - 2][k] dc[p][co] for ALL 16 taps in one CTA, so xs
//             and dc are each read once; split-K over pixel ranges with red.global.add into dwsub, then stem_dw_gather_kernel
//             moves the 4x4 gradient back into the [co][7][7][c] master layout.
#include <string.h>

#include <algorithm>

#include "pcb_tc_epi.cuh"

namespace {

constexpr int SK = 4;              // sub-kernel size

size_t rup256(size_t v) { return (v + 255) / 256 * 256; }
int rup64(int v) { return (v + 63) / 64 * 64; }
size_t s2d_bytes(const pcb_conv *c, int sc) { return rup256(static_cast<size_t>(c->n) * (c->h / 2) * (c->w / 2) * sc * sizeof(bf16)); }
size_t dwsub_bytes(const pcb_conv *c, int sc) { return rup256(sizeof(float) * c->cout * SK * SK * sc); }

}  // namespace

StemPlan pcb_stem_plan(const pcb_conv *c) {
    StemPlan K;
    memset(&K, 0, sizeof(K));
    if (c->dtype != PCB_BF16 || c->groups != 1 || c->nparts != 1 || c->kh != 7 || c->kw != 7 || c->stride != 2 || c->pad_h != 3 || c->pad_w != 3 ||
        c->dil != 1) return K;
    const pcb_part &p = c->parts[0];
    if (p.x_up || p.c > 8 || p.x_cstride != 8 || (p.mask && p.mask_up != 0) || ((c->h | c->w) & 1)) return K;
    if (p.x && (reinterpret_cast<uintptr_t>(p.x) & 15)) return K;
    if (c->ho != c->h / 2 || c->wo != c->w / 2 || c->cout < 32 || (c->cout & 7)) return K;
    // the 32-bit index bounds of the tensor-core kernels, for the 4x4 problem's outputs and its widest space-to-depth image
    const long long lim = (1ll << 31) - 1, cells = static_cast<long long>(c->n) * c->ho * c->wo;
    if (cells * rup64(c->cout) > lim || cells * 32 > lim) return K;
    K.sc = p.c <= 4 ? 16 : 32;
    // The operand and workspace sizes a stem layer reports through the C ABI stay those of the earlier layout, which callers
    // allocate and the dispatch fixture (tests/golden/conv_dispatch.json) pins: a 4x4 problem over 32-channel cells on the
    // general tensor-core kernels, sized by conv_tc.cu's layout_of() (forward operand rup(cout, bn_f) rows x 16 taps x one
    // 64-wide K block, bn_f = 128 for multiples of 128, else 64) and tc_plan() (one tap-validity word per output pixel), plus
    // the fp32 staging of its weights, the 32-channel image and dwsub.  The kernels here use a prefix of each buffer:
    // rup(cout, 64) x 16 sc bf16 weights (about a third of the operand), the image and dwsub at sc channels.  Nothing reads
    // the tap-word part any more.
    const int bn_f = (c->cout % 128 == 0) ? 128 : 64;
    K.fwd_extra = static_cast<size_t>((c->cout + bn_f - 1) / bn_f * bn_f) * SK * SK * 64 + 2 * static_cast<size_t>(c->cout) * SK * SK * 32;
    K.workspace = s2d_bytes(c, 32) + dwsub_bytes(c, 32) + rup256(static_cast<size_t>(cells) * sizeof(uint64_t));
    K.ok = true;
    return K;
}

namespace {

// one thread per (cell, a): two horizontally adjacent pixels -> 2 cc channels of the cell, times the hole mask
__global__ void s2d_kernel(const bf16 *__restrict__ x, const uint8_t *__restrict__ mask, bf16 *__restrict__ xs, int n, int h, int w, int cc) {
    const int hs = h >> 1, ws = w >> 1;
    const long long total = static_cast<long long>(n) * hs * ws * 2;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int a = static_cast<int>(i & 1);
        const long long cell = i >> 1;
        const int sx = static_cast<int>(cell % ws);
        const long long t = cell / ws;
        const int sy = static_cast<int>(t % hs), img = static_cast<int>(t / hs);
        const long long q = (static_cast<long long>(img) * h + 2 * sy + a) * w + 2 * sx;
        const bool k0 = !mask || mask[q] != 0, k1 = !mask || mask[q + 1] != 0;
        bf16 *dst = xs + cell * 4 * cc + a * 2 * cc;
        if (cc == 4) {
            const uint2 z = make_uint2(0u, 0u);
            const uint2 v0 = k0 ? __ldg(reinterpret_cast<const uint2 *>(x + q * 8)) : z, v1 = k1 ? __ldg(reinterpret_cast<const uint2 *>(x + q * 8 + 8)) : z;
            *reinterpret_cast<uint4 *>(dst) = make_uint4(v0.x, v0.y, v1.x, v1.y);
        } else {
            const uint4 z = make_uint4(0u, 0u, 0u, 0u);
            reinterpret_cast<uint4 *>(dst)[0] = k0 ? __ldg(reinterpret_cast<const uint4 *>(x + q * 8)) : z;
            reinterpret_cast<uint4 *>(dst)[1] = k1 ? __ldg(reinterpret_cast<const uint4 *>(x + q * 8 + 8)) : z;
        }
    }
}

// (ja, jb, a, b, ch) of K index k of the 4x4 problem (k < 16 sc)
struct StemK { int ja, jb, a, b, ch; };
__host__ __device__ __forceinline__ StemK stem_k(int k, int sc) {
    const int cc = sc >> 2;
    StemK r;
    r.ja = k / (4 * sc); r.jb = (k / sc) & 3; r.a = (k / (2 * cc)) & 1; r.b = (k / cc) & 1; r.ch = k % cc;
    return r;
}

// wst[co][k] = w[co][2 ja + a - 1][2 jb + b - 1][ch] in bf16, rows padded to a multiple of 64 with zeros (every element written)
__global__ void stem_weight_kernel(const float *__restrict__ w, bf16 *__restrict__ wst, int cout, int rows, int cin, int sc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * SK * SK * sc) return;
    const int co = i / (SK * SK * sc);
    const StemK k = stem_k(i % (SK * SK * sc), sc);
    const int ty = 2 * k.ja + k.a - 1, tx = 2 * k.jb + k.b - 1;
    const bool in = co < cout && ty >= 0 && ty < 7 && tx >= 0 && tx < 7 && k.ch < cin;
    wst[i] = __float2bfloat16_rn(in ? w[((static_cast<long long>(co) * 7 + ty) * 7 + tx) * cin + k.ch] : 0.f);
}

// dw[co][ty][tx][ch] += dwsub[co][k] of the k with 2 ja + a - 1 = ty, 2 jb + b - 1 = tx
__global__ void stem_dw_gather_kernel(const float *__restrict__ dwsub, float *__restrict__ dw, int cout, int cin, int sc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cout * 49 * cin) return;
    const int ch = i % cin, tx = (i / cin) % 7, ty = (i / (cin * 7)) % 7, co = i / (cin * 49);
    const int ja = (ty + 1) >> 1, a = (ty + 1) & 1, jb = (tx + 1) >> 1, b = (tx + 1) & 1;
    dw[i] += dwsub[static_cast<long long>(co) * SK * SK * sc + (ja * SK + jb) * sc + (a * 2 + b) * (sc >> 2) + ch];
}

// cp.async of one 16-byte chunk of an im2row row: K elements [kidx, kidx + 8) of output pixel (img, oy, ox) -> dst (zero
// outside the space-to-depth image)
__device__ __forceinline__ void im2row_chunk(const bf16 *xs, int hs, int ws, int sc, bool rv, int img, int oy, int ox, int kidx, uint32_t dst) {
    const int ja = kidx / (4 * sc), rem = kidx - ja * 4 * sc, jb = rem / sc, ch0 = rem - jb * sc;
    const int y = oy + ja - 2, x = ox + jb - 2;
    const bool ok = rv && y >= 0 && y < hs && x >= 0 && x < ws;
    const bf16 *src = ok ? xs + ((static_cast<long long>(img) * hs + y) * ws + x) * sc + ch0 : xs;
    ptx::cp_async_16_ca(dst, src, ok);
}

// ---- forward -------------------------------------------------------------------------------------------------------------
// 512 threads: warps 0-7 two consumer warpgroups (wgmma of their 64 rows, then the forward element math into the bf16 staging
// tile), warps 8-11 the im2row gather, warps 12-15 the epilogue warps of the TMA-fed kernels.  CTA b owns N tile b % n_tiles
// (its 64 output channels' weights stay in shared memory) and walks M tiles of 128 output pixels.  One ring stage is the
// [128 px][64 K] tile of one K block (a kernel row at SC = 16, half of one at SC = 32).
constexpr int STEM_THREADS = MMA_THREADS + 4 * 32 + EPI_WARPS * 32;
constexpr int STEM_PROD_THREADS = 128;
constexpr int STEM_EPI_WARP0 = MMA_WARPS + 4;
constexpr uint32_t STEM_W_BLOCK = 64 * 128;           // [64 co][64 K] bf16

struct StemFwdParams {
    TcParams P;                    // epilogue fields (m_total, msum, no_guard, bias, y, BatchNorm statistics, ep_*, abort_flag)
    const bf16 *xs, *wst;
    int hs, ws, sc, nkb, n_tiles, stages;
};

__global__ void __launch_bounds__(STEM_THREADS, 1) stem_fwd_kernel(const __grid_constant__ StemFwdParams A) {
    const TcParams &P = A.P;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    uint8_t *smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
    const int S = A.stages, nkb = A.nkb;
    const uint32_t sW = smem_base, sA = sW + nkb * STEM_W_BLOCK;
    const uint32_t sBar = sA + S * A_STAGE_BYTES;
    const uint32_t bar_full = sBar, bar_empty = sBar + 8 * MAX_RING;
    const uint32_t acc_full = sBar + 16 * MAX_RING, acc_empty = acc_full + 8;
    const uint32_t s_stat_addr = sBar + TMA_BAR_BYTES;
    bf16 *acc_stage = reinterpret_cast<bf16 *>(smem_gen + (s_stat_addr + EPI_STAT_SMEM_BYTES - smem_base));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int n0 = (blockIdx.x % A.n_tiles) * 64;
    const int tile0 = blockIdx.x / A.n_tiles, tstep = gridDim.x / A.n_tiles;
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) { ptx::mbar_init(bar_full + 8 * s, STEM_PROD_THREADS); ptx::mbar_init(bar_empty + 8 * s, 2); }
        ptx::mbar_init(acc_full, MMA_WARPS); ptx::mbar_init(acc_empty, EPI_WARPS);     // one arrival per warp
        ptx::fence_mbar_init();
    }
    // resident weights: rows [n0, n0 + 64) of wst as nkb K-major [64 co][128 B] blocks, 128B-swizzled
    const int kw = SK * SK * A.sc;
    for (int i = threadIdx.x; i < nkb * 64 * 8; i += STEM_THREADS) {
        const int kb = i >> 9, r = (i >> 3) & 63, ch = i & 7;
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(A.wst + static_cast<long long>(n0 + r) * kw + kb * 64 + ch * 8));
        *reinterpret_cast<uint4 *>(smem_gen + kb * STEM_W_BLOCK + r * 128 + ((ch ^ (r & 7)) << 4)) = v;
    }
    ptx::fence_proxy_async_smem();                        // st.shared (generic proxy) -> wgmma (async proxy)
    __syncthreads();

    if (warp < MMA_WARPS) {
        // ================================ consumer warpgroups ================================
        const int e = warp, g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint64_t desc_a0 = ptx::make_smem_desc(sA + g * 64 * 128, 16, 1024);     // this warpgroup's 64 rows
        const uint64_t desc_w0 = ptx::make_smem_desc(sW, 16, 1024);
        int s = 0;
        uint32_t ph = 0, aph = 1;                                      // aph: first pass, the staging tile is free
        bool dead = false;
        for (int mt = tile0; mt < m_tiles && !dead; mt += tstep) {
            const ConsRows cr = cons_rows<0>(P, mt * BLOCK_M, e, lane);
            float acc[32];
            zero_acc(acc);
            int held = -1;
            for (int kb = 0; kb < nkb; ++kb) {
                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 131))) { dead = true; break; }
                ptx::fence_proxy_async_smem();                     // cp.async (generic proxy) data -> wgmma (async proxy)
                const uint64_t da = desc_a0 + static_cast<uint64_t>(s * (A_STAGE_BYTES >> 4));
                const uint64_t dw = desc_w0 + static_cast<uint64_t>(kb * (STEM_W_BLOCK >> 4));
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) ptx::wgmma_bf16<64, 0, 0>(acc, da + 2 * k, dw + 2 * k);
                ptx::wgmma_commit();
                // keep one K block in flight: the previous stage is released once its MMAs completed
                ptx::wgmma_wait<1>();
                if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
                held = s;
                if (++s == S) { s = 0; ph ^= 1; }
            }
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(acc);
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            if (dead) break;
            // The element math runs here, between two tiles' MMAs.  Two accumulator sets that issue tile i+1's MMAs before
            // staging tile i were measured slower (DESIGN 4.5), so this is not what bounds the kernel.
            if (!tma_stage_tile<64, 0>(P, acc, acc_stage, acc_full, acc_empty, aph, e, lane, n0, cr, 132)) break;
        }
    } else if (warp < STEM_EPI_WARP0) {
        // ================================ im2row gather ================================
        // thread t: 16-byte chunk t & 7 of rows t / 8 + 16 i; every row of a thread has the same swizzle phase
        const int t = threadIdx.x - MMA_THREADS, chunk = t & 7, r0 = t >> 3;
        const uint32_t sw = static_cast<uint32_t>((chunk ^ (r0 & 7)) << 4);
        const int plane = A.hs * A.ws;
        int s = 0;
        uint32_t ph = 1;                                               // first pass over the ring: stages are free
        bool dead = false;
        for (int mt = tile0; mt < m_tiles && !dead; mt += tstep) {
            int img[8], oy[8], ox[8];
            bool rv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int m = mt * BLOCK_M + r0 + 16 * i;
                rv[i] = m < P.m_total;
                const int mm = rv[i] ? m : 0;
                img[i] = mm / plane;
                const int rem = mm - img[i] * plane;
                oy[i] = rem / A.ws; ox[i] = rem - oy[i] * A.ws;
            }
            for (int kb = 0; kb < nkb; ++kb) {
                if (!ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 133)) { dead = true; break; }
                const uint32_t dst = sA + s * A_STAGE_BYTES + r0 * 128 + sw;
#pragma unroll
                for (int i = 0; i < 8; ++i) im2row_chunk(A.xs, A.hs, A.ws, A.sc, rv[i], img[i], oy[i], ox[i], kb * 64 + chunk * 8, dst + i * 16 * 128);
                ptx::cp_async_mbar_arrive(bar_full + 8 * s);
                ptx::mbar_arrive(bar_full + 8 * s);
                if (++s == S) { s = 0; ph ^= 1; }
            }
        }
        ptx::cp_async_wait<0>();
    } else {
        // ================================ epilogue warps ================================
        const int w = warp - STEM_EPI_WARP0;
        float *s_stat = P.bn_sums != nullptr ? reinterpret_cast<float *>(smem_gen + (s_stat_addr - smem_base)) + w * EPI_STAT_SLICE : nullptr;
        int stat_n0 = -1;
        auto origin = [&](int mt, int &m0, int &tn0) { m0 = mt * BLOCK_M; tn0 = n0; };
        tma_epilogue_warps<64, 0>(P, tile0, tstep, m_tiles, origin, acc_stage, acc_full, acc_empty, s_stat, stat_n0, w, lane, 134);
        ptx::named_sync(1, EPI_WARPS * 32);                   // all four statistics slices are complete
        if (s_stat != nullptr && stat_n0 >= 0) tc_stats_final<64>(P, s_stat - w * EPI_STAT_SLICE, w, lane, stat_n0);
    }
}

// ---- weight gradient -----------------------------------------------------------------------------------------------------
// 384 threads: warps 0-7 two consumer warpgroups, warps 8-11 the gather.  A CTA owns a range of K blocks of 64 output pixels
// and the 64 output channels [n0, n0 + 64).  Per K block one stage holds the 16 SC / 64 im2row tiles [64 px][64 K] (both
// operands MN-major: a 128-byte row is one pixel) and the dc tile [64 px][64 co]; warpgroup g accumulates the MB 64-row
// blocks [g MB, g MB + MB) of D = all 16 taps x SC channels, 32 MB fp32 registers per thread.
constexpr int STEM_WG_THREADS = MMA_THREADS + 4 * 32;

struct StemWgParams {
    const bf16 *xs, *dc;
    float *dwsub;                  // [cout][16 sc] fp32, pre-zeroed
    int *abort_flag;
    int hs, ws, sc, cin, cout, dc_cstride, m_total, kb_per_cta, stages;
};

template <int MB>
__global__ void __launch_bounds__(STEM_WG_THREADS, 1) stem_wgrad_kernel(const __grid_constant__ StemWgParams W) {
    constexpr uint32_t BLK = 64 * 128;
    constexpr uint32_t A_BYTES = 2 * MB * BLK, STAGE = A_BYTES + BLK;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int S = W.stages;
    const uint32_t bar_full = smem_base + S * STAGE, bar_empty = bar_full + 8 * MAX_RING;
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int n0 = blockIdx.y * 64;
    const int total_kb = (W.m_total + 63) / 64;
    const int kb_begin = blockIdx.x * W.kb_per_cta;
    const int num_kb = max(0, min(total_kb, kb_begin + W.kb_per_cta) - kb_begin);

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) { ptx::mbar_init(bar_full + 8 * s, STEM_PROD_THREADS); ptx::mbar_init(bar_empty + 8 * s, 2); }
        ptx::fence_mbar_init();
    }
    __syncthreads();
    if (warp < MMA_WARPS) {
        // ================================ consumer warpgroups ================================
        const int g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + g * MB * BLK, BLK, 1024);
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_BYTES, BLK, 1024);
        float acc[MB][32];
#pragma unroll
        for (int j = 0; j < MB; ++j) zero_acc(acc[j]);
        int s = 0, held = -1;
        uint32_t ph = 0;
        bool dead = false;
        for (int it = 0; it < num_kb; ++it) {
            if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full + 8 * s, ph, W.abort_flag, 231))) { dead = true; break; }
            ptx::fence_proxy_async_smem();
            const uint64_t da = desc_a0 + static_cast<uint64_t>(s * (STAGE >> 4)), db = desc_b0 + static_cast<uint64_t>(s * (STAGE >> 4));
            ptx::wgmma_fence();
#pragma unroll
            for (int j = 0; j < MB; ++j)
#pragma unroll
                for (int k = 0; k < 4; ++k)                       // 16 pixels (two 8-row atoms = 2048 bytes) per step
                    ptx::wgmma_m64n64<1, 1>(acc[j], da + j * (BLK >> 4) + 128 * k, db + 128 * k);
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            held = s;
            if (++s == S) { s = 0; ph ^= 1; }
        }
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < MB; ++j) ptx::wgmma_fence_regs(acc[j]);
        if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
        // ---- D[k][co] -> red.global.add into dwsub[co][k]; rows of taps outside the 7x7 kernel and of padding channels are
        // never read back and are skipped
        if (!dead && num_kb > 0) {
            const int kw = SK * SK * W.sc;
#pragma unroll
            for (int j = 0; j < MB; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int k = (g * MB + j) * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h;
                    const StemK q = stem_k(k, W.sc);
                    const int ty = 2 * q.ja + q.a - 1, tx = 2 * q.jb + q.b - 1;
                    if (ty < 0 || ty >= 7 || tx < 0 || tx >= 7 || q.ch >= W.cin) continue;
#pragma unroll
                    for (int i = 2 * h; i < 32; i += 4)
#pragma unroll
                        for (int l = 0; l < 2; ++l) {
                            const int co = n0 + 8 * (i >> 2) + 2 * (lane & 3) + l;
                            if (co < W.cout) atomicAdd(W.dwsub + static_cast<long long>(co) * kw + k, acc[j][i + l]);
                        }
                }
        }
    } else {
        // ================================ gather: im2row tiles and the dc tile ================================
        const int t = threadIdx.x - MMA_THREADS, chunk = t & 7, r0 = t >> 3;
        const uint32_t sw = static_cast<uint32_t>((chunk ^ (r0 & 7)) << 4);
        const int plane = W.hs * W.ws;
        const int co = n0 + chunk * 8;
        int s = 0;
        uint32_t ph = 1;
        for (int it = 0; it < num_kb; ++it) {
            if (!ptx::mbar_wait(bar_empty + 8 * s, ph, W.abort_flag, 233)) break;
            const uint32_t dst = smem_base + s * STAGE + r0 * 128 + sw;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = (kb_begin + it) * 64 + r0 + 16 * i;
                const bool rv = m < W.m_total;
                const int mm = rv ? m : 0, img = mm / plane, rem = mm - img * plane, oy = rem / W.ws, ox = rem - oy * W.ws;
                const uint32_t d = dst + i * 16 * 128;
#pragma unroll
                for (int b = 0; b < 2 * MB; ++b) im2row_chunk(W.xs, W.hs, W.ws, W.sc, rv, img, oy, ox, b * 64 + chunk * 8, d + b * BLK);
                const bool ok = rv && co < W.cout;
                ptx::cp_async_16(d + A_BYTES, ok ? W.dc + static_cast<long long>(mm) * W.dc_cstride + co : W.dc, ok);
            }
            ptx::cp_async_mbar_arrive(bar_full + 8 * s);
            ptx::mbar_arrive(bar_full + 8 * s);
            if (++s == S) { s = 0; ph ^= 1; }
        }
        ptx::cp_async_wait<0>();
    }
}

int run_s2d(const pcb_conv *c, int sc, bf16 *xs, cudaStream_t st) {
    const pcb_part &p = c->parts[0];
    PCB_CHECK(p.x != nullptr, "space-to-depth stem: null x");
    const long long total = static_cast<long long>(c->n) * (c->h / 2) * (c->w / 2) * 2;
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, 16ll * pcb_num_sms())));
    s2d_kernel<<<grid, 256, 0, st>>>(static_cast<const bf16 *>(p.x), p.mask, xs, c->n, c->h, c->w, sc / 4);
    PCB_LAUNCH_CHECK();
    return 0;
}

constexpr size_t STEM_MAX_SMEM = 227 * 1024;

}  // namespace

int pcb_stem_weight_prepare(const pcb_conv *c, const StemPlan &K, const float *w_master, void *w_fwd_extra, bool, cudaStream_t st) {
    PCB_CHECK(K.ok && w_fwd_extra, "space-to-depth stem: weight prepare on a layer that does not take this path");
    const int rows = rup64(c->cout), total = rows * SK * SK * K.sc;
    stem_weight_kernel<<<(total + 255) / 256, 256, 0, st>>>(w_master, static_cast<bf16 *>(w_fwd_extra), c->cout, rows, c->cin, K.sc);
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_stem_forward(const pcb_conv *c, const StemPlan &K, const void *w_fwd_extra, const float *bias, void *y, int y_cstride,
                     const float *msum, void *workspace, double *bn_sums, const pcb_ep *ep, cudaStream_t st) {
    PCB_CHECK(K.ok && workspace, "space-to-depth stem forward: wrong layer / no workspace");
    PCB_CHECK((reinterpret_cast<uintptr_t>(y) & 15) == 0, "space-to-depth stem forward: y must be 16-byte aligned");
    int *flag = pcb_tc_abort_flag();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    bf16 *xs = static_cast<bf16 *>(workspace);
    if (int rc = run_s2d(c, K.sc, xs, st)) return rc;
    StemFwdParams A;
    memset(&A, 0, sizeof(A));
    TcParams &P = A.P;
    P.n = c->n; P.h = P.ho = c->ho; P.w = P.wo = c->wo; P.cout = c->cout; P.m_total = c->n * c->ho * c->wo;
    P.nparts = 1; P.no_guard = c->no_guard; P.sub = 1; P.fh = c->ho; P.fw = c->wo;
    P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride; P.abort_flag = flag;
    P.bn_sums = bn_sums; P.bn_c = c->cout;
    if (ep != nullptr) { P.ep_on = 1; P.ep_scale = ep->scale; P.ep_shift = ep->shift; P.ep_act = ep->act; P.ep_slope = ep->slope; }
    A.xs = xs; A.wst = static_cast<const bf16 *>(w_fwd_extra);
    A.hs = c->ho; A.ws = c->wo; A.sc = K.sc; A.nkb = K.sc / 4; A.n_tiles = rup64(c->cout) / 64;
    const size_t fixed = 1024 + static_cast<size_t>(A.nkb) * STEM_W_BLOCK + TMA_BAR_BYTES + EPI_STAT_SMEM_BYTES + bf16_stage_bytes(64);
    A.stages = static_cast<int>(std::min<size_t>(MAX_RING, (STEM_MAX_SMEM - fixed) / A_STAGE_BYTES));
    PCB_CHECK(A.stages >= 2, "space-to-depth stem forward: the ring does not fit");
    const size_t smem = fixed + static_cast<size_t>(A.stages) * A_STAGE_BYTES;
    PCB_SMEM_OPT_IN(stem_fwd_kernel, STEM_MAX_SMEM);
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int per_n = std::max(1, std::min(m_tiles, pcb_num_sms() / A.n_tiles));
    stem_fwd_kernel<<<per_n * A.n_tiles, STEM_THREADS, smem, st>>>(A);
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_stem_wgrad(const pcb_conv *c, const StemPlan &K, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw,
                   cudaStream_t st) {
    PCB_CHECK(K.ok && workspace, "space-to-depth stem wgrad: wrong layer / no workspace");
    PCB_CHECK((reinterpret_cast<uintptr_t>(dc) & 15) == 0, "space-to-depth stem wgrad: dc must be 16-byte aligned");
    int *flag = pcb_tc_abort_flag();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * c->cout * 49 * c->cin, st));
    uint8_t *ws = static_cast<uint8_t *>(workspace);
    bf16 *xs = reinterpret_cast<bf16 *>(ws);
    float *dwsub = reinterpret_cast<float *>(ws + s2d_bytes(c, K.sc));
    if (int rc = run_s2d(c, K.sc, xs, st)) return rc;
    PCB_CUDA(cudaMemsetAsync(dwsub, 0, sizeof(float) * c->cout * SK * SK * K.sc, st));
    StemWgParams W;
    memset(&W, 0, sizeof(W));
    W.xs = xs; W.dc = static_cast<const bf16 *>(dc); W.dwsub = dwsub; W.abort_flag = flag;
    W.hs = c->ho; W.ws = c->wo; W.sc = K.sc; W.cin = c->cin; W.cout = c->cout; W.dc_cstride = dc_cstride; W.m_total = c->n * c->ho * c->wo;
    const size_t stage = static_cast<size_t>(K.sc / 4 + 1) * 64 * 128;
    W.stages = static_cast<int>(std::min<size_t>(MAX_RING, (STEM_MAX_SMEM - 1024 - 16 * MAX_RING) / stage));
    const size_t smem = 1024 + W.stages * stage + 16 * MAX_RING;
    const int co_tiles = rup64(c->cout) / 64;
    const int total_kb = (W.m_total + 63) / 64;
    const int ctas = std::max(1, std::min(total_kb, pcb_num_sms() / co_tiles));
    W.kb_per_cta = (total_kb + ctas - 1) / ctas;
    dim3 grid((total_kb + W.kb_per_cta - 1) / W.kb_per_cta, co_tiles);
    if (K.sc == 16) {
        PCB_SMEM_OPT_IN(stem_wgrad_kernel<2>, STEM_MAX_SMEM);
        stem_wgrad_kernel<2><<<grid, STEM_WG_THREADS, smem, st>>>(W);
    } else {
        PCB_SMEM_OPT_IN(stem_wgrad_kernel<4>, STEM_MAX_SMEM);
        stem_wgrad_kernel<4><<<grid, STEM_WG_THREADS, smem, st>>>(W);
    }
    PCB_LAUNCH_CHECK();
    const int total = c->cout * 49 * c->cin;
    stem_dw_gather_kernel<<<(total + 255) / 256, 256, 0, st>>>(dwsub, dw, c->cout, c->cin, K.sc);
    PCB_LAUNCH_CHECK();
    return 0;
}

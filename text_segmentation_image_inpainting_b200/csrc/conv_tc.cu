// conv_tc.cu -- partial convolution as implicit GEMM on the Hopper tensor cores (wgmma / TMA / mbarrier).
//
// Replaces (per layer) the reference's pair of dense convolutions + ~9 elementwise passes
// (models/partial_convolution.py:49-80): `feature_conv(x*mask)`, the all-ones `mask_conv`, `==0`,
// `masked_fill_`, `(out-b)/mask_sum+b`, `masked_fill_`, `ones_like`+`masked_fill_` -- and, in the U-Net
// decoders, the `nn.Upsample` + `torch.cat` in front of it (models/image_inpainting.py:183-185).
//
// Two generations of kernels live in this file:
//
// (1) TMA-FED kernels (pconv_tc_tma_kernel, pconv_tc_wgrad_tma_kernel) -- the shipped hot path for power-of-two pixel grids.
//     GEMM view   M = output pixels (n*ho*wo) [fwd]  or input pixels (n*h*w) [dgrad];  N = cout [fwd] / input channels [dgrad];
//                 K walked tap-major in 64-element blocks.
//     A operand   the im2col rows of a tap are ONE 4-D TMA tile of the NHWC tensor (a 128-pixel M tile is a box of the
//                 pixel grid): padding = out-of-range zero fill, stride 2 = traversal stride, channel padding = map extent.
//                 Holes (x*mask) are zeroed in the landed tile by fixer warps.  Row-halo tiles serve the kw taps of a kernel row
//                 through row-shifted SWIZZLE_128B descriptors.  2x-upsampled sources are first copied densely into the
//                 workspace (TMA cannot replicate pixels).
//     B operand   weights [N][K] bf16 (K padded to the same block structure), TMA 2D tiles (SWIZZLE_128B).
//     MMA         wgmma.mma_async m64nNk16 bf16 -> fp32, N in {32, 64, 128, 256}: two consumer warpgroups each own 64 rows of
//                 the 128-row tile and hold its accumulators in registers; stages are released through mbarriers once
//                 wgmma.wait_group reports the MMAs that read them complete.
//     epilogue    registers -> fwd: y = hole ? 0 : acc / s + bias (s = mask box sum) in the consumers -> bf16 staging tile ->
//                 one thread per row, dgrad: dx_part = staged value * input-mask of that part; bf16 NHWC stores.
//                 Stride-2 dgrad = four stride-1 parity classes.
//     wgrad       D[k][co] (+)= sum_pixels x[p+tap][k] * dc[p][co]: both operands MN-major "pixel row x 128-byte channel chunk"
//                 tiles by TMA, split-K over pixels with fp32 red.global.add into the (logical, unpadded) KRSC gradient.
//
// (2) cp.async-GATHER kernels (pconv_tc_persistent_kernel, pconv_tc_wgrad_kernel) -- the first generation, kept for shapes (1)
//     does not take: arbitrary pixel grids, and the row-packed small-Cin mode (cin <= 8, e.g. the RGB stem: one K block = one
//     kernel ROW, its eight 16-byte chunks are the taps of that row, so a 7x7x3 stem costs 7 K blocks, not 49).  Their A
//     operand is gathered by 4 producer warps with 16-byte zero-filling cp.async from up to 2 concatenated, optionally
//     2x-upsampled sources, driven by per-pixel tap-validity words (tapmask_kernel).
//
// DESIGN.md section 4 has the anatomy and the reasons behind these choices.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "pcb_common.cuh"
#include "pcb_ptx.cuh"
#include "pcb_tc_epi.cuh"

namespace {

// 32 values per lane, 32 lanes: returns in lane l the sum over all lanes of v[l] (a transposing butterfly: 31 shuffles)
__device__ __forceinline__ float warp_transpose_sum(float (&v)[32], int lane) {
#pragma unroll
    for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (i < (n >> 1)) {
                const float send = upper ? v[i] : v[i + (n >> 1)];
                const float keep = upper ? v[i + (n >> 1)] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
    }
    return v[0];
}

// -------------------------------------------------------------------------------------------------
// epilogue shared by the forward / dgrad kernels: staged fp32 accumulators -> renormalise / mask -> bf16 NHWC
// -------------------------------------------------------------------------------------------------
// `acc_row` is the row of the staging tile that holds GEMM row `er.m`.  Columns [cb, ce) of the tile (multiples of 32).  s_stat:
// this warp's accumulators [sums of its columns | squares at offset sq_off].
__device__ __forceinline__ void load_acc32(const float *src, uint32_t (&r)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 v = reinterpret_cast<const uint4 *>(src)[j];
        r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
    }
}

template <int BLOCK_N, int MODE>
__device__ __forceinline__ void tc_epilogue(const TcParams &P, const EpiRow &er, const float *acc_row, int lane, int n0, float *s_stat,
                                            int cb, int ce, int sq_off) {
                const bool rvalid = er.rvalid, hole = er.hole;
                const long long mo = er.mo;
    #pragma unroll 1
                for (int c0 = cb; c0 < ce; c0 += 32) {
                    uint32_t r[32];
                    load_acc32(acc_row + c0, r);
                    const int col = n0 + c0;
                    bf16 *orow = nullptr;
                    int nstore = 0;                      // channels to store from this 32-column chunk (multiple of 8)
                    float scale = er.inv;
                    if (MODE == 0) {
                        if (rvalid && col < P.y_cstride) { orow = P.y + mo * P.y_cstride + col; nstore = min(32, P.y_cstride - col); }
                    } else {
                        scale = 1.f;
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            if (p >= P.nparts) break;
                            const TcPart &pt = P.parts[p];
                            const int local = col - pt.koff;
                            if (local >= 0 && local < pt.kext && pt.dx != nullptr && local < pt.c8 && rvalid) {
                                orow = pt.dx + mo * pt.dx_cstride + local;
                                nstore = min(32, pt.c8 - local);
                                scale = er.dscale[p];
                            }
                        }
                    }
                    const bool stats = (MODE == 0) && (s_stat != nullptr);
                    // warp-uniform: the block below shuffles (bias broadcast, statistics butterfly); lanes of rows past the end of the
                    // tensor have nothing to store but must take part
                    if (__any_sync(0xffffffffu, nstore > 0) || stats) {
                        uint4 o[4];
                        __nv_bfloat162 *ob = reinterpret_cast<__nv_bfloat162 *>(o);
                        // The per-element work is kept to a multiply-add, a select and the conversion: the epilogue of the K <= 512
                        // problems is ISSUE-bound (per-element bias loads and bounds tests would dominate it), so everything uniform
                        // over the chunk is decided here.  Lane l fetches the bias of column col + l
                        // once; elements get theirs by shuffle.  Columns past cout only exist in the last chunk of a layer.
                        float bl = 0.f;
                        const bool has_bias = (MODE == 0) && (P.bias != nullptr);
                        if (has_bias && col + lane < P.cout) bl = P.bias[col + lane];
                        const bool edge = (MODE == 0) && (col + 32 > P.cout);
                        // eval-mode BatchNorm + activation: scale / shift fetched like the bias (one load per lane, then shuffles)
                        const bool ep = (MODE == 0) && (P.ep_on != 0);
                        float el = 1.f, eh = 0.f;
                        if (ep && P.ep_scale != nullptr && col + lane < P.cout) { el = P.ep_scale[col + lane]; eh = P.ep_shift[col + lane]; }
    #pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            float a = __uint_as_float(r[2 * j]), b = __uint_as_float(r[2 * j + 1]);
                            if (MODE == 0) {
                                const float b0 = has_bias ? __shfl_sync(0xffffffffu, bl, 2 * j) : 0.f;
                                const float b1 = has_bias ? __shfl_sync(0xffffffffu, bl, 2 * j + 1) : 0.f;
                                a = hole ? 0.f : fmaf(a, scale, b0);
                                b = hole ? 0.f : fmaf(b, scale, b1);
                                if (ep) {                  // holes become apply_act(shift): the BatchNorm sees the zeros written above
                                    a = apply_act(fmaf(a, __shfl_sync(0xffffffffu, el, 2 * j), __shfl_sync(0xffffffffu, eh, 2 * j)), P.ep_act, P.ep_slope);
                                    b = apply_act(fmaf(b, __shfl_sync(0xffffffffu, el, 2 * j + 1), __shfl_sync(0xffffffffu, eh, 2 * j + 1)), P.ep_act, P.ep_slope);
                                }
                                if (edge) {
                                    if (col + 2 * j >= P.cout) a = 0.f;
                                    if (col + 2 * j + 1 >= P.cout) b = 0.f;
                                }
                            } else {
                                a *= scale; b *= scale;
                            }
                            ob[j] = __floats2bfloat162_rn(a, b);
                        }
                        if (nstore > 0) {
                            // a lane owns one output row: its 64 bytes of this chunk go out as four 16-byte stores
                            uint4 *dst = reinterpret_cast<uint4 *>(orow);
    #pragma unroll
                            for (int j = 0; j < 4; ++j)
                                if (j * 8 < nstore) dst[j] = o[j];
                        }
                        if (stats) {
                            // per-channel sum and sum of squares of what was just stored (rows past the tensor contribute 0)
                            float v[32], q[32];
                            const float live = rvalid ? 1.f : 0.f;          // rows past the end of the tensor (last M tile only)
    #pragma unroll
                            for (int j = 0; j < 16; ++j) {
                                const float2 f = __bfloat1622float2(ob[j]);
                                v[2 * j] = f.x * live; v[2 * j + 1] = f.y * live;
                                q[2 * j] = v[2 * j] * v[2 * j]; q[2 * j + 1] = v[2 * j + 1] * v[2 * j + 1];
                            }
                            const float cs = warp_transpose_sum(v, lane), cq = warp_transpose_sum(q, lane);
                            s_stat[c0 - cb + lane] += cs;                     // this warp's private accumulators: no atomics needed
                            s_stat[sq_off + c0 - cb + lane] += cq;
                        }
                    }
                }
}

// The two consumer warpgroups' share of the forward / dgrad epilogue.  Epilogue warp e (0..7) = warp e of the consumer
// warpgroups: warpgroup g = e / 4 owns rows [64 g, 64 g + 64), i.e. row quadrants 2 g and 2 g + 1, and each quadrant is drained
// by two warps that split the columns.
template <int BLOCK_N>
struct EpiRole {
    static constexpr int HN = (BLOCK_N >= 64) ? BLOCK_N / 2 : BLOCK_N;
    int q, half, cb, ce;
    __device__ __forceinline__ explicit EpiRole(int e) {
        q = 2 * (e >> 2) + (e & 1);
        half = (e & 3) >> 1;
        cb = half * HN;
        ce = (cb + HN <= BLOCK_N) ? cb + HN : cb;        // a 32-column tile is not split: the second warp only waits
    }
    __device__ __forceinline__ int slice() const { return half * 4 + q; }
};

// register accumulators of consumer warp e (fragment layout: see ptx::wgmma_bf16) -> its 16 rows of the staging tile
template <int BLOCK_N>
__device__ __forceinline__ void stage_acc(const float (&acc)[BLOCK_N / 2], float *stage, int e, int lane) {
    constexpr int PITCH = acc_pitch(BLOCK_N);
    const int r0 = 64 * (e >> 2) + 16 * (e & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c0;
        *reinterpret_cast<float2 *>(stage + row * PITCH + col) = make_float2(acc[i], acc[i + 1]);
    }
}

// register accumulators of warpgroup g -> staging tile -> tc_epilogue of this warp's 32 rows x column half.  Both named barriers
// span the warpgroup only: the other one keeps its own pace.
template <int BLOCK_N, int MODE>
__device__ __forceinline__ void mma_epilogue(const TcParams &P, const float (&acc)[BLOCK_N / 2], float *stage, int e, int lane, int m0, int n0,
                                             float *s_stat) {
    constexpr int PITCH = acc_pitch(BLOCK_N);
    const int g = e >> 2;
    stage_acc<BLOCK_N>(acc, stage, e, lane);
    ptx::named_sync(1 + g, 128);
    const EpiRole<BLOCK_N> R(e);
    const EpiRow er = tc_epi_row<MODE>(P, m0 + R.q * 32 + lane);
    tc_epilogue<BLOCK_N, MODE>(P, er, stage + (R.q * 32 + lane) * PITCH, lane, n0, s_stat, R.cb, R.ce, 128);
    ptx::named_sync(1 + g, 128);                          // the staging rows are free for the next tile
}

// -------------------------------------------------------------------------------------------------
// forward (MODE 0) / data gradient (MODE 1): PERSISTENT, warp-specialised implicit GEMM.
//
// One CTA per SM loops over output tiles (128 pixels x BLOCK_N channels).  Roles:
//   warps 0-3   A producers : im2col gather with zero-filling cp.async (padding AND holes), 32-bit offsets
//   warps 4-11  consumers   : two warpgroups, wgmma into register accumulators, then the epilogue of their 64 rows
//   warp  12    B producer  : weight tiles by TMA (SWIZZLE_128B)
// so the producers' per-tile latencies (mask-word loads, pipeline fill) of tile i+1 overlap the epilogue of tile i.
//
// A operand: per tap, a [128 pixel x 64 channel] tile in the 128B-swizzled K-major layout (any stride / dilation; also the
// row-packed small-Cin mode: K block = kernel row, chunk = tap column).
// -------------------------------------------------------------------------------------------------
constexpr int PERSIST_THREADS = 4 * 32 + MMA_THREADS + 32;
template <int BLOCK_N, int MODE>
__global__ void __launch_bounds__(PERSIST_THREADS, 1)
pconv_tc_persistent_kernel(const __grid_constant__ TcParams P, const __grid_constant__ CUtensorMap tmap_w) {
    constexpr int B_STAGE_BYTES = BLOCK_N * 128;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int SA = P.ring_a, SB = P.ring_b;
    const uint32_t sB = smem_base;
    const uint32_t sA = sB + SB * B_STAGE_BYTES;                      // stays 1024-aligned (B stages are multiples of 1024)
    const uint32_t sBar = (sA + SA * A_STAGE_BYTES + 15u) & ~15u;
    const uint32_t bar_full_a = sBar, bar_empty_a = sBar + 8 * MAX_RING;
    const uint32_t bar_full_b = sBar + 16 * MAX_RING, bar_empty_b = sBar + 24 * MAX_RING;
    const uint32_t s_stat_addr = sBar + 32 * MAX_RING;                                  // BatchNorm statistics slices
    const uint32_t s_acc = (s_stat_addr + STAT_SMEM_BYTES + 15u) & ~15u;               // epilogue staging tile
    float *acc_stage = reinterpret_cast<float *>(smem_raw + (s_acc - ptx::smem_u32(smem_raw)));

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int taps = P.kh * P.kw;
    const int np = (MODE == 0) ? P.nparts : 1;
    const int n_tiles = P.ncols / BLOCK_N;
    const int num_tiles = ((P.m_total + BLOCK_M - 1) / BLOCK_M) * n_tiles;

    // dgrad: N tiles none of whose parts wants a gradient are skipped (same decision in every role)
    auto tile_active = [&](int n0) -> bool {
        if (MODE == 0) return true;
        for (int p = 0; p < P.nparts; ++p)
            if (P.parts[p].dx && n0 < P.parts[p].koff + P.parts[p].kext && n0 + BLOCK_N > P.parts[p].koff) return true;
        return false;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) {      // empty barriers: one arrival per consumer warpgroup
            ptx::mbar_init(bar_full_a + 8 * s, NUM_PRODUCER_THREADS); ptx::mbar_init(bar_empty_a + 8 * s, 2);
            ptx::mbar_init(bar_full_b + 8 * s, 1); ptx::mbar_init(bar_empty_b + 8 * s, 2);
        }
        ptx::fence_mbar_init();
    }
    if (warp == 12 && lane == 0) ptx::prefetch_tmap(&tmap_w);
    __syncthreads();

    if (warp < 4) {
        // ================================ A producers ================================
        const int t = threadIdx.x;
        const int chunk = t & 7, r0 = t >> 3;
        const int plane = (MODE == 0) ? P.ho * P.wo : P.h * P.w;
        const int pwid = (MODE == 0) ? P.wo : P.w;
        int it = 0;
        bool dead = false;
        // Tap-validity words of the NEXT tile are loaded while the current tile's items stream (software pipelining across
        // tiles): their global-load latency would otherwise stall all gathers at the start of every tile.
        uint64_t wnext[TC_MAX_PARTS][8];
        auto issue_mask_loads = [&](int tl) {
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p)
#pragma unroll
                for (int i = 0; i < 8; ++i) wnext[p][i] = 0ull;
            if (MODE != 0 || tl >= num_tiles) return;
            const int tm0 = (tl / n_tiles) * BLOCK_M;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int idx = tm0 + r0 + 16 * i;
                if (idx >= P.m_total) continue;
#pragma unroll
                for (int p = 0; p < TC_MAX_PARTS; ++p)
                    if (p < P.nparts) wnext[p][i] = __ldg(P.parts[p].tapmask + idx);
            }
        };
        issue_mask_loads(blockIdx.x);
        for (int tile = blockIdx.x; tile < num_tiles && !dead; tile += gridDim.x) {
            const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
            uint64_t wcur[TC_MAX_PARTS][8];
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p)
#pragma unroll
                for (int i = 0; i < 8; ++i) wcur[p][i] = wnext[p][i];
            issue_mask_loads(tile + gridDim.x);
            if (!tile_active(n0)) continue;
            const uint32_t sw = static_cast<uint32_t>((chunk ^ (r0 & 7)) << 4);   // (r & 7) == (r0 & 7) for all rows of a thread
            int ph[8], pw[8];
            int ibase[TC_MAX_PARTS][8];                 // element offset of the row's image inside each source (+ chunk)
            bool prow[8];
            const int ls = 31 - __clz(P.stride);        // dgrad: stride is a power of two on this path (host-checked)
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int m = m0 + r0 + 16 * i;
                prow[i] = m < P.m_total;
                const int mm = prow[i] ? m : 0;
                const int nn = mm / plane, rem = mm - nn * plane;
                const int hh = rem / pwid, ww = rem - hh * pwid;
                if (MODE == 0) {
                    ph[i] = hh * P.stride - P.pad_h; pw[i] = ww * P.stride - P.pad_w;
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p)
                        ibase[p][i] = (p < P.nparts) ? nn * (P.h >> P.parts[p].xup) * (P.w >> P.parts[p].xup) * P.parts[p].cstride + chunk * 8 : 0;
                } else {
                    ph[i] = hh + P.pad_h; pw[i] = ww + P.pad_w;
                    ibase[0][i] = nn * P.ho * P.wo * P.dc_cstride + chunk * 8;
#pragma unroll
                    for (int p = 1; p < TC_MAX_PARTS; ++p) ibase[p][i] = 0;
                }
            }
            uint64_t tmv[TC_MAX_PARTS][8];              // per-row tap-validity bits (bounds + holes), prefetched one tile ahead
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p)
#pragma unroll
                for (int i = 0; i < 8; ++i) tmv[p][i] = wcur[p][i];

            auto push = [&](const bf16 *base, const int (&off)[8], const bool (&ok)[8]) -> bool {
                const int s = it % SA;
                if (!ptx::mbar_wait(bar_empty_a + 8 * s, ((it / SA) & 1) ^ 1, P.abort_flag, 101)) return false;
                const uint32_t dst = sA + s * A_STAGE_BYTES + r0 * 128 + sw;
#pragma unroll
                for (int i = 0; i < 8; ++i) ptx::cp_async_16(dst + i * (16 * 128), base + off[i], ok[i]);
                ptx::cp_async_mbar_arrive(bar_full_a + 8 * s);
                ptx::mbar_arrive(bar_full_a + 8 * s);
                ++it;
                return true;
            };
            if (MODE == 0 && P.rowpack) {
                // small-Cin mode: K block = kernel row `tr`; chunk = tap column; the source pixel shifts with the chunk
                const TcPart &pt = P.parts[0];
                const int cs = pt.cstride, rowpitch = P.w * cs;
                for (int tr = 0; tr < P.kh && !dead; ++tr) {
                    int off[8];
                    bool ok[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const bool v = (chunk < P.kw) && ((tmv[0][i] >> (tr * P.kw + chunk)) & 1ull);
                        off[i] = v ? (ibase[0][i] - chunk * 8) + (ph[i] + tr * P.dil) * rowpitch + (pw[i] + chunk * P.dil) * cs : 0;
                        ok[i] = v;
                    }
                    if (!push(pt.x, off, ok)) dead = true;
                }
            } else {
                for (int tap = 0; tap < taps && !dead; ++tap) {
                    const int tr = tap / P.kw, tc = tap - tr * P.kw;
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) {
                        if (p >= np || dead) break;
                        const TcPart &pt = P.parts[p];
                        const bf16 *src = (MODE == 0) ? pt.x : P.dc;
                        const int cs = (MODE == 0) ? pt.cstride : P.dc_cstride;
                        const int xup = (MODE == 0) ? pt.xup : 0;
                        const int rowpitch = ((MODE == 0) ? (P.w >> xup) : P.wo) * cs;
                        int base[8];
                        bool rv[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            bool v;
                            int hi, wi;
                            if (MODE == 0) {
                                v = (tmv[p][i] >> tap) & 1ull;                  // bounds + hole (0 for rows past m_total)
                                hi = (ph[i] + tr * P.dil) >> xup; wi = (pw[i] + tc * P.dil) >> xup;
                            } else {
                                const int th = ph[i] - tr * P.dil, tw = pw[i] - tc * P.dil;
                                hi = th >> ls; wi = tw >> ls;
                                v = prow[i] && th >= 0 && tw >= 0 && ((th | tw) & (P.stride - 1)) == 0 && hi < P.ho && wi < P.wo;
                            }
                            base[i] = v ? ibase[p][i] + hi * rowpitch + wi * cs : 0;
                            rv[i] = v;
                        }
                        const int nb = ((MODE == 0) ? pt.kext : P.dc_kext) / BLOCK_K;
                        const int c8 = (MODE == 0) ? pt.c8 : P.dc_c8;
                        for (int cb = 0; cb < nb; ++cb) {
                            const bool cv = cb * BLOCK_K + chunk * 8 < c8;       // channel padding of the part: zero-fill
                            int off[8];
                            bool ok[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i) { ok[i] = rv[i] && cv; off[i] = ok[i] ? base[i] + cb * BLOCK_K : 0; }
                            if (!push(src, off, ok)) { dead = true; break; }
                        }
                    }
                }
            }
        }
        ptx::cp_async_wait<0>();
    } else if (warp == 12) {
        // ================================ B producer: weight tiles by TMA ================================
        if (lane == 0) {
            int itb = 0;
            bool dead = false;
            auto load = [&](int kidx, int n0) -> bool {
                const int s = itb % SB;
                if (!ptx::mbar_wait(bar_empty_b + 8 * s, ((itb / SB) & 1) ^ 1, P.abort_flag, 103)) return false;
                ptx::mbar_arrive_expect_tx(bar_full_b + 8 * s, B_STAGE_BYTES);
                ptx::tma_load_2d(sB + s * B_STAGE_BYTES, &tmap_w, kidx, n0, bar_full_b + 8 * s);
                ++itb;
                return true;
            };
            for (int tile = blockIdx.x; tile < num_tiles && !dead; tile += gridDim.x) {
                const int n0 = (tile % n_tiles) * BLOCK_N;
                if (!tile_active(n0)) continue;
                const int num_kb = (MODE == 0) ? (P.rowpack ? P.kh : taps * (P.ktap / BLOCK_K)) : taps * (P.dc_kext / BLOCK_K);
                for (int kb = 0; kb < num_kb; ++kb)
                    if (!load(kb * BLOCK_K, n0)) { dead = true; break; }
            }
        }
    } else {
        // ================================ consumer warpgroups (warps 4-11) ================================
        const int e = warp - 4, g = e >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const int num_a = (MODE == 0) ? (P.rowpack ? P.kh : taps * (P.ktap / BLOCK_K)) : taps * (P.dc_kext / BLOCK_K);
        const uint32_t a_rows = 64u * 128u;             // this warpgroup's 64 rows of 128 bytes further into the A stage
        float *s_stat = (MODE == 0 && P.bn_sums != nullptr)
                            ? reinterpret_cast<float *>(smem_raw + (s_stat_addr - ptx::smem_u32(smem_raw))) : nullptr;
        const EpiRole<BLOCK_N> R(e);
        float *my_stat = s_stat ? s_stat + R.slice() * STAT_SLICE : nullptr;
        int stat_n0 = -1;
        if (my_stat) {
            for (int i = lane; i < STAT_SLICE; i += 32) my_stat[i] = 0.f;
            __syncwarp();
        }
        int ita = 0, itb = 0;
        bool dead = false;
        for (int tile = blockIdx.x; tile < num_tiles && !dead; tile += gridDim.x) {
            const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
            if (!tile_active(n0)) continue;
            if (my_stat && n0 != stat_n0) {
                if (stat_n0 >= 0) tc_stats_flush<BLOCK_N>(P, my_stat, lane, stat_n0, R.cb, R.ce, 128);
                stat_n0 = n0;
            }
            float acc[BLOCK_N / 2];
            zero_acc(acc);
            for (int a = 0; a < num_a && !dead; ++a, ++ita) {
                const int sa = ita % SA;
                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full_a + 8 * sa, (ita / SA) & 1, P.abort_flag, 104))) { dead = true; break; }
                ptx::fence_proxy_async_smem();                   // cp.async (generic proxy) data -> wgmma (async proxy)
                const int sb = itb % SB;
                if (__all_sync(0xffffffffu, ptx::mbar_wait(bar_full_b + 8 * sb, (itb / SB) & 1, P.abort_flag, 105))) {
                    const uint64_t db = ptx::make_smem_desc(sB + sb * B_STAGE_BYTES, 16, 1024);
                    ptx::wgmma_fence();
                    const uint64_t da = ptx::make_smem_desc(sA + sa * A_STAGE_BYTES + g * a_rows, 16, 1024);
#pragma unroll
                    for (int k = 0; k < BLOCK_K / 16; ++k)                                  // +32 bytes per K=16 step inside the swizzle row
                        ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + 2 * k, db + 2 * k);
                    ptx::wgmma_commit();
                    ++itb;
                } else {
                    dead = true;
                }
                // the A item and its weight tile are released once this warpgroup's MMAs on them completed
                ptx::wgmma_wait<0>();
                ptx::wgmma_fence_regs(acc);
                if (leader) {
                    ptx::mbar_arrive(bar_empty_b + 8 * sb);
                    ptx::mbar_arrive(bar_empty_a + 8 * sa);
                }
            }
            if (dead) { stat_n0 = -1; break; }
            mma_epilogue<BLOCK_N, MODE>(P, acc, acc_stage, e, lane, m0, n0, my_stat);
        }
        if (my_stat && stat_n0 >= 0) tc_stats_flush<BLOCK_N>(P, my_stat, lane, stat_n0, R.cb, R.ce, 128);
    }
}


// -------------------------------------------------------------------------------------------------
// forward (MODE 0) / stride-1 data gradient (MODE 1), TMA-FED: the im2col rows are not gathered by threads at all.
//
// An M tile of 128 consecutive output pixels is a box {box_w, box_h, box_n} of the (x, y, image) grid (all extents powers
// of two here), so the A operand of tap (tr, tc) / channel block cb is ONE 4-D TMA tile {64 ch, box_w, box_h, box_n} of
// the NHWC source at coordinates shifted by the tap -- negative / past-the-edge coordinates are zero-filled by the TMA
// unit (the convolution padding), stride-2 layers use the tensor map's traversal stride, channel padding is the map's
// channel extent.  TMA writes exactly the 128B-swizzled K-major image wgmma reads.  What TMA cannot know are the HOLES
// (x*mask, models/partial_convolution.py:51): three "fixer" warps (each thread loops over tile rows) test the rows'
// tap-validity bits and overwrite hole rows of the landed tile with zeros before handing the stage to the MMA thread
// (generic-proxy stores -> fence.proxy.async -> mbarrier).  Plain convolutions / dgrad skip the fixers.
//
//   warpgroups 0-1 consumers  : 4 x wgmma (K=16) per K block and weight tile, then the element math of their 64 rows -> staging
//   warpgroup 2    warp 8      TMA producer : per K block one A tile (4-D) + the weight tiles (2-D) onto the same mbarrier
//                  warps 9-11  fixers       : hole rows -> 0   (MODE 0 with masks only)
//   warpgroup 3    epilogue   : staging tile -> dgrad input mask -> bf16 NHWC stores (+ BatchNorm statistics)
// The roles are whole warpgroups so that setmaxnreg can move registers to the consumers: a 128 x 256 tile is 64 x 256 fp32
// accumulators = 128 registers per consumer thread (2 x 128 x TMA_CONSUMER_REGS + 2 x 128 x TMA_SUPPORT_REGS = 65,536).
// Every per-K-block loop of the producer is a handful of instructions: index arithmetic there (the old kernels did integer
// divisions) directly delays the stages the tensor cores wait for.
// The epilogue of tile i overlaps the MMAs of tile i+1 through ONE staging tile and two mbarriers: the consumers wait on
// acc_empty before they write it and arrive on acc_full after; the epilogue warps wait on acc_full and arrive on acc_empty once
// they have read it.  The consumers fetch their rows' mask sums, the epilogue warps the dgrad mask bytes, before the K loop /
// the wait.
// -------------------------------------------------------------------------------------------------
// HALO = true (stride 1, tiles that are one image-row segment of 128 pixels): per kernel ROW one A tile of
// 128 + (kw-1)*dil pixel rows is loaded, and the kw taps of that row are kw wgmma descriptors whose start address is
// shifted by whole 128-byte rows (the 128B swizzle is a function of the absolute smem address, so a row-shifted start
// reads the same image) -- kw x less A traffic from L2 and kw x fewer barrier round trips per MMA.  K steps that only cover
// channel padding (c8 <= 16*k) are skipped.
template <int BLOCK_N, int MODE, bool HALO>
__global__ void __maxnreg__(TMA_REGS)
pconv_tc_tma_kernel(const __grid_constant__ TcParams P, const __grid_constant__ CUtensorMap tmap_w,
                    const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1) {
    constexpr uint32_t B_BYTES = BLOCK_N * 128;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int S = P.stages;
    const int nB = HALO ? P.kw : 1;                                    // weight tiles (taps) per stage
    const int hx = HALO ? (P.kw - 1) * P.dil : 0;                      // extra pixel rows of a halo tile
    const uint32_t A_BYTES = static_cast<uint32_t>(BLOCK_M + hx) * 128u;
    const uint32_t A_ROOM = (A_BYTES + 1023u) & ~1023u;
    const uint32_t STAGE = A_ROOM + nB * B_BYTES;                      // multiple of 1024
    const uint32_t STAGE_TX = A_BYTES + nB * B_BYTES;
    const uint32_t sBar = smem_base + S * STAGE;
    const uint32_t bar_full = sBar, bar_fixed = sBar + 8 * MAX_RING, bar_empty = sBar + 16 * MAX_RING;
    const uint32_t acc_full = sBar + 24 * MAX_RING, acc_empty = acc_full + 8;
    const uint32_t s_stat_addr = sBar + TMA_BAR_BYTES;
    const uint32_t s_acc = s_stat_addr + EPI_STAT_SMEM_BYTES;
    uint8_t *smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform by construction
    const int np = (MODE == 0) ? P.nparts : 1;
    const int n_tiles = P.ncols / BLOCK_N;
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * n_tiles;                           // tile index = m tile * n_tiles + n tile
    const int tile0 = static_cast<int>(blockIdx.x), tstep = static_cast<int>(gridDim.x);
    auto m0_of = [&](int mt) -> int { return mt * BLOCK_M; };
    const bool fix = (MODE == 0) && P.use_fix;
    const int kwi = HALO ? 1 : P.kw;                                   // A items per kernel row

    auto tile_active = [&](int n0) -> bool {
        if (MODE == 0) return true;
        for (int p = 0; p < P.nparts; ++p)
            if (P.parts[p].dx && n0 < P.parts[p].koff + P.parts[p].kext && n0 + BLOCK_N > P.parts[p].koff) return true;
        return false;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) {      // empty: one arrival per consumer warpgroup
            ptx::mbar_init(bar_full + 8 * s, 1); ptx::mbar_init(bar_fixed + 8 * s, TMA_FIX_THREADS / 32); ptx::mbar_init(bar_empty + 8 * s, 2);
        }
        ptx::mbar_init(acc_full, MMA_WARPS); ptx::mbar_init(acc_empty, EPI_WARPS);     // one arrival per warp
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_w); ptx::prefetch_tmap(&tmap_a0); if (np > 1) ptx::prefetch_tmap(&tmap_a1); }
    __syncthreads();

    // The producer runs WARP-CONVERGED (all 32 lanes walk the loops and wait on the barriers; the warp index is a shuffle
    // broadcast so the compiler knows the role branch is uniform) and only the TMA instructions sit inside an elect.sync region.
    float *s_stat = nullptr;                                          // epilogue warps: private BatchNorm-statistics accumulators
    int stat_n0 = -1;                                                  // N tile they currently belong to (-1: none / aborted)
    bf16 *acc_stage = reinterpret_cast<bf16 *>(smem_gen + (s_acc - smem_base));
    if (warp < MMA_WARPS) {
        ptx::setmaxnreg_inc<TMA_CONSUMER_REGS>();
        // ================================ consumer warpgroups ================================
        const int e = warp, g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t ready = fix ? bar_fixed : bar_full;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + g * 64 * 128, 16, 1024);     // this warpgroup's 64 rows
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_ROOM, 16, 1024);
        const uint32_t stage16 = STAGE >> 4;
        // dgrad walks tap columns right to left inside a halo tile
        const int shift0 = (HALO && MODE == 1) ? hx * 8 : 0;           // in 16-byte units: one pixel row = 128 B = 8 units
        const int dshift = HALO ? ((MODE == 1) ? -P.dil * 8 : P.dil * 8) : 0;
        const int rows_a = P.kh * kwi;                                 // (kernel row, A item) pairs per tile
        // per part: K blocks, and the K steps of the last block that hold real channels (channel padding is skipped)
        int nb0, nb1 = 0, kl0, kl1 = 4;
        {
            const int kext = (MODE == 0) ? P.parts[0].kext : P.dc_kext, c8 = (MODE == 0) ? P.parts[0].c8 : P.dc_c8;
            nb0 = kext / BLOCK_K; kl0 = min(4, (c8 - (nb0 - 1) * BLOCK_K + 15) >> 4);
            if (MODE == 0 && np > 1) { nb1 = P.parts[1].kext / BLOCK_K; kl1 = min(4, (P.parts[1].c8 - (nb1 - 1) * BLOCK_K + 15) >> 4); }
        }
        int s = 0;
        uint32_t ph = 0, aph = 1;                                      // aph: first pass, the staging tile is free
        bool dead = false;
        for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
            const int n0 = (tile % n_tiles) * BLOCK_N;
            if (!tile_active(n0)) continue;
            const ConsRows cr = cons_rows<MODE>(P, m0_of(tile / n_tiles), e, lane);
            float acc[BLOCK_N / 2];
            zero_acc(acc);
            int held = -1;                                             // stage whose MMAs may still be reading it
            for (int r = 0; r < rows_a && !dead; ++r) {
#pragma unroll
                for (int p = 0; p < TC_MAX_PARTS; ++p) {
                    const int nbp = (p == 0) ? nb0 : nb1, klast = (p == 0) ? kl0 : kl1;
                    for (int cb = 0; cb < nbp; ++cb) {
                        if (!__all_sync(0xffffffffu, ptx::mbar_wait(ready + 8 * s, ph, P.abort_flag, 124))) { dead = true; break; }
                        uint64_t da = desc_a0 + static_cast<uint64_t>(s * stage16 + shift0), db = desc_b0 + static_cast<uint64_t>(s * stage16);
                        const int ksteps = (cb + 1 < nbp) ? 4 : klast;
                        ptx::wgmma_fence();
                        for (int tc = 0; tc < nB; ++tc, da += dshift, db += B_BYTES >> 4) {
                            if (ksteps == 4) {
#pragma unroll
                                for (int k = 0; k < 4; ++k) ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + 2 * k, db + 2 * k);
                            } else {
                                for (int k = 0; k < ksteps; ++k) ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + 2 * k, db + 2 * k);
                            }
                        }
                        ptx::wgmma_commit();
                        // keep one K block in flight: the previous stage is released once its MMAs completed
                        ptx::wgmma_wait<1>();
                        if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
                        held = s;
                        if (++s == S) { s = 0; ph ^= 1; }
                    }
                    if (dead) break;
                }
            }
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(acc);
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            if (dead) break;
            if (!tma_stage_tile<BLOCK_N, MODE>(P, acc, acc_stage, acc_full, acc_empty, aph, e, lane, n0, cr, 125)) break;
        }
    } else {
        ptx::setmaxnreg_dec<TMA_SUPPORT_REGS>();       // warpgroups 2 and 3, fixers included when there are no holes
        if (warp >= EPI_WARP0) {
            // ================================ epilogue warps ================================
            const int w = warp - EPI_WARP0;
            s_stat = (MODE == 0 && P.bn_sums != nullptr)
                         ? reinterpret_cast<float *>(smem_gen + (s_stat_addr - smem_base)) + w * EPI_STAT_SLICE : nullptr;
            auto origin = [&](int tile, int &m0, int &n0) {
                m0 = m0_of(tile / n_tiles); n0 = (tile % n_tiles) * BLOCK_N;
                if (!tile_active(n0)) n0 = -1;
            };
            tma_epilogue_warps<BLOCK_N, MODE>(P, tile0, tstep, num_tiles, origin, acc_stage, acc_full, acc_empty, s_stat, stat_n0, w, lane, 126);
            // last N tile's statistics: all four slices are complete once the epilogue warpgroup passed this barrier (no CTA-wide
            // barrier: the warpgroups run under different register limits, setmaxnreg regions must not meet again)
            ptx::named_sync(1, EPI_WARPS * 32);
            if (s_stat != nullptr && stat_n0 >= 0) tc_stats_final<BLOCK_N>(P, s_stat - w * EPI_STAT_SLICE, w, lane, stat_n0);
        } else if (warp == 8) {
            // ================================ TMA producer ================================
            int s = 0;
            uint32_t ph = 1;                                               // first pass over the ring: stages are free
            const int plane = (MODE == 0) ? P.ho * P.wo : P.h * P.w;
            const int pwid = (MODE == 0) ? P.wo : P.w;
            const int kext0 = (MODE == 0) ? P.parts[0].kext : P.dc_kext, kext1 = (MODE == 0 && np > 1) ? P.parts[1].kext : 0;
            const int dstep = (MODE == 0) ? P.dil : -P.dil;
            const int row_k = P.wk_row, col_k = P.wk_col;
            bool dead = false;
            for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                const int m0 = m0_of(tile / n_tiles), n0 = (tile % n_tiles) * BLOCK_N;
                if (!tile_active(n0)) continue;
                const int img = m0 / plane, rem = m0 - img * plane;
                const int oy = rem / pwid, ox = rem - oy * pwid;
                // leftmost / topmost source coordinate of tap column 0 (fwd) -- dgrad walks its taps right to left
                const int x_org = (MODE == 0) ? ox * P.stride - P.pad_w : (HALO ? ox + P.pad_w - hx : ox + P.pad_w);
                const int y_org = (MODE == 0) ? oy * P.stride - P.pad_h : oy + P.pad_h;
                int krow = P.wk_base;                                      // weight K index of (tr, tap column 0, part 0, block 0)
                for (int tr = 0, y = y_org; tr < P.kh && !dead; ++tr, y += dstep, krow += row_k)
                    for (int ti = 0, x = x_org, kidx = krow; ti < kwi && !dead; ++ti, x += dstep, kidx = krow + ti * col_k) {
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            const int kext = (p == 0) ? kext0 : kext1;
                            const CUtensorMap *ma = (p == 0) ? &tmap_a0 : &tmap_a1;
                            for (int c0 = 0; c0 < kext; c0 += BLOCK_K, kidx += BLOCK_K) {
                                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 121))) { dead = true; break; }
                                if (ptx::elect_one()) {
                                    const uint32_t full = bar_full + 8 * s, dst = smem_base + s * STAGE;
                                    ptx::mbar_arrive_expect_tx(full, STAGE_TX);
                                    ptx::tma_load_4d(dst, ma, c0, x, y, img, full);
                                    uint32_t bdst = dst + A_ROOM;
                                    for (int tc = 0, kb = kidx; tc < nB; ++tc, kb += col_k, bdst += B_BYTES)
                                        ptx::tma_load_2d(bdst, &tmap_w, kb, n0, full);
                                }
                                __syncwarp();
                                if (++s == S) { s = 0; ph ^= 1; }
                            }
                            if (dead) break;
                        }
                    }
            }
        } else {
            // ================================ fixers: zero the hole rows of every landed A tile ================================
            // thread t owns tile rows t, t + 96 (and t + 192: halo rows up to 256)
            if (fix) {
                constexpr int FR = HALO ? 3 : 2;
                const int t = (warp - 9) * 32 + lane;
                int s = 0;
                uint32_t ph = 0;
                bool dead = false;
                auto zero_row = [&](int row) {
                    uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + row * 128);
                    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                    for (int k = 0; k < 8; ++k) r[k] = z;
                };
                if (!HALO) {
                    // validity = the row's tap bit (bounds + hole)
                    uint64_t wnext[FR][TC_MAX_PARTS];
                    auto load_words = [&](int tl) {
#pragma unroll
                        for (int r = 0; r < FR; ++r)
#pragma unroll
                            for (int p = 0; p < TC_MAX_PARTS; ++p) {
                                wnext[r][p] = 0ull;
                                const int m = m0_of(tl / n_tiles) + t + TMA_FIX_THREADS * r;
                                if (p < P.nparts && tl < num_tiles && t + TMA_FIX_THREADS * r < BLOCK_M && m < P.m_total)
                                    wnext[r][p] = __ldg(P.parts[p].tapmask + m);
                            }
                    };
                    load_words(tile0);
                    for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                        uint64_t wcur[FR][TC_MAX_PARTS];
#pragma unroll
                        for (int r = 0; r < FR; ++r)
#pragma unroll
                            for (int p = 0; p < TC_MAX_PARTS; ++p) wcur[r][p] = wnext[r][p];
                        load_words(tile + tstep);                      // next tile's words travel while this tile streams
                        if (MODE == 1 && !tile_active((tile % n_tiles) * BLOCK_N)) continue;
                        const int taps = P.kh * P.kw;
                        for (int tap = 0; tap < taps && !dead; ++tap) {
#pragma unroll
                            for (int p = 0; p < TC_MAX_PARTS; ++p) {
                                if (p >= np) break;
                                bool hole[FR], mine = false;
#pragma unroll
                                for (int r = 0; r < FR; ++r) {      // rows past the tile (t + 96 >= 128) are not rows
                                    hole[r] = t + TMA_FIX_THREADS * r < BLOCK_M && ((wcur[r][p] >> tap) & 1ull) == 0ull;
                                    mine = mine || hole[r];
                                }
                                const bool any_hole = __any_sync(0xffffffffu, mine);
                                const int nb = ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
                                for (int cb = 0; cb < nb; ++cb) {
                                    if (!ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 122)) { dead = true; break; }
                                    if (any_hole) {
#pragma unroll
                                        for (int r = 0; r < FR; ++r)
                                            if (hole[r]) zero_row(t + TMA_FIX_THREADS * r);
                                        ptx::fence_proxy_async_smem();
                                    }
                                    __syncwarp();
                                    if (lane == 0) ptx::mbar_arrive(bar_fixed + 8 * s);
                                    if (++s == S) { s = 0; ph ^= 1; }
                                }
                                if (dead) break;
                            }
                        }
                    }
                } else {
                    // validity = the source mask at the halo pixel row (rows < 128 + hx)
                    const int plane = P.ho * P.wo;
                    auto load_bits = [&](int tl, uint32_t (&b)[FR]) {       // bit (p*8 + tr) of b[r]: pixel row t + 96 r is a hole
#pragma unroll
                        for (int r = 0; r < FR; ++r) b[r] = 0;
                        if (tl >= num_tiles) return;
                        const int m0 = m0_of(tl / n_tiles);
                        const int img = m0 / plane, rem = m0 - img * plane;
                        const int oy = rem / P.wo, ox = rem - oy * P.wo;
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            if (p >= P.nparts || P.parts[p].mask == nullptr) continue;
                            const int mup = P.parts[p].mup;
                            const uint8_t *mk = P.parts[p].mask + static_cast<long long>(img) * (P.h >> mup) * (P.w >> mup);
                            for (int tr = 0; tr < P.kh; ++tr) {
                                const int y = oy - P.pad_h + tr * P.dil;
                                if (y < 0 || y >= P.h) continue;            // rows outside the image were zero-filled by TMA
#pragma unroll
                                for (int r = 0; r < FR; ++r) {
                                    const int row = t + TMA_FIX_THREADS * r, x = ox - P.pad_w + row;
                                    if (row < BLOCK_M + hx && x >= 0 && x < P.w && __ldg(mk + (y >> mup) * (P.w >> mup) + (x >> mup)) == 0)
                                        b[r] |= 1u << (p * 8 + tr);
                                }
                            }
                        }
                    };
                    uint32_t nb_bits[FR];
                    load_bits(tile0, nb_bits);
                    for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                        uint32_t cb_bits[FR];
#pragma unroll
                        for (int r = 0; r < FR; ++r) cb_bits[r] = nb_bits[r];
                        load_bits(tile + tstep, nb_bits);
                        if (MODE == 1 && !tile_active((tile % n_tiles) * BLOCK_N)) continue;
                        for (int tr = 0; tr < P.kh && !dead; ++tr) {
#pragma unroll
                            for (int p = 0; p < TC_MAX_PARTS; ++p) {
                                if (p >= np) break;
                                bool hole[FR], mine = false;
#pragma unroll
                                for (int r = 0; r < FR; ++r) { hole[r] = (cb_bits[r] >> (p * 8 + tr)) & 1u; mine = mine || hole[r]; }
                                const bool any_hole = __any_sync(0xffffffffu, mine);
                                const int nb = ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
                                for (int cb = 0; cb < nb; ++cb) {
                                    if (!ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 122)) { dead = true; break; }
                                    if (any_hole) {
#pragma unroll
                                        for (int r = 0; r < FR; ++r)
                                            if (hole[r]) zero_row(t + TMA_FIX_THREADS * r);
                                        ptx::fence_proxy_async_smem();
                                    }
                                    __syncwarp();
                                    if (lane == 0) ptx::mbar_arrive(bar_fixed + 8 * s);
                                    if (++s == S) { s = 0; ph ^= 1; }
                                }
                                if (dead) break;
                            }
                        }
                    }
                }
            }
        }
    }

}


// -------------------------------------------------------------------------------------------------
// SUB-PIXEL data gradient: for convolutions whose input is cat([nearest-2x-upsample(x0), x1]) (models/image_inpainting.py:183-185)
// the gradient w.r.t. x0 is computed directly at SOURCE resolution -- neither the full-resolution gradient of the upsampled
// part nor the 2x2 reduction pass over it exists.
//
// Output pixel (2k+py, 2j+px) of a k x k convolution over up2x(x0) reads source pixel (k + floor((py + tr*d - p)/2), ...): within
// one parity class (py, px) the convolution over the upsampled part IS a convolution over the SOURCE with a smaller kernel whose
// taps are sums of the original taps (3x3, pad 1: 2x2 effective taps).  So dx0 = sum over the classes and their effective taps
// of dc read with a traversal stride of 2 times the transposed effective weights -- 16/36 of the multiplications of
// "full-resolution gradient + 2x2 sum".  The M tiles are boxes of the source grid [n][h/2][w/2]; what each K step loads is
// listed in a small table built on the host:
//     item = { (dx, dy) added to twice the tile origin (dc coordinates), weight K index }
// Roles / pipeline / epilogue as in pconv_tc_tma_kernel; dc has no holes, so the fixer warps stay idle.
// -------------------------------------------------------------------------------------------------
constexpr int SP_MAX_ITEMS = 40;
struct SpItem { int dx, dy, wk; };
struct SpTable {
    int n_items;
    SpItem it[SP_MAX_ITEMS];
};

template <int BLOCK_N>
__global__ void __maxnreg__(TMA_REGS)
pconv_tc_sp_kernel(const __grid_constant__ TcParams P, const __grid_constant__ SpTable TB, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ CUtensorMap tmap_a) {
    constexpr uint32_t B_BYTES = BLOCK_N * 128;
    constexpr uint32_t STAGE = A_STAGE_BYTES + B_BYTES;               // multiple of 1024
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int S = P.stages;
    // shared-memory layout of pconv_tc_tma_kernel (tma_fixed_smem), the fixed-barrier and statistics slots unused
    const uint32_t sBar = smem_base + S * STAGE;
    const uint32_t bar_full = sBar, bar_empty = sBar + 16 * MAX_RING;
    const uint32_t acc_full = sBar + 24 * MAX_RING, acc_empty = acc_full + 8;
    const uint32_t s_acc = sBar + TMA_BAR_BYTES + EPI_STAT_SMEM_BYTES;
    bf16 *acc_stage = reinterpret_cast<bf16 *>(smem_raw + (s_acc - ptx::smem_u32(smem_raw)));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int n_tiles = P.ncols / BLOCK_N;
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * n_tiles;
    const int tile0 = static_cast<int>(blockIdx.x), tstep = static_cast<int>(gridDim.x);
    // the tile grid is the source grid [n][P.h][P.w]
    const int plane = P.w * P.h;
    // 64-channel K blocks of dc and the K steps of the last block that hold real channels
    const int nbk = P.dc_kext / BLOCK_K;
    const int klast = min(4, (P.dc_c8 - (nbk - 1) * BLOCK_K + 15) >> 4);

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) { ptx::mbar_init(bar_full + 8 * s, 1); ptx::mbar_init(bar_empty + 8 * s, 2); }
        ptx::mbar_init(acc_full, MMA_WARPS); ptx::mbar_init(acc_empty, EPI_WARPS);     // one arrival per warp
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_w); ptx::prefetch_tmap(&tmap_a); }
    __syncthreads();

    if (warp < MMA_WARPS) {
        ptx::setmaxnreg_inc<TMA_CONSUMER_REGS>();
        // ================================ consumer warpgroups ================================
        const int e = warp, g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + g * 64 * 128, 16, 1024);     // this warpgroup's 64 rows
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_STAGE_BYTES, 16, 1024);
        const uint32_t stage16 = STAGE >> 4;
        int s = 0;
        uint32_t ph = 0, aph = 1;                                      // aph: first pass, the staging tile is free
        bool dead = false;
        for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
            float acc[BLOCK_N / 2];
            zero_acc(acc);
            int held = -1;
            for (int i = 0; i < TB.n_items && !dead; ++i) {
                for (int cb = 0; cb < nbk; ++cb) {
                    if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 324))) { dead = true; break; }
                    const uint64_t da = desc_a0 + static_cast<uint64_t>(s * stage16), db = desc_b0 + static_cast<uint64_t>(s * stage16);
                    const int ksteps = (cb + 1 < nbk) ? 4 : klast;
                    ptx::wgmma_fence();
                    for (int k = 0; k < ksteps; ++k) ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + 2 * k, db + 2 * k);
                    ptx::wgmma_commit();
                    ptx::wgmma_wait<1>();
                    if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
                    held = s;
                    if (++s == S) { s = 0; ph ^= 1; }
                }
            }
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_regs(acc);
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            if (dead) break;
            if (!tma_stage_tile<BLOCK_N, 1>(P, acc, acc_stage, acc_full, acc_empty, aph, e, lane, (tile % n_tiles) * BLOCK_N, ConsRows{}, 325)) break;
        }
    } else {
        ptx::setmaxnreg_dec<TMA_SUPPORT_REGS>();       // warpgroups 2 and 3, the idle fixer warps included
        if (warp >= EPI_WARP0) {
            // ================================ epilogue warps ================================
            int stat_n0 = -1;
            auto origin = [&](int tile, int &m0, int &n0) { m0 = (tile / n_tiles) * BLOCK_M; n0 = (tile % n_tiles) * BLOCK_N; };
            tma_epilogue_warps<BLOCK_N, 1>(P, tile0, tstep, num_tiles, origin, acc_stage, acc_full, acc_empty, nullptr, stat_n0,
                                           warp - EPI_WARP0, lane, 326);
        } else if (warp == 8) {
            // ================================ TMA producer ================================
            int s = 0;
            uint32_t ph = 1;
            bool dead = false;
            for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
                const int img = m0 / plane, rem = m0 - img * plane;
                const int oy = rem / P.w, ox = rem - oy * P.w;
                for (int i = 0; i < TB.n_items && !dead; ++i) {
                    const SpItem it = TB.it[i];
                    const int x = 2 * ox + it.dx, y = 2 * oy + it.dy;
                    for (int cb = 0; cb < nbk; ++cb) {
                        if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 321))) { dead = true; break; }
                        if (ptx::elect_one()) {
                            const uint32_t full = bar_full + 8 * s, dst = smem_base + s * STAGE;
                            ptx::mbar_arrive_expect_tx(full, STAGE);
                            ptx::tma_load_4d(dst, &tmap_a, cb * BLOCK_K, x, y, img, full);
                            ptx::tma_load_2d(dst + A_STAGE_BYTES, &tmap_w, it.wk + cb * BLOCK_K, n0, full);
                        }
                        __syncwarp();
                        if (++s == S) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
    }
}

// nearest 2x upsample of one convolution source into a dense [n, 2hs, 2ws, c8] buffer (TMA cannot replicate pixels)
__global__ void upsample_part_kernel(const bf16 *__restrict__ src, int cstride, int c8, long long pixels_src, int hs, int ws, bf16 *__restrict__ dst) {
    const int chunks = c8 >> 3;
    const long long total = pixels_src * chunks;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % chunks);
        const long long pix = i / chunks;
        const int x = static_cast<int>(pix % ws);
        const long long t = pix / ws;
        const int y = static_cast<int>(t % hs);
        const long long n = t / hs;
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(src + pix * cstride + ch * 8));
        bf16 *d = dst + ((n * (2 * hs) + 2 * y) * (2ll * ws) + 2 * x) * c8 + ch * 8;
        uint4 *d0 = reinterpret_cast<uint4 *>(d), *d1 = reinterpret_cast<uint4 *>(d + 2ll * ws * c8);
        d0[0] = v; *reinterpret_cast<uint4 *>(d + c8) = v;
        d1[0] = v; *reinterpret_cast<uint4 *>(d + 2ll * ws * c8 + c8) = v;
    }
}

// -------------------------------------------------------------------------------------------------
// weight gradient
// -------------------------------------------------------------------------------------------------
struct WgParams {
    int n, h, w, cin, cout, kh, kw, stride, pad_h, pad_w, dil, ho, wo;
    int m_total;              // n*ho*wo : the reduction (K) extent
    int nparts, rowpack;
    int ktap;                 // gathered-operand extent per tap group (sum of part kext; rowpack: 64)
    int ntaps;                // tap groups walked: kh*kw, or kh in rowpack mode
    TcPart parts[TC_MAX_PARTS];
    int tap_groups;
    int ci_tiles;             // ceil(ktap / 128)
    int kb_per_split;
    float *dw;                // [cout][kh*kw][cin] fp32, pre-zeroed
    int *abort_flag;
    // TMA-fed kernel: a K block of 64 consecutive output pixels is the box {box_w, box_h, box_n}; use_fix: some part has holes
    int box_w, box_h, box_n, stages, use_fix;
};

// Both weight-gradient kernels: warps 0-7 are two consumer warpgroups; warpgroup g computes rows [64 g, 64 g + 64) of
// D[k][co] (k = the tile's 128 gathered channels) for every tap of the CTA and adds them into dw from its registers.
constexpr int WGRAD_THREADS = MMA_THREADS + 5 * 32;

// red.global.add of a consumer thread's accumulators: element i of tap tl is row r0 + 8 ((i / 2) & 1), column 8 (i / 4) +
// 2 (lane % 4) + (i & 1) of the tile.  ci[h] / tap[h][tl]: input channel (-1: none) and kernel tap of the thread's two rows.
// Only the first `ncols` (64 or BLOCK_N) columns were computed.
template <int BLOCK_N, int T>
__device__ __forceinline__ void wgrad_store(const WgParams &P, const float (&acc)[T][BLOCK_N / 2], int ntap, int lane, int n0,
                                            int ncols, const int (&ci)[2], const int (&tap)[2][T]) {
    const int taps_full = P.kh * P.kw;
#pragma unroll
    for (int tl = 0; tl < T; ++tl) {
        if (tl >= ntap) break;
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) {
            if (2 * i >= ncols) break;
            const int h = (i >> 1) & 1;
            const int co = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
            if (ci[h] >= 0 && co < P.cout)
                atomicAdd(P.dw + (static_cast<long long>(co) * taps_full + tap[h][tl]) * P.cin + ci[h], acc[tl][i]);
        }
    }
}

template <int BLOCK_N, int T, int STAGES>
__global__ void __launch_bounds__(WGRAD_THREADS, 1)
pconv_tc_wgrad_kernel(const __grid_constant__ WgParams P, const __grid_constant__ CUtensorMap tmap_dc) {
    constexpr int B_STAGE_BYTES = BLOCK_N * 128;            // [64 px][BLOCK_N co] as BLOCK_N/64 blocks of 8 KB
    constexpr int A_TAP_BYTES = 16384;                      // [64 px][128 k] as 2 blocks of 8 KB
    constexpr int A_STAGE = T * A_TAP_BYTES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const uint32_t sA = smem_base;
    const uint32_t sB = sA + STAGES * A_STAGE;
    const uint32_t sBar = sB + STAGES * B_STAGE_BYTES;
    const uint32_t bar_full_a = sBar, bar_full_b = sBar + 8 * STAGES, bar_empty = sBar + 16 * STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // blockIdx.x = ((co_tile * tap_groups) + tap_group) * ci_tiles + ci_tile ; blockIdx.y = K split
    int bx = blockIdx.x;
    const int ci_tile = bx % P.ci_tiles; bx /= P.ci_tiles;
    const int tap_group = bx % P.tap_groups;
    const int co_tile = bx / P.tap_groups;
    const int taps_full = P.kh * P.kw;
    const int tap0 = tap_group * T;
    const int ntap = min(T, P.ntaps - tap0);
    const int n0 = co_tile * BLOCK_N;
    const int total_kb = (P.m_total + 63) / 64;
    const int kb_begin = blockIdx.y * P.kb_per_split;
    const int kb_end = min(total_kb, kb_begin + P.kb_per_split);
    const int num_kb = max(0, kb_end - kb_begin);

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            ptx::mbar_init(bar_full_a + 8 * s, NUM_PRODUCER_THREADS);
            ptx::mbar_init(bar_full_b + 8 * s, 1);
            ptx::mbar_init(bar_empty + 8 * s, 2);
        }
        ptx::fence_mbar_init();
    }
    if (warp == 12 && lane == 0) ptx::prefetch_tmap(&tmap_dc);
    __syncthreads();

    if (warp >= MMA_WARPS && warp < MMA_WARPS + 4) {
        // ============ A producers (warps 8-11): gather x rows (K = pixels) for each tap, 2 x 64-element blocks ============
        const int t = threadIdx.x - MMA_THREADS;
        const int chunk = t & 7, r0 = t >> 3;
        const uint32_t sw = static_cast<uint32_t>((chunk ^ (r0 & 7)) << 4);
        // the two 64-element blocks of this k tile -> (part, channel offset inside the part, chunk readable?)
        int blk_part[2], blk_off[2];
        bool blk_cv[2];
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
            const int kpos = ci_tile * 128 + hb * 64;
            blk_part[hb] = -1; blk_off[hb] = 0; blk_cv[hb] = false;
            if (P.rowpack) {
                if (kpos == 0) { blk_part[hb] = 0; blk_cv[hb] = chunk < P.kw; }
            } else {
                for (int p = 0; p < P.nparts; ++p)
                    if (kpos >= P.parts[p].koff && kpos < P.parts[p].koff + P.parts[p].kext) {
                        blk_part[hb] = p; blk_off[hb] = kpos - P.parts[p].koff;
                        blk_cv[hb] = blk_off[hb] + chunk * 8 < P.parts[p].c8;
                    }
            }
        }
        const int plane = P.ho * P.wo;
        bool dead = false;
        // per-CTA constants of the gather (32-bit element offsets): tap displacements and per-block source geometry
        int dtr[T], dtc[T], tbit[T];
#pragma unroll
        for (int tl = 0; tl < T; ++tl) {
            const int tg = tap0 + tl;
            if (P.rowpack) { dtr[tl] = tg * P.dil; dtc[tl] = chunk * P.dil; tbit[tl] = tg * P.kw + chunk; }
            else { const int tr = tg / P.kw, tc = tg - tr * P.kw; dtr[tl] = tr * P.dil; dtc[tl] = tc * P.dil; tbit[tl] = tg; }
        }
        const bf16 *bsrc[2];
        int bcs[2], brow[2], bimg[2], bxup[2], boff[2];
#pragma unroll
        for (int hb = 0; hb < 2; ++hb) {
            const TcPart &pt = P.parts[blk_part[hb] >= 0 ? blk_part[hb] : 0];
            bsrc[hb] = pt.x; bcs[hb] = pt.cstride; bxup[hb] = pt.xup;
            brow[hb] = (P.w >> pt.xup) * pt.cstride;
            bimg[hb] = (P.h >> pt.xup) * brow[hb];
            boff[hb] = P.rowpack ? 0 : blk_off[hb] + chunk * 8;
        }
        const bool fastrow = P.wo >= 64;
        // tap-validity words are prefetched one k-block ahead so their latency hides behind the barrier wait
        uint64_t tm_next[4][2];
        auto load_tm = [&](int kb, uint64_t (&dst)[4][2]) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int m = kb * 64 + r0 + 16 * i;
#pragma unroll
                for (int hb = 0; hb < 2; ++hb)
                    dst[i][hb] = (m < P.m_total && blk_part[hb] >= 0 && blk_cv[hb]) ? __ldg(P.parts[blk_part[hb]].tapmask + m) : 0ull;
            }
        };
        if (num_kb > 0) load_tm(kb_begin, tm_next);
        for (int it = 0; it < num_kb && !dead; ++it) {
            const int kb = kb_begin + it;
            const int s = it % STAGES;
            const uint32_t parity = ((it / STAGES) & 1) ^ 1;
            uint64_t tm_cur[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) { tm_cur[i][0] = tm_next[i][0]; tm_cur[i][1] = tm_next[i][1]; }
            if (it + 1 < num_kb) load_tm(kb + 1, tm_next);
            // coordinates of the k-block's first pixel (two divisions per k-block, not per row)
            const int mf = kb * 64;
            const int nf = mf / plane, remf = mf - nf * plane;
            const int ohf = remf / P.wo, owf = remf - ohf * P.wo;
            if (!ptx::mbar_wait(bar_empty + 8 * s, parity, P.abort_flag, 201)) { dead = true; break; }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = r0 + 16 * i;
                int nn = nf, oh = ohf, ow = owf + r;
                if (fastrow) {
                    if (ow >= P.wo) { ow -= P.wo; if (++oh >= P.ho) { oh = 0; ++nn; } }
                } else {
                    const int mm = min(mf + r, P.m_total - 1);
                    nn = mm / plane; const int rem = mm - nn * plane; oh = rem / P.wo; ow = rem - oh * P.wo;
                }
                const int hb0 = oh * P.stride - P.pad_h, wb0 = ow * P.stride - P.pad_w;
#pragma unroll
                for (int tl = 0; tl < T; ++tl) {
                    if (tl >= ntap) break;
                    const int hi = hb0 + dtr[tl], wi = wb0 + dtc[tl];
#pragma unroll
                    for (int hb = 0; hb < 2; ++hb) {
                        const bool v = (tm_cur[i][hb] >> tbit[tl]) & 1ull;     // 0 unless the block / chunk exists and the tap is valid
                        const int off = v ? nn * bimg[hb] + (hi >> bxup[hb]) * brow[hb] + (wi >> bxup[hb]) * bcs[hb] + boff[hb] : 0;
                        const uint32_t dst = sA + s * A_STAGE + tl * A_TAP_BYTES + hb * 8192 + r * 128 + sw;
                        ptx::cp_async_16(dst, bsrc[hb] + off, v);
                    }
                }
            }
            ptx::cp_async_mbar_arrive(bar_full_a + 8 * s);
            ptx::mbar_arrive(bar_full_a + 8 * s);
        }
        ptx::cp_async_wait<0>();
    } else if (warp == 12) {
        // ============ B producer: dc tiles [64 px][BLOCK_N co] via TMA, BLOCK_N/64 boxes of {64 co, 64 px} ============
        if (lane == 0) {
            for (int it = 0; it < num_kb; ++it) {
                const int kb = kb_begin + it;
                const int s = it % STAGES;
                const uint32_t parity = ((it / STAGES) & 1) ^ 1;
                if (!ptx::mbar_wait(bar_empty + 8 * s, parity, P.abort_flag, 203)) break;
                ptx::mbar_arrive_expect_tx(bar_full_b + 8 * s, B_STAGE_BYTES);
#pragma unroll
                for (int j = 0; j < BLOCK_N / 64; ++j)
                    ptx::tma_load_2d(sB + s * B_STAGE_BYTES + j * 8192, &tmap_dc, n0 + j * 64, kb * 64, bar_full_b + 8 * s);
            }
        }
    } else if (warp < MMA_WARPS && num_kb > 0) {
        // ============ consumer warpgroups: both operands MN-major; warpgroup g takes the tile's 64-channel block g ============
        const int g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        float acc[T][BLOCK_N / 2];
#pragma unroll
        for (int tl = 0; tl < T; ++tl) zero_acc(acc[tl]);
        bool dead = false;
        int held = -1;
        for (int it = 0; it < num_kb && !dead; ++it) {
            const int s = it % STAGES;
            const uint32_t parity = (it / STAGES) & 1;
            if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full_a + 8 * s, parity, P.abort_flag, 204) &&
                                             ptx::mbar_wait(bar_full_b + 8 * s, parity, P.abort_flag, 205))) { dead = true; break; }
            ptx::fence_proxy_async_smem();                       // cp.async (generic proxy) data -> wgmma (async proxy)
            ptx::wgmma_fence();
#pragma unroll
            for (int tl = 0; tl < T; ++tl) {
                if (tl >= ntap) break;
#pragma unroll
                for (int k = 0; k < 4; ++k) {     // 16 pixels (2 atoms of 8 k-rows = 2048 bytes) per step
                    const uint64_t da = ptx::make_smem_desc(sA + s * A_STAGE + tl * A_TAP_BYTES + g * 8192 + k * 2048, 8192, 1024);
                    const uint64_t db = ptx::make_smem_desc(sB + s * B_STAGE_BYTES + k * 2048, 8192, 1024);
                    ptx::wgmma_bf16<BLOCK_N, 1, 1>(acc[tl], da, db);
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            held = s;
        }
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int tl = 0; tl < T; ++tl) ptx::wgmma_fence_regs(acc[tl]);
        if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
        // ============ epilogue: D[k][co] per tap -> red.global.add into dw[co][tap][ci] ============
        if (!dead) {
            int ci[2], tap[2][T];
            for (int h = 0; h < 2; ++h) {
                const int row = 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * h;
                const int kpos = ci_tile * 128 + row;
                ci[h] = -1;
#pragma unroll
                for (int tl = 0; tl < T; ++tl) tap[h][tl] = tap0 + tl;
                if (P.rowpack) {
                    const int tc = row >> 3, ch = row & 7;
                    if (row < 64 && ci_tile == 0 && tc < P.kw && ch < P.cin) {
                        ci[h] = ch;
#pragma unroll
                        for (int tl = 0; tl < T; ++tl) tap[h][tl] = (tap0 + tl) * P.kw + tc;
                    }
                } else {
                    for (int p = 0; p < P.nparts; ++p) {
                        const int local = kpos - P.parts[p].koff;
                        if (local >= 0 && local < P.parts[p].c) ci[h] = P.parts[p].choff + local;
                    }
                }
            }
            wgrad_store<BLOCK_N, T>(P, acc, ntap, lane, n0, BLOCK_N, ci, tap);
        }
    }
}


// -------------------------------------------------------------------------------------------------
// weight gradient, TMA-FED.  Same GEMM as pconv_tc_wgrad_kernel (D[ci][co] per tap, K = output pixels, split-K with fp32
// red.global.add) but the gathered operand is no longer gathered: a K block of 64 consecutive output pixels is a box of the
// pixel grid, so the x rows of tap (tr, tc) / 64-channel block are one 4-D TMA tile (padding = out-of-range zero fill,
// stride-2 layers = traversal stride), written as exactly the MN-major 128B-swizzled block wgmma reads.  Holes are zeroed
// in the landed tile by three fixer warps (the tap-validity words of the block's pixels).
//   HALO (stride 1, K block = one image-row segment): a CTA owns one kernel ROW; one tile of 64 + (kw-1)*dil pixel rows per
//   channel block serves the kw taps of the row through row-shifted descriptors (T = kw register accumulators).
//   otherwise: a CTA owns T taps, one tile per tap.
//   warpgroups 0-1 consumers (MMA, then the red.global.add epilogue) | warpgroup 2: warp 8 TMA producer, warps 9-11 fixers
// BLOCK_N = 128 needs T x 64 fp32 accumulators per consumer thread: setmaxnreg moves registers from warpgroup 2 to the
// consumers (2 x 128 x 224 + 128 x 56 = 64,512 of the SM's 65,536; the kernel launches at 168 = 64,512 / 384).
// Who computes what: with both 64-channel blocks of the M tile present, warpgroup g takes block g for all BLOCK_N output
// channels.  With one block, a 128-wide tile gives warpgroup g output channels [64 g, 64 g + 64) of it; a 64-wide tile
// (cout <= 64) leaves warpgroup 1 idle.  Both warpgroups release every stage.
// -------------------------------------------------------------------------------------------------
constexpr int WGRAD_TMA_THREADS = 384;
constexpr int WGRAD_FIX_THREADS = 96;
constexpr int WGRAD_TMA_REGS = 168;                           // per thread at launch: setmaxnreg needs a fixed count
constexpr int WGRAD_CONSUMER_REGS = 224, WGRAD_SUPPORT_REGS = 56;
static_assert(2 * 128 * WGRAD_CONSUMER_REGS + 128 * WGRAD_SUPPORT_REGS == WGRAD_TMA_THREADS * WGRAD_TMA_REGS &&
              WGRAD_TMA_THREADS * WGRAD_TMA_REGS <= 65536, "wgrad register budget");

template <int BLOCK_N, int T, bool HALO>
__global__ void __maxnreg__(WGRAD_TMA_REGS)
pconv_tc_wgrad_tma_kernel(const __grid_constant__ WgParams P, const __grid_constant__ CUtensorMap tmap_dc,
                          const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1) {
    constexpr uint32_t B_BYTES = BLOCK_N * 128;               // [64 px][BLOCK_N co] as BLOCK_N/64 blocks of 8 KB
    constexpr int FIX_ROWS = HALO ? 3 : 1;                    // A-block rows per fixer thread: rows_a <= 256 (launch_wgrad_tma)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    uint8_t *smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));
    const int S = P.stages;
    const int hx = HALO ? (P.kw - 1) * P.dil : 0;
    const int rows_a = 64 + hx;                                // pixel rows of one A block
    const uint32_t A_BLK = (static_cast<uint32_t>(rows_a) * 128u + 1023u) & ~1023u;
    const uint32_t A_BYTES = (HALO ? 1 : T) * 2 * A_BLK;       // per stage: [tap][channel block]
    const uint32_t STAGE = A_BYTES + B_BYTES;
    const uint32_t sBar = smem_base + S * STAGE;
    const uint32_t bar_full = sBar, bar_fixed = sBar + 8 * MAX_RING, bar_empty = sBar + 16 * MAX_RING;

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    // blockIdx.x = ((co_tile * tap_groups) + tap_group) * ci_tiles + ci_tile ; blockIdx.y = K split
    int bx = blockIdx.x;
    const int ci_tile = bx % P.ci_tiles; bx /= P.ci_tiles;
    const int tap_group = bx % P.tap_groups;
    const int co_tile = bx / P.tap_groups;
    const int taps_full = P.kh * P.kw;
    const int tap0 = tap_group * T;                             // HALO: tap_group = kernel row, T = kw
    const int ntap = HALO ? T : min(T, taps_full - tap0);
    const int n0 = co_tile * BLOCK_N;
    const int total_kb = (P.m_total + 63) / 64;
    const int kb_begin = blockIdx.y * P.kb_per_split;
    const int num_kb = max(0, min(total_kb, kb_begin + P.kb_per_split) - kb_begin);
    // the two 64-channel blocks of this M tile: part and first channel (-1: block does not exist)
    int blk_part[2], blk_c0[2];
#pragma unroll
    for (int hb = 0; hb < 2; ++hb) {
        const int kpos = ci_tile * 128 + hb * 64;
        blk_part[hb] = -1; blk_c0[hb] = 0;
        for (int p = 0; p < P.nparts; ++p)
            if (kpos >= P.parts[p].koff && kpos < P.parts[p].koff + P.parts[p].kext && kpos - P.parts[p].koff < P.parts[p].c8) {
                blk_part[hb] = p; blk_c0[hb] = kpos - P.parts[p].koff;
            }
    }
    const int nblk = (blk_part[0] >= 0 ? 1 : 0) + (blk_part[1] >= 0 ? 1 : 0);
    const int solo = nblk == 1 ? (blk_part[0] >= 0 ? 0 : 1) : -1;      // the only channel block, or -1
    const bool fix = P.use_fix != 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) {
            ptx::mbar_init(bar_full + 8 * s, 1);
            ptx::mbar_init(bar_fixed + 8 * s, WGRAD_FIX_THREADS / 32);
            ptx::mbar_init(bar_empty + 8 * s, 2);                     // one arrival per consumer warpgroup
        }
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_dc); ptx::prefetch_tmap(&tmap_a0); ptx::prefetch_tmap(&tmap_a1); }
    __syncthreads();
    if (warp < MMA_WARPS) {
        ptx::setmaxnreg_inc<WGRAD_CONSUMER_REGS>();
        // ================================ consumer warpgroups: both operands MN-major ================================
        // warpgroup g multiplies channel block ablk of the A tile by output channels [nc0, nc0 + ncols) of the B tile; a
        // 64-wide tile with one channel block leaves warpgroup 1 idle (it still releases every stage)
        const int g = warp >> 2;
        const int ablk = solo >= 0 ? solo : g;
        const bool split_n = solo >= 0 && BLOCK_N == 128;
        const bool live = !(solo >= 0 && BLOCK_N == 64) || g == 0;
        const int nc0 = split_n ? 64 * g : 0, ncols = split_n ? 64 : BLOCK_N;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t ready = fix ? bar_fixed : bar_full;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + ablk * A_BLK, A_BLK, 1024);
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_BYTES + nc0 * 128, 8192, 1024);
        const uint32_t stage16 = STAGE >> 4;
        const uint32_t tap16 = HALO ? static_cast<uint32_t>(P.dil * 8) : (2 * A_BLK) >> 4;   // per tap: row shift (halo) or next tile
        float acc[T][BLOCK_N / 2];
#pragma unroll
        for (int tl = 0; tl < T; ++tl) zero_acc(acc[tl]);
        int s = 0, held = -1;
        uint32_t ph = 0;
        bool dead = false;
        for (int it = 0; it < num_kb; ++it) {
            if (!__all_sync(0xffffffffu, ptx::mbar_wait(ready + 8 * s, ph, P.abort_flag, 224))) { dead = true; break; }
            if (!live) {
                if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
                held = s;
                if (++s == S) { s = 0; ph ^= 1; }
                continue;
            }
            uint64_t da = desc_a0 + static_cast<uint64_t>(s * stage16);
            const uint64_t db = desc_b0 + static_cast<uint64_t>(s * stage16);
            ptx::wgmma_fence();
            if (BLOCK_N == 128 && split_n) {
#pragma unroll
                for (int tl = 0; tl < T; ++tl, da += tap16) {
                    if (tl >= ntap) break;
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        ptx::wgmma_m64n64<1, 1>(acc[tl], da + 128 * k, db + 128 * k);     // columns 0-63 of acc
                }
            } else {
#pragma unroll
                for (int tl = 0; tl < T; ++tl, da += tap16) {
                    if (tl >= ntap) break;
#pragma unroll
                    for (int k = 0; k < 4; ++k)                  // 16 pixels (two 8-row atoms = 2048 bytes) per step
                        ptx::wgmma_bf16<BLOCK_N, 1, 1>(acc[tl], da + 128 * k, db + 128 * k);
                }
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();
            if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
            held = s;
            if (++s == S) { s = 0; ph ^= 1; }
        }
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int tl = 0; tl < T; ++tl) ptx::wgmma_fence_regs(acc[tl]);
        if (held >= 0 && leader) ptx::mbar_arrive(bar_empty + 8 * held);
        // ---- epilogue: D[ci][co] per tap -> red.global.add into dw[co][tap][ci]
        if (!dead && live && num_kb > 0) {
            int ci[2], tap[2][T];
            for (int h = 0; h < 2; ++h) {
                const int kpos = ci_tile * 128 + 64 * ablk + 16 * (warp & 3) + (lane >> 2) + 8 * h;
                ci[h] = -1;
                for (int p = 0; p < P.nparts; ++p) {
                    const int local = kpos - P.parts[p].koff;
                    if (local >= 0 && local < P.parts[p].c) ci[h] = P.parts[p].choff + local;
                }
#pragma unroll
                for (int tl = 0; tl < T; ++tl) tap[h][tl] = tap0 + tl;
            }
            wgrad_store<BLOCK_N, T>(P, acc, ntap, lane, n0 + nc0, ncols, ci, tap);
        }
    } else {
        ptx::setmaxnreg_dec<WGRAD_SUPPORT_REGS>();      // the whole of warpgroup 2, fixers included when there are no holes
        if (warp == 8) {
            // ================================ TMA producer ================================
            const int plane = P.ho * P.wo;
            const uint32_t tx_bytes = static_cast<uint32_t>((HALO ? 1 : ntap) * nblk * rows_a * 128) + B_BYTES;
            int s = 0;
            uint32_t ph = 1;
            for (int it = 0; it < num_kb; ++it) {
                const int m0 = (kb_begin + it) * 64;
                const int img = m0 / plane, rem = m0 - img * plane;
                const int oy = rem / P.wo, ox = rem - oy * P.wo;
                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 221))) break;
                if (ptx::elect_one()) {
                    const uint32_t full = bar_full + 8 * s, dst = smem_base + s * STAGE;
                    ptx::mbar_arrive_expect_tx(full, tx_bytes);
                    for (int tl = 0; tl < (HALO ? 1 : ntap); ++tl) {
                        const int tap = tap0 + tl;
                        const int tr = HALO ? tap_group : tap / P.kw, tc = HALO ? 0 : tap - tr * P.kw;
                        const int y = oy * P.stride - P.pad_h + tr * P.dil, x = ox * P.stride - P.pad_w + tc * P.dil;
#pragma unroll
                        for (int hb = 0; hb < 2; ++hb)
                            if (blk_part[hb] >= 0)
                                ptx::tma_load_4d(dst + (tl * 2 + hb) * A_BLK, blk_part[hb] == 0 ? &tmap_a0 : &tmap_a1, blk_c0[hb], x, y, img, full);
                    }
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 64; ++j)
                        ptx::tma_load_2d(dst + A_BYTES + j * 8192, &tmap_dc, n0 + j * 64, m0, full);
                }
                __syncwarp();
                if (++s == S) { s = 0; ph ^= 1; }
            }
        } else if (fix) {
            // ================================ fixers (hole rows -> 0) ================================
            // thread fi owns pixel rows fi + 96 j of the A blocks.  A row takes the tap-validity word of the output pixel that
            // reads it (halo rows past 63 belong to a later tap column).
            const int fi = (warp - 9) * 32 + lane;
            int jpix[FIX_ROWS], bit[FIX_ROWS];
#pragma unroll
            for (int j = 0; j < FIX_ROWS; ++j) {
                const int f = fi + WGRAD_FIX_THREADS * j;
                const int tcs = (HALO && f > 63) ? (f - 63 + P.dil - 1) / P.dil : 0;
                jpix[j] = f < rows_a ? f - tcs * P.dil : -1;
                bit[j] = HALO ? tap_group * P.kw + tcs : tap0;
            }
            uint64_t wnext[FIX_ROWS][2];
            auto load_words = [&](int kb) {
#pragma unroll
                for (int j = 0; j < FIX_ROWS; ++j) {
                    const int m = kb * 64 + jpix[j];
#pragma unroll
                    for (int hb = 0; hb < 2; ++hb)
                        wnext[j][hb] = (jpix[j] >= 0 && blk_part[hb] >= 0 && m < P.m_total && kb < kb_begin + num_kb) ? __ldg(P.parts[blk_part[hb]].tapmask + m) : 0ull;
                }
            };
            load_words(kb_begin);
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < num_kb; ++it) {
                uint32_t hole = 0;                                   // bit (j * 2 + hb) * T + tl: row j of tile (tl, hb) -> 0
#pragma unroll
                for (int j = 0; j < FIX_ROWS; ++j)
#pragma unroll
                    for (int hb = 0; hb < 2; ++hb)
#pragma unroll
                        for (int tl = 0; tl < (HALO ? 1 : T); ++tl)
                            if (tl < ntap && jpix[j] >= 0 && blk_part[hb] >= 0 && ((wnext[j][hb] >> (bit[j] + tl)) & 1ull) == 0ull)
                                hole |= 1u << ((j * 2 + hb) * T + tl);
                load_words(kb_begin + it + 1);
                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 222))) break;
                if (hole) {
#pragma unroll
                    for (int j = 0; j < FIX_ROWS; ++j)
#pragma unroll
                        for (int hb = 0; hb < 2; ++hb)
#pragma unroll
                            for (int tl = 0; tl < (HALO ? 1 : T); ++tl)
                                if ((hole >> ((j * 2 + hb) * T + tl)) & 1u) {
                                    uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + (tl * 2 + hb) * A_BLK + (fi + WGRAD_FIX_THREADS * j) * 128);
                                    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                                    for (int k = 0; k < 8; ++k) r[k] = z;
                                }
                }
                if (__any_sync(0xffffffffu, hole != 0)) ptx::fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) ptx::mbar_arrive(bar_fixed + 8 * s);
                if (++s == S) { s = 0; ph ^= 1; }
            }
        }
    }
}

// -------------------------------------------------------------------------------------------------
// tap-validity bitmasks: bit t of tapmask[p][m] = tap t of output pixel m is in bounds and not a hole
// -------------------------------------------------------------------------------------------------
struct TapMaskParams {
    int n, h, w, kh, kw, stride, pad_h, pad_w, dil, ho, wo, m_total, nparts;
    const uint8_t *mask[TC_MAX_PARTS];
    int mup[TC_MAX_PARTS];
    uint64_t *out;   // [nparts][m_total]
};

__global__ void tapmask_kernel(const TapMaskParams P) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= P.m_total) return;
    const int plane = P.ho * P.wo;
    const int nn = m / plane, rem = m - nn * plane, oh = rem / P.wo, ow = rem - oh * P.wo;
#pragma unroll
    for (int p = 0; p < TC_MAX_PARTS; ++p) {
        if (p >= P.nparts) break;
        const uint8_t *mk = P.mask[p];
        const int u = P.mup[p];
        uint64_t bits = 0;
        int tap = 0;
        for (int tr = 0; tr < P.kh; ++tr)
            for (int tc = 0; tc < P.kw; ++tc, ++tap) {
                const int hi = oh * P.stride - P.pad_h + tr * P.dil, wi = ow * P.stride - P.pad_w + tc * P.dil;
                bool v = hi >= 0 && hi < P.h && wi >= 0 && wi < P.w;
                if (v && mk) v = mk[(static_cast<long long>(nn) * (P.h >> u) + (hi >> u)) * (P.w >> u) + (wi >> u)] != 0;
                bits |= (v ? 1ull : 0ull) << tap;
            }
        P.out[static_cast<long long>(p) * P.m_total + m] = bits;
    }
}

// -------------------------------------------------------------------------------------------------
// weight re-layout: fp32 master KRSC [cout][taps][cin] -> padded bf16 operands of the two GEMMs
//   w_fwd  [rows_f][kf] : row = co ; k = tap*ktap + koff_p + local        (rowpack: tr*64 + tc*8 + ci)
//   w_dg   [ktap][kd]   : row = koff_p + local ; k = tap*cout64 + co      (not built in rowpack mode)
// -------------------------------------------------------------------------------------------------
struct WPrepParams {
    int cout, taps, cin, kw, rowpack, nparts, ktap, cout64;
    int choff[TC_MAX_PARTS], c[TC_MAX_PARTS], koff[TC_MAX_PARTS];
    long long kf, kd;
};

// tiled variant: a block converts a [32 cout][32 cin] tile of one tap through shared memory, so the master is read and both
// operand matrices are written along their contiguous dimension (w_dg is the transpose: written along cout)
__global__ void __launch_bounds__(256) tc_weight_prepare_tiled_kernel(const float *__restrict__ wm, const WPrepParams P, bf16 *__restrict__ w_fwd,
                                                                      bf16 *__restrict__ w_dg) {
    __shared__ float tile[32][33];
    const int tap = blockIdx.z, co0 = blockIdx.y * 32, ci0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int co = co0 + ty + 8 * i, ci = ci0 + tx;
        float v = 0.f;
        if (co < P.cout && ci < P.cin) v = wm[(static_cast<long long>(co) * P.taps + tap) * P.cin + ci];
        tile[ty + 8 * i][tx] = v;
    }
    __syncthreads();
    {
        const int ci = ci0 + tx;
        if (ci < P.cin) {
            int p = 0;
            while (p + 1 < P.nparts && ci >= P.choff[p] + P.c[p]) ++p;
            const int kpos = P.koff[p] + (ci - P.choff[p]);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int co = co0 + ty + 8 * i;
                if (co < P.cout) w_fwd[static_cast<long long>(co) * P.kf + static_cast<long long>(tap) * P.ktap + kpos] = __float2bfloat16_rn(tile[ty + 8 * i][tx]);
            }
        }
    }
    if (w_dg) {
        const int co = co0 + tx;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int ci = ci0 + ty + 8 * i;
            if (co < P.cout && ci < P.cin) {
                int p = 0;
                while (p + 1 < P.nparts && ci >= P.choff[p] + P.c[p]) ++p;
                const int kpos = P.koff[p] + (ci - P.choff[p]);
                w_dg[static_cast<long long>(kpos) * P.kd + static_cast<long long>(tap) * P.cout64 + co] = __float2bfloat16_rn(tile[tx][ty + 8 * i]);
            }
        }
    }
}

__global__ void tc_weight_prepare_kernel(const float *__restrict__ wm, const WPrepParams P, bf16 *__restrict__ w_fwd, bf16 *__restrict__ w_dg) {
    const long long total = static_cast<long long>(P.cout) * P.taps * P.cin;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % P.cin);
        const long long t = i / P.cin;
        const int tap = static_cast<int>(t % P.taps), co = static_cast<int>(t / P.taps);
        const bf16 v = __float2bfloat16_rn(wm[i]);
        if (P.rowpack) {
            const int tr = tap / P.kw, tc = tap - tr * P.kw;
            w_fwd[static_cast<long long>(co) * P.kf + tr * 64 + tc * 8 + ci] = v;
        } else {
            int p = 0;
            while (p + 1 < P.nparts && ci >= P.choff[p] + P.c[p]) ++p;
            const int kpos = P.koff[p] + (ci - P.choff[p]);
            w_fwd[static_cast<long long>(co) * P.kf + static_cast<long long>(tap) * P.ktap + kpos] = v;
            if (w_dg) w_dg[static_cast<long long>(kpos) * P.kd + static_cast<long long>(tap) * P.cout64 + co] = v;
        }
    }
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// 2D bf16 row-major [rows][cols] tensor (row pitch `pitch_elems`), box {64 cols (128 bytes), box_rows}, SWIZZLE_128B
int make_tmap_2d(CUtensorMap *tm, const void *base, long long rows, long long cols, long long pitch_elems, int box_rows) {
    EncodeTiledFn enc = get_encode_fn();
    PCB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch_elems) * 2};
    cuuint32_t box[2] = {64, static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PCB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld pitch=%lld box_rows=%d base=%p", (int)r,
              rows, cols, pitch_elems, box_rows, base);
    return 0;
}

// 4D bf16 NHWC tensor viewed as (channels, x, y, image); box {64 ch, bx, by, bn} pixels visited with traversal stride `es`
// along x and y.  `channels` may be smaller than 64: the rest of the 128-byte row is zero-filled (channel padding).
int make_tmap_nhwc(CUtensorMap *tm, const void *base, int channels, int w, int h, int n, long long cstride, int bx, int by, int bn, int es) {
    EncodeTiledFn enc = get_encode_fn();
    PCB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(channels), static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h), static_cast<cuuint64_t>(n)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(cstride) * 2, static_cast<cuuint64_t>(w) * cstride * 2, static_cast<cuuint64_t>(h) * w * cstride * 2};
    cuuint32_t box[4] = {64, static_cast<cuuint32_t>(bx * es), static_cast<cuuint32_t>(by * es), static_cast<cuuint32_t>(bn)};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(es), static_cast<cuuint32_t>(es), 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    PCB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(4D) failed (%d) c=%d w=%d h=%d n=%d cstride=%lld box=%d,%d,%d es=%d base=%p", (int)r,
              channels, w, h, n, cstride, bx, by, bn, es, base);
    return 0;
}

// one abort flag per device (a flag allocated on the first-used device is an illegal address on every other one)
int *abort_flag_ptr() {
    static int *flag[PCB_MAX_DEVICES] = {};
    const int dev = pcb_cur_device();
    if (!flag[dev]) {
        if (cudaMalloc(&flag[dev], sizeof(int)) != cudaSuccess) { flag[dev] = nullptr; return nullptr; }
        cudaMemset(flag[dev], 0, sizeof(int));
    }
    return flag[dev];
}

bool is_rowpack(const pcb_conv *c) { return c->nparts == 1 && c->cin <= 8 && c->kw <= 8 && c->parts[0].x_up == 0; }

bool common_ok(const pcb_conv *c) {
    if (c->dtype != PCB_BF16 || c->groups != 1 || c->kh * c->kw > 64) return false;
    if (c->stride & (c->stride - 1)) return false;                               // shifts instead of divisions in the gather
    // the gathers use 32-bit element offsets
    const long long lim = (1ll << 31) - 1;
    if (static_cast<long long>(c->n) * c->ho * c->wo * rup(c->cout, 64) > lim) return false;
    if (c->nparts < 1 || c->nparts > TC_MAX_PARTS) return false;
    for (int p = 0; p < c->nparts; ++p) {
        const pcb_part &pt = c->parts[p];
        if (pt.x_cstride % 8 != 0 || pt.x_cstride < rup(pt.c, 8)) return false;     // 16-byte chunks must be readable
        if (static_cast<long long>(c->n) * (c->h >> pt.x_up) * (c->w >> pt.x_up) * pt.x_cstride > lim) return false;
        if (pt.x && (reinterpret_cast<uintptr_t>(pt.x) & 15)) return false;
    }
    if (is_rowpack(c)) return c->cout >= 16;
    // tensor cores pay off once the reduction is reasonably wide; tiny-channel layers stay on the generic kernels
    return c->cin >= 32 || c->cout >= 32;
}

struct Layout {
    int rowpack, ktap, cout64, rows_f, bn_f;
    long long kf, kd;
    int koff[TC_MAX_PARTS], kext[TC_MAX_PARTS];
};

Layout layout_of(const pcb_conv *c) {
    Layout L;
    memset(&L, 0, sizeof(L));
    L.rowpack = is_rowpack(c);
    const int taps = c->kh * c->kw;
    if (L.rowpack) {
        L.ktap = 64; L.koff[0] = 0; L.kext[0] = 64;
        L.kf = static_cast<long long>(c->kh) * 64;
    } else {
        int off = 0;
        for (int p = 0; p < c->nparts; ++p) { L.koff[p] = off; L.kext[p] = rup(c->parts[p].c, 64); off += L.kext[p]; }
        L.ktap = off;
        L.kf = static_cast<long long>(taps) * L.ktap;
    }
    L.cout64 = rup(c->cout, 64);
    L.bn_f = (c->cout % 128 == 0) ? 128 : 64;
    L.rows_f = rup(c->cout, L.bn_f);
    L.kd = static_cast<long long>(taps) * L.cout64;
    return L;
}

void fill_parts(const pcb_conv *c, const Layout &L, TcPart *out, const uint64_t *tapmask, long long m_total) {
    int off = 0;
    for (int p = 0; p < c->nparts; ++p) {
        out[p].x = static_cast<const bf16 *>(c->parts[p].x);
        out[p].tapmask = tapmask ? tapmask + static_cast<long long>(p) * m_total : nullptr;
        out[p].mask = c->parts[p].mask;
        out[p].dx = nullptr; out[p].dx_cstride = 0;
        out[p].c = c->parts[p].c;
        out[p].c8 = rup(c->parts[p].c, 8);
        out[p].kext = L.kext[p];
        out[p].koff = L.koff[p];
        out[p].choff = off;
        out[p].cstride = c->parts[p].x_cstride;
        out[p].xup = c->parts[p].x_up;
        out[p].mup = c->parts[p].mask_up;
        off += c->parts[p].c;
    }
}

int launch_tapmask(const pcb_conv *c, uint64_t *out, cudaStream_t st) {
    TapMaskParams T;
    memset(&T, 0, sizeof(T));
    T.n = c->n; T.h = c->h; T.w = c->w; T.kh = c->kh; T.kw = c->kw; T.stride = c->stride; T.pad_h = c->pad_h;
    T.pad_w = c->pad_w; T.dil = c->dil; T.ho = c->ho; T.wo = c->wo; T.m_total = c->n * c->ho * c->wo; T.nparts = c->nparts;
    for (int p = 0; p < c->nparts; ++p) { T.mask[p] = c->parts[p].mask; T.mup[p] = c->parts[p].mask_up; }
    T.out = out;
    tapmask_kernel<<<(T.m_total + 255) / 256, 256, 0, st>>>(T);
    PCB_LAUNCH_CHECK();
    return 0;
}

void set_ep(TcParams &P, const pcb_ep *ep) {
    if (ep == nullptr) return;
    P.ep_on = 1; P.ep_scale = ep->scale; P.ep_shift = ep->shift; P.ep_act = ep->act; P.ep_slope = ep->slope;
}

void base_params(TcParams &P, const pcb_conv *c, const Layout &L) {
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.cin = c->cin; P.cout = c->cout; P.kh = c->kh; P.kw = c->kw; P.stride = c->stride;
    P.pad_h = c->pad_h; P.pad_w = c->pad_w; P.dil = c->dil; P.ho = c->ho; P.wo = c->wo;
    P.nparts = c->nparts; P.no_guard = c->no_guard; P.rowpack = L.rowpack; P.ktap = L.ktap;
    P.sub = 1; P.py = 0; P.px = 0; P.fh = c->h; P.fw = c->w;
}

// H100: 227 KB of shared memory per block.  The rings get what the epilogue staging tile, the statistics and the barriers leave.
constexpr size_t MAX_SMEM = 227 * 1024;
constexpr size_t RING_BUDGET = 208 * 1024;

template <int BLOCK_N, int MODE>
int launch_persistent(TcParams &P, const CUtensorMap &tm, cudaStream_t st) {
    const size_t a_stage = A_STAGE_BYTES;
    const size_t b_stage = BLOCK_N * 128;
    const size_t budget = RING_BUDGET - acc_stage_bytes(BLOCK_N);
    P.ring_b = 6;
    P.ring_a = 6;
    while (P.ring_a * a_stage + P.ring_b * b_stage > budget && P.ring_b > 3) --P.ring_b;
    while (P.ring_a * a_stage + P.ring_b * b_stage > budget && P.ring_a > 2) --P.ring_a;
    const size_t smem = 1024 + P.ring_a * a_stage + P.ring_b * b_stage + 32 * MAX_RING + 16 + STAT_SMEM_BYTES + acc_stage_bytes(BLOCK_N);
    PCB_CHECK(smem <= MAX_SMEM, "tensor-core conv: %zu bytes of shared memory do not fit", smem);
    auto kern = pconv_tc_persistent_kernel<BLOCK_N, MODE>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    const int num_tiles = ((P.m_total + BLOCK_M - 1) / BLOCK_M) * (P.ncols / BLOCK_N);
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, PERSIST_THREADS, smem, st>>>(P, tm);
    PCB_LAUNCH_CHECK();
    return 0;
}


// ---- TMA-fed path: eligibility, tile box, launch -------------------------------------------------
// 128 consecutive pixels of a [n][ht][wt] grid as a box {bw, bh, bn}: possible when the extents nest in powers of two
bool tile_box(int wt, int ht, int *bw, int *bh, int *bn) {
    if (wt < 4) return false;
    if (wt % 128 == 0) { *bw = 128; *bh = 1; *bn = 1; return true; }
    if (128 % wt) return false;
    const int rows = 128 / wt;
    *bw = wt;
    if (ht % rows == 0) { *bh = rows; *bn = 1; return true; }
    if (rows % ht) return false;
    *bh = ht; *bn = rows / ht;
    return true;
}

// 64 consecutive pixels of a [n][ht][wt] grid as a box {bw, bh, bn} (the K blocks of the weight gradient)
bool kblock_box(int wt, int ht, int *bw, int *bh, int *bn) {
    if (wt < 4) return false;
    if (wt % 64 == 0) { *bw = 64; *bh = 1; *bn = 1; return true; }
    if (64 % wt) return false;
    const int rows = 64 / wt;
    *bw = wt;
    if (ht % rows == 0) { *bh = rows; *bn = 1; return true; }
    if (rows % ht) return false;
    *bh = ht; *bn = rows / ht;
    return true;
}

bool even_upsampled_parts(const pcb_conv *c) {
    for (int p = 0; p < c->nparts; ++p)
        if (c->parts[p].x_up && ((c->h | c->w) & 1)) return false;
    return true;
}

// the TMA-fed kernels of each direction take the problem when its M tile box exists (the row-packed layout has no TMA path)
bool tma_fwd_ok(const pcb_conv *c, int *bw, int *bh, int *bn) {
    if (is_rowpack(c) || !tile_box(c->wo, c->ho, bw, bh, bn)) return false;
    if (c->stride > 2 || *bw * c->stride > 256 || *bh * c->stride > 256) return false;
    return even_upsampled_parts(c);
}

// stride-2 data gradient of a layer that is not row-packed as four stride-1 parity-class problems (see pcb_tc_dgrad)
bool tma_dgrad_s2_ok(const pcb_conv *c, int *bw, int *bh, int *bn) {
    if (c->stride != 2 || c->dil != 1 || c->kh < 2 || c->kw < 2 || ((c->h | c->w) & 1) || c->ho != c->h / 2 || c->wo != c->w / 2) return false;
    return tile_box(c->w / 2, c->h / 2, bw, bh, bn);
}

// kernel columns of the parity class with input column parity px: the taps with (px + pad - tc) even
int class_kw(const pcb_conv *c, int px) { return (c->kw - ((px + c->pad_w) & 1) + 1) / 2; }

bool tma_wgrad_ok(const pcb_conv *c, int *bw, int *bh, int *bn) {
    return !is_rowpack(c) && c->stride <= 2 && kblock_box(c->wo, c->ho, bw, bh, bn) && even_upsampled_parts(c);
}

size_t up_bytes(const pcb_conv *c, int p) {
    return (static_cast<size_t>(c->n) * c->h * c->w * rup(c->parts[p].c, 8) * 2 + 255) / 256 * 256;
}
size_t tapmask_bytes(const pcb_conv *c) {
    return (static_cast<size_t>(c->nparts) * c->n * c->ho * c->wo * sizeof(uint64_t) + 255) / 256 * 256;
}

// shared memory of a TMA-fed fwd / dgrad / sub-pixel launch outside its ring: alignment slack, barriers, statistics slices and
// the bf16 staging tile; the ring gets the rest of the opt-in maximum
size_t tma_fixed_smem(int block_n) {
    return 1024 + TMA_BAR_BYTES + EPI_STAT_SMEM_BYTES + bf16_stage_bytes(block_n);
}

template <int BLOCK_N, int MODE, bool HALO>
int launch_tma_n(TcParams &P, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, cudaStream_t st) {
    const int nb = HALO ? P.kw : 1;
    const size_t a_room = (static_cast<size_t>(BLOCK_M + (HALO ? (P.kw - 1) * P.dil : 0)) * 128 + 1023) / 1024 * 1024;
    const size_t stage = a_room + static_cast<size_t>(nb) * BLOCK_N * 128;
    const size_t fixed = tma_fixed_smem(BLOCK_N);
    P.stages = static_cast<int>(std::min<size_t>(MAX_RING, (MAX_SMEM - fixed) / stage));
    PCB_CHECK(P.stages >= 2, "TMA-fed conv: stage of %zu bytes does not fit twice", stage);
    const size_t smem = fixed + P.stages * stage;
    auto kern = pconv_tc_tma_kernel<BLOCK_N, MODE, HALO>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * (P.ncols / BLOCK_N);
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, TMA_THREADS, smem, st>>>(P, tw, ta0, ta1);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <int MODE>
int launch_tma(TcParams &P, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, int bn, bool halo, cudaStream_t st) {
    PCB_CHECK(!(halo && bn == 256), "TMA-fed conv: no 256-wide row-halo tiles");
    if (halo) {
        if (bn == 128) return launch_tma_n<128, MODE, true>(P, tw, ta0, ta1, st);
        if (bn == 64) return launch_tma_n<64, MODE, true>(P, tw, ta0, ta1, st);
        return launch_tma_n<32, MODE, true>(P, tw, ta0, ta1, st);
    }
    if (bn == 256) return launch_tma_n<256, MODE, false>(P, tw, ta0, ta1, st);
    if (bn == 128) return launch_tma_n<128, MODE, false>(P, tw, ta0, ta1, st);
    if (bn == 64) return launch_tma_n<64, MODE, false>(P, tw, ta0, ta1, st);
    return launch_tma_n<32, MODE, false>(P, tw, ta0, ta1, st);
}

// at least three stages of (halo tile of 128 + (kw-1)*dil pixel rows + kw weight tiles) fit in shared memory next to the
// epilogue staging tile of an N tile of block_n columns.  The test keeps the fp32 staging size and ring budget it was
// introduced with although the tiles now stage bf16: halo tiles sum a layer's K blocks in another order, so moving this
// boundary would change which layers' outputs round differently.
bool halo_stages_fit(int kw, int dil, int block_n) {
    const size_t stage = (static_cast<size_t>(128 + (kw - 1) * dil) * 128 + 1023) / 1024 * 1024 + static_cast<size_t>(kw) * block_n * 128;
    return 3 * stage + acc_stage_bytes(block_n) <= RING_BUDGET;
}

// row-halo tiles of the TMA-fed forward / data gradient for a (stride-1) kernel row of kw taps: the M tile is one image-row
// segment, a kernel row's halo fits the 256-pixel TMA box, and the stages fit
bool halo_ok(int kw, int dil, int bw, int bh, int bn, int block_n) {
    return bw == 128 && bh == 1 && bn == 1 && kw >= 2 && 128 + (kw - 1) * dil <= 256 && halo_stages_fit(kw, dil, block_n);
}

// widest N tile that divides `cols` and still leaves at least one tile per SM; low-resolution layers (a handful of M tiles
// against a multi-megabyte weight matrix) get NARROWER N tiles: each CTA's operand stream is latency-bound (a ring of a few
// stages), so the time of such a layer is (bytes per CTA) / that rate -- more, smaller CTAs stream the weights in parallel
// (a consumer warpgroup holds 64 rows x N fp32 accumulators in registers).
// 256-wide tiles pull a quarter fewer operand bytes from L2 per FLOP and give every ring stage twice the MMA work.  The
// persistent CTAs walk the tiles in waves of one tile per SM, so 256 columns can only win when their (twice as long) waves are
// at most half as many as those of 128-wide tiles.  Measured per layer on ImageFillOrigin 512^2, batch 8 (tools/tc_layers.py,
// H100 at 700 W, 128 forced vs this rule): the data gradients win wherever that holds (dec1 1024 columns, 256 tiles: 0.137 ->
// 0.133 ms; dec5 768 columns, 768 tiles: 0.262 -> 0.252 ms), the forward only where 256 columns take ONE wave instead of two
// (dec1, 128 tiles: 0.199 -> 0.191 ms).  With more waves the forward lost (enc2 and dec5, 256 tiles: 0.164 -> 0.172 and
// 0.271 -> 0.295 ms; enc3: 0.082 -> 0.089 ms): its consumers also do the epilogue's element math, twice as much per tile.
int pick_bn(int cols, long long m_total, bool fwd, int sms) {
    const long long m_tiles = (m_total + BLOCK_M - 1) / BLOCK_M;
    if (cols <= 32) return 32;
    auto waves = [&](int b) { return (m_tiles * (cols / b) + sms - 1) / sms; };
    if (cols % 256 == 0 && 2 * waves(256) <= waves(128) && (!fwd || waves(256) == 1)) return 256;
    int bn = (cols % 128 == 0) ? 128 : 64;
    while (bn > 32 && cols % (bn / 2) == 0 && m_tiles * (cols / bn) < sms / 2) bn /= 2;
    return bn;
}

template <int MODE>
int launch_tc(TcParams &P, const CUtensorMap &tm, int bn, cudaStream_t st) {
    return (bn == 128) ? launch_persistent<128, MODE>(P, tm, st) : launch_persistent<64, MODE>(P, tm, st);
}

// internal streams for the four parity-class launches of low-resolution layers: one set per device AND per host thread (two
// host threads driving data gradients on two streams must not share the fork / join events)
struct ClassStreams { cudaStream_t aux[3]; cudaEvent_t ev_fork, ev_join[3]; bool ready; };
int class_streams(ClassStreams **out) {
    static thread_local ClassStreams cs_all[PCB_MAX_DEVICES] = {};
    ClassStreams &CS = cs_all[pcb_cur_device()];
    if (!CS.ready) {
        for (int i = 0; i < 3; ++i) {
            PCB_CUDA(cudaStreamCreateWithFlags(&CS.aux[i], cudaStreamNonBlocking));
            PCB_CUDA(cudaEventCreateWithFlags(&CS.ev_join[i], cudaEventDisableTiming));
        }
        PCB_CUDA(cudaEventCreateWithFlags(&CS.ev_fork, cudaEventDisableTiming));
        CS.ready = true;
    }
    *out = &CS;
    return 0;
}

// ---- sub-pixel data gradient: plan, weights, launch ---------------------------------------------------
// one spatial axis: for output parity q, tap t of a (k, dilation d, padding p) kernel over the 2x-upsampled source reads source
// offset floor((q + t*d - p) / 2); the distinct offsets e0 .. e0+ne-1 are the effective taps, tapbits[q][e] the original taps
// that collapse onto effective tap e
struct SpAxis { int e0[2], ne[2], tapbits[2][4]; bool ok; };

int floordiv2(int v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); }

SpAxis sp_axis(int k, int d, int p) {
    SpAxis A;
    memset(&A, 0, sizeof(A));
    A.ok = k <= 4;
    for (int q = 0; q < 2 && A.ok; ++q) {
        A.e0[q] = floordiv2(q - p);
        const int last = floordiv2(q + (k - 1) * d - p);
        A.ne[q] = last - A.e0[q] + 1;
        if (A.ne[q] < 1 || A.ne[q] > 4) { A.ok = false; break; }
        for (int t = 0; t < k; ++t) A.tapbits[q][floordiv2(q + t * d - p) - A.e0[q]] |= 1 << t;
        for (int e = 0; e < A.ne[q]; ++e)
            if (!A.tapbits[q][e]) A.ok = false;               // a gap between effective taps (dilation > 2): not handled here
    }
    return A;
}

struct SpPlan {
    bool ok;                         // the data gradient of the upsampled part takes the sub-pixel kernel (see sp_plan)
    int pu, ps;                      // the upsampled part and the other one (-1: none)
    SpAxis ay, ax;
    int net[4], eoff[4], net_total;  // effective taps of the upsampled part per class (class = py * 2 + px)
    int kext_u, c8_u;
    long long sp_dg_elems, kd_sp;
    int bw, bh, bn;                  // M tile box of the source grid [n][h/2][w/2]
    int block_n;                     // N tile width (at most 64)
};

// for a tensor-core problem that is neither row-packed nor small-Cout
SpPlan sp_plan(const pcb_conv *c, const Layout &L, int sms) {
    SpPlan S;
    memset(&S, 0, sizeof(S));
    S.pu = S.ps = -1;
    if (c->stride != 1 || c->ho != c->h || c->wo != c->w || ((c->h | c->w) & 1) || c->nparts > 2) return S;
    for (int p = 0; p < c->nparts; ++p) {
        if (c->parts[p].x_up) { if (S.pu >= 0) return S; S.pu = p; }
        else { if (S.ps >= 0) return S; S.ps = p; }
    }
    if (S.pu < 0) return S;
    // the hole mask of each part must live at the part's own resolution (HoleMask.upsampled keeps them together)
    if (c->parts[S.pu].mask && c->parts[S.pu].mask_up != 1) return S;
    if (S.ps >= 0 && c->parts[S.ps].mask && c->parts[S.ps].mask_up != 0) return S;
    S.ay = sp_axis(c->kh, c->dil, c->pad_h);
    S.ax = sp_axis(c->kw, c->dil, c->pad_w);
    if (!S.ay.ok || !S.ax.ok) return S;
    if (!tile_box(c->w / 2, c->h / 2, &S.bw, &S.bh, &S.bn)) return S;
    S.kext_u = L.kext[S.pu]; S.c8_u = rup(c->parts[S.pu].c, 8);
    int eo = 0;
    for (int cls = 0; cls < 4; ++cls) {
        S.net[cls] = S.ay.ne[cls >> 1] * S.ax.ne[cls & 1];
        S.eoff[cls] = eo; eo += S.net[cls];
    }
    S.net_total = eo;
    if (S.net_total > SP_MAX_ITEMS) return S;
    S.kd_sp = static_cast<long long>(S.net_total) * L.cout64;
    // one launch over the source grid replaces the full-resolution gradient of the upsampled part AND its 2x2 reduction pass; it
    // is used wherever the source grid has at least a third of a wave of tiles -- low-resolution layers keep the regular kernel
    // (their launches are latency-bound either way)
    const long long m_src = static_cast<long long>(c->n) * (c->h / 2) * (c->w / 2);
    S.ok = (m_src + BLOCK_M - 1) / BLOCK_M >= sms / 3;
    S.sp_dg_elems = static_cast<long long>(rup(S.kext_u, 128)) * S.kd_sp;
    S.block_n = std::min(pick_bn(S.kext_u, m_src, true, sms), 64);
    return S;
}

struct SpWParams {
    int cout, taps, cin, kw, cout64, choff_u;
    int eoff[4], nex[4];                         // per class: the prefix of its effective taps, its effective columns
    int ybits[2][4], xbits[2][4];
    long long kd_sp;
};

// transposed effective-tap weights: one block per (input channel of the upsampled part, effective tap of a class), threads over
// cout -> coalesced writes of the transposed matrix (the master reads are strided but L2-resident)
__global__ void sp_weight_dg_kernel(const float *__restrict__ wm, const SpWParams W, bf16 *__restrict__ w_d) {
    const int ci = blockIdx.x;
    int slot = blockIdx.y, cls = 0;
    while (cls < 3 && slot >= W.eoff[cls + 1]) ++cls;
    slot -= W.eoff[cls];
    const int ey = slot / W.nex[cls], ex = slot - ey * W.nex[cls];
    const int yb = W.ybits[cls >> 1][ey], xb = W.xbits[cls & 1][ex];
    for (int co = threadIdx.x; co < W.cout; co += blockDim.x) {
        const float *wrow = wm + static_cast<long long>(co) * W.taps * W.cin + W.choff_u + ci;
        float v = 0.f;
        for (int tr = 0; tr < 4; ++tr)
            if ((yb >> tr) & 1)
                for (int tc = 0; tc < 4; ++tc)
                    if ((xb >> tc) & 1) v += wrow[static_cast<long long>(tr * W.kw + tc) * W.cin];
        w_d[static_cast<long long>(ci) * W.kd_sp + static_cast<long long>(W.eoff[cls] + slot) * W.cout64 + co] = __float2bfloat16_rn(v);
    }
}

int sp_weight_prepare(const pcb_conv *c, const SpPlan &S, const Layout &L, const float *w_master, bf16 *w_d, cudaStream_t st) {
    SpWParams W;
    memset(&W, 0, sizeof(W));
    W.cout = c->cout; W.taps = c->kh * c->kw; W.cin = c->cin; W.kw = c->kw; W.cout64 = L.cout64; W.kd_sp = S.kd_sp;
    for (int p = 0; p < S.pu; ++p) W.choff_u += c->parts[p].c;
    for (int cls = 0; cls < 4; ++cls) { W.eoff[cls] = S.eoff[cls]; W.nex[cls] = S.ax.ne[cls & 1]; }
    for (int q = 0; q < 2; ++q)
        for (int e = 0; e < 4; ++e) { W.ybits[q][e] = S.ay.tapbits[q][e]; W.xbits[q][e] = S.ax.tapbits[q][e]; }
    sp_weight_dg_kernel<<<dim3(c->parts[S.pu].c, S.net_total), 128, 0, st>>>(w_master, W, w_d);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <int BLOCK_N>
int launch_sp_n(TcParams &P, const SpTable &TB, const CUtensorMap &tw, const CUtensorMap &ta, cudaStream_t st) {
    const size_t stage = A_STAGE_BYTES + static_cast<size_t>(BLOCK_N) * 128;
    const size_t fixed = tma_fixed_smem(BLOCK_N);
    P.stages = static_cast<int>(std::min<size_t>(MAX_RING, (MAX_SMEM - fixed) / stage));
    PCB_CHECK(P.stages >= 2, "sub-pixel conv: stage of %zu bytes does not fit twice", stage);
    const size_t smem = fixed + P.stages * stage;
    auto kern = pconv_tc_sp_kernel<BLOCK_N>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    const int num_tiles = ((P.m_total + BLOCK_M - 1) / BLOCK_M) * (P.ncols / BLOCK_N);
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, TMA_THREADS, smem, st>>>(P, TB, tw, ta);
    PCB_LAUNCH_CHECK();
    return 0;
}

// data gradient w.r.t. the upsampled part, written directly at SOURCE resolution: dx_u[k][j] = mask_u[k][j] * sum over classes and
// effective taps of dc[2(k - ey) + py][2(j - ex) + px] . Weff^T
int sp_dgrad_up(const pcb_conv *c, const SpPlan &S, const Layout &L, const void *dc, int dc_cstride, const bf16 *w_sp_dg, void *dx_u, int dx_cstride,
                int *flag, cudaStream_t st) {
    const int hs = c->h / 2, ws = c->w / 2;
    const long long m_src = static_cast<long long>(c->n) * hs * ws;
    TcParams P;
    base_params(P, c, L);
    P.h = hs; P.w = ws; P.m_total = static_cast<int>(m_src);
    P.sub = 1; P.py = 0; P.px = 0; P.fh = hs; P.fw = ws;
    P.nparts = 1;
    memset(P.parts, 0, sizeof(P.parts));
    TcPart &pt = P.parts[0];
    pt.c = c->parts[S.pu].c; pt.c8 = S.c8_u; pt.kext = S.kext_u; pt.koff = 0; pt.mask = c->parts[S.pu].mask; pt.mup = 0;
    pt.dx = static_cast<bf16 *>(dx_u); pt.dx_cstride = dx_cstride;
    PCB_CHECK(dx_cstride % 8 == 0 && dx_cstride >= S.c8_u && (reinterpret_cast<uintptr_t>(dx_u) & 15) == 0, "sub-pixel dgrad: dx must be 16-byte aligned with a channel stride that is a multiple of 8");
    P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.dc_c8 = rup(c->cout, 8); P.dc_kext = L.cout64;
    P.abort_flag = flag;
    P.ncols = S.kext_u;
    P.box_w = S.bw; P.box_h = S.bh; P.box_n = S.bn;
    const int bn = S.block_n;
    SpTable TB;
    memset(&TB, 0, sizeof(TB));
    int ni = 0;
    for (int cls = 0; cls < 4; ++cls) {
        const int py = cls >> 1, px = cls & 1;
        const int ney = S.ay.ne[py], nex = S.ax.ne[px];
        for (int e = 0; e < ney; ++e)
            for (int f = 0; f < nex; ++f) {
                SpItem &it = TB.it[ni++];
                it.dx = px - 2 * (S.ax.e0[px] + f); it.dy = py - 2 * (S.ay.e0[py] + e);
                it.wk = (S.eoff[cls] + e * nex + f) * L.cout64;
            }
    }
    TB.n_items = ni;
    CUtensorMap ta, tw;
    if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, S.bw, S.bh, S.bn, 2)) return rc;
    if (int rc = make_tmap_2d(&tw, w_sp_dg, rup(S.kext_u, 128), S.kd_sp, S.kd_sp, bn)) return rc;
    return (bn == 64) ? launch_sp_n<64>(P, TB, tw, ta, st) : launch_sp_n<32>(P, TB, tw, ta, st);
}

// ---- the plan ---------------------------------------------------------------------------------------------------------------
// Every choice the tensor-core path makes for one problem, taken once from the descriptor and the SM count: the kernel of each
// direction and its tiles, where the extra operands sit in the weight buffers, and the layout of the workspace.  Every pcb_tc_*
// entry point works from this plan, so the mask pass, the workspace and the weight layout agree with the kernels that use them.
enum TcRoute { ROUTE_NONE, ROUTE_STEM, ROUTE_K2R, ROUTE_SMALLCO, ROUTE_TMA, ROUTE_TMA_S2, ROUTE_GATHER };

struct DirPlan {
    TcRoute route;
    int box_w, box_h, box_n;           // M tile box of the TMA-fed kernels
    int bn;                            // N tile width
    bool halo;                         // TMA-fed row-halo tiles
};

struct TcPlan {
    bool ok;                           // the tensor-core path takes the problem
    Layout L;
    long long m_out, m_in;             // output / input pixels
    size_t fwd_elems, dg_elems;        // operand buffer sizes (bf16 elements)
    size_t extra_fwd_off, extra_dg_off;  // the operands of the stem's / the tail's sub-problem follow the layer's own
    size_t sp_off;                     // the sub-pixel matrices follow the regular data-gradient operand
    size_t workspace;                  // tap-validity words first, then the dense copies of the 2x-upsampled parts
    size_t up_off[TC_MAX_PARTS];       // workspace offset of each 2x-upsampled part's copy
    DirPlan fwd, dg, wg;
    bool fwd_tapmask, wg_tapmask;      // the forward / weight-gradient kernel reads tap-validity words from the workspace
    StemPlan stem;                     // ROUTE_STEM: the 4x4 problem over the space-to-depth image (conv_stem.cu)
    K2rPlan k2r;                       // ROUTE_K2R: the 1x1 problem at source resolution (conv_k2r.cu)
    SpPlan sp;                         // the data gradient of the 2x-upsampled part at source resolution (sp.ok)
    bool cls_halo[4];                  // ROUTE_TMA_S2: row-halo tiles per parity class (py * 2 + px)
    bool cls_fork;                     // ROUTE_TMA_S2: one class does not fill the GPU, the four run concurrently
    bool fuses_epilogue;               // the forward accumulates the BatchNorm statistics / applies the eval-mode epilogue
    bool dg_fuses_relu;                // the data gradient applies the ReLU backward of the layer's input
    bool dg_at_source;                 // see pcb_conv_dgrad_at_source_resolution
};

TcPlan tc_plan(const pcb_conv *c) {
    TcPlan T;
    memset(&T, 0, sizeof(T));
    T.sp.pu = T.sp.ps = -1;
    if (!common_ok(c)) return T;
    T.ok = true;
    const int sms = pcb_num_sms();
    T.L = layout_of(c);
    const Layout &L = T.L;
    T.m_out = static_cast<long long>(c->n) * c->ho * c->wo;
    T.m_in = static_cast<long long>(c->n) * c->h * c->w;
    bool any_mask = false;
    for (int p = 0; p < c->nparts; ++p) any_mask = any_mask || (c->parts[p].mask != nullptr);
    const bool smallco = !L.rowpack && pcb_smallco_eligible(c);
    if (L.rowpack) T.stem = pcb_stem_plan(c);
    if (smallco) T.k2r = pcb_k2r_plan(c);
    const bool stem = T.stem.ok, k2r = T.k2r.ok;
    if (!L.rowpack && !smallco) T.sp = sp_plan(c, L, sms);

    T.fwd_elems = static_cast<size_t>(L.rows_f) * L.kf;
    T.sp_off = static_cast<size_t>(rup(L.ktap, 128)) * L.kd;
    T.dg_elems = L.rowpack ? 0 : T.sp_off;
    if (T.sp.ok) T.dg_elems += static_cast<size_t>(T.sp.sp_dg_elems);
    T.extra_fwd_off = (T.fwd_elems + 63) / 64 * 64;
    T.extra_dg_off = (T.sp_off + 63) / 64 * 64;
    if (k2r) {
        T.fwd_elems = T.extra_fwd_off + T.k2r.fwd_extra;
        T.dg_elems = T.extra_dg_off + T.k2r.dg_extra;
    }
    if (stem) T.fwd_elems = T.extra_fwd_off + T.stem.fwd_extra;

    int bw, bh, bn;
    const bool fwd_tma = tma_fwd_ok(c, &bw, &bh, &bn);
    DirPlan &F = T.fwd;
    if (stem) F.route = ROUTE_STEM;                      // (the stem applies its mask in the space-to-depth pass)
    else if (k2r) F.route = ROUTE_K2R;
    else if (smallco) F.route = ROUTE_SMALLCO;
    else if (fwd_tma) {
        F.route = ROUTE_TMA;
        F.box_w = bw; F.box_h = bh; F.box_n = bn;
        F.bn = pick_bn(c->cout <= 32 ? 32 : L.rows_f, T.m_out, true, sms);
        F.halo = c->stride == 1 && c->kh <= 8 && halo_ok(c->kw, c->dil, bw, bh, bn, F.bn);
        // without holes TMA's out-of-range zero fill is all the validity there is; row-halo tiles read the mask planes themselves
        T.fwd_tapmask = any_mask && !F.halo;
    } else {
        F.route = ROUTE_GATHER;
        F.bn = L.bn_f;
        T.fwd_tapmask = true;
    }

    DirPlan &D = T.dg;
    if (k2r) D.route = ROUTE_K2R;
    else if (smallco) D.route = ROUTE_SMALLCO;
    else if (L.rowpack) D.route = ROUTE_NONE;            // row-packed layers take their data gradient on the generic kernels
    else if (c->stride == 1 && tile_box(c->w, c->h, &bw, &bh, &bn)) {
        D.route = ROUTE_TMA;
        D.box_w = bw; D.box_h = bh; D.box_n = bn;
        D.bn = pick_bn(L.ktap, T.m_in, false, sms);
        D.halo = c->kh <= 8 && halo_ok(c->kw, c->dil, bw, bh, bn, D.bn);
    } else if (tma_dgrad_s2_ok(c, &bw, &bh, &bn)) {
        D.route = ROUTE_TMA_S2;
        D.box_w = bw; D.box_h = bh; D.box_n = bn;
        const long long m_class = static_cast<long long>(c->n) * (c->h / 2) * (c->w / 2);
        D.bn = pick_bn(L.ktap, m_class, false, sms);
        for (int cls = 0; cls < 4; ++cls) T.cls_halo[cls] = halo_ok(class_kw(c, cls & 1), 1, bw, bh, bn, D.bn);
        T.cls_fork = ((m_class + BLOCK_M - 1) / BLOCK_M) * (L.ktap / D.bn) < sms;
    } else {
        D.route = ROUTE_GATHER;
        D.bn = (L.ktap % 128 == 0) ? 128 : 64;
    }

    const bool wg_tma = tma_wgrad_ok(c, &bw, &bh, &bn);
    DirPlan &W = T.wg;
    if (stem) W.route = ROUTE_STEM;
    else if (k2r) W.route = ROUTE_K2R;
    else if (smallco) W.route = ROUTE_SMALLCO;
    else if (wg_tma) {
        W.route = ROUTE_TMA;
        W.box_w = bw; W.box_h = bh; W.box_n = bn;
        // row-halo tiles for kw == 3: the three taps of a kernel row are three 64 x 64 register accumulators per consumer thread
        W.halo = c->stride == 1 && c->kw == 3 && bw == 64 && bh == 1 && bn == 1 && 64 + (c->kw - 1) * c->dil <= 256;
        // 128 output channels per tile, except for layers with at most 64 and for short reductions (< 128 K blocks of 64
        // pixels): there each CTA has few K blocks and its red.global.add epilogue, twice as long at 128 columns, dominates
        W.bn = (c->cout > 64 && T.m_out >= 128 * 64) ? 128 : 64;
        T.wg_tapmask = any_mask;                         // without holes the TMA-fed kernel needs no validity words
    } else {
        W.route = ROUTE_GATHER;
        T.wg_tapmask = true;
    }

    if (k2r) T.workspace = T.k2r.workspace;
    else if (stem) T.workspace = std::max(T.stem.workspace, tapmask_bytes(c));
    else {
        T.workspace = tapmask_bytes(c);
        // dense copies of the 2x-upsampled sources for the TMA-fed kernels (TMA cannot replicate pixels), reserved wherever the
        // geometry allows them (small-Cout layers included)
        if (fwd_tma || wg_tma)
            for (int p = 0; p < c->nparts; ++p)
                if (c->parts[p].x_up) { T.up_off[p] = T.workspace; T.workspace += up_bytes(c, p); }
    }

    T.fuses_epilogue = !smallco;                         // the small-Cout / RGB-tail kernels have no such epilogue
    T.dg_fuses_relu = c->nparts == 1 && !T.sp.ok && D.route == ROUTE_TMA;
    T.dg_at_source = smallco ? k2r : T.sp.ok;
    return T;
}

// A-operand tensor maps of the TMA-fed forward and weight gradient, one per part (the second repeats a single part): a
// 2x-upsampled part is first copied densely into the workspace at the plan's offset.  *use_fix is set when a part has holes.
int a_operand_maps(const pcb_conv *c, const TcPlan &T, void *workspace, int bx, int by, int bn, CUtensorMap (&ta)[TC_MAX_PARTS],
                   int *use_fix, cudaStream_t st) {
    memset(ta, 0, sizeof(ta));
    for (int p = 0; p < c->nparts; ++p) {
        const pcb_part &pt = c->parts[p];
        const void *src = pt.x;
        long long cs = pt.x_cstride;
        const int c8 = rup(pt.c, 8);
        if (pt.x_up) {
            bf16 *up = reinterpret_cast<bf16 *>(static_cast<uint8_t *>(workspace) + T.up_off[p]);
            const long long pix = static_cast<long long>(c->n) * (c->h >> 1) * (c->w >> 1);
            const long long work = pix * (c8 >> 3);
            const int grid = static_cast<int>(std::min<long long>((work + 255) / 256, 16ll * pcb_num_sms()));
            upsample_part_kernel<<<grid, 256, 0, st>>>(static_cast<const bf16 *>(pt.x), pt.x_cstride, c8, pix, c->h >> 1, c->w >> 1, up);
            PCB_LAUNCH_CHECK();
            src = up; cs = c8;
        }
        if (pt.mask) *use_fix = 1;
        if (int rc = make_tmap_nhwc(&ta[p], src, c8, c->w, c->h, c->n, cs, bx, by, bn, c->stride)) return rc;
    }
    if (c->nparts < 2) ta[1] = ta[0];
    return 0;
}

pcb_smallco_layout smallco_layout(const Layout &L) {
    pcb_smallco_layout S;
    S.ktap = L.ktap; S.koff[0] = L.koff[0]; S.koff[1] = L.koff[1]; S.cout64 = L.cout64; S.kf = L.kf; S.kd = L.kd;
    return S;
}

}  // namespace

// ---- entry points --------------------------------------------------------------------------------------------------------
bool pcb_tc_eligible(const pcb_conv *c) { return common_ok(c); }

size_t pcb_tc_workspace(const pcb_conv *c) { return tc_plan(c).workspace; }

void pcb_tc_weight_layout(const pcb_conv *c, size_t *fwd_elems, size_t *dgrad_elems) {
    const TcPlan T = tc_plan(c);
    *fwd_elems = T.fwd_elems;
    *dgrad_elems = T.dg_elems;
}

// true when the data gradient of the 2x-upsampled part is delivered at that part's own (source) resolution
bool pcb_tc_subpixel(const pcb_conv *c) { return tc_plan(c).dg_at_source; }

void pcb_tc_routes(const pcb_conv *c, int32_t routes[3]) {
    static const int32_t code[] = {PCB_ROUTE_NONE, PCB_ROUTE_STEM, PCB_ROUTE_K2R, PCB_ROUTE_SMALLCO, PCB_ROUTE_TMA, PCB_ROUTE_TMA_S2,
                                   PCB_ROUTE_GATHER};
    const TcPlan T = tc_plan(c);
    routes[0] = code[T.fwd.route]; routes[1] = code[T.dg.route]; routes[2] = code[T.wg.route];
}

int pcb_tc_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd, void *w_dgrad, bool zero_padding, cudaStream_t st) {
    const TcPlan T = tc_plan(c);
    const Layout &L = T.L;
    const size_t fe = T.fwd_elems, de = T.dg_elems;
    if (zero_padding) {                                  // a refresh of buffers filled before leaves the (never written) padding alone
        PCB_CUDA(cudaMemsetAsync(w_fwd, 0, fe * 2, st));
        if (w_dgrad && de) PCB_CUDA(cudaMemsetAsync(w_dgrad, 0, de * 2, st));
    }
    WPrepParams W;
    memset(&W, 0, sizeof(W));
    W.cout = c->cout; W.taps = c->kh * c->kw; W.cin = c->cin; W.kw = c->kw; W.rowpack = L.rowpack; W.nparts = c->nparts;
    W.ktap = L.ktap; W.cout64 = L.cout64; W.kf = L.kf; W.kd = L.kd;
    int off = 0;
    for (int p = 0; p < c->nparts; ++p) { W.choff[p] = off; W.c[p] = c->parts[p].c; W.koff[p] = L.koff[p]; off += c->parts[p].c; }
    bf16 *wf = static_cast<bf16 *>(w_fwd), *wd = static_cast<bf16 *>(w_dgrad);
    if (!L.rowpack && W.taps <= 65535 && c->cout >= 32 && c->cin >= 32) {
        dim3 tg((c->cin + 31) / 32, (c->cout + 31) / 32, W.taps);
        tc_weight_prepare_tiled_kernel<<<tg, 256, 0, st>>>(w_master, W, wf, (w_dgrad && de) ? wd : nullptr);
    } else {
        const long long total = static_cast<long long>(c->cout) * W.taps * c->cin;
        const int grid = static_cast<int>(std::min<long long>((total + 1023) / 1024, 8ll * pcb_num_sms()));
        tc_weight_prepare_kernel<<<grid < 1 ? 1 : grid, 256, 0, st>>>(w_master, W, wf, (w_dgrad && de) ? wd : nullptr);
    }
    PCB_LAUNCH_CHECK();
    if (T.fwd.route == ROUTE_STEM) return pcb_stem_weight_prepare(c, T.stem, w_master, wf + T.extra_fwd_off, zero_padding, st);
    if (T.fwd.route == ROUTE_K2R) {
        PCB_CHECK(w_dgrad != nullptr, "kernel-to-row weights need the dgrad operand buffer");
        return pcb_k2r_weight_prepare(c, T.k2r, w_master, wf + T.extra_fwd_off, wd + T.extra_dg_off, zero_padding, st);
    }
    if (T.sp.ok) {
        PCB_CHECK(w_dgrad != nullptr, "sub-pixel weights need the dgrad operand buffer");
        return sp_weight_prepare(c, T.sp, L, w_master, wd + T.sp_off, st);
    }
    return 0;
}

// the part of the forward that only depends on the masks: tap-validity words for the kernels that want them
int pcb_tc_forward_mask_pass(const pcb_conv *c, uint64_t *tapmask, cudaStream_t st) {
    const TcPlan T = tc_plan(c);
    PCB_CHECK(T.m_out < (1ll << 31), "problem too large");
    return T.fwd_tapmask ? launch_tapmask(c, tapmask, st) : 0;
}

// true when pcb_tc_forward_ws can accumulate the BatchNorm statistics of its output / apply an eval-mode BatchNorm + activation
// in its epilogue
bool pcb_tc_fuses_epilogue(const pcb_conv *c) { return tc_plan(c).fuses_epilogue; }

int pcb_tc_forward_ws(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, const float *msum,
                      uint64_t *tapmask, bool mask_pass_done, double *bn_sums, const pcb_ep *ep, cudaStream_t st) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    const TcPlan T = tc_plan(c);
    const Layout &L = T.L;
    const DirPlan &F = T.fwd;
    PCB_CHECK(T.m_out < (1ll << 31), "problem too large");
    PCB_CHECK(y_cstride % 8 == 0 && y_cstride >= c->cout, "tensor-core forward: y channel stride must be a multiple of 8 and >= cout");
    PCB_CHECK(bn_sums == nullptr || T.fuses_epilogue, "fused BatchNorm statistics requested from a kernel that does not produce them");
    PCB_CHECK(ep == nullptr || T.fuses_epilogue, "fused BatchNorm + activation requested from a kernel that does not apply it");
    if (!mask_pass_done && T.fwd_tapmask)
        if (int rc = launch_tapmask(c, tapmask, st)) return rc;
    const bf16 *wf = static_cast<const bf16 *>(w_fwd);
    if (F.route == ROUTE_STEM) return pcb_stem_forward(c, T.stem, wf + T.extra_fwd_off, bias, y, y_cstride, msum, tapmask, bn_sums, ep, st);
    if (F.route == ROUTE_K2R) return pcb_k2r_forward(c, T.k2r, smallco_layout(L), w_fwd, wf + T.extra_fwd_off, bias, y, y_cstride, msum, tapmask, st);
    if (F.route == ROUTE_SMALLCO) return pcb_smallco_forward(c, smallco_layout(L), w_fwd, bias, y, y_cstride, msum, st);
    TcParams P;
    base_params(P, c, L);
    P.m_total = static_cast<int>(T.m_out);
    fill_parts(c, L, P.parts, tapmask, T.m_out);
    P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride; P.abort_flag = flag;
    P.bn_sums = bn_sums; P.bn_c = c->cout;
    set_ep(P, ep);
    P.ncols = L.rows_f;
    CUtensorMap tm;
    if (int rc = make_tmap_2d(&tm, w_fwd, L.rows_f, L.kf, L.kf, F.bn)) return rc;
    if (F.route == ROUTE_TMA) {
        P.box_w = F.box_w; P.box_h = F.box_h; P.box_n = F.box_n;
        CUtensorMap ta[TC_MAX_PARTS];
        if (int rc = a_operand_maps(c, T, tapmask, F.box_w + (F.halo ? (c->kw - 1) * c->dil : 0), F.box_h, F.box_n, ta, &P.use_fix, st)) return rc;
        P.ncols = (c->cout <= 32) ? 32 : L.rows_f;
        P.wk_base = 0; P.wk_col = L.ktap; P.wk_row = c->kw * L.ktap;
        return launch_tma<0>(P, tm, ta[0], ta[1], F.bn, F.halo, st);
    }
    return launch_tc<0>(P, tm, F.bn, st);
}

// the data-gradient problems whose kernel can apply the ReLU backward of the layer's input in its epilogue: the TMA-fed
// stride-1 kernel on a single-part layer (not the small-Cout, sub-pixel or gather kernels)
bool pcb_tc_dgrad_fuses_relu(const pcb_conv *c) { return tc_plan(c).dg_fuses_relu; }

int pcb_tc_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_dgrad, void *const *dx, const int *dx_cstride,
                 cudaStream_t st, const void *relu_x, int relu_cstride) {
    const TcPlan T = tc_plan(c);
    const Layout &L = T.L;
    const DirPlan &D = T.dg;
    PCB_CHECK(D.route != ROUTE_NONE, "data gradient of a row-packed (cin <= 8) tensor-core layer: set force_generic and pass KRSC weights");
    PCB_CHECK(w_dgrad != nullptr && (reinterpret_cast<uintptr_t>(dc) & 15) == 0, "pcb_pconv_backward_data: w_dgrad required / dc misaligned");
    PCB_CHECK(relu_x == nullptr || (T.dg_fuses_relu && relu_cstride % 8 == 0 && relu_cstride >= rup(c->cin, 8) &&
                                    (reinterpret_cast<uintptr_t>(relu_x) & 15) == 0),
              "tensor-core dgrad: the ReLU backward is fused only on the TMA-fed stride-1 kernel (16-byte aligned input, channel stride %% 8 == 0)");
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    PCB_CHECK(T.m_in < (1ll << 31), "problem too large");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= rup(c->cout, 8), "tensor-core dgrad: dc channel stride must be a multiple of 8");
    const bf16 *wd = static_cast<const bf16 *>(w_dgrad);
    if (D.route == ROUTE_K2R) return pcb_k2r_dgrad(c, T.k2r, smallco_layout(L), dc, dc_cstride, w_dgrad, wd + T.extra_dg_off, dx, dx_cstride, st);
    if (D.route == ROUTE_SMALLCO) return pcb_smallco_dgrad(c, smallco_layout(L), dc, dc_cstride, w_dgrad, dx, dx_cstride, st);
    // sub-pixel path: the gradient of the upsampled part is computed directly at source resolution (dx[pu] is a SOURCE-resolution
    // buffer, see pcb_conv_dgrad_at_source_resolution); the other part goes through the regular kernel below
    const SpPlan &SPL = T.sp;
    void *dx_local[TC_MAX_PARTS] = {nullptr, nullptr};
    for (int p = 0; p < c->nparts && p < TC_MAX_PARTS; ++p) dx_local[p] = dx[p];
    if (SPL.ok) {
        if (dx[SPL.pu] != nullptr)
            if (int rc = sp_dgrad_up(c, SPL, L, dc, dc_cstride, wd + T.sp_off, dx[SPL.pu], dx_cstride[SPL.pu], flag, st)) return rc;
        dx_local[SPL.pu] = nullptr;
        if (SPL.ps < 0 || dx[SPL.ps] == nullptr) return 0;
    }
    dx = dx_local;
    TcParams P;
    base_params(P, c, L);
    P.m_total = static_cast<int>(T.m_in);
    fill_parts(c, L, P.parts, nullptr, 0);
    for (int p = 0; p < c->nparts; ++p) {
        P.parts[p].dx = static_cast<bf16 *>(dx[p]);
        P.parts[p].dx_cstride = dx_cstride[p];
        PCB_CHECK(!dx[p] || (dx_cstride[p] % 8 == 0 && dx_cstride[p] >= P.parts[p].c8 && (reinterpret_cast<uintptr_t>(dx[p]) & 15) == 0),
                  "tensor-core dgrad: dx[%d] must be 16-byte aligned with a channel stride that is a multiple of 8", p);
    }
    P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.dc_c8 = rup(c->cout, 8); P.dc_kext = L.cout64;
    P.relu_x = static_cast<const bf16 *>(relu_x); P.relu_cstride = relu_cstride;
    P.abort_flag = flag;
    P.ncols = L.ktap;
    CUtensorMap tm;
    if (int rc = make_tmap_2d(&tm, w_dgrad, rup(L.ktap, 128), L.kd, L.kd, D.bn)) return rc;
    if (D.route == ROUTE_TMA) {
        P.box_w = D.box_w; P.box_h = D.box_h; P.box_n = D.box_n;
        P.wk_base = 0; P.wk_col = L.cout64; P.wk_row = c->kw * L.cout64;
        CUtensorMap ta;
        if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, D.box_w + (D.halo ? (c->kw - 1) * c->dil : 0), D.box_h, D.box_n, 1)) return rc;
        return launch_tma<1>(P, tm, ta, ta, D.bn, D.halo, st);
    }
    if (D.route == ROUTE_TMA_S2) {
        // Stride 2: an input pixel (y, x) only sees the taps with (y + pad - tr) even, so the four parity classes
        // (y & 1, x & 1) are four independent STRIDE-1 problems on the half-resolution grid -- which is dc's own grid --
        // each with its subset of taps (3x3 / 3x2 / 2x3 / 2x2 for a 5x5 kernel) and no multiplications by inserted zeros.
        const int hh = c->h / 2, hw = c->w / 2;
        P.box_w = D.box_w; P.box_h = D.box_h; P.box_n = D.box_n;
        // The classes write disjoint pixels.  When one class does not fill the GPU (low-resolution layers) the four launches
        // run concurrently: fork onto three internal streams after an event on `st`, join before returning (also valid
        // inside a stream capture: the internal streams join the capture and leave it again).
        const bool fork = T.cls_fork;
        ClassStreams *CS = nullptr;
        if (fork) {
            if (int rc = class_streams(&CS)) return rc;
            PCB_CUDA(cudaEventRecord(CS->ev_fork, st));
        }
        for (int cls = 0; cls < 4; ++cls) {
            TcParams Q = P;
            const int py = cls >> 1, px = cls & 1;
            const int tr0 = (py + c->pad_h) & 1, tc0 = (px + c->pad_w) & 1;
            Q.kh = (c->kh - tr0 + 1) / 2; Q.kw = class_kw(c, px);
            Q.pad_h = (py + c->pad_h - tr0) / 2; Q.pad_w = (px + c->pad_w - tc0) / 2;
            Q.h = hh; Q.w = hw; Q.stride = 1; Q.dil = 1;
            Q.m_total = static_cast<int>(static_cast<long long>(c->n) * hh * hw);
            Q.sub = 2; Q.py = py; Q.px = px; Q.fh = c->h; Q.fw = c->w;
            Q.wk_base = (tr0 * c->kw + tc0) * L.cout64; Q.wk_row = 2 * c->kw * L.cout64; Q.wk_col = 2 * L.cout64;
            const bool halo = T.cls_halo[cls];
            CUtensorMap ta;
            if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, Q.box_w + (halo ? Q.kw - 1 : 0), Q.box_h, Q.box_n, 1)) return rc;
            cudaStream_t cs = (fork && cls > 0) ? CS->aux[cls - 1] : st;
            if (fork && cls > 0) PCB_CUDA(cudaStreamWaitEvent(cs, CS->ev_fork, 0));
            if (int rc = launch_tma<1>(Q, tm, ta, ta, D.bn, halo, cs)) return rc;
            if (fork && cls > 0) {
                PCB_CUDA(cudaEventRecord(CS->ev_join[cls - 1], cs));
                PCB_CUDA(cudaStreamWaitEvent(st, CS->ev_join[cls - 1], 0));
            }
        }
        return 0;
    }
    return launch_tc<1>(P, tm, D.bn, st);
}


// ---- TMA-fed weight gradient ---------------------------------------------------------------------
template <int BLOCK_N, int T, bool HALO>
int launch_wgrad_tma(WgParams &P, const CUtensorMap &tdc, const CUtensorMap &ta0, const CUtensorMap &ta1, cudaStream_t st) {
    const int rows_a = 64 + (HALO ? (P.kw - 1) * P.dil : 0);
    PCB_CHECK(rows_a <= (HALO ? 3 : 1) * WGRAD_FIX_THREADS, "TMA-fed wgrad: %d-row A blocks exceed the fixer warps", rows_a);
    const size_t a_blk = (static_cast<size_t>(rows_a) * 128 + 1023) / 1024 * 1024;
    const size_t stage = (HALO ? 1 : T) * 2 * a_blk + static_cast<size_t>(BLOCK_N) * 128;
    P.stages = static_cast<int>(std::min<size_t>(MAX_RING, RING_BUDGET / stage));
    PCB_CHECK(P.stages >= 2, "TMA-fed wgrad: stage of %zu bytes does not fit twice", stage);
    const size_t smem = 1024 + P.stages * stage + 24 * MAX_RING;
    auto kern = pconv_tc_wgrad_tma_kernel<BLOCK_N, T, HALO>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    P.tap_groups = HALO ? P.kh : (P.kh * P.kw + T - 1) / T;
    P.ci_tiles = (P.ktap + 127) / 128;
    const int co_tiles = (P.cout + BLOCK_N - 1) / BLOCK_N;
    const int base_ctas = co_tiles * P.tap_groups * P.ci_tiles;
    const int total_kb = (P.m_total + 63) / 64;
    // one CTA per SM at a time: ~2 waves (measured faster than one wave for the large layers at 128-wide tiles)
    int splits = (2 * pcb_num_sms() + base_ctas - 1) / base_ctas;
    splits = std::max(1, std::min(splits, total_kb));
    splits = std::min(splits, 65535);
    P.kb_per_split = (total_kb + splits - 1) / splits;
    splits = (total_kb + P.kb_per_split - 1) / P.kb_per_split;
    dim3 grid(base_ctas, splits);
    kern<<<grid, WGRAD_TMA_THREADS, smem, st>>>(P, tdc, ta0, ta1);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <int BLOCK_N, int T, int STAGES>
static int launch_wgrad(WgParams &P, const CUtensorMap &tm, int cout, cudaStream_t st) {
    constexpr size_t smem = 1024 + STAGES * (T * 16384 + BLOCK_N * 128) + 24 * STAGES;
    auto kern = pconv_tc_wgrad_kernel<BLOCK_N, T, STAGES>;
    PCB_SMEM_OPT_IN(kern, (int)smem);
    P.tap_groups = (P.ntaps + T - 1) / T;
    P.ci_tiles = (P.ktap + 127) / 128;
    const int co_tiles = (cout + BLOCK_N - 1) / BLOCK_N;
    const int base_ctas = co_tiles * P.tap_groups * P.ci_tiles;
    const int total_kb = (P.m_total + 63) / 64;
    int splits = (4 * pcb_num_sms() + base_ctas - 1) / base_ctas;      // aim at ~4 CTAs per SM worth of work
    splits = std::max(1, std::min(splits, total_kb));
    splits = std::min(splits, 65535);
    P.kb_per_split = (total_kb + splits - 1) / splits;
    splits = (total_kb + P.kb_per_split - 1) / P.kb_per_split;
    dim3 grid(base_ctas, splits);
    kern<<<grid, WGRAD_THREADS, smem, st>>>(P, tm);
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_tc_wgrad(const pcb_conv *c, const void *dc, int dc_cstride, float *dw, void *workspace, bool zero_dw, cudaStream_t st) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    PCB_CHECK(workspace != nullptr, "pcb_tc_wgrad: workspace required");
    const TcPlan T = tc_plan(c);
    const Layout &L = T.L;
    const DirPlan &W = T.wg;
    PCB_CHECK(T.m_out < (1ll << 31), "problem too large");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= c->cout, "tensor-core wgrad: dc channel stride must be a multiple of 8");
    if (W.route == ROUTE_STEM) return pcb_stem_wgrad(c, T.stem, dc, dc_cstride, dw, workspace, zero_dw, st);
    if (W.route == ROUTE_K2R) return pcb_k2r_wgrad(c, T.k2r, dc, dc_cstride, dw, workspace, zero_dw, st);
    if (W.route == ROUTE_SMALLCO) return pcb_smallco_wgrad(c, smallco_layout(L), dc, dc_cstride, dw, zero_dw, st);
    uint64_t *tapmask = static_cast<uint64_t *>(workspace);
    if (T.wg_tapmask)
        if (int rc = launch_tapmask(c, tapmask, st)) return rc;
    const size_t dw_bytes = sizeof(float) * c->cout * c->kh * c->kw * c->cin;
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, dw_bytes, st));
    WgParams P;
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.cin = c->cin; P.cout = c->cout; P.kh = c->kh; P.kw = c->kw; P.stride = c->stride;
    P.pad_h = c->pad_h; P.pad_w = c->pad_w; P.dil = c->dil; P.ho = c->ho; P.wo = c->wo; P.m_total = static_cast<int>(T.m_out);
    P.nparts = c->nparts; P.rowpack = L.rowpack; P.ktap = L.ktap; P.ntaps = L.rowpack ? c->kh : c->kh * c->kw;
    fill_parts(c, L, P.parts, tapmask, T.m_out);
    P.dw = dw; P.abort_flag = flag;
    CUtensorMap tm;
    if (int rc = make_tmap_2d(&tm, dc, T.m_out, c->cout, dc_cstride, 64)) return rc;
    if (W.route == ROUTE_TMA) {
        P.box_w = W.box_w; P.box_h = W.box_h; P.box_n = W.box_n;
        CUtensorMap ta[TC_MAX_PARTS];
        if (int rc = a_operand_maps(c, T, workspace, W.box_w + (W.halo ? (c->kw - 1) * c->dil : 0), W.box_h, W.box_n, ta, &P.use_fix, st)) return rc;
        if (W.bn == 128) return W.halo ? launch_wgrad_tma<128, 3, true>(P, tm, ta[0], ta[1], st) : launch_wgrad_tma<128, 3, false>(P, tm, ta[0], ta[1], st);
        return W.halo ? launch_wgrad_tma<64, 3, true>(P, tm, ta[0], ta[1], st) : launch_wgrad_tma<64, 3, false>(P, tm, ta[0], ta[1], st);
    }
    return launch_wgrad<64, 3, 3>(P, tm, c->cout, st);
}

int *pcb_tc_abort_flag() { return abort_flag_ptr(); }

// abort flag query used by api.cu after synchronising debug runs
int pcb_tc_read_abort_flag(int *value) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "no abort flag");
    PCB_CUDA(cudaMemcpy(value, flag, sizeof(int), cudaMemcpyDeviceToHost));
    if (*value != 0) cudaMemset(flag, 0, sizeof(int));
    return 0;
}

// pcb_tc_epi.cuh -- what the tensor-core convolution kernels share: the kernel parameter block, the tile constants and the
// forward / data-gradient epilogue of the TMA-fed kernels (consumer-side element math into a bf16 staging tile, dedicated
// epilogue warps that store it and accumulate the BatchNorm statistics).  Used by conv_tc.cu and by the space-to-depth stem
// kernels of conv_stem.cu, so both apply the same epilogue arithmetic.
#pragma once
#include <cuda.h>

#include "pcb_common.cuh"
#include "pcb_ptx.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                 // bf16 elements = 128 bytes = one swizzle row
constexpr int A_STAGE_BYTES = BLOCK_M * 128;
constexpr int NUM_PRODUCER_THREADS = 128;
constexpr int TC_MAX_PARTS = 2;             // U-Net inputs are cat([upsampled, skip]) at most
// Every tensor-core kernel computes its 128-row tile with TWO consumer warpgroups: warpgroup g issues the m64 wgmmas of rows
// [64 g, 64 g + 64) into register accumulators and then stages them for the epilogue (run by the same warps in the cp.async-gather
// kernel, by dedicated epilogue warps in the TMA-fed kernels).  wgmma reads shared memory through
// the async proxy, so data written by cp.async / st.shared is made visible to it with fence.proxy.async after the consumer
// acquired the stage's mbarrier.
constexpr int MMA_WARPS = 8;
constexpr int MMA_THREADS = MMA_WARPS * 32;
// fp32 staging tile of the forward / dgrad epilogue: [128 rows][BLOCK_N + 4] (the pad spreads the rows over the banks)
constexpr int acc_pitch(int block_n) { return block_n + 4; }
constexpr int acc_stage_bytes(int block_n) { return BLOCK_M * acc_pitch(block_n) * 4; }

inline int rup(int v, int m) { return (v + m - 1) / m * m; }

struct TcPart {
    const bf16 *x;            // first channel of the part (fwd / wgrad gather source)
    const uint64_t *tapmask;  // [m_total] bit t = tap t is in-bounds and not a hole (fwd / wgrad)
    const uint8_t *mask;      // input hole plane (dgrad epilogue), may be null
    bf16 *dx;                 // dgrad output of this part [n,h,w,dx_cstride] (null: not needed)
    int c, c8, kext, koff, choff, cstride, xup, mup, dx_cstride;
};

struct TcParams {
    int n, h, w, cin, cout, kh, kw, stride, pad_h, pad_w, dil, ho, wo;
    int m_total;              // GEMM M
    int nparts, no_guard, rowpack;
    int ncols;                // GEMM N extent covered by the grid (multiple of BLOCK_N)
    int ring_a, ring_b;       // smem ring depths (A items / weight tiles): 8-byte aligned, the gather kernel loads them as a pair
    int ktap;                 // K extent of one tap (sum of part kext); rowpack: 64 per kernel row
    TcPart parts[TC_MAX_PARTS];
    // fwd epilogue
    const float *bias; const float *msum; bf16 *y; int y_cstride;
    // dgrad gather source
    const bf16 *dc; int dc_cstride, dc_c8, dc_kext;
    // dgrad (TMA-fed kernel, one part): backward of the in-place ReLU that produced the layer's input -- the stored gradient is 0
    // where relu_x <= 0 (torch's threshold_backward).  null: off.
    const bf16 *relu_x; int relu_cstride;
    int *abort_flag;
    // TMA-fed kernel: the 128 pixels of an M tile form the box {box_w, box_h, box_n} of the (x, y, image) pixel grid
    int box_w, box_h, box_n, stages, use_fix;
    int wk_base, wk_row, wk_col;   // weight-matrix K index of tap (a, b) of this launch: wk_base + a*wk_row + b*wk_col (+ part / block offset)
    // dgrad output addressing: the tile grid (h, w above) is every `sub`-th pixel of the full-resolution [fh, fw] gradient,
    // starting at (py, px) -- sub = 2 for the parity classes of a stride-2 layer, 1 otherwise
    int sub, py, px, fh, fw;
    // fused BatchNorm statistics (forward, MODE 0): per-channel sum / sum of squares of the bf16-ROUNDED outputs are accumulated
    // into bn_sums[0][co] / bn_sums[1][co] (doubles, pre-zeroed by the caller, row pitch bn_c = cout) -- the separate statistics
    // pass over y (nn.BatchNorm2d in training mode, partial_convolution.py:193-197) disappears.  null: off.
    double *bn_sums;
    int bn_c;
    // fused eval-mode BatchNorm + activation (forward, MODE 0, inference): the stored value is
    // apply_act(v * ep_scale[co] + ep_shift[co]) with v = the renormalised output (0 at holes), rounded to bf16 once.
    // ep_scale == null: activation only (scale 1, shift 0).  ep_on == 0: off (the training path).
    const float *ep_scale, *ep_shift;
    int ep_on, ep_act;
    float ep_slope;
};

// fused BatchNorm statistics: private slices of [128 sums | 128 squares], one per epilogue warp -- eight in the cp.async-gather
// kernel (row quadrant x column half), four in the TMA-fed kernels (row quadrant, all BLOCK_N <= 128 columns)
constexpr int STAT_SLICE = 256;
constexpr int STAT_SMEM_BYTES = MMA_WARPS * STAT_SLICE * 4 + 16;
// TMA-fed kernels: four dedicated epilogue warps; warp w drains rows [32 w, 32 w + 32) of the staging tile.  Their statistics
// slices are [256 sums | 256 squares] (all BLOCK_N <= 256 columns).
constexpr int EPI_WARPS = 4;
constexpr int EPI_STAT_SLICE = 512;
constexpr int EPI_STAT_SQ = EPI_STAT_SLICE / 2;
constexpr int EPI_STAT_SMEM_BYTES = EPI_WARPS * EPI_STAT_SLICE * 4;
// TMA-fed kernels: the consumers finish the element math and stage bf16 [128 rows][BLOCK_N + 8] (a row is an odd number of
// 16-byte units, so the epilogue warps' one-row-per-lane 16-byte loads are conflict-free)
constexpr int bf16_pitch(int block_n) { return block_n + 8; }
constexpr int bf16_stage_bytes(int block_n) { return BLOCK_M * bf16_pitch(block_n) * 2; }

// 16 values per lane, 32 lanes: returns in lane l the sum over all lanes of v[l & 15].  The reduction tree is the one
// warp_transpose_sum builds for the same column (lanes paired across bit 4 first, then bits 3 .. 0), so the sums are bitwise
// equal to it; the first level keeps all 16 values (both partners hold the same sums).
__device__ __forceinline__ float warp_transpose_sum16(float (&v)[16], int lane) {
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], 16);
#pragma unroll
    for (int off = 8, n = 16; off >= 1; off >>= 1, n >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (i < (n >> 1)) {
                const float send = upper ? v[i] : v[i + (n >> 1)];
                const float keep = upper ? v[i + (n >> 1)] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
    }
    return v[0];
}

__device__ __forceinline__ uint32_t align1024(uint32_t a) { return (a + 1023u) & ~1023u; }

// What the epilogue of one row needs from global memory and the pixel arithmetic.  The dedicated epilogue warps fetch it
// before they wait for the tile's accumulators, so the load latency is hidden behind the MMAs.
struct EpiRow {
    long long mo;                 // pixel index in the full-resolution output (fwd) / gradient (dgrad)
    int m;
    bool rvalid, hole;
    float inv;                    // fwd: 1 / mask box sum
    float dscale[TC_MAX_PARTS];   // dgrad: input mask of part p at this pixel (1 / 0; 1 without a mask)
};

// renorm = false: leave inv / hole unset (the TMA-fed kernels' consumers apply the renormalisation themselves)
template <int MODE>
__device__ __forceinline__ EpiRow tc_epi_row(const TcParams &P, int m, bool renorm = true) {
    EpiRow er;
    er.m = m;
    er.rvalid = m < P.m_total;
    er.inv = 0.f;
    er.hole = false;
    er.mo = m;
    int en = 0, eh = 0, ew = 0;
    if (MODE == 1 && er.rvalid) {
        en = m / (P.h * P.w); const int rem = m - en * P.h * P.w; eh = rem / P.w; ew = rem - eh * P.w;
        eh = eh * P.sub + P.py; ew = ew * P.sub + P.px;
        er.mo = (static_cast<long long>(en) * P.fh + eh) * P.fw + ew;
    }
    if (MODE == 0 && er.rvalid && renorm) {
        const float s = P.msum ? P.msum[er.mo] : 1.f;               // null: plain convolution (renormaliser 1)
        er.hole = (s == 0.f) && !P.no_guard;
        er.inv = er.hole ? 0.f : 1.0f / s;        // no_guard: 1/0 = inf -> 0*inf = NaN like the reference
    }
#pragma unroll
    for (int p = 0; p < TC_MAX_PARTS; ++p) {
        er.dscale[p] = 1.f;
        if (MODE == 1 && p < P.nparts) {
            const TcPart &pt = P.parts[p];
            if (er.rvalid && pt.dx != nullptr && pt.mask != nullptr)      // dx = acc * input mask of this part
                er.dscale[p] = pt.mask[(static_cast<long long>(en) * (P.fh >> pt.mup) + (eh >> pt.mup)) * (P.fw >> pt.mup) + (ew >> pt.mup)] ? 1.f : 0.f;
        }
    }
    return er;
}

// flush one warp's per-column statistics of the N tile starting at n0 into the global fp64 sums, and clear them
template <int BLOCK_N>
__device__ __forceinline__ void tc_stats_flush(const TcParams &P, float *s_stat, int lane, int n0, int cb, int ce, int sq_off) {
    __syncwarp();
    for (int c0 = cb; c0 < ce; c0 += 32) {
        const int co = n0 + c0 + lane;
        if (co < P.bn_c) {
            atomicAdd(P.bn_sums + co, static_cast<double>(s_stat[c0 - cb + lane]));
            atomicAdd(P.bn_sums + P.bn_c + co, static_cast<double>(s_stat[sq_off + c0 - cb + lane]));
        }
        s_stat[c0 - cb + lane] = 0.f; s_stat[sq_off + c0 - cb + lane] = 0.f;
    }
    __syncwarp();
}

// TMA-fed kernels: last N tile's BatchNorm statistics.  The EPI_WARPS epilogue warps' partials (slice w = [sums of the tile's
// columns | squares at offset 128]) are summed after a CTA-wide barrier, so the global sums receive ONE atomic per channel per
// CTA.  `stat_base`: slice 0.
template <int BLOCK_N>
__device__ __forceinline__ void tc_stats_final(const TcParams &P, const float *stat_base, int w, int lane, int stat_n0) {
    for (int col = w * 32 + lane; col < BLOCK_N; col += EPI_WARPS * 32) {
        const int co = stat_n0 + col;
        if (co < P.bn_c) {
            float a = 0.f, q = 0.f;
#pragma unroll
            for (int w4 = 0; w4 < EPI_WARPS; ++w4) { a += stat_base[w4 * EPI_STAT_SLICE + col]; q += stat_base[w4 * EPI_STAT_SLICE + EPI_STAT_SQ + col]; }
            atomicAdd(P.bn_sums + co, static_cast<double>(a));
            atomicAdd(P.bn_sums + P.bn_c + co, static_cast<double>(q));
        }
    }
}

template <int R> __device__ __forceinline__ void zero_acc(float (&a)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) a[i] = 0.f;
}

constexpr int MAX_RING = 8;

constexpr int EPI_WARP0 = MMA_WARPS + 4;
constexpr int TMA_THREADS = (EPI_WARP0 + EPI_WARPS) * 32;
constexpr int TMA_FIX_THREADS = 96;
constexpr int TMA_REGS = 128;                                  // per thread at launch: setmaxnreg needs a fixed count
constexpr int TMA_CONSUMER_REGS = 192, TMA_SUPPORT_REGS = 64;
static_assert(TMA_THREADS == 512 && 2 * 128 * TMA_CONSUMER_REGS + 2 * 128 * TMA_SUPPORT_REGS == TMA_THREADS * TMA_REGS &&
              TMA_THREADS * TMA_REGS <= 65536, "TMA-fed fwd / dgrad register budget");

// shared memory behind the TMA-fed kernels' rings: full / fixed / empty barriers, acc_full / acc_empty, the statistics slices
constexpr size_t TMA_BAR_BYTES = 24 * MAX_RING + 16;

// bf16-staged epilogue of one row (TMA-fed kernels): the consumers already applied the forward's renormalisation, bias, eval
// BatchNorm + activation and the zeroing of columns >= cout, and rounded once; what is left is the dgrad input mask, the
// 16-byte stores and the BatchNorm statistics of the stored values (same values, same reduction order as tc_epilogue).
// dgrad: the staged value is bf16(acc), multiplied here by the 0 / 1 mask -- equal to rounding acc * mask except where |acc|
// is finite but rounds to bf16 infinity (inf * 0 = NaN instead of 0).
template <int BLOCK_N, int MODE>
__device__ __forceinline__ void tc_epilogue_bf16(const TcParams &P, const EpiRow &er, const bf16 *srow, int lane, int n0, float *s_stat) {
    const bool stats = (MODE == 0) && (s_stat != nullptr);
#pragma unroll 1
    for (int c0 = 0; c0 < BLOCK_N; c0 += 32) {
        const int col = n0 + c0;
        bf16 *orow = nullptr;
        int nstore = 0;                                  // channels to store from this 32-column chunk (multiple of 8)
        int xlocal = 0;                                  // dgrad: channel of the part's input that column col is
        float scale = 1.f;
        if (MODE == 0) {
            if (er.rvalid && col < P.y_cstride) { orow = P.y + er.mo * P.y_cstride + col; nstore = min(32, P.y_cstride - col); }
        } else {
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p) {
                if (p >= P.nparts) break;
                const TcPart &pt = P.parts[p];
                const int local = col - pt.koff;
                if (local >= 0 && local < pt.kext && pt.dx != nullptr && local < pt.c8 && er.rvalid) {
                    orow = pt.dx + er.mo * pt.dx_cstride + local;
                    nstore = min(32, pt.c8 - local);
                    scale = er.dscale[p];
                    xlocal = local;
                }
            }
        }
        if (nstore == 0 && !stats) continue;
        uint4 o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = reinterpret_cast<const uint4 *>(srow + c0)[j];
        if (MODE == 1 && scale != 1.f) {
            __nv_bfloat162 *ob = reinterpret_cast<__nv_bfloat162 *>(o);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float2 f = __bfloat1622float2(ob[j]);
                ob[j] = __floats2bfloat162_rn(f.x * scale, f.y * scale);
            }
        }
        if (MODE == 1 && P.relu_x != nullptr && nstore > 0) {
            // in-place ReLU backward: one 16-byte load of the layer's input per 8 channels, a select per element
            const uint4 *xr = reinterpret_cast<const uint4 *>(P.relu_x + er.mo * P.relu_cstride + xlocal);
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                if (j * 8 >= nstore) break;
                const uint4 xv = xr[j];
                const __nv_bfloat162 *xb = reinterpret_cast<const __nv_bfloat162 *>(&xv);
                __nv_bfloat162 *ob = reinterpret_cast<__nv_bfloat162 *>(&o[j]);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 xf = __bfloat1622float2(xb[k]);
                    const __nv_bfloat162 z = __float2bfloat162_rn(0.f);
                    ob[k] = __halves2bfloat162(xf.x <= 0.f ? z.x : ob[k].x, xf.y <= 0.f ? z.y : ob[k].y);
                }
            }
        }
        if (nstore > 0) {
            uint4 *dst = reinterpret_cast<uint4 *>(orow);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j * 8 < nstore) dst[j] = o[j];
        }
        if (stats) {
            // per-channel sum and sum of squares of what was just stored (rows past the tensor contribute 0), 16 columns at a
            // time: lane l ends up with column c0 + l.  The values are read again from the staging row (the forward stores them
            // unchanged) and the halves are not unrolled: holding o[] and both halves in registers makes the 64-register
            // epilogue warps spill.
            const float live = er.rvalid ? 1.f : 0.f;
            const __nv_bfloat162 *ob = reinterpret_cast<const __nv_bfloat162 *>(srow + c0);
            float cs = 0.f, cq = 0.f;
#pragma unroll 1
            for (int h = 0; h < 2; ++h) {
                float v[16];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 f = __bfloat1622float2(ob[8 * h + j]);
                    v[2 * j] = f.x * live; v[2 * j + 1] = f.y * live;
                }
                const float s = warp_transpose_sum16(v, lane);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float2 f = __bfloat1622float2(ob[8 * h + j]);
                    const float a = f.x * live, b = f.y * live;
                    v[2 * j] = a * a; v[2 * j + 1] = b * b;
                }
                const float q = warp_transpose_sum16(v, lane);
                if ((lane >> 4) == h) { cs = s; cq = q; }
            }
            s_stat[c0 + lane] += cs;                     // this warp's private accumulators: no atomics needed
            s_stat[EPI_STAT_SQ + c0 + lane] += cq;
        }
    }
}

// epilogue warp w of the TMA-fed kernels: drains rows [32 w, 32 w + 32) x all columns of every tile the consumers stage (same
// tile walk), one row per thread.  `tile_origin(tile, m0, n0)` gives a tile's origin, n0 < 0 for a tile the consumers skip.
// stat_n0: N tile the statistics slice s_stat currently belongs to (-1: none / aborted).
template <int BLOCK_N, int MODE, typename TileFn>
__device__ __forceinline__ void tma_epilogue_warps(const TcParams &P, int tile0, int tstep, int num_tiles, TileFn tile_origin,
                                                   const bf16 *stage, uint32_t acc_full, uint32_t acc_empty, float *s_stat,
                                                   int &stat_n0, int w, int lane, int code) {
    const int row = w * 32 + lane;
    if (s_stat) {
        for (int i = lane; i < EPI_STAT_SLICE; i += 32) s_stat[i] = 0.f;
        __syncwarp();
    }
    uint32_t ph = 0;
    for (int tile = tile0; tile < num_tiles; tile += tstep) {
        int m0, n0;
        tile_origin(tile, m0, n0);
        if (n0 < 0) continue;
        if (s_stat && n0 != stat_n0) {
            if (stat_n0 >= 0) tc_stats_flush<BLOCK_N>(P, s_stat, lane, stat_n0, 0, BLOCK_N, EPI_STAT_SQ);
            stat_n0 = n0;
        }
        const EpiRow er = tc_epi_row<MODE>(P, m0 + row, false);     // the consumers staged renormalised values
        if (!__all_sync(0xffffffffu, ptx::mbar_wait(acc_full, ph, P.abort_flag, code))) { stat_n0 = -1; return; }
        ph ^= 1;
        tc_epilogue_bf16<BLOCK_N, MODE>(P, er, stage + row * bf16_pitch(BLOCK_N), lane, n0, s_stat);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(acc_empty);
    }
}

// What a consumer thread needs for the forward element math of its two rows per m64 block (rows r0 and r0 + 8 of the
// accumulator fragment): fetched when the tile starts, so the loads hide behind the K loop.
struct ConsRows {
    float inv[2];
    bool hole[2];
};
template <int MODE>
__device__ __forceinline__ ConsRows cons_rows(const TcParams &P, int m0, int e, int lane) {
    ConsRows cr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        cr.inv[h] = 0.f; cr.hole[h] = false;
        if (MODE == 0) {
            const EpiRow er = tc_epi_row<0>(P, m0 + 64 * (e >> 2) + 16 * (e & 3) + (lane >> 2) + 8 * h);
            cr.inv[h] = er.inv; cr.hole[h] = er.hole;
        }
    }
    return cr;
}

// register accumulators of consumer warp e -> its 16 rows of the bf16 staging tile, with the fp32 element math of the forward
// epilogue (the expression tc_epilogue evaluates, in the same order) done here, rounded to bf16 once:
//   y = hole ? 0 : acc * (1 / mask sum) + bias;  eval: y = act(y * scale + shift);  columns >= cout: 0
// dgrad stages bf16(acc).  Bias / scale / shift: one pair of columns per fragment column block, from L1.
template <int BLOCK_N, int MODE>
__device__ __forceinline__ void stage_acc_bf16(const TcParams &P, const float (&acc)[BLOCK_N / 2], bf16 *stage, int e, int lane, int n0,
                                               const ConsRows &cr) {
    constexpr int PITCH = bf16_pitch(BLOCK_N);
    const int r0 = 64 * (e >> 2) + 16 * (e & 3) + (lane >> 2), c0 = 2 * (lane & 3);
    const bool has_bias = (MODE == 0) && (P.bias != nullptr);
    const bool ep = (MODE == 0) && (P.ep_on != 0);
    const bool ep_aff = ep && (P.ep_scale != nullptr);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + 8 * j + c0;
        float b0 = 0.f, b1 = 0.f, s0 = 1.f, s1 = 1.f, t0 = 0.f, t1 = 0.f;
        if (MODE == 0) {
            const bool in0 = col < P.cout, in1 = col + 1 < P.cout;
            if (has_bias) { if (in0) b0 = __ldg(P.bias + col); if (in1) b1 = __ldg(P.bias + col + 1); }
            if (ep_aff) {
                if (in0) { s0 = __ldg(P.ep_scale + col); t0 = __ldg(P.ep_shift + col); }
                if (in1) { s1 = __ldg(P.ep_scale + col + 1); t1 = __ldg(P.ep_shift + col + 1); }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float a = acc[4 * j + 2 * h], b = acc[4 * j + 2 * h + 1];
            if (MODE == 0) {
                a = cr.hole[h] ? 0.f : fmaf(a, cr.inv[h], b0);
                b = cr.hole[h] ? 0.f : fmaf(b, cr.inv[h], b1);
                if (ep) {                          // holes become apply_act(shift): the BatchNorm sees the zeros written above
                    a = apply_act(fmaf(a, s0, t0), P.ep_act, P.ep_slope);
                    b = apply_act(fmaf(b, s1, t1), P.ep_act, P.ep_slope);
                }
                if (col >= P.cout) a = 0.f;
                if (col + 1 >= P.cout) b = 0.f;
            }
            *reinterpret_cast<__nv_bfloat162 *>(stage + (r0 + 8 * h) * PITCH + 8 * j + c0) = __floats2bfloat162_rn(a, b);
        }
    }
}

// consumer warp e after a tile's K loop: wait until the epilogue warps have read the staging tile, write this warp's rows into
// it (bf16, with the element math), hand it over.  false: aborted.
template <int BLOCK_N, int MODE>
__device__ __forceinline__ bool tma_stage_tile(const TcParams &P, const float (&acc)[BLOCK_N / 2], bf16 *stage, uint32_t acc_full,
                                               uint32_t acc_empty, uint32_t &ph, int e, int lane, int n0, const ConsRows &cr, int code) {
    if (!__all_sync(0xffffffffu, ptx::mbar_wait(acc_empty, ph, P.abort_flag, code))) return false;
    ph ^= 1;
    stage_acc_bf16<BLOCK_N, MODE>(P, acc, stage, e, lane, n0, cr);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(acc_full);
    return true;
}

}  // namespace

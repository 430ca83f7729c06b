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
//     MMA         wgmma.mma_async m64nNk16 bf16 -> fp32, N in {32, 64, 128}: two consumer warpgroups each own 64 rows of the
//                 128-row tile and hold its accumulators in registers; stages are released through mbarriers once
//                 wgmma.wait_group reports the MMAs that read them complete.
//     epilogue    registers -> shared staging tile -> one thread per row, fwd: y = hole ? 0 : acc / s + bias (s = mask box sum),
//                 dgrad: dx_part = acc * input-mask of that part; bf16 NHWC stores.  Stride-2 dgrad = four stride-1 parity classes.
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

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;                 // bf16 elements = 128 bytes = one swizzle row
constexpr int A_STAGE_BYTES = BLOCK_M * 128;
constexpr int NUM_PRODUCER_THREADS = 128;
constexpr int TC_MAX_PARTS = 2;             // U-Net inputs are cat([upsampled, skip]) at most
// Every tensor-core kernel computes its 128-row tile with TWO consumer warpgroups: warpgroup g issues the m64 wgmmas of rows
// [64 g, 64 g + 64) into register accumulators and then runs the epilogue of those rows.  wgmma reads shared memory through
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
    int hg;                   // row-halo mode: input pixels staged per group of 8 output pixels = 8 + (kw-1)*dil
    int ring_a, ring_b;       // smem ring depths (A items / weight tiles)
    int ktap;                 // K extent of one tap (sum of part kext); rowpack: 64 per kernel row
    int ncols;                // GEMM N extent covered by the grid (multiple of BLOCK_N)
    TcPart parts[TC_MAX_PARTS];
    // fwd epilogue
    const float *bias; const float *msum; bf16 *y; int y_cstride;
    // dgrad gather source
    const bf16 *dc; int dc_cstride, dc_c8, dc_kext;
    int *abort_flag;
    int l2pf;                 // TMA-fed fwd/dgrad: request the next tile's A boxes into L2 one tile ahead (PCB_TMA_L2_PREFETCH)
    // TMA-fed kernel: the 128 pixels of an M tile form the box {box_w, box_h, box_n} of the (x, y, image) pixel grid
    int box_w, box_h, box_n, stages, use_fix;
    int wk_base, wk_row, wk_col;   // weight-matrix K index of tap (a, b) of this launch: wk_base + a*wk_row + b*wk_col (+ part / block offset)
    // dgrad output addressing: the tile grid (h, w above) is every `sub`-th pixel of the full-resolution [fh, fw] gradient,
    // starting at (py, px) -- sub = 2 for the parity classes of a stride-2 layer, 1 otherwise
    int sub, py, px, fh, fw;
    // split-K (layers with too few output tiles to fill the GPU): the 64-channel K blocks of every tap are dealt round-robin to
    // `ksplit` CTAs per tile, which add their raw fp32 accumulators into `partial` [m_total][ncols]; a finish kernel applies
    // the epilogue.  ksplit = 1: `partial` is null and the epilogue runs in the kernel.
    int ksplit;
    float *partial;
    // fused BatchNorm statistics (forward, MODE 0): per-channel sum / sum of squares of the bf16-ROUNDED outputs are accumulated
    // into bn_sums[0][co] / bn_sums[1][co] (doubles, pre-zeroed by the caller, row pitch bn_c = cout) -- the separate statistics
    // pass over y (nn.BatchNorm2d in training mode, partial_convolution.py:193-197) disappears.  null: off.
    double *bn_sums;
    int bn_c;
};

// fused BatchNorm statistics: eight private slices of [128 sums | 128 squares], one per epilogue warp (row quadrant x column half)
constexpr int STAT_SLICE = 256;
constexpr int STAT_SMEM_BYTES = MMA_WARPS * STAT_SLICE * 4 + 16;

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

__device__ __forceinline__ uint32_t align1024(uint32_t a) { return (a + 1023u) & ~1023u; }

// -------------------------------------------------------------------------------------------------
// epilogue shared by the forward / dgrad kernels: staged fp32 accumulators -> renormalise / mask -> bf16 NHWC
// -------------------------------------------------------------------------------------------------
// `acc_row` is this lane's row of the staging tile (row warp * 32 + lane).  Columns [cb, ce) of the tile (multiples of 32): each
// row quadrant is drained by two warps that split the columns.  s_stat: this warp's accumulators [sums of its columns | squares
// at offset sq_off].
__device__ __forceinline__ void load_acc32(const float *src, uint32_t (&r)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 v = reinterpret_cast<const uint4 *>(src)[j];
        r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
    }
}

template <int BLOCK_N, int MODE>
__device__ __forceinline__ void tc_epilogue(const TcParams &P, const float *acc_row, int warp, int lane, int m0, int n0, float *s_stat,
                                            int cb, int ce, int sq_off) {
                const int row = warp * 32 + lane;
                const int m = m0 + row;
                const bool rvalid = m < P.m_total;
                float inv = 0.f;
                bool hole = false;
                int en = 0, eh = 0, ew = 0;
                long long mo = m;                         // pixel index in the full-resolution output (fwd) / gradient (dgrad)
                if (MODE == 1 && rvalid) {
                    en = m / (P.h * P.w); const int rem = m - en * P.h * P.w; eh = rem / P.w; ew = rem - eh * P.w;
                    eh = eh * P.sub + P.py; ew = ew * P.sub + P.px;
                    mo = (static_cast<long long>(en) * P.fh + eh) * P.fw + ew;
                }
                if (MODE == 0 && rvalid && P.sub != 1) {  // sub-pixel class launch: the tile grid is every `sub`-th output pixel
                    en = m / (P.ho * P.wo); const int rem = m - en * P.ho * P.wo; eh = rem / P.wo; ew = rem - eh * P.wo;
                    mo = (static_cast<long long>(en) * P.fh + eh * P.sub + P.py) * P.fw + ew * P.sub + P.px;
                }
                if (MODE == 0 && rvalid) {
                    const float s = P.msum ? P.msum[mo] : 1.f;               // null: plain convolution (renormaliser 1)
                    hole = (s == 0.f) && !P.no_guard;
                    inv = hole ? 0.f : 1.0f / s;         // no_guard: 1/0 = inf -> 0*inf = NaN like the reference
                }
                if (P.partial != nullptr) {                // split-K: raw accumulators, reduced across CTAs with fp32 adds
    #pragma unroll 1
                    for (int c0 = cb; c0 < ce; c0 += 32) {
                        uint32_t r[32];
                        load_acc32(acc_row + c0, r);
                        if (rvalid) {
                            float *dst = P.partial + static_cast<long long>(m) * P.ncols + n0 + c0;
    #pragma unroll
                            for (int j = 0; j < 32; ++j) atomicAdd(dst + j, __uint_as_float(r[j]));
                        }
                    }
                    return;
                }
    #pragma unroll 1
                for (int c0 = cb; c0 < ce; c0 += 32) {
                    uint32_t r[32];
                    load_acc32(acc_row + c0, r);
                    const int col = n0 + c0;
                    bf16 *orow = nullptr;
                    int nstore = 0;                      // channels to store from this 32-column chunk (multiple of 8)
                    float scale = inv;
                    if (MODE == 0) {
                        if (rvalid && col < P.y_cstride) { orow = P.y + mo * P.y_cstride + col; nstore = min(32, P.y_cstride - col); }
                    } else {
                        scale = 1.f;
                        for (int p = 0; p < P.nparts; ++p) {
                            const TcPart &pt = P.parts[p];
                            const int local = col - pt.koff;
                            if (local >= 0 && local < pt.kext && pt.dx != nullptr && local < pt.c8 && rvalid) {
                                orow = pt.dx + mo * pt.dx_cstride + local;
                                nstore = min(32, pt.c8 - local);
                                if (pt.mask != nullptr)          // dx = acc * input mask of this part
                                    scale = pt.mask[(static_cast<long long>(en) * (P.fh >> pt.mup) + (eh >> pt.mup)) * (P.fw >> pt.mup) + (ew >> pt.mup)] ? 1.f : 0.f;
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
    #pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            float a = __uint_as_float(r[2 * j]), b = __uint_as_float(r[2 * j + 1]);
                            if (MODE == 0) {
                                const float b0 = has_bias ? __shfl_sync(0xffffffffu, bl, 2 * j) : 0.f;
                                const float b1 = has_bias ? __shfl_sync(0xffffffffu, bl, 2 * j + 1) : 0.f;
                                a = hole ? 0.f : fmaf(a, scale, b0);
                                b = hole ? 0.f : fmaf(b, scale, b1);
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

// register accumulators of warpgroup g (fragment layout: see ptx::wgmma_bf16) -> staging tile -> tc_epilogue of this warp's
// 32 rows x column half.  Both named barriers span the warpgroup only: the other one keeps its own pace.
template <int BLOCK_N, int MODE>
__device__ __forceinline__ void mma_epilogue(const TcParams &P, const float (&acc)[BLOCK_N / 2], float *stage, int e, int lane, int m0, int n0,
                                             float *s_stat) {
    constexpr int PITCH = acc_pitch(BLOCK_N);
    const int g = e >> 2;
    const int r0 = 64 * g + 16 * (e & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c0;
        *reinterpret_cast<float2 *>(stage + row * PITCH + col) = make_float2(acc[i], acc[i + 1]);
    }
    ptx::named_sync(1 + g, 128);
    const EpiRole<BLOCK_N> R(e);
    tc_epilogue<BLOCK_N, MODE>(P, stage + (R.q * 32 + lane) * PITCH, R.q, lane, m0, n0, s_stat, R.cb, R.ce, 128);
    ptx::named_sync(1 + g, 128);                          // the staging rows are free for the next tile
}

// last N tile's BatchNorm statistics: the eight epilogue warps' partials are summed after a CTA-wide barrier, so the global sums
// receive ONE atomic per channel per CTA.  `stat_base`: slice 0.
template <int BLOCK_N>
__device__ __forceinline__ void tc_stats_final(const TcParams &P, const float *stat_base, int e, int lane, int stat_n0) {
    constexpr int HN = EpiRole<BLOCK_N>::HN;
    for (int col = e * 32 + lane; col < BLOCK_N; col += MMA_THREADS) {
        const int co = stat_n0 + col;
        if (co < P.bn_c) {
            const int h = col / HN, lc = col - h * HN;
            float a = 0.f, q = 0.f;
#pragma unroll
            for (int w4 = 0; w4 < 4; ++w4) { a += stat_base[(h * 4 + w4) * STAT_SLICE + lc]; q += stat_base[(h * 4 + w4) * STAT_SLICE + 128 + lc]; }
            atomicAdd(P.bn_sums + co, static_cast<double>(a));
            atomicAdd(P.bn_sums + P.bn_c + co, static_cast<double>(q));
        }
    }
}

template <int R> __device__ __forceinline__ void zero_acc(float (&a)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) a[i] = 0.f;
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
// Two A-operand layouts:
//   HALO = false : per tap, a [128 pixel x 64 channel] tile in the 128B-swizzled K-major layout (any stride / dilation;
//                  also the row-packed small-Cin mode: K block = kernel row, chunk = tap column).
//   HALO = true  : stride-1 layers.  Per kernel ROW, each group of 8 consecutive output pixels stages its
//                  8 + (kw-1)*dil input pixels once in the canonical NO-SWIZZLE K-major layout
//                  addr(slot, chunk) = chunk*LBO + slot*16; the kw taps of the row are kw wgmma descriptors whose start
//                  address is shifted by tap*dil slots (SBO = HG*16 between 8-row groups): kw x fewer gathers.
// -------------------------------------------------------------------------------------------------
constexpr int HALO_MAX_HG = 12;
constexpr int PERSIST_THREADS = 4 * 32 + MMA_THREADS + 32;
constexpr int MAX_RING = 8;

template <int BLOCK_N, int MODE, bool HALO>
__global__ void __launch_bounds__(PERSIST_THREADS, 1)
pconv_tc_persistent_kernel(const __grid_constant__ TcParams P, const __grid_constant__ CUtensorMap tmap_w) {
    constexpr int B_STAGE_BYTES = BLOCK_N * 128;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int SA = P.ring_a, SB = P.ring_b;
    const int HG = P.hg;
    const uint32_t LBO = 16u * (16u * HG + 1u);                       // halo: byte distance between 8-channel chunks
    const uint32_t A_STAGE = HALO ? ((8u * LBO + 127u) & ~127u) : static_cast<uint32_t>(A_STAGE_BYTES);
    const uint32_t sB = smem_base;
    const uint32_t sA = sB + SB * B_STAGE_BYTES;                      // stays 1024-aligned (B stages are multiples of 1024)
    const uint32_t sBar = (sA + SA * A_STAGE + 15u) & ~15u;
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
    const int nB = HALO ? P.kw : 1;                                   // weight tiles consumed per A item

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
        constexpr int NW = HALO ? HALO_MAX_HG : 8;
        uint64_t wnext[TC_MAX_PARTS][NW];
        auto issue_mask_loads = [&](int tl) {
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p)
#pragma unroll
                for (int i = 0; i < NW; ++i) wnext[p][i] = 0ull;
            if (MODE != 0 || tl >= num_tiles) return;
            const int tm0 = (tl / n_tiles) * BLOCK_M;
#pragma unroll
            for (int i = 0; i < NW; ++i) {
                int idx;
                if (HALO) {
                    if (i >= HG) continue;
                    const int S = r0 + 16 * i;
                    const int g = S / HG, sl = S - g * HG;
                    const int tcs = sl > 7 ? (sl - 7 + P.dil - 1) / P.dil : 0;
                    idx = tm0 + g * 8 + (sl - tcs * P.dil);
                    if (tm0 + g * 8 >= P.m_total) continue;
                } else {
                    idx = tm0 + r0 + 16 * i;
                    if (idx >= P.m_total) continue;
                }
#pragma unroll
                for (int p = 0; p < TC_MAX_PARTS; ++p)
                    if (p < P.nparts) wnext[p][i] = __ldg(P.parts[p].tapmask + idx);
            }
        };
        issue_mask_loads(blockIdx.x);
        for (int tile = blockIdx.x; tile < num_tiles && !dead; tile += gridDim.x) {
            const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
            uint64_t wcur[TC_MAX_PARTS][NW];
#pragma unroll
            for (int p = 0; p < TC_MAX_PARTS; ++p)
#pragma unroll
                for (int i = 0; i < NW; ++i) wcur[p][i] = wnext[p][i];
            issue_mask_loads(tile + gridDim.x);
            if (!tile_active(n0)) continue;
            if (HALO) {
                int ph[HALO_MAX_HG];                              // row coordinate of the slot at kernel row 0
                int cterm[TC_MAX_PARTS][HALO_MAX_HG];             // image base + column*cstride + chunk*8 (element offset)
                uint32_t vb[TC_MAX_PARTS][HALO_MAX_HG];           // bit tr = slot valid (bounds [+ hole]) for kernel row tr
#pragma unroll
                for (int i = 0; i < HALO_MAX_HG; ++i) {
                    ph[i] = 0;
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) { vb[p][i] = 0; cterm[p][i] = 0; }
                    if (i >= HG) continue;
                    const int S = r0 + 16 * i;
                    const int g = S / HG, sl = S - g * HG;
                    const int m = m0 + g * 8;               // first pixel of the group (groups never straddle image rows)
                    const bool ok = m < P.m_total;
                    const int mm = ok ? m : 0;
                    const int nn = mm / plane, rem = mm - nn * plane;
                    const int hh = rem / pwid, ww = rem - hh * pwid;
                    if (MODE == 0) {
                        ph[i] = hh - P.pad_h;
                        const int col = ww - P.pad_w + sl;
                        // the (pixel j of the group, tap column tc) pair that looks at this slot: sl == j + tc*dil
                        const int tcs = sl > 7 ? (sl - 7 + P.dil - 1) / P.dil : 0;
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            if (p >= P.nparts || !ok) continue;
                            const TcPart &pt = P.parts[p];
                            const uint64_t word = wcur[p][i];
                            uint32_t bits = 0;
                            for (int tr = 0; tr < P.kh; ++tr) bits |= static_cast<uint32_t>((word >> (tr * P.kw + tcs)) & 1ull) << tr;
                            vb[p][i] = bits;
                            const int colc = min(max(col, 0), P.w - 1) >> pt.xup;   // clamped: only dereferenced when valid
                            cterm[p][i] = (nn * (P.h >> pt.xup) * (P.w >> pt.xup) + colc) * pt.cstride + chunk * 8;
                        }
                    } else {
                        ph[i] = hh + P.pad_h;
                        const int col = ww + P.pad_w - (P.kw - 1) * P.dil + sl;
                        const bool cok = ok && col >= 0 && col < P.wo;
                        uint32_t bits = 0;
                        for (int tr = 0; tr < P.kh; ++tr) { const int hi = ph[i] - tr * P.dil; bits |= (cok && hi >= 0 && hi < P.ho ? 1u : 0u) << tr; }
                        vb[0][i] = bits;
                        cterm[0][i] = (nn * P.ho * P.wo + min(max(col, 0), P.wo - 1)) * P.dc_cstride + chunk * 8;
                    }
                }
                for (int tr = 0; tr < P.kh && !dead; ++tr) {
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) {
                        if (p >= np || dead) break;
                        const TcPart &pt = P.parts[p];
                        const bf16 *src = (MODE == 0) ? pt.x : P.dc;
                        const int xup = (MODE == 0) ? pt.xup : 0;
                        const int hmax = ((MODE == 0) ? (P.h >> xup) : P.ho) - 1;
                        const int rowpitch = (MODE == 0) ? (P.w >> xup) * pt.cstride : P.wo * P.dc_cstride;
                        const int nb = ((MODE == 0) ? pt.kext : P.dc_kext) / BLOCK_K;
                        const int c8 = (MODE == 0) ? pt.c8 : P.dc_c8;
                        int rterm[HALO_MAX_HG];
#pragma unroll
                        for (int i = 0; i < HALO_MAX_HG; ++i) {
                            const int hi = (MODE == 0) ? ((ph[i] + tr * P.dil) >> xup) : (ph[i] - tr * P.dil);
                            rterm[i] = cterm[p][i] + min(max(hi, 0), hmax) * rowpitch;
                        }
                        for (int cb = 0; cb < nb; ++cb, ++it) {
                            const int s = it % SA;
                            if (!ptx::mbar_wait(bar_empty_a + 8 * s, ((it / SA) & 1) ^ 1, P.abort_flag, 111)) { dead = true; break; }
                            const bool cv = cb * BLOCK_K + chunk * 8 < c8;
                            const uint32_t dst0 = sA + s * A_STAGE + chunk * LBO + r0 * 16;
                            const bf16 *srcb = src + cb * BLOCK_K;
#pragma unroll
                            for (int i = 0; i < HALO_MAX_HG; ++i) {
                                if (i >= HG) break;
                                ptx::cp_async_16(dst0 + i * 256, srcb + rterm[i], cv && ((vb[p][i] >> tr) & 1u));   // slot r0 + 16*i
                            }
                            ptx::cp_async_mbar_arrive(bar_full_a + 8 * s);
                            ptx::mbar_arrive(bar_full_a + 8 * s);
                        }
                    }
                }
            } else {
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
                    const uint32_t dst = sA + s * A_STAGE + r0 * 128 + sw;
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
                if (HALO) {
                    for (int tr = 0; tr < P.kh && !dead; ++tr)
                        for (int p = 0; p < np && !dead; ++p) {
                            const int nb = ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
                            for (int cb = 0; cb < nb && !dead; ++cb)
                                for (int tc = 0; tc < P.kw; ++tc) {
                                    const int tap = tr * P.kw + tc;
                                    const int kidx = (MODE == 0) ? tap * P.ktap + P.parts[p].koff + cb * BLOCK_K : tap * P.dc_kext + cb * BLOCK_K;
                                    if (!load(kidx, n0)) { dead = true; break; }
                                }
                        }
                } else {
                    const int num_kb = (MODE == 0) ? (P.rowpack ? P.kh : taps * (P.ktap / BLOCK_K)) : taps * (P.dc_kext / BLOCK_K);
                    for (int kb = 0; kb < num_kb; ++kb)
                        if (!load(kb * BLOCK_K, n0)) { dead = true; break; }
                }
            }
        }
    } else {
        // ================================ consumer warpgroups (warps 4-11) ================================
        const int e = warp - 4, g = e >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        int num_a = 0;
        if (HALO) {
            for (int p = 0; p < np; ++p) num_a += ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
            num_a *= P.kh;
        } else {
            num_a = (MODE == 0) ? (P.rowpack ? P.kh : taps * (P.ktap / BLOCK_K)) : taps * (P.dc_kext / BLOCK_K);
        }
        // this warpgroup's 64 rows: 8 groups of 8 rows further into the A stage
        const uint32_t a_rows = HALO ? 8u * HG * 16u : 64u * 128u;
        float *s_stat = (MODE == 0 && P.bn_sums != nullptr && P.partial == nullptr)
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
                const int sb0 = itb % SB;
                for (int tc = 0; tc < nB; ++tc, ++itb) {
                    const int sb = itb % SB;
                    if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full_b + 8 * sb, (itb / SB) & 1, P.abort_flag, 105))) { dead = true; break; }
                    const uint64_t db = ptx::make_smem_desc(sB + sb * B_STAGE_BYTES, 16, 1024);
                    ptx::wgmma_fence();
                    if (HALO) {
                        const int shift = ((MODE == 0) ? tc : (P.kw - 1 - tc)) * P.dil;    // slots
                        const uint32_t a0 = sA + sa * A_STAGE + g * a_rows + shift * 16;
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 16; ++k)                              // 2 chunks (16 channels) per MMA
                            ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, ptx::make_smem_desc_noswizzle(a0 + k * 2 * LBO, LBO, HG * 16), db + 2 * k);
                    } else {
                        const uint64_t da = ptx::make_smem_desc(sA + sa * A_STAGE + g * a_rows, 16, 1024);
#pragma unroll
                        for (int k = 0; k < BLOCK_K / 16; ++k)                              // +32 bytes per K=16 step inside the swizzle row
                            ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + 2 * k, db + 2 * k);
                    }
                    ptx::wgmma_commit();
                }
                // the A item and its weight tiles are released once this warpgroup's MMAs on them completed
                ptx::wgmma_wait<0>();
                ptx::wgmma_fence_regs(acc);
                if (leader) {
                    for (int tc = 0; tc < nB; ++tc) ptx::mbar_arrive(bar_empty_b + 8 * ((sb0 + tc) % SB));
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
// (x*mask, models/partial_convolution.py:51): four "fixer" warps (one thread per tile row) test the row's tap-validity
// bit and overwrite hole rows of the landed tile with zeros before handing the stage to the MMA thread
// (generic-proxy stores -> fence.proxy.async -> mbarrier).  Plain convolutions / dgrad skip the fixers.
//
//   warps 0-7  consumers  : two warpgroups, 4 x wgmma (K=16) per K block and weight tile, then the epilogue of their 64 rows
//   warp 8     TMA producer : per K block one A tile (4-D) + the weight tiles (2-D) onto the same mbarrier
//   warps 9-12 fixers     : hole rows -> 0   (MODE 0 with masks only)
// Every per-K-block loop of the producer is a handful of instructions: index arithmetic there (the old kernels did integer
// divisions) directly delays the stages the tensor cores wait for.
// -------------------------------------------------------------------------------------------------
constexpr int TMA_THREADS = MMA_THREADS + 5 * 32;

// HALO = true (stride 1, tiles that are one image-row segment of 128 pixels): per kernel ROW one A tile of
// 128 + (kw-1)*dil pixel rows is loaded, and the kw taps of that row are kw wgmma descriptors whose start address is
// shifted by whole 128-byte rows (the 128B swizzle is a function of the absolute smem address, so a row-shifted start
// reads the same image) -- kw x less A traffic from L2 and kw x fewer barrier round trips per MMA.  K steps that only cover
// channel padding (c8 <= 16*k) are skipped.
template <int BLOCK_N, int MODE, bool HALO>
__global__ void __launch_bounds__(TMA_THREADS, 1)
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
    const uint32_t s_stat_addr = sBar + 24 * MAX_RING;
    const uint32_t s_acc = (s_stat_addr + STAT_SMEM_BYTES + 15u) & ~15u;
    uint8_t *smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform by construction
    const int np = (MODE == 0) ? P.nparts : 1;
    const int n_tiles = P.ncols / BLOCK_N;
    const int KS = P.ksplit;                                            // tile index = (m tile * n_tiles + n tile) * KS + split
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * n_tiles * KS;
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
            ptx::mbar_init(bar_full + 8 * s, 1); ptx::mbar_init(bar_fixed + 8 * s, 4); ptx::mbar_init(bar_empty + 8 * s, 2);
        }
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_w); ptx::prefetch_tmap(&tmap_a0); if (np > 1) ptx::prefetch_tmap(&tmap_a1); }
    __syncthreads();

    // The producer runs WARP-CONVERGED (all 32 lanes walk the loops and wait on the barriers; the warp index is a shuffle
    // broadcast so the compiler knows the role branch is uniform) and only the TMA instructions sit inside an elect.sync region.
    float *s_stat = nullptr;                                          // consumer warps: private BatchNorm-statistics accumulators
    int stat_n0 = -1;                                                  // N tile they currently belong to (-1: none / aborted)
    if (warp == 8) {
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
            const int sp = tile % KS, mn = tile / KS;
            const int m0 = m0_of(mn / n_tiles), n0 = (mn % n_tiles) * BLOCK_N;
            if (!tile_active(n0)) continue;
            const int img = m0 / plane, rem = m0 - img * plane;
            const int oy = rem / pwid, ox = rem - oy * pwid;
            // leftmost / topmost source coordinate of tap column 0 (fwd) -- dgrad walks its taps right to left
            const int x_org = (MODE == 0) ? ox * P.stride - P.pad_w : (HALO ? ox + P.pad_w - hx : ox + P.pad_w);
            const int y_org = (MODE == 0) ? oy * P.stride - P.pad_h : oy + P.pad_h;
            // optional L2 prefetch (P.l2pf): while tile t is loaded, the A boxes of this CTA's NEXT tile are requested into L2, one
            // tile's worth of stages ahead, so that their loads find L2 instead of DRAM (the ring is round-trip-latency bound)
            int nx_org = 0, ny_org = 0, nimg = -1;
            if (P.l2pf && tile + tstep < num_tiles) {
                const int nmn = (tile + tstep) / KS;
                const int nm0 = m0_of(nmn / n_tiles);
                if (nm0 != m0) {
                    nimg = nm0 / plane;
                    const int nrem = nm0 - nimg * plane, noy = nrem / pwid, nox = nrem - noy * pwid;
                    nx_org = (MODE == 0) ? nox * P.stride - P.pad_w : (HALO ? nox + P.pad_w - hx : nox + P.pad_w);
                    ny_org = (MODE == 0) ? noy * P.stride - P.pad_h : noy + P.pad_h;
                }
            }
            int krow = P.wk_base;                                      // weight K index of (tr, tap column 0, part 0, block 0)
            for (int tr = 0, y = y_org; tr < P.kh && !dead; ++tr, y += dstep, krow += row_k)
                for (int ti = 0, x = x_org, kidx = krow; ti < kwi && !dead; ++ti, x += dstep, kidx = krow + ti * col_k) {
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) {
                        const int kext = (p == 0) ? kext0 : kext1;
                        const CUtensorMap *ma = (p == 0) ? &tmap_a0 : &tmap_a1;
                        const int gb0 = (p == 0) ? 0 : kext0 / BLOCK_K;          // global K-block index of the part's first block
                        for (int c0 = 0; c0 < kext; c0 += BLOCK_K, kidx += BLOCK_K) {
                            if (KS > 1 && (gb0 + c0 / BLOCK_K) % KS != sp) continue;
                            if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 121))) { dead = true; break; }
                            if (ptx::elect_one()) {
                                const uint32_t full = bar_full + 8 * s, dst = smem_base + s * STAGE;
                                ptx::mbar_arrive_expect_tx(full, STAGE_TX);
                                ptx::tma_load_4d(dst, ma, c0, x, y, img, full);
                                uint32_t bdst = dst + A_ROOM;
                                for (int tc = 0, kb = kidx; tc < nB; ++tc, kb += col_k, bdst += B_BYTES)
                                    ptx::tma_load_2d(bdst, &tmap_w, kb, n0, full);
                                if (nimg >= 0) ptx::tma_prefetch_4d(ma, c0, nx_org + ti * dstep, ny_org + tr * dstep, nimg);
                            }
                            __syncwarp();
                            if (++s == S) { s = 0; ph ^= 1; }
                        }
                        if (dead) break;
                    }
                }
        }
    } else if (warp < MMA_WARPS) {
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
        const EpiRole<BLOCK_N> R(e);
        s_stat = (MODE == 0 && P.bn_sums != nullptr && P.partial == nullptr)
                     ? reinterpret_cast<float *>(smem_gen + (s_stat_addr - smem_base)) + R.slice() * STAT_SLICE : nullptr;
        if (s_stat) {
            for (int i = lane; i < STAT_SLICE; i += 32) s_stat[i] = 0.f;
            __syncwarp();
        }
        float *acc_stage = reinterpret_cast<float *>(smem_gen + (s_acc - smem_base));
        int s = 0;
        uint32_t ph = 0;
        bool dead = false;
        for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
            const int sp = tile % KS, mn = tile / KS;
            const int m0 = m0_of(mn / n_tiles), n0 = (mn % n_tiles) * BLOCK_N;
            if (!tile_active(n0)) continue;
            if (s_stat && n0 != stat_n0) {
                if (stat_n0 >= 0) tc_stats_flush<BLOCK_N>(P, s_stat, lane, stat_n0, R.cb, R.ce, 128);
                stat_n0 = n0;
            }
            float acc[BLOCK_N / 2];
            zero_acc(acc);
            int held = -1;                                             // stage whose MMAs may still be reading it
            for (int r = 0; r < rows_a && !dead; ++r) {
#pragma unroll
                for (int p = 0; p < TC_MAX_PARTS; ++p) {
                    const int nbp = (p == 0) ? nb0 : nb1, klast = (p == 0) ? kl0 : kl1;
                    const int gb0 = (p == 0) ? 0 : nb0;
                    for (int cb = 0; cb < nbp; ++cb) {
                        if (KS > 1 && (gb0 + cb) % KS != sp) continue;
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
            if (dead) { stat_n0 = -1; break; }
            mma_epilogue<BLOCK_N, MODE>(P, acc, acc_stage, e, lane, m0, n0, s_stat);
        }
    } else if (warp > 8) {
        // ================================ fixers: zero the hole rows of every landed A tile ================================
        if (fix) {
            const int t = (warp - 9) * 32 + lane;
            int s = 0;
            uint32_t ph = 0;
            bool dead = false;
            if (!HALO) {
                // one thread per tile row; validity = the row's tap bit (bounds + hole)
                uint64_t wnext[TC_MAX_PARTS];
                auto load_words = [&](int tl) {
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) {
                        wnext[p] = 0ull;
                        const int m = m0_of(tl / KS / n_tiles) + t;
                        if (fix && p < P.nparts && tl < num_tiles && m < P.m_total) wnext[p] = __ldg(P.parts[p].tapmask + m);
                    }
                };
                load_words(tile0);
                for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                    const int sp = tile % KS;
                    uint64_t wcur[TC_MAX_PARTS];
#pragma unroll
                    for (int p = 0; p < TC_MAX_PARTS; ++p) wcur[p] = wnext[p];
                    load_words(tile + tstep);                      // next tile's words travel while this tile streams
                    if (MODE == 1 && !tile_active(((tile / KS) % n_tiles) * BLOCK_N)) continue;
                    const int taps = P.kh * P.kw;
                    for (int tap = 0; tap < taps && !dead; ++tap) {
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            if (p >= np) break;
                            const bool hole = fix && ((wcur[p] >> tap) & 1ull) == 0ull;
                            const bool any_hole = __any_sync(0xffffffffu, hole);
                            const int nb = ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
                            const int gb0 = (p == 0) ? 0 : P.parts[0].kext / BLOCK_K;
                            for (int cb = 0; cb < nb; ++cb) {
                                if (KS > 1 && (gb0 + cb) % KS != sp) continue;
                                if (!ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 122)) { dead = true; break; }
                                if (any_hole) {
                                    if (hole) {
                                        uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + t * 128);
                                        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                                        for (int k = 0; k < 8; ++k) r[k] = z;
                                    }
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
                // one thread per halo pixel row (threads < hx own a second one); validity = the source mask at that pixel
                const int plane = P.ho * P.wo;
                auto load_bits = [&](int tl, uint32_t &b0, uint32_t &b1) {       // bit (p*8 + tr): pixel row is a hole
                    b0 = b1 = 0;
                    if (!fix || tl >= num_tiles) return;
                    const int m0 = m0_of(tl / KS / n_tiles);
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
                            const int x0 = ox - P.pad_w + t, x1 = x0 + 128;
                            if (x0 >= 0 && x0 < P.w && __ldg(mk + (y >> mup) * (P.w >> mup) + (x0 >> mup)) == 0) b0 |= 1u << (p * 8 + tr);
                            if (t < hx && x1 < P.w && __ldg(mk + (y >> mup) * (P.w >> mup) + (x1 >> mup)) == 0) b1 |= 1u << (p * 8 + tr);
                        }
                    }
                };
                uint32_t n0b, n1b;
                load_bits(tile0, n0b, n1b);
                for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                    const int sp = tile % KS;
                    const uint32_t c0b = n0b, c1b = n1b;
                    load_bits(tile + tstep, n0b, n1b);
                    if (MODE == 1 && !tile_active(((tile / KS) % n_tiles) * BLOCK_N)) continue;
                    for (int tr = 0; tr < P.kh && !dead; ++tr) {
#pragma unroll
                        for (int p = 0; p < TC_MAX_PARTS; ++p) {
                            if (p >= np) break;
                            const bool h0 = (c0b >> (p * 8 + tr)) & 1u, h1 = (c1b >> (p * 8 + tr)) & 1u;
                            const bool any_hole = __any_sync(0xffffffffu, h0 || h1);
                            const int nb = ((MODE == 0) ? P.parts[p].kext : P.dc_kext) / BLOCK_K;
                            const int gb0 = (p == 0) ? 0 : P.parts[0].kext / BLOCK_K;
                            for (int cb = 0; cb < nb; ++cb) {
                                if (KS > 1 && (gb0 + cb) % KS != sp) continue;
                                if (!ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 122)) { dead = true; break; }
                                if (any_hole) {
                                    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
                                    if (h0) {
                                        uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + t * 128);
#pragma unroll
                                        for (int k = 0; k < 8; ++k) r[k] = z;
                                    }
                                    if (h1) {
                                        uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + (t + 128) * 128);
#pragma unroll
                                        for (int k = 0; k < 8; ++k) r[k] = z;
                                    }
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

    __syncthreads();
    if (s_stat != nullptr && stat_n0 >= 0) tc_stats_final<BLOCK_N>(P, s_stat - EpiRole<BLOCK_N>(warp).slice() * STAT_SLICE, warp, lane, stat_n0);
}


// -------------------------------------------------------------------------------------------------
// SUB-PIXEL (table-driven) variant of the TMA-fed kernel: convolutions whose input is cat([nearest-2x-upsample(x0), x1])
// (models/image_inpainting.py:183-185) WITHOUT materialising the upsampled tensor and WITHOUT multiplying by replicated pixels.
//
// Output pixel (2k+py, 2j+px) of a k x k convolution over up2x(x0) reads source pixel (k + floor((py + tr*d - p)/2), ...): within
// one parity class (py, px) the convolution over the upsampled part IS a convolution over the SOURCE with a smaller kernel whose
// taps are sums of the original taps (3x3, pad 1: 2x2 effective taps -- 4/9 of the multiplications); the skip part x1 keeps its
// k x k taps and is read with a traversal stride of 2.  The hole mask of the upsampled part was upsampled with it
// (HoleMask.upsampled), so masking commutes.  One launch computes one class: its M tiles are boxes of the class grid
// [n][h/2][w/2]; what each K step loads is listed in a small table built on the host:
//     item = { part (tensor map), (dx, dy) added to the tile origin scaled by the part's step, nb weight tiles (taps served by
//              one A tile through row-shifted descriptors), weight K index of the first, step between them }
// The same kernel computes the data gradient w.r.t. x0 directly at SOURCE resolution (MODE 1): its A operand is dc read with a
// traversal stride of 2 per (class, effective tap) item -- 16/36 of the multiplications of "full-resolution gradient + 2x2 sum",
// and neither the full-resolution gradient nor the reduction pass exists.
// Roles / pipeline / epilogue exactly as in pconv_tc_tma_kernel (no split-K).
// -------------------------------------------------------------------------------------------------
constexpr int SP_MAX_ITEMS = 40;
struct SpItem { int part, dx, dy, wk, nb, wk_step, shift0, dshift; };
struct SpTable {
    int n_items;
    int step[TC_MAX_PARTS];         // tile origin (class grid) -> part coordinates: origin * step + (dx, dy)
    int es[TC_MAX_PARTS];           // traversal stride of the part's tensor map (pixels between consecutive tile rows)
    int ph[TC_MAX_PARTS], pw[TC_MAX_PARTS];     // the part's own pixel grid (its mask plane has exactly this resolution)
    int arows[TC_MAX_PARTS];        // pixel rows one TMA tile of the part delivers (128 + the halo of the part's tensor-map box)
    int rows_max;                   // pixel rows of the largest A tile
    SpItem it[SP_MAX_ITEMS];
};

template <int BLOCK_N, int MODE>
__global__ void __launch_bounds__(TMA_THREADS, 1)
pconv_tc_sp_kernel(const __grid_constant__ TcParams P, const __grid_constant__ SpTable TB, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1) {
    constexpr uint32_t B_BYTES = BLOCK_N * 128;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = align1024(ptx::smem_u32(smem_raw));
    const int S = P.stages;
    int nb_max = 1;
    for (int i = 0; i < TB.n_items; ++i) nb_max = max(nb_max, TB.it[i].nb);
    const uint32_t A_ROOM = (static_cast<uint32_t>(TB.rows_max) * 128u + 1023u) & ~1023u;
    const uint32_t STAGE = A_ROOM + nb_max * B_BYTES;
    const uint32_t sBar = smem_base + S * STAGE;
    const uint32_t bar_full = sBar, bar_fixed = sBar + 8 * MAX_RING, bar_empty = sBar + 16 * MAX_RING;
    const uint32_t s_stat_addr = sBar + 24 * MAX_RING;
    const uint32_t s_acc = (s_stat_addr + STAT_SMEM_BYTES + 15u) & ~15u;
    uint8_t *smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    const int n_tiles = P.ncols / BLOCK_N;
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * n_tiles;
    const int tile0 = static_cast<int>(blockIdx.x), tstep = static_cast<int>(gridDim.x);
    const bool fix = P.use_fix != 0;
    // the tile grid: [n][gh][gw] = the class grid (MODE 0: P.ho x P.wo) or the source grid (MODE 1: P.h x P.w)
    const int gw = (MODE == 0) ? P.wo : P.w, gh = (MODE == 0) ? P.ho : P.h;
    const int plane = gw * gh;
    // per part: 64-channel K blocks and the K steps of the last block that hold real channels
    int nbk[TC_MAX_PARTS], klast[TC_MAX_PARTS];
#pragma unroll
    for (int p = 0; p < TC_MAX_PARTS; ++p) {
        const int kext = (MODE == 0) ? P.parts[p].kext : P.dc_kext, c8 = (MODE == 0) ? P.parts[p].c8 : P.dc_c8;
        nbk[p] = (p < ((MODE == 0) ? P.nparts : 1)) ? kext / BLOCK_K : 0;
        klast[p] = nbk[p] ? min(4, (c8 - (nbk[p] - 1) * BLOCK_K + 15) >> 4) : 4;
    }

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) { ptx::mbar_init(bar_full + 8 * s, 1); ptx::mbar_init(bar_fixed + 8 * s, 4); ptx::mbar_init(bar_empty + 8 * s, 2); }
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_w); ptx::prefetch_tmap(&tmap_a0); ptx::prefetch_tmap(&tmap_a1); }
    __syncthreads();

    float *s_stat = nullptr;
    int stat_n0 = -1;
    if (warp == 8) {
        // ================================ TMA producer ================================
        int s = 0;
        uint32_t ph = 1;
        bool dead = false;
        for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
            const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
            const int img = m0 / plane, rem = m0 - img * plane;
            const int oy = rem / gw, ox = rem - oy * gw;
            for (int i = 0; i < TB.n_items && !dead; ++i) {
                const SpItem it = TB.it[i];
                const CUtensorMap *ma = (it.part == 0) ? &tmap_a0 : &tmap_a1;
                const int x = ox * TB.step[it.part] + it.dx, y = oy * TB.step[it.part] + it.dy;
                const uint32_t a_bytes = static_cast<uint32_t>(TB.arows[it.part]) * 128u;      // what the part's box delivers
                for (int cb = 0; cb < nbk[it.part]; ++cb) {
                    if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_empty + 8 * s, ph, P.abort_flag, 321))) { dead = true; break; }
                    if (ptx::elect_one()) {
                        const uint32_t full = bar_full + 8 * s, dst = smem_base + s * STAGE;
                        ptx::mbar_arrive_expect_tx(full, a_bytes + it.nb * B_BYTES);
                        ptx::tma_load_4d(dst, ma, cb * BLOCK_K, x, y, img, full);
                        uint32_t bdst = dst + A_ROOM;
                        for (int tc = 0, kb = it.wk + cb * BLOCK_K; tc < it.nb; ++tc, kb += it.wk_step, bdst += B_BYTES)
                            ptx::tma_load_2d(bdst, &tmap_w, kb, n0, full);
                    }
                    __syncwarp();
                    if (++s == S) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp < MMA_WARPS) {
        // ================================ consumer warpgroups ================================
        const int e = warp, g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t ready = fix ? bar_fixed : bar_full;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + g * 64 * 128, 16, 1024);     // this warpgroup's 64 rows
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_ROOM, 16, 1024);
        const uint32_t stage16 = STAGE >> 4;
        const EpiRole<BLOCK_N> R(e);
        s_stat = (MODE == 0 && P.bn_sums != nullptr) ? reinterpret_cast<float *>(smem_gen + (s_stat_addr - smem_base)) + R.slice() * STAT_SLICE : nullptr;
        if (s_stat) {
            for (int i = lane; i < STAT_SLICE; i += 32) s_stat[i] = 0.f;
            __syncwarp();
        }
        float *acc_stage = reinterpret_cast<float *>(smem_gen + (s_acc - smem_base));
        int s = 0;
        uint32_t ph = 0;
        bool dead = false;
        for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
            const int m0 = (tile / n_tiles) * BLOCK_M, n0 = (tile % n_tiles) * BLOCK_N;
            if (s_stat && n0 != stat_n0) {
                if (stat_n0 >= 0) tc_stats_flush<BLOCK_N>(P, s_stat, lane, stat_n0, R.cb, R.ce, 128);
                stat_n0 = n0;
            }
            float acc[BLOCK_N / 2];
            zero_acc(acc);
            int held = -1;
            for (int i = 0; i < TB.n_items && !dead; ++i) {
                const SpItem it = TB.it[i];
                for (int cb = 0; cb < nbk[it.part]; ++cb) {
                    if (!__all_sync(0xffffffffu, ptx::mbar_wait(ready + 8 * s, ph, P.abort_flag, 324))) { dead = true; break; }
                    uint64_t da = desc_a0 + static_cast<uint64_t>(s * stage16 + it.shift0), db = desc_b0 + static_cast<uint64_t>(s * stage16);
                    const int ksteps = (cb + 1 < nbk[it.part]) ? 4 : klast[it.part];
                    ptx::wgmma_fence();
                    for (int tc = 0; tc < it.nb; ++tc, da += it.dshift, db += B_BYTES >> 4)
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
            if (dead) { stat_n0 = -1; break; }
            mma_epilogue<BLOCK_N, MODE>(P, acc, acc_stage, e, lane, m0, n0, s_stat);
        }
    } else if (warp > 8) {
        // ================================ fixers: zero the hole rows of every landed A tile ================================
        if (fix) {
            const int t = (warp - 9) * 32 + lane;
            int s = 0;
            uint32_t ph = 0;
            bool dead = false;
            // bit i of b0 / b1: row t / row t + 128 of item i's A tile is a hole (rows outside the image were zero-filled by TMA)
            auto load_bits = [&](int tl, uint64_t &b0, uint64_t &b1) {
                b0 = b1 = 0ull;
                if (tl >= num_tiles) return;
                const int m0 = (tl / n_tiles) * BLOCK_M;
                const int img = m0 / plane, rem = m0 - img * plane;
                const int oy = rem / gw, ox = rem - oy * gw;
                for (int i = 0; i < TB.n_items; ++i) {
                    const SpItem it = TB.it[i];
                    const uint8_t *mk = P.parts[it.part].mask;
                    if (mk == nullptr) continue;
                    const int pwid = TB.pw[it.part], phei = TB.ph[it.part], es = TB.es[it.part];
                    const int hrows = TB.arows[it.part] - BLOCK_M;
                    const int x0 = ox * TB.step[it.part] + it.dx, y0 = oy * TB.step[it.part] + it.dy;
                    int tx, ty, tn;
                    if (hrows > 0 || (P.box_h == 1 && P.box_n == 1)) { tx = t; ty = 0; tn = 0; }
                    else { tx = t % P.box_w; ty = (t / P.box_w) % P.box_h; tn = t / (P.box_w * P.box_h); }
                    const int X = x0 + tx * es, Y = y0 + ty * es, IM = img + tn;
                    if (X >= 0 && X < pwid && Y >= 0 && Y < phei && IM < P.n &&
                        __ldg(mk + (static_cast<long long>(IM) * phei + Y) * pwid + X) == 0) b0 |= 1ull << i;
                    if (t < hrows) {
                        const int X1 = x0 + (t + 128) * es;
                        if (X1 >= 0 && X1 < pwid && Y >= 0 && Y < phei && __ldg(mk + (static_cast<long long>(IM) * phei + Y) * pwid + X1) == 0) b1 |= 1ull << i;
                    }
                }
            };
            uint64_t n0b, n1b;
            load_bits(tile0, n0b, n1b);
            for (int tile = tile0; tile < num_tiles && !dead; tile += tstep) {
                const uint64_t c0b = n0b, c1b = n1b;
                load_bits(tile + tstep, n0b, n1b);
                for (int i = 0; i < TB.n_items && !dead; ++i) {
                    const bool h0 = (c0b >> i) & 1ull, h1 = (c1b >> i) & 1ull;
                    const bool any_hole = __any_sync(0xffffffffu, h0 || h1);
                    const int nb_i = nbk[TB.it[i].part];
                    for (int cb = 0; cb < nb_i; ++cb) {
                        if (!ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 322)) { dead = true; break; }
                        if (any_hole) {
                            const uint4 z = make_uint4(0u, 0u, 0u, 0u);
                            if (h0) {
                                uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + t * 128);
#pragma unroll
                                for (int k = 0; k < 8; ++k) r[k] = z;
                            }
                            if (h1) {
                                uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + (t + 128) * 128);
#pragma unroll
                                for (int k = 0; k < 8; ++k) r[k] = z;
                            }
                            ptx::fence_proxy_async_smem();
                        }
                        __syncwarp();
                        if (lane == 0) ptx::mbar_arrive(bar_fixed + 8 * s);
                        if (++s == S) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
    }

    __syncthreads();
    if (s_stat != nullptr && stat_n0 >= 0) tc_stats_final<BLOCK_N>(P, s_stat - EpiRole<BLOCK_N>(warp).slice() * STAT_SLICE, warp, lane, stat_n0);
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
template <int BLOCK_N, int T>
__device__ __forceinline__ void wgrad_store(const WgParams &P, const float (&acc)[T][BLOCK_N / 2], int ntap, int lane, int n0,
                                            const int (&ci)[2], const int (&tap)[2][T]) {
    const int taps_full = P.kh * P.kw;
#pragma unroll
    for (int tl = 0; tl < T; ++tl) {
        if (tl >= ntap) break;
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) {
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
            wgrad_store<BLOCK_N, T>(P, acc, ntap, lane, n0, ci, tap);
        }
    }
}


// -------------------------------------------------------------------------------------------------
// weight gradient, TMA-FED.  Same GEMM as pconv_tc_wgrad_kernel (D[ci][co] per tap, K = output pixels, split-K with fp32
// red.global.add) but the gathered operand is no longer gathered: a K block of 64 consecutive output pixels is a box of the
// pixel grid, so the x rows of tap (tr, tc) / 64-channel block are one 4-D TMA tile (padding = out-of-range zero fill,
// stride-2 layers = traversal stride), written as exactly the MN-major 128B-swizzled block wgmma reads.  Holes are zeroed
// in the landed tile by four fixer warps (the tap-validity words of the block's pixels), which then run the epilogue.
//   HALO (stride 1, K block = one image-row segment): a CTA owns one kernel ROW; one tile of 64 + (kw-1)*dil pixel rows per
//   channel block serves the kw taps of the row through row-shifted descriptors (T = kw register accumulators).
//   otherwise: a CTA owns T taps, one tile per tap.
//   warps 0-7 consumer warpgroups (MMA, then epilogue) | warp 8 TMA producer | warps 9-12 fixers
// -------------------------------------------------------------------------------------------------
template <int BLOCK_N, int T, bool HALO>
__global__ void __launch_bounds__(WGRAD_THREADS, 1)
pconv_tc_wgrad_tma_kernel(const __grid_constant__ WgParams P, const __grid_constant__ CUtensorMap tmap_dc,
                          const __grid_constant__ CUtensorMap tmap_a0, const __grid_constant__ CUtensorMap tmap_a1) {
    constexpr uint32_t B_BYTES = BLOCK_N * 128;               // [64 px][BLOCK_N co] as BLOCK_N/64 blocks of 8 KB
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
    const bool fix = P.use_fix != 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < MAX_RING; ++s) { ptx::mbar_init(bar_full + 8 * s, 1); ptx::mbar_init(bar_fixed + 8 * s, 4); ptx::mbar_init(bar_empty + 8 * s, 2); }
        ptx::fence_mbar_init();
    }
    if (warp == 8 && lane == 0) { ptx::prefetch_tmap(&tmap_dc); ptx::prefetch_tmap(&tmap_a0); ptx::prefetch_tmap(&tmap_a1); }
    __syncthreads();

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
    } else if (warp < MMA_WARPS) {
        // ================================ consumer warpgroups: both operands MN-major ================================
        // warpgroup g takes the tile's 64-channel block g (nothing to compute when that block does not exist)
        const int g = warp >> 2;
        const bool leader = (threadIdx.x & 127) == 0, live = blk_part[g] >= 0;
        const uint32_t ready = fix ? bar_fixed : bar_full;
        const uint64_t desc_a0 = ptx::make_smem_desc(smem_base + g * A_BLK, A_BLK, 1024);
        const uint64_t desc_b0 = ptx::make_smem_desc(smem_base + A_BYTES, 8192, 1024);
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
            if (live) {
                uint64_t da = desc_a0 + static_cast<uint64_t>(s * stage16);
                const uint64_t db = desc_b0 + static_cast<uint64_t>(s * stage16);
                ptx::wgmma_fence();
#pragma unroll
                for (int tl = 0; tl < T; ++tl, da += tap16) {
                    if (tl >= ntap) break;
#pragma unroll
                    for (int k = 0; k < 4; ++k)                  // 16 pixels (two 8-row atoms = 2048 bytes) per step
                        ptx::wgmma_bf16<BLOCK_N, 1, 1>(acc[tl], da + 128 * k, db + 128 * k);
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();
            }
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
                const int kpos = ci_tile * 128 + 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * h;
                ci[h] = -1;
                for (int p = 0; p < P.nparts; ++p) {
                    const int local = kpos - P.parts[p].koff;
                    if (local >= 0 && local < P.parts[p].c) ci[h] = P.parts[p].choff + local;
                }
#pragma unroll
                for (int tl = 0; tl < T; ++tl) tap[h][tl] = tap0 + tl;
            }
            wgrad_store<BLOCK_N, T>(P, acc, ntap, lane, n0, ci, tap);
        }
    } else {
        // ================================ fixers (hole rows -> 0) ================================
        const int f = (warp - 9) * 32 + lane;                   // pixel row of the A blocks owned by this thread
        if (fix) {
            // tap-validity word of the output pixel that looks at this row (halo rows past 63 belong to a later tap column)
            int jpix = f, tcs = 0;
            if (HALO && f > 63) { tcs = (f - 63 + P.dil - 1) / P.dil; jpix = f - tcs * P.dil; }
            const bool row_used = f < rows_a;
            uint64_t wnext[2];
            auto load_words = [&](int kb) {
                const int m = kb * 64 + jpix;
#pragma unroll
                for (int hb = 0; hb < 2; ++hb)
                    wnext[hb] = (row_used && blk_part[hb] >= 0 && m < P.m_total && kb < kb_begin + num_kb) ? __ldg(P.parts[blk_part[hb]].tapmask + m) : 0ull;
            };
            load_words(kb_begin);
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < num_kb; ++it) {
                const uint64_t w0 = wnext[0], w1 = wnext[1];
                load_words(kb_begin + it + 1);
                if (!__all_sync(0xffffffffu, ptx::mbar_wait(bar_full + 8 * s, ph, P.abort_flag, 222))) break;
                bool wrote = false;
                if (row_used) {
                    for (int tl = 0; tl < (HALO ? 1 : ntap); ++tl) {
                        const int bit = HALO ? tap_group * P.kw + tcs : tap0 + tl;
#pragma unroll
                        for (int hb = 0; hb < 2; ++hb) {
                            if (blk_part[hb] < 0) continue;
                            if ((((hb ? w1 : w0) >> bit) & 1ull) == 0ull) {
                                uint4 *r = reinterpret_cast<uint4 *>(smem_gen + s * STAGE + (tl * 2 + hb) * A_BLK + f * 128);
                                const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
                                for (int k = 0; k < 8; ++k) r[k] = z;
                                wrote = true;
                            }
                        }
                    }
                }
                if (__any_sync(0xffffffffu, wrote)) ptx::fence_proxy_async_smem();
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

void base_params(TcParams &P, const pcb_conv *c, const Layout &L) {
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.cin = c->cin; P.cout = c->cout; P.kh = c->kh; P.kw = c->kw; P.stride = c->stride;
    P.pad_h = c->pad_h; P.pad_w = c->pad_w; P.dil = c->dil; P.ho = c->ho; P.wo = c->wo;
    P.nparts = c->nparts; P.no_guard = c->no_guard; P.rowpack = L.rowpack; P.ktap = L.ktap;
    P.sub = 1; P.py = 0; P.px = 0; P.fh = c->h; P.fw = c->w;
    P.l2pf = getenv("PCB_TMA_L2_PREFETCH") != nullptr;
}

// row-halo eligibility: stride 1, output rows made of whole groups of 8 pixels, halo small enough
int halo_hg(const pcb_conv *c, bool rowpack) {
    if (rowpack || c->stride != 1 || getenv("PCB_DISABLE_HALO")) return 0;
    const int hg = 8 + (c->kw - 1) * c->dil;
    if (c->kw < 2 || hg > HALO_MAX_HG || c->kh > 8) return 0;
    if (c->wo % 8 != 0 || c->w % 8 != 0 || c->wo != c->w) return 0;
    return hg;
}

// H100: 227 KB of shared memory per block.  The rings get what the epilogue staging tile, the statistics and the barriers leave.
constexpr size_t MAX_SMEM = 227 * 1024;
constexpr size_t RING_BUDGET = 208 * 1024;

template <int BLOCK_N, int MODE, bool HALO>
int launch_persistent(TcParams &P, const CUtensorMap &tm, cudaStream_t st) {
    const size_t a_stage = HALO ? ((8 * 16 * (16 * P.hg + 1) + 127) / 128 * 128) : A_STAGE_BYTES;
    const size_t b_stage = BLOCK_N * 128;
    const size_t budget = RING_BUDGET - acc_stage_bytes(BLOCK_N);
    P.ring_b = 6;
    P.ring_a = HALO ? 3 : 6;
    while (P.ring_a * a_stage + P.ring_b * b_stage > budget && P.ring_b > 3) --P.ring_b;
    while (P.ring_a * a_stage + P.ring_b * b_stage > budget && P.ring_a > 2) --P.ring_a;
    const size_t smem = 1024 + P.ring_a * a_stage + P.ring_b * b_stage + 32 * MAX_RING + 16 + STAT_SMEM_BYTES + acc_stage_bytes(BLOCK_N);
    PCB_CHECK(smem <= MAX_SMEM, "tensor-core conv: %zu bytes of shared memory do not fit", smem);
    auto kern = pconv_tc_persistent_kernel<BLOCK_N, MODE, HALO>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    const int num_tiles = ((P.m_total + BLOCK_M - 1) / BLOCK_M) * (P.ncols / BLOCK_N);
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, PERSIST_THREADS, smem, st>>>(P, tm);
    PCB_LAUNCH_CHECK();
    return 0;
}


// ---- split-K: scratch buffer and finish kernels --------------------------------------------------
// (opt-in debug path, PCB_SPLITK=1: one scratch buffer per device, single host thread / stream per device assumed)
float *splitk_scratch(size_t bytes) {
    static float *buf[PCB_MAX_DEVICES] = {};
    static size_t cap[PCB_MAX_DEVICES] = {};
    const int dev = pcb_cur_device();
    if (bytes > cap[dev]) {
        // the previous (smaller) buffer is deliberately not freed: a captured CUDA graph may still point into it
        const size_t want = std::max<size_t>(bytes, 16u << 20);
        float *fresh = nullptr;
        if (cudaMalloc(&fresh, want) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        buf[dev] = fresh; cap[dev] = want;
    }
    return buf[dev];
}

// y = hole ? 0 : acc / s + b over [m_total][y_cstride] (8 channels per thread)
__global__ void splitk_finish_fwd_kernel(const float *__restrict__ part, int ncols, const float *__restrict__ msum, const float *__restrict__ bias, int cout,
                                         int no_guard, long long m_total, bf16 *__restrict__ y, int y_cstride) {
    const int cv = y_cstride >> 3;
    const long long total = m_total * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long m = i / cv;
        const int col = static_cast<int>(i - m * cv) * 8;
        const float s = msum ? msum[m] : 1.f;
        const bool hole = (s == 0.f) && !no_guard;
        const float inv = hole ? 0.f : 1.0f / s;
        uint4 o;
        __nv_bfloat162 *ob = reinterpret_cast<__nv_bfloat162 *>(&o);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int co = col + 2 * j;
            float a = (co < ncols) ? part[m * ncols + co] : 0.f, b = (co + 1 < ncols) ? part[m * ncols + co + 1] : 0.f;
            a = (hole || co >= cout) ? 0.f : a * inv + (bias ? bias[co] : 0.f);
            b = (hole || co + 1 >= cout) ? 0.f : b * inv + (bias ? bias[co + 1] : 0.f);
            ob[j] = __floats2bfloat162_rn(a, b);
        }
        *reinterpret_cast<uint4 *>(y + m * y_cstride + col) = o;
    }
}

// dx_part = acc * input mask of the part (8 channels per thread); the tile grid may be a parity class of the gradient
__global__ void splitk_finish_dgrad_kernel(const float *__restrict__ part, const TcParams P) {
    const int cv = P.ncols >> 3;
    const long long total = static_cast<long long>(P.m_total) * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i / cv);
        const int col = static_cast<int>(i - static_cast<long long>(m) * cv) * 8;
        const int en = m / (P.h * P.w), rem = m - en * P.h * P.w;
        const int eh = (rem / P.w) * P.sub + P.py, ew = (rem % P.w) * P.sub + P.px;
        const long long mo = (static_cast<long long>(en) * P.fh + eh) * P.fw + ew;
        for (int p = 0; p < P.nparts; ++p) {
            const TcPart &pt = P.parts[p];
            const int local = col - pt.koff;
            if (local < 0 || local >= pt.c8 || pt.dx == nullptr) continue;
            float scale = 1.f;
            if (pt.mask != nullptr)
                scale = pt.mask[(static_cast<long long>(en) * (P.fh >> pt.mup) + (eh >> pt.mup)) * (P.fw >> pt.mup) + (ew >> pt.mup)] ? 1.f : 0.f;
            const float *src = part + static_cast<long long>(m) * P.ncols + col;
            uint4 o;
            __nv_bfloat162 *ob = reinterpret_cast<__nv_bfloat162 *>(&o);
#pragma unroll
            for (int j = 0; j < 4; ++j) ob[j] = __floats2bfloat162_rn(src[2 * j] * scale, src[2 * j + 1] * scale);
            *reinterpret_cast<uint4 *>(pt.dx + mo * pt.dx_cstride + local) = o;
        }
    }
}

// how many CTAs should share the K loop of one output tile
int pick_ksplit(long long m_total, int ncols, int bn, int blocks_per_tap) {
    // the shorter K loop of the low-resolution layers is paid back by the memset + finish kernels, so the split is opt-in
    // (PCB_SPLITK=1; the parity tests set it)
    if (!getenv("PCB_SPLITK")) return 1;
    const long long tiles = ((m_total + BLOCK_M - 1) / BLOCK_M) * (ncols / bn);
    const int sms = pcb_num_sms();
    if (tiles * 2 > sms) return 1;
    int ks = static_cast<int>(std::min<long long>(16, sms / tiles));
    ks = std::min(ks, blocks_per_tap);                   // every split keeps at least one K block per tap
    return ks < 2 ? 1 : ks;
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

bool tma_fwd_ok(const pcb_conv *c) {
    if (getenv("PCB_DISABLE_TMA") || is_rowpack(c)) return false;
    int bw, bh, bn;
    if (!tile_box(c->wo, c->ho, &bw, &bh, &bn)) return false;
    if (c->stride > 2 || bw * c->stride > 256 || bh * c->stride > 256) return false;
    for (int p = 0; p < c->nparts; ++p)
        if (c->parts[p].x_up && ((c->h | c->w) & 1)) return false;
    return true;
}

bool tma_dgrad_ok(const pcb_conv *c) {
    if (getenv("PCB_DISABLE_TMA") || is_rowpack(c) || c->stride != 1) return false;
    int bw, bh, bn;
    return tile_box(c->w, c->h, &bw, &bh, &bn);
}

// stride-2 data gradient as four stride-1 parity-class problems (see pcb_tc_dgrad)
bool tma_dgrad_s2_ok(const pcb_conv *c) {
    if (getenv("PCB_DISABLE_TMA") || getenv("PCB_DISABLE_TMA_S2") || is_rowpack(c)) return false;
    if (c->stride != 2 || c->dil != 1 || c->kh < 2 || c->kw < 2 || ((c->h | c->w) & 1) || c->ho != c->h / 2 || c->wo != c->w / 2) return false;
    int bw, bh, bn;
    return tile_box(c->w / 2, c->h / 2, &bw, &bh, &bn);
}

size_t up_bytes(const pcb_conv *c, int p) {
    return (static_cast<size_t>(c->n) * c->h * c->w * rup(c->parts[p].c, 8) * 2 + 255) / 256 * 256;
}
size_t tapmask_bytes(const pcb_conv *c) {
    return (static_cast<size_t>(c->nparts) * c->n * c->ho * c->wo * sizeof(uint64_t) + 255) / 256 * 256;
}

template <int BLOCK_N, int MODE, bool HALO>
int launch_tma_n(TcParams &P, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, cudaStream_t st) {
    const int nb = HALO ? P.kw : 1;
    const size_t a_room = (static_cast<size_t>(BLOCK_M + (HALO ? (P.kw - 1) * P.dil : 0)) * 128 + 1023) / 1024 * 1024;
    const size_t stage = a_room + static_cast<size_t>(nb) * BLOCK_N * 128;
    P.stages = static_cast<int>(std::min<size_t>(MAX_RING, (RING_BUDGET - acc_stage_bytes(BLOCK_N)) / stage));
    PCB_CHECK(P.stages >= 2, "TMA-fed conv: stage of %zu bytes does not fit twice", stage);
    const size_t smem = 1024 + P.stages * stage + 24 * MAX_RING + 16 + STAT_SMEM_BYTES + acc_stage_bytes(BLOCK_N);
    auto kern = pconv_tc_tma_kernel<BLOCK_N, MODE, HALO>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    if (P.ksplit < 1) P.ksplit = 1;
    const int m_tiles = (P.m_total + BLOCK_M - 1) / BLOCK_M;
    const int num_tiles = m_tiles * (P.ncols / BLOCK_N) * P.ksplit;
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, TMA_THREADS, smem, st>>>(P, tw, ta0, ta1);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <int MODE>
int launch_tma(TcParams &P, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, int bn, bool halo, cudaStream_t st) {
    if (halo) {
        if (bn == 128) return launch_tma_n<128, MODE, true>(P, tw, ta0, ta1, st);
        if (bn == 64) return launch_tma_n<64, MODE, true>(P, tw, ta0, ta1, st);
        return launch_tma_n<32, MODE, true>(P, tw, ta0, ta1, st);
    }
    if (bn == 128) return launch_tma_n<128, MODE, false>(P, tw, ta0, ta1, st);
    if (bn == 64) return launch_tma_n<64, MODE, false>(P, tw, ta0, ta1, st);
    return launch_tma_n<32, MODE, false>(P, tw, ta0, ta1, st);
}

// at least three stages of (halo tile of 128 + (kw-1)*dil pixel rows + kw weight tiles) fit in shared memory next to the
// epilogue staging tile of an N tile of block_n columns
bool halo_stages_fit(int kw, int dil, int block_n) {
    const size_t stage = (static_cast<size_t>(128 + (kw - 1) * dil) * 128 + 1023) / 1024 * 1024 + static_cast<size_t>(kw) * block_n * 128;
    return 3 * stage + acc_stage_bytes(block_n) <= RING_BUDGET;
}

// halo tiles: stride 1, the M tile is one image-row segment, a kernel row's halo fits the 256-pixel TMA box, and the stages fit
bool tma_halo_ok(const pcb_conv *c, int bw, int bh, int bn, int block_n) {
    if (getenv("PCB_DISABLE_TMA_HALO")) return false;
    if (!(c->stride == 1 && bw == 128 && bh == 1 && bn == 1 && c->kw >= 2 && 128 + (c->kw - 1) * c->dil <= 256 && c->kh <= 8)) return false;
    return halo_stages_fit(c->kw, c->dil, block_n);
}

// widest N tile that divides `cols` and still leaves at least one tile per SM; low-resolution layers (a handful of M tiles
// against a multi-megabyte weight matrix) get NARROWER N tiles: each CTA's operand stream is latency-bound (a ring of a few
// stages), so the time of such a layer is (bytes per CTA) / that rate -- more, smaller CTAs stream the weights in parallel
// (at most 128 columns: a consumer warpgroup holds 64 rows x N fp32 accumulators in registers)
int pick_bn(int cols, long long m_total) {
    const long long m_tiles = (m_total + BLOCK_M - 1) / BLOCK_M;
    if (cols <= 32) return 32;
    int bn = (cols % 128 == 0) ? 128 : 64;
    if (!getenv("PCB_NO_NARROW_N"))
        while (bn > 32 && cols % (bn / 2) == 0 && m_tiles * (cols / bn) < pcb_num_sms() / 2) bn /= 2;
    return bn;
}

template <int MODE>
int launch_tc(TcParams &P, const CUtensorMap &tm, int bn, cudaStream_t st) {
    if (P.hg) return (bn == 128) ? launch_persistent<128, MODE, true>(P, tm, st) : launch_persistent<64, MODE, true>(P, tm, st);
    return (bn == 128) ? launch_persistent<128, MODE, false>(P, tm, st) : launch_persistent<64, MODE, false>(P, tm, st);
}

}  // namespace

static bool smallco_ok(const pcb_conv *c);
namespace {

// ---- sub-pixel path: plan, weights, launches -------------------------------------------------------
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
    bool ok;                         // geometry admits the decomposition
    bool fwd, dgrad;                 // which passes use it (see sp_plan)
    int pu, ps;                      // the upsampled part and the other one (-1: none)
    SpAxis ay, ax;
    int net[4], eoff[4], net_total;  // effective taps of the upsampled part per class (class = py * 2 + px)
    int kext_u, kext_s, c8_u, c8_s;
    long long kc[4], clsoff[4], sp_fwd_elems, sp_dg_elems, kd_sp;
    int bw, bh, bn;                  // M tile box of the class grid [n][h/2][w/2]
};

SpPlan sp_plan(const pcb_conv *c) {
    SpPlan S;
    memset(&S, 0, sizeof(S));
    S.pu = S.ps = -1;
    if (getenv("PCB_DISABLE_SUBPIXEL") || getenv("PCB_DISABLE_TMA") || !common_ok(c) || is_rowpack(c)) return S;
    if (c->stride != 1 || c->ho != c->h || c->wo != c->w || ((c->h | c->w) & 1) || c->nparts > 2) return S;
    for (int p = 0; p < c->nparts; ++p) {
        if (c->parts[p].x_up) { if (S.pu >= 0) return S; S.pu = p; }
        else { if (S.ps >= 0) return S; S.ps = p; }
    }
    if (S.pu < 0) return S;
    // the hole mask of each part must live at the part's own resolution (HoleMask.upsampled keeps them together)
    if (c->parts[S.pu].mask && c->parts[S.pu].mask_up != 1) return S;
    if (S.ps >= 0 && c->parts[S.ps].mask && c->parts[S.ps].mask_up != 0) return S;
    if (smallco_ok(c)) return S;
    S.ay = sp_axis(c->kh, c->dil, c->pad_h);
    S.ax = sp_axis(c->kw, c->dil, c->pad_w);
    if (!S.ay.ok || !S.ax.ok) return S;
    if (!tile_box(c->w / 2, c->h / 2, &S.bw, &S.bh, &S.bn)) return S;
    const Layout L = layout_of(c);
    S.kext_u = L.kext[S.pu]; S.c8_u = rup(c->parts[S.pu].c, 8);
    S.kext_s = S.ps >= 0 ? L.kext[S.ps] : 0; S.c8_s = S.ps >= 0 ? rup(c->parts[S.ps].c, 8) : 0;
    const int taps = c->kh * c->kw;
    long long off = 0;
    int eo = 0;
    for (int cls = 0; cls < 4; ++cls) {
        S.net[cls] = S.ay.ne[cls >> 1] * S.ax.ne[cls & 1];
        S.eoff[cls] = eo; eo += S.net[cls];
        S.kc[cls] = static_cast<long long>(S.net[cls]) * S.kext_u + static_cast<long long>(S.ps >= 0 ? taps : 0) * S.kext_s;
        S.clsoff[cls] = off; off += static_cast<long long>(L.rows_f) * S.kc[cls];
        // worst-case item count of one class launch (no halo re-use)
        if (S.net[cls] + (S.ps >= 0 ? taps : 0) > SP_MAX_ITEMS) return S;
    }
    S.net_total = eo;
    if (S.net_total > SP_MAX_ITEMS) return S;
    S.kd_sp = static_cast<long long>(S.net_total) * L.cout64;
    S.ok = true;
    //  * DATA GRADIENT: one launch over the source grid replaces the full-resolution gradient of the upsampled part AND its 2x2
    //    reduction pass; it is used wherever the source grid has at least a third of a wave of tiles -- low-resolution layers keep
    //    the regular kernel (their launches are latency-bound either way).
    //  * FORWARD: 37 % fewer MMAs but MORE tile rows per output pixel (the skip part is read with a traversal stride of 2, which
    //    costs the TMA unit two rows per delivered row, and row-halo re-use is lost where the class grid is narrower than 128).
    //    Off by default (PCB_SUBPIXEL_FWD=1 enables it; parity-tested either way).
    const long long src_tiles = (static_cast<long long>(c->n) * (c->h / 2) * (c->w / 2) + BLOCK_M - 1) / BLOCK_M;
    S.dgrad = src_tiles >= pcb_num_sms() / 3 || getenv("PCB_SUBPIXEL_ALL") != nullptr;
    S.fwd = getenv("PCB_SUBPIXEL_FWD") != nullptr || getenv("PCB_SUBPIXEL_ALL") != nullptr;
    S.sp_fwd_elems = S.fwd ? off : 0;
    S.sp_dg_elems = S.dgrad ? static_cast<long long>(rup(S.kext_u, 128)) * S.kd_sp : 0;
    if (!S.fwd && !S.dgrad) S.ok = false;
    return S;
}

struct SpWParams {
    int cout, taps, cin, kw, cout64, rows_f;
    int choff_u, c_u, kext_u, choff_s, c_s, kext_s, has_skip;
    int net[4], eoff[4], nex[4], slot0[4];       // per class: eff taps, their prefix, eff columns, first slot index
    int ybits[2][4], xbits[2][4];
    long long kc[4], clsoff[4], kd_sp;
    int want_fwd, want_dg;
};

// slot = (class, effective tap of the upsampled part | original tap of the skip part); one block per (cout, slot)
__global__ void sp_weight_prepare_kernel(const float *__restrict__ wm, const SpWParams W, bf16 *__restrict__ w_f, bf16 *__restrict__ w_d) {
    const int co = blockIdx.x;
    int slot = blockIdx.y, cls = 0;
    while (cls < 3 && slot >= W.slot0[cls + 1]) ++cls;
    slot -= W.slot0[cls];
    const float *wrow = wm + static_cast<long long>(co) * W.taps * W.cin;
    if (slot < W.net[cls]) {
        const int ey = slot / W.nex[cls], ex = slot - ey * W.nex[cls];
        const int yb = W.ybits[cls >> 1][ey], xb = W.xbits[cls & 1][ex];
        for (int ci = threadIdx.x; ci < W.c_u; ci += blockDim.x) {
            float v = 0.f;
            for (int tr = 0; tr < 4; ++tr)
                if ((yb >> tr) & 1)
                    for (int tc = 0; tc < 4; ++tc)
                        if ((xb >> tc) & 1) v += wrow[static_cast<long long>(tr * W.kw + tc) * W.cin + W.choff_u + ci];
            const bf16 b = __float2bfloat16_rn(v);
            if (W.want_fwd) w_f[W.clsoff[cls] + static_cast<long long>(co) * W.kc[cls] + static_cast<long long>(slot) * W.kext_u + ci] = b;
            if (W.want_dg) w_d[static_cast<long long>(ci) * W.kd_sp + static_cast<long long>(W.eoff[cls] + slot) * W.cout64 + co] = b;
        }
    } else if (W.has_skip && W.want_fwd) {
        const int tap = slot - W.net[cls];
        for (int ci = threadIdx.x; ci < W.c_s; ci += blockDim.x)
            w_f[W.clsoff[cls] + static_cast<long long>(co) * W.kc[cls] + static_cast<long long>(W.net[cls]) * W.kext_u + static_cast<long long>(tap) * W.kext_s + ci] =
                __float2bfloat16_rn(wrow[static_cast<long long>(tap) * W.cin + W.choff_s + ci]);
    }
}

// dgrad-only variant: one block per (input channel of the upsampled part, slot), threads over cout -> coalesced writes of the
// transposed matrix (the master reads are strided but L2-resident)
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

int sp_weight_prepare(const pcb_conv *c, const SpPlan &S, const Layout &L, const float *w_master, bf16 *w_f, bf16 *w_d, cudaStream_t st) {
    SpWParams W;
    memset(&W, 0, sizeof(W));
    W.cout = c->cout; W.taps = c->kh * c->kw; W.cin = c->cin; W.kw = c->kw; W.cout64 = L.cout64; W.rows_f = L.rows_f;
    int off = 0;
    for (int p = 0; p < c->nparts; ++p) {
        if (p == S.pu) { W.choff_u = off; W.c_u = c->parts[p].c; }
        if (p == S.ps) { W.choff_s = off; W.c_s = c->parts[p].c; }
        off += c->parts[p].c;
    }
    W.kext_u = S.kext_u; W.kext_s = S.kext_s; W.has_skip = S.ps >= 0; W.kd_sp = S.kd_sp;
    W.want_fwd = S.fwd; W.want_dg = S.dgrad;
    int slot = 0;
    for (int cls = 0; cls < 4; ++cls) {
        W.net[cls] = S.net[cls]; W.eoff[cls] = S.eoff[cls]; W.nex[cls] = S.ax.ne[cls & 1]; W.slot0[cls] = slot;
        slot += S.net[cls] + (S.ps >= 0 ? W.taps : 0);
        W.kc[cls] = S.kc[cls]; W.clsoff[cls] = S.clsoff[cls];
    }
    for (int q = 0; q < 2; ++q)
        for (int e = 0; e < 4; ++e) { W.ybits[q][e] = S.ay.tapbits[q][e]; W.xbits[q][e] = S.ax.tapbits[q][e]; }
    if (S.fwd) {
        sp_weight_prepare_kernel<<<dim3(c->cout, slot), 128, 0, st>>>(w_master, W, w_f, w_d);
        PCB_LAUNCH_CHECK();
    } else if (S.dgrad) {
        sp_weight_dg_kernel<<<dim3(W.c_u, S.net_total), 128, 0, st>>>(w_master, W, w_d);
        PCB_LAUNCH_CHECK();
    }
    return 0;
}

// sub-pixel tiles are at most 64 columns wide: two stages of (A tile + up to four weight tiles) must fit next to the staging tile
int sp_bn(int cols, long long m_total) { return std::min(pick_bn(cols, m_total), 64); }

template <int BLOCK_N, int MODE>
int launch_sp_n(TcParams &P, const SpTable &TB, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, cudaStream_t st) {
    int nb_max = 1;
    for (int i = 0; i < TB.n_items; ++i) nb_max = std::max(nb_max, TB.it[i].nb);
    const size_t a_room = (static_cast<size_t>(TB.rows_max) * 128 + 1023) / 1024 * 1024;
    const size_t stage = a_room + static_cast<size_t>(nb_max) * BLOCK_N * 128;
    P.stages = static_cast<int>(std::min<size_t>(MAX_RING, (RING_BUDGET - acc_stage_bytes(BLOCK_N)) / stage));
    PCB_CHECK(P.stages >= 2, "sub-pixel conv: stage of %zu bytes does not fit twice", stage);
    const size_t smem = 1024 + P.stages * stage + 24 * MAX_RING + 16 + STAT_SMEM_BYTES + acc_stage_bytes(BLOCK_N);
    auto kern = pconv_tc_sp_kernel<BLOCK_N, MODE>;
    PCB_SMEM_OPT_IN(kern, MAX_SMEM);
    const int num_tiles = ((P.m_total + BLOCK_M - 1) / BLOCK_M) * (P.ncols / BLOCK_N);
    const int grid = std::min(num_tiles, pcb_num_sms());
    kern<<<grid, TMA_THREADS, smem, st>>>(P, TB, tw, ta0, ta1);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <int MODE>
int launch_sp(TcParams &P, const SpTable &TB, const CUtensorMap &tw, const CUtensorMap &ta0, const CUtensorMap &ta1, int bn, cudaStream_t st) {
    if (bn == 64) return launch_sp_n<64, MODE>(P, TB, tw, ta0, ta1, st);
    return launch_sp_n<32, MODE>(P, TB, tw, ta0, ta1, st);
}

// internal streams for the four class launches of low-resolution layers (one set per device and host thread)
struct ClassStreams4 { cudaStream_t aux[3]; cudaEvent_t ev_fork, ev_join[3]; bool ready; };
int class_streams(ClassStreams4 **out) {
    static thread_local ClassStreams4 cs_all[PCB_MAX_DEVICES] = {};
    ClassStreams4 &CS = cs_all[pcb_cur_device()];
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

// forward over cat([up2x(x_u), x_s]): four class launches (see pconv_tc_sp_kernel)
int sp_forward(const pcb_conv *c, const SpPlan &S, const Layout &L, const bf16 *w_sp, const float *bias, void *y, int y_cstride, const float *msum,
               double *bn_sums, int *flag, cudaStream_t st) {
    const int hc = c->h / 2, wc = c->w / 2;
    const long long m_class = static_cast<long long>(c->n) * hc * wc;
    TcParams P;
    base_params(P, c, L);
    fill_parts(c, L, P.parts, nullptr, 0);
    P.ho = hc; P.wo = wc; P.m_total = static_cast<int>(m_class);
    P.sub = 2; P.fh = c->ho; P.fw = c->wo;
    P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride; P.abort_flag = flag;
    P.bn_sums = bn_sums; P.bn_c = c->cout;
    P.box_w = S.bw; P.box_h = S.bh; P.box_n = S.bn;
    const int cols = (c->cout <= 32) ? 32 : L.rows_f;
    const int bn = sp_bn(cols, m_class);
    P.ncols = cols;
    for (int p = 0; p < c->nparts; ++p)
        if (c->parts[p].mask) P.use_fix = 1;
    const bool row_tiles = S.bw == 128 && S.bh == 1 && S.bn == 1;       // halo re-use possible for the traversal-stride-1 part
    const int taps = c->kh * c->kw;
    const long long class_tiles = ((m_class + BLOCK_M - 1) / BLOCK_M) * (cols / bn);
    const bool fork = class_tiles < pcb_num_sms() && !getenv("PCB_DISABLE_CLASS_STREAMS");
    ClassStreams4 *CS = nullptr;
    if (fork) {
        if (int rc = class_streams(&CS)) return rc;
        PCB_CUDA(cudaEventRecord(CS->ev_fork, st));
    }
    for (int cls = 0; cls < 4; ++cls) {
        const int py = cls >> 1, px = cls & 1;
        const int ney = S.ay.ne[py], nex = S.ax.ne[px], ey0 = S.ay.e0[py], ex0 = S.ax.e0[px];
        SpTable TB;
        memset(&TB, 0, sizeof(TB));
        const int pu = S.pu, ps = S.ps;
        TB.step[pu] = 1; TB.es[pu] = 1; TB.ph[pu] = hc; TB.pw[pu] = wc;
        const bool halo_u = row_tiles && nex > 1 && !getenv("PCB_DISABLE_TMA_HALO");
        TB.arows[pu] = BLOCK_M + (halo_u ? nex - 1 : 0);
        int ni = 0;
        for (int e = 0; e < ney; ++e) {
            if (halo_u) {
                SpItem &it = TB.it[ni++];
                it.part = pu; it.dx = ex0; it.dy = ey0 + e; it.nb = nex; it.wk = (e * nex) * S.kext_u; it.wk_step = S.kext_u; it.shift0 = 0; it.dshift = 8;
            } else {
                for (int f = 0; f < nex; ++f) {
                    SpItem &it = TB.it[ni++];
                    it.part = pu; it.dx = ex0 + f; it.dy = ey0 + e; it.nb = 1; it.wk = (e * nex + f) * S.kext_u; it.wk_step = 0; it.shift0 = 0; it.dshift = 0;
                }
            }
        }
        if (ps >= 0) {
            TB.step[ps] = 2; TB.es[ps] = 2; TB.ph[ps] = c->h; TB.pw[ps] = c->w;
            TB.arows[ps] = BLOCK_M;                                      // (a 129-pixel box at traversal stride 2 would exceed the 256-element TMA box limit)
            for (int tr = 0; tr < c->kh; ++tr)
                for (int tc = 0; tc < c->kw; ++tc) {
                    SpItem &it = TB.it[ni++];
                    it.part = ps; it.dx = px + tc * c->dil - c->pad_w; it.dy = py + tr * c->dil - c->pad_h; it.nb = 1;
                    it.wk = S.net[cls] * S.kext_u + (tr * c->kw + tc) * S.kext_s; it.wk_step = 0; it.shift0 = 0; it.dshift = 0;
                }
        }
        TB.n_items = ni;
        TB.rows_max = std::max(TB.arows[pu], ps >= 0 ? TB.arows[ps] : 0);
        PCB_CHECK(ni <= SP_MAX_ITEMS, "sub-pixel conv: too many items");
        CUtensorMap ta[TC_MAX_PARTS], tw;
        memset(ta, 0, sizeof(ta));
        if (int rc = make_tmap_nhwc(&ta[pu], c->parts[pu].x, S.c8_u, wc, hc, c->n, c->parts[pu].x_cstride, S.bw + (halo_u ? nex - 1 : 0), S.bh, S.bn, 1)) return rc;
        if (ps >= 0) {
            if (int rc = make_tmap_nhwc(&ta[ps], c->parts[ps].x, S.c8_s, c->w, c->h, c->n, c->parts[ps].x_cstride, S.bw, S.bh, S.bn, 2)) return rc;
        } else ta[1 - pu] = ta[pu];
        if (int rc = make_tmap_2d(&tw, w_sp + S.clsoff[cls], L.rows_f, S.kc[cls], S.kc[cls], bn)) return rc;
        TcParams Q = P;
        Q.py = py; Q.px = px;
        cudaStream_t cs = (fork && cls > 0) ? CS->aux[cls - 1] : st;
        if (fork && cls > 0) PCB_CUDA(cudaStreamWaitEvent(cs, CS->ev_fork, 0));
        if (int rc = launch_sp<0>(Q, TB, tw, ta[0], ta[1], bn, cs)) return rc;
        if (fork && cls > 0) {
            PCB_CUDA(cudaEventRecord(CS->ev_join[cls - 1], cs));
            PCB_CUDA(cudaStreamWaitEvent(st, CS->ev_join[cls - 1], 0));
        }
    }
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
    const int bn = sp_bn(S.kext_u, m_src);
    SpTable TB;
    memset(&TB, 0, sizeof(TB));
    TB.step[0] = 2; TB.es[0] = 2; TB.ph[0] = c->ho; TB.pw[0] = c->wo; TB.arows[0] = BLOCK_M; TB.rows_max = BLOCK_M;
    int ni = 0;
    for (int cls = 0; cls < 4; ++cls) {
        const int py = cls >> 1, px = cls & 1;
        const int ney = S.ay.ne[py], nex = S.ax.ne[px];
        for (int e = 0; e < ney; ++e)
            for (int f = 0; f < nex; ++f) {
                SpItem &it = TB.it[ni++];
                it.part = 0; it.dx = px - 2 * (S.ax.e0[px] + f); it.dy = py - 2 * (S.ay.e0[py] + e); it.nb = 1;
                it.wk = (S.eoff[cls] + e * nex + f) * L.cout64; it.wk_step = 0; it.shift0 = 0; it.dshift = 0;
            }
    }
    TB.n_items = ni;
    CUtensorMap ta, tw;
    if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, S.bw, S.bh, S.bn, 2)) return rc;
    if (int rc = make_tmap_2d(&tw, w_sp_dg, rup(S.kext_u, 128), S.kd_sp, S.kd_sp, bn)) return rc;
    return launch_sp<1>(P, TB, tw, ta, ta, bn, st);
}

}  // namespace

static bool smallco_ok(const pcb_conv *c) { return common_ok(c) && !is_rowpack(c) && pcb_smallco_eligible(c); }
static pcb_smallco_layout smallco_layout(const Layout &L) {
    pcb_smallco_layout S;
    S.ktap = L.ktap; S.koff[0] = L.koff[0]; S.koff[1] = L.koff[1]; S.cout64 = L.cout64; S.kf = L.kf; S.kd = L.kd;
    return S;
}

// ---- eligibility / layouts -----------------------------------------------------------------------
bool pcb_tc_eligible(const pcb_conv *c) { return common_ok(c) && !getenv("PCB_DISABLE_TC"); }

static bool tma_wgrad_ok(const pcb_conv *c);

// kernel-to-row tails (conv_k2r.cu): their 1x1 operands follow the layer's regular ones, at 64-element boundaries
static void k2r_bases(const Layout &L, size_t *fe, size_t *de) {
    *fe = (static_cast<size_t>(L.rows_f) * L.kf + 63) / 64 * 64;
    *de = (static_cast<size_t>(rup(L.ktap, 128)) * L.kd + 63) / 64 * 64;
}

// space-to-depth stems (conv_stem.cu): the 4x4 problem's operand (+ staging) follows the row-packed operand
static bool stem_ok(const pcb_conv *c) { return common_ok(c) && is_rowpack(c) && pcb_stem_ok(c); }
static size_t stem_base(const Layout &L) { return (static_cast<size_t>(L.rows_f) * L.kf + 63) / 64 * 64; }

size_t pcb_tc_workspace(const pcb_conv *c) {
    if (smallco_ok(c) && pcb_k2r_ok(c)) return pcb_k2r_workspace(c);
    if (stem_ok(c)) return std::max(pcb_stem_workspace(c), tapmask_bytes(c));
    size_t bytes = tapmask_bytes(c);
    if (tma_fwd_ok(c) || tma_wgrad_ok(c))                // dense copies of the 2x-upsampled sources (TMA cannot replicate pixels)
        for (int p = 0; p < c->nparts; ++p)
            if (c->parts[p].x_up) bytes += up_bytes(c, p);
    return bytes;
}

void pcb_tc_weight_layout(const pcb_conv *c, size_t *fwd_elems, size_t *dgrad_elems) {
    const Layout L = layout_of(c);
    *fwd_elems = static_cast<size_t>(L.rows_f) * L.kf;
    *dgrad_elems = L.rowpack ? 0 : static_cast<size_t>(rup(L.ktap, 128)) * L.kd;
    // sub-pixel path (conv over a 2x-upsampled source): the per-class effective-tap matrices follow the regular operands
    const SpPlan S = sp_plan(c);
    if (S.ok) { *fwd_elems += static_cast<size_t>(S.sp_fwd_elems); *dgrad_elems += static_cast<size_t>(S.sp_dg_elems); }
    if (smallco_ok(c) && pcb_k2r_ok(c)) {
        size_t fb, db, fx, dx;
        k2r_bases(L, &fb, &db);
        pcb_k2r_weight_layout(c, &fx, &dx);
        *fwd_elems = fb + fx; *dgrad_elems = db + dx;
    }
    if (stem_ok(c)) *fwd_elems = stem_base(L) + pcb_stem_weight_extra(c);
}

// true when the data gradient of the 2x-upsampled part is delivered at that part's own (source) resolution
bool pcb_tc_subpixel(const pcb_conv *c) {
    if (smallco_ok(c)) return pcb_k2r_ok(c);
    const SpPlan S = sp_plan(c);
    return S.ok && S.dgrad;
}

int pcb_tc_weight_prepare(const pcb_conv *c, const float *w_master, void *w_fwd, void *w_dgrad, bool zero_padding, cudaStream_t st) {
    const Layout L = layout_of(c);
    size_t fe, de;
    pcb_tc_weight_layout(c, &fe, &de);
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
    if (!L.rowpack && W.taps <= 65535 && c->cout >= 32 && c->cin >= 32) {
        dim3 tg((c->cin + 31) / 32, (c->cout + 31) / 32, W.taps);
        tc_weight_prepare_tiled_kernel<<<tg, 256, 0, st>>>(w_master, W, static_cast<bf16 *>(w_fwd), (w_dgrad && de) ? static_cast<bf16 *>(w_dgrad) : nullptr);
        PCB_LAUNCH_CHECK();
        const SpPlan S = sp_plan(c);
        if (S.ok) {
            PCB_CHECK(w_dgrad != nullptr, "sub-pixel weights need the dgrad operand buffer");
            return sp_weight_prepare(c, S, L, w_master, static_cast<bf16 *>(w_fwd) + static_cast<size_t>(L.rows_f) * L.kf,
                                     static_cast<bf16 *>(w_dgrad) + static_cast<size_t>(rup(L.ktap, 128)) * L.kd, st);
        }
        return 0;
    }
    const long long total = static_cast<long long>(c->cout) * W.taps * c->cin;
    const int grid = static_cast<int>(std::min<long long>((total + 1023) / 1024, 8ll * pcb_num_sms()));
    tc_weight_prepare_kernel<<<grid < 1 ? 1 : grid, 256, 0, st>>>(w_master, W, static_cast<bf16 *>(w_fwd),
                                                                   (w_dgrad && de) ? static_cast<bf16 *>(w_dgrad) : nullptr);
    PCB_LAUNCH_CHECK();
    if (stem_ok(c)) return pcb_stem_weight_prepare(c, w_master, static_cast<bf16 *>(w_fwd) + stem_base(L), zero_padding, st);
    if (smallco_ok(c) && pcb_k2r_ok(c)) {
        PCB_CHECK(w_dgrad != nullptr, "kernel-to-row weights need the dgrad operand buffer");
        size_t fb, db;
        k2r_bases(L, &fb, &db);
        return pcb_k2r_weight_prepare(c, w_master, static_cast<bf16 *>(w_fwd) + fb, static_cast<bf16 *>(w_dgrad) + db, zero_padding, st);
    }
    const SpPlan S = sp_plan(c);
    if (S.ok) {
        PCB_CHECK(w_dgrad != nullptr, "sub-pixel weights need the dgrad operand buffer");
        return sp_weight_prepare(c, S, L, w_master, static_cast<bf16 *>(w_fwd) + static_cast<size_t>(L.rows_f) * L.kf,
                                 static_cast<bf16 *>(w_dgrad) + static_cast<size_t>(rup(L.ktap, 128)) * L.kd, st);
    }
    return 0;
}

// the part of the forward that only depends on the masks: tap-validity words for the kernels that want them
int pcb_tc_forward_mask_pass(const pcb_conv *c, uint64_t *tapmask, cudaStream_t st) {
    const long long m_total = static_cast<long long>(c->n) * c->ho * c->wo;
    PCB_CHECK(m_total < (1ll << 31), "problem too large");
    const Layout L = layout_of(c);
    if (smallco_ok(c) || stem_ok(c)) return 0;            // (the stem applies its mask in the space-to-depth pass)
    { const SpPlan S = sp_plan(c); if (S.ok && S.fwd) return 0; }   // sub-pixel forward: its fixers read the mask planes themselves
    bool any_mask = false;
    for (int p = 0; p < c->nparts; ++p) any_mask = any_mask || (c->parts[p].mask != nullptr);
    if (tma_fwd_ok(c) && !any_mask) return 0;            // no holes: TMA's out-of-range zero fill is all the validity there is
    if (tma_fwd_ok(c)) {                                  // row-halo tiles: the fixers read the mask planes themselves
        int bw, bh, bn;
        tile_box(c->wo, c->ho, &bw, &bh, &bn);
        if (tma_halo_ok(c, bw, bh, bn, pick_bn(c->cout <= 32 ? 32 : L.rows_f, m_total))) return 0;
    }
    return launch_tapmask(c, tapmask, st);
}

// true when pcb_tc_forward_ws accumulates the BatchNorm statistics of its output itself (tensor-core kernels, no split-K)
bool pcb_tc_fuses_bn_stats(const pcb_conv *c) {
    return pcb_tc_eligible(c) && !smallco_ok(c) && !getenv("PCB_SPLITK") && !getenv("PCB_DISABLE_FUSED_BN_STATS");
}

int pcb_tc_forward_ws(const pcb_conv *c, const void *w_fwd, const float *bias, void *y, int y_cstride, const float *msum,
                      uint64_t *tapmask, bool mask_pass_done, double *bn_sums, cudaStream_t st) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    const long long m_total = static_cast<long long>(c->n) * c->ho * c->wo;
    PCB_CHECK(m_total < (1ll << 31), "problem too large");
    PCB_CHECK(y_cstride % 8 == 0 && y_cstride >= c->cout, "tensor-core forward: y channel stride must be a multiple of 8 and >= cout");
    const Layout L = layout_of(c);
    if (!mask_pass_done)
        if (int rc = pcb_tc_forward_mask_pass(c, tapmask, st)) return rc;
    if (stem_ok(c)) {
        PCB_CHECK(bn_sums == nullptr || pcb_tc_fuses_bn_stats(c), "fused BatchNorm statistics requested from a kernel that does not produce them");
        return pcb_stem_forward(c, static_cast<const bf16 *>(w_fwd) + stem_base(L), bias, y, y_cstride, msum, tapmask, bn_sums, st);
    }
    if (smallco_ok(c)) {
        if (pcb_k2r_ok(c)) {
            size_t fb, db;
            k2r_bases(L, &fb, &db);
            return pcb_k2r_forward(c, smallco_layout(L), w_fwd, static_cast<const bf16 *>(w_fwd) + fb, bias, y, y_cstride, msum, tapmask, st);
        }
        return pcb_smallco_forward(c, smallco_layout(L), w_fwd, bias, y, y_cstride, msum, st);
    }
    {
        const SpPlan S = sp_plan(c);
        if (S.ok && S.fwd) {
            PCB_CHECK(bn_sums == nullptr || pcb_tc_fuses_bn_stats(c), "fused BatchNorm statistics requested from a kernel that does not produce them");
            return sp_forward(c, S, L, static_cast<const bf16 *>(w_fwd) + static_cast<size_t>(L.rows_f) * L.kf, bias, y, y_cstride, msum, bn_sums, flag, st);
        }
    }
    TcParams P;
    base_params(P, c, L);
    P.m_total = static_cast<int>(m_total);
    fill_parts(c, L, P.parts, tapmask, m_total);
    P.bias = bias; P.msum = msum; P.y = static_cast<bf16 *>(y); P.y_cstride = y_cstride; P.abort_flag = flag;
    PCB_CHECK(bn_sums == nullptr || pcb_tc_fuses_bn_stats(c), "fused BatchNorm statistics requested from a kernel that does not produce them");
    P.bn_sums = bn_sums; P.bn_c = c->cout;
    P.ncols = L.rows_f;
    CUtensorMap tm;
    if (tma_fwd_ok(c)) {
        tile_box(c->wo, c->ho, &P.box_w, &P.box_h, &P.box_n);
        const int bn = pick_bn(c->cout <= 32 ? 32 : L.rows_f, m_total);
        const bool halo = tma_halo_ok(c, P.box_w, P.box_h, P.box_n, bn);
        const int hx = halo ? (c->kw - 1) * c->dil : 0;
        CUtensorMap ta[TC_MAX_PARTS];
        memset(ta, 0, sizeof(ta));
        uint8_t *extra = reinterpret_cast<uint8_t *>(tapmask) + tapmask_bytes(c);
        for (int p = 0; p < c->nparts; ++p) {
            const pcb_part &pt = c->parts[p];
            const void *src = pt.x;
            long long cs = pt.x_cstride;
            const int c8 = rup(pt.c, 8);
            if (pt.x_up) {
                const long long pix = static_cast<long long>(c->n) * (c->h >> 1) * (c->w >> 1);
                const long long work = pix * (c8 >> 3);
                const int grid = static_cast<int>(std::min<long long>((work + 255) / 256, 16ll * pcb_num_sms()));
                upsample_part_kernel<<<grid, 256, 0, st>>>(static_cast<const bf16 *>(pt.x), pt.x_cstride, c8, pix, c->h >> 1, c->w >> 1, reinterpret_cast<bf16 *>(extra));
                PCB_LAUNCH_CHECK();
                src = extra; cs = c8;
                extra += up_bytes(c, p);
            }
            if (pt.mask) P.use_fix = 1;
            if (int rc = make_tmap_nhwc(&ta[p], src, c8, c->w, c->h, c->n, cs, P.box_w + hx, P.box_h, P.box_n, c->stride)) return rc;
        }
        if (c->nparts < 2) ta[1] = ta[0];
        P.ncols = (c->cout <= 32) ? 32 : L.rows_f;
        P.wk_base = 0; P.wk_col = L.ktap; P.wk_row = c->kw * L.ktap;
        if (int rc = make_tmap_2d(&tm, w_fwd, L.rows_f, L.kf, L.kf, bn)) return rc;
        P.ksplit = pick_ksplit(m_total, P.ncols, bn, L.ktap / BLOCK_K);
        if (P.ksplit > 1) {
            const size_t bytes = static_cast<size_t>(m_total) * P.ncols * sizeof(float);
            P.partial = splitk_scratch(bytes);
            PCB_CHECK(P.partial != nullptr, "split-K scratch allocation failed");
            PCB_CUDA(cudaMemsetAsync(P.partial, 0, bytes, st));
            if (int rc = launch_tma<0>(P, tm, ta[0], ta[1], bn, halo, st)) return rc;
            const long long work = m_total * (y_cstride / 8);
            splitk_finish_fwd_kernel<<<static_cast<int>(std::min<long long>((work + 255) / 256, 8ll * pcb_num_sms())), 256, 0, st>>>(
                P.partial, P.ncols, msum, bias, c->cout, c->no_guard, m_total, static_cast<bf16 *>(y), y_cstride);
            PCB_LAUNCH_CHECK();
            return 0;
        }
        return launch_tma<0>(P, tm, ta[0], ta[1], bn, halo, st);
    }
    if (int rc = make_tmap_2d(&tm, w_fwd, L.rows_f, L.kf, L.kf, L.bn_f)) return rc;
    P.hg = halo_hg(c, L.rowpack);
    return launch_tc<0>(P, tm, L.bn_f, st);
}

bool pcb_tc_dgrad_supported(const pcb_conv *c) { return pcb_tc_eligible(c) && !is_rowpack(c); }

int pcb_tc_dgrad(const pcb_conv *c, const void *dc, int dc_cstride, const void *w_dgrad, void *const *dx, const int *dx_cstride,
                 cudaStream_t st) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "cudaMalloc(abort flag) failed");
    const long long m_total = static_cast<long long>(c->n) * c->h * c->w;
    PCB_CHECK(m_total < (1ll << 31), "problem too large");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= rup(c->cout, 8), "tensor-core dgrad: dc channel stride must be a multiple of 8");
    const Layout L = layout_of(c);
    if (smallco_ok(c)) {
        if (pcb_k2r_ok(c)) {
            size_t fb, db;
            k2r_bases(L, &fb, &db);
            return pcb_k2r_dgrad(c, smallco_layout(L), dc, dc_cstride, w_dgrad, static_cast<const bf16 *>(w_dgrad) + db, dx, dx_cstride, st);
        }
        return pcb_smallco_dgrad(c, smallco_layout(L), dc, dc_cstride, w_dgrad, dx, dx_cstride, st);
    }
    // sub-pixel path: the gradient of the upsampled part is computed directly at source resolution (dx[pu] is a SOURCE-resolution
    // buffer, see pcb_conv_dgrad_at_source_resolution); the other part goes through the regular kernel below
    const SpPlan SPL = sp_plan(c);
    void *dx_local[TC_MAX_PARTS] = {nullptr, nullptr};
    for (int p = 0; p < c->nparts && p < TC_MAX_PARTS; ++p) dx_local[p] = dx[p];
    if (SPL.ok && SPL.dgrad) {
        if (dx[SPL.pu] != nullptr)
            if (int rc = sp_dgrad_up(c, SPL, L, dc, dc_cstride, static_cast<const bf16 *>(w_dgrad) + static_cast<size_t>(rup(L.ktap, 128)) * L.kd,
                                     dx[SPL.pu], dx_cstride[SPL.pu], flag, st)) return rc;
        dx_local[SPL.pu] = nullptr;
        if (SPL.ps < 0 || dx[SPL.ps] == nullptr) return 0;
    }
    dx = dx_local;
    TcParams P;
    base_params(P, c, L);
    P.m_total = static_cast<int>(m_total);
    fill_parts(c, L, P.parts, nullptr, 0);
    for (int p = 0; p < c->nparts; ++p) {
        P.parts[p].dx = static_cast<bf16 *>(dx[p]);
        P.parts[p].dx_cstride = dx_cstride[p];
        PCB_CHECK(!dx[p] || (dx_cstride[p] % 8 == 0 && dx_cstride[p] >= P.parts[p].c8 && (reinterpret_cast<uintptr_t>(dx[p]) & 15) == 0),
                  "tensor-core dgrad: dx[%d] must be 16-byte aligned with a channel stride that is a multiple of 8", p);
    }
    P.dc = static_cast<const bf16 *>(dc); P.dc_cstride = dc_cstride; P.dc_c8 = rup(c->cout, 8); P.dc_kext = L.cout64;
    P.abort_flag = flag;
    int bn = (L.ktap % 128 == 0) ? 128 : 64;
    P.ncols = L.ktap;
    CUtensorMap tm;
    if (tma_dgrad_ok(c)) {
        tile_box(c->w, c->h, &P.box_w, &P.box_h, &P.box_n);
        bn = pick_bn(L.ktap, m_total);
        const bool halo = tma_halo_ok(c, P.box_w, P.box_h, P.box_n, bn);
        P.wk_base = 0; P.wk_col = L.cout64; P.wk_row = c->kw * L.cout64;
        CUtensorMap ta;
        if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, P.box_w + (halo ? (c->kw - 1) * c->dil : 0), P.box_h, P.box_n, 1)) return rc;
        if (int rc = make_tmap_2d(&tm, w_dgrad, rup(L.ktap, 128), L.kd, L.kd, bn)) return rc;
        P.ksplit = pick_ksplit(m_total, P.ncols, bn, L.cout64 / BLOCK_K);
        if (P.ksplit > 1) {
            const size_t bytes = static_cast<size_t>(m_total) * P.ncols * sizeof(float);
            P.partial = splitk_scratch(bytes);
            PCB_CHECK(P.partial != nullptr, "split-K scratch allocation failed");
            PCB_CUDA(cudaMemsetAsync(P.partial, 0, bytes, st));
            if (int rc = launch_tma<1>(P, tm, ta, ta, bn, halo, st)) return rc;
            const long long work = m_total * (P.ncols / 8);
            splitk_finish_dgrad_kernel<<<static_cast<int>(std::min<long long>((work + 255) / 256, 8ll * pcb_num_sms())), 256, 0, st>>>(P.partial, P);
            PCB_LAUNCH_CHECK();
            return 0;
        }
        return launch_tma<1>(P, tm, ta, ta, bn, halo, st);
    }
    if (tma_dgrad_s2_ok(c)) {
        // Stride 2: an input pixel (y, x) only sees the taps with (y + pad - tr) even, so the four parity classes
        // (y & 1, x & 1) are four independent STRIDE-1 problems on the half-resolution grid -- which is dc's own grid --
        // each with its subset of taps (3x3 / 3x2 / 2x3 / 2x2 for a 5x5 kernel) and no multiplications by inserted zeros.
        const int hh = c->h / 2, hw = c->w / 2;
        const long long m_class = static_cast<long long>(c->n) * hh * hw;
        tile_box(hw, hh, &P.box_w, &P.box_h, &P.box_n);
        bn = pick_bn(L.ktap, m_class);
        if (int rc = make_tmap_2d(&tm, w_dgrad, rup(L.ktap, 128), L.kd, L.kd, bn)) return rc;
        // The classes write disjoint pixels.  When one class does not fill the GPU (low-resolution layers) the four launches
        // run concurrently: fork onto three internal streams after an event on `st`, join before returning (also valid
        // inside a stream capture: the internal streams join the capture and leave it again).
        const long long class_tiles = ((m_class + BLOCK_M - 1) / BLOCK_M) * (L.ktap / bn);
        const bool fork = class_tiles < pcb_num_sms() && !getenv("PCB_DISABLE_CLASS_STREAMS");
        // internal streams / events: one set per device AND per host thread (two host threads driving dgrads on two streams
        // must not share the fork / join events)
        struct ClassStreams { cudaStream_t aux[3]; cudaEvent_t ev_fork, ev_join[3]; bool ready; };
        static thread_local ClassStreams cs_all[PCB_MAX_DEVICES] = {};
        ClassStreams &CS = cs_all[pcb_cur_device()];
        cudaStream_t *aux = CS.aux;
        cudaEvent_t *ev_join = CS.ev_join;
        if (fork && !CS.ready) {
            for (int i = 0; i < 3; ++i) {
                PCB_CUDA(cudaStreamCreateWithFlags(&aux[i], cudaStreamNonBlocking));
                PCB_CUDA(cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming));
            }
            PCB_CUDA(cudaEventCreateWithFlags(&CS.ev_fork, cudaEventDisableTiming));
            CS.ready = true;
        }
        cudaEvent_t ev_fork = CS.ev_fork;
        if (fork) PCB_CUDA(cudaEventRecord(ev_fork, st));
        for (int cls = 0; cls < 4; ++cls) {
            TcParams Q = P;
            const int py = cls >> 1, px = cls & 1;
            const int tr0 = (py + c->pad_h) & 1, tc0 = (px + c->pad_w) & 1;
            Q.kh = (c->kh - tr0 + 1) / 2; Q.kw = (c->kw - tc0 + 1) / 2;
            Q.pad_h = (py + c->pad_h - tr0) / 2; Q.pad_w = (px + c->pad_w - tc0) / 2;
            Q.h = hh; Q.w = hw; Q.stride = 1; Q.dil = 1;
            Q.m_total = static_cast<int>(m_class);
            Q.sub = 2; Q.py = py; Q.px = px; Q.fh = c->h; Q.fw = c->w;
            Q.wk_base = (tr0 * c->kw + tc0) * L.cout64; Q.wk_row = 2 * c->kw * L.cout64; Q.wk_col = 2 * L.cout64;
            const bool halo = !getenv("PCB_DISABLE_TMA_HALO") && Q.box_w == 128 && Q.box_h == 1 && Q.box_n == 1 && Q.kw >= 2 &&
                              halo_stages_fit(Q.kw, 1, bn);
            CUtensorMap ta;
            if (int rc = make_tmap_nhwc(&ta, dc, P.dc_c8, c->wo, c->ho, c->n, dc_cstride, Q.box_w + (halo ? Q.kw - 1 : 0), Q.box_h, Q.box_n, 1)) return rc;
            cudaStream_t cs = (fork && cls > 0) ? aux[cls - 1] : st;
            if (fork && cls > 0) PCB_CUDA(cudaStreamWaitEvent(cs, ev_fork, 0));
            if (int rc = launch_tma<1>(Q, tm, ta, ta, bn, halo, cs)) return rc;
            if (fork && cls > 0) {
                PCB_CUDA(cudaEventRecord(ev_join[cls - 1], cs));
                PCB_CUDA(cudaStreamWaitEvent(st, ev_join[cls - 1], 0));
            }
        }
        return 0;
    }
    if (int rc = make_tmap_2d(&tm, w_dgrad, rup(L.ktap, 128), L.kd, L.kd, bn)) return rc;
    P.hg = halo_hg(c, L.rowpack);
    return launch_tc<1>(P, tm, bn, st);
}


// ---- TMA-fed weight gradient ---------------------------------------------------------------------
// 64 consecutive pixels of a [n][ht][wt] grid as a box {bw, bh, bn}
static bool kblock_box(int wt, int ht, int *bw, int *bh, int *bn) {
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

static bool tma_wgrad_ok(const pcb_conv *c) {
    if (getenv("PCB_DISABLE_TMA") || getenv("PCB_DISABLE_TMA_WGRAD") || is_rowpack(c) || c->stride > 2) return false;
    int bw, bh, bn;
    if (!kblock_box(c->wo, c->ho, &bw, &bh, &bn)) return false;
    for (int p = 0; p < c->nparts; ++p)
        if (c->parts[p].x_up && ((c->h | c->w) & 1)) return false;
    return true;
}

template <int BLOCK_N, int T, bool HALO>
int launch_wgrad_tma(WgParams &P, const CUtensorMap &tdc, const CUtensorMap &ta0, const CUtensorMap &ta1, cudaStream_t st) {
    const size_t a_blk = (static_cast<size_t>(64 + (HALO ? (P.kw - 1) * P.dil : 0)) * 128 + 1023) / 1024 * 1024;
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
    int splits = (2 * pcb_num_sms() + base_ctas - 1) / base_ctas;      // one CTA per SM at a time: ~2 waves
    splits = std::max(1, std::min(splits, total_kb));
    splits = std::min(splits, 65535);
    P.kb_per_split = (total_kb + splits - 1) / splits;
    splits = (total_kb + P.kb_per_split - 1) / P.kb_per_split;
    dim3 grid(base_ctas, splits);
    kern<<<grid, WGRAD_THREADS, smem, st>>>(P, tdc, ta0, ta1);
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
    const long long m_total = static_cast<long long>(c->n) * c->ho * c->wo;
    PCB_CHECK(m_total < (1ll << 31), "problem too large");
    PCB_CHECK(dc_cstride % 8 == 0 && dc_cstride >= c->cout, "tensor-core wgrad: dc channel stride must be a multiple of 8");
    if (stem_ok(c)) return pcb_stem_wgrad(c, dc, dc_cstride, dw, workspace, zero_dw, st);
    if (smallco_ok(c)) {
        if (pcb_k2r_ok(c)) return pcb_k2r_wgrad(c, dc, dc_cstride, dw, workspace, zero_dw, st);
        return pcb_smallco_wgrad(c, smallco_layout(layout_of(c)), dc, dc_cstride, dw, zero_dw, st);
    }
    uint64_t *tapmask = static_cast<uint64_t *>(workspace);
    bool any_mask = false;
    for (int p = 0; p < c->nparts; ++p) any_mask = any_mask || (c->parts[p].mask != nullptr);
    if (any_mask || !tma_wgrad_ok(c))                     // the TMA-fed kernel without holes needs no validity words
        if (int rc = launch_tapmask(c, tapmask, st)) return rc;
    const size_t dw_bytes = sizeof(float) * c->cout * c->kh * c->kw * c->cin;
    if (zero_dw) PCB_CUDA(cudaMemsetAsync(dw, 0, dw_bytes, st));
    const Layout L = layout_of(c);
    WgParams P;
    memset(&P, 0, sizeof(P));
    P.n = c->n; P.h = c->h; P.w = c->w; P.cin = c->cin; P.cout = c->cout; P.kh = c->kh; P.kw = c->kw; P.stride = c->stride;
    P.pad_h = c->pad_h; P.pad_w = c->pad_w; P.dil = c->dil; P.ho = c->ho; P.wo = c->wo; P.m_total = static_cast<int>(m_total);
    P.nparts = c->nparts; P.rowpack = L.rowpack; P.ktap = L.ktap; P.ntaps = L.rowpack ? c->kh : c->kh * c->kw;
    fill_parts(c, L, P.parts, tapmask, m_total);
    P.dw = dw; P.abort_flag = flag;
    CUtensorMap tm;
    if (int rc = make_tmap_2d(&tm, dc, m_total, c->cout, dc_cstride, 64)) return rc;
    if (tma_wgrad_ok(c)) {
        kblock_box(c->wo, c->ho, &P.box_w, &P.box_h, &P.box_n);
        // row-halo tiles for kw == 3: the three taps of a kernel row are three 64 x 64 register accumulators per consumer thread
        const bool halo = !getenv("PCB_DISABLE_TMA_HALO") && c->stride == 1 && c->kw == 3 && P.box_w == 64 &&
                          P.box_h == 1 && P.box_n == 1 && 64 + (c->kw - 1) * c->dil <= 256;
        const int hx = halo ? (c->kw - 1) * c->dil : 0;
        CUtensorMap ta[TC_MAX_PARTS];
        memset(ta, 0, sizeof(ta));
        uint8_t *extra = reinterpret_cast<uint8_t *>(workspace) + tapmask_bytes(c);
        for (int p = 0; p < c->nparts; ++p) {
            const pcb_part &pt = c->parts[p];
            const void *src = pt.x;
            long long cs = pt.x_cstride;
            const int c8 = rup(pt.c, 8);
            if (pt.x_up) {
                const long long pix = static_cast<long long>(c->n) * (c->h >> 1) * (c->w >> 1);
                const long long work = pix * (c8 >> 3);
                const int grid = static_cast<int>(std::min<long long>((work + 255) / 256, 16ll * pcb_num_sms()));
                upsample_part_kernel<<<grid, 256, 0, st>>>(static_cast<const bf16 *>(pt.x), pt.x_cstride, c8, pix, c->h >> 1, c->w >> 1, reinterpret_cast<bf16 *>(extra));
                PCB_LAUNCH_CHECK();
                src = extra; cs = c8;
                extra += up_bytes(c, p);
            }
            if (pt.mask) P.use_fix = 1;
            if (int rc = make_tmap_nhwc(&ta[p], src, c8, c->w, c->h, c->n, cs, P.box_w + hx, P.box_h, P.box_n, c->stride)) return rc;
        }
        if (c->nparts < 2) ta[1] = ta[0];
        if (halo) return launch_wgrad_tma<64, 3, true>(P, tm, ta[0], ta[1], st);
        return launch_wgrad_tma<64, 3, false>(P, tm, ta[0], ta[1], st);
    }
    return launch_wgrad<64, 3, 3>(P, tm, c->cout, st);
}

// abort flag query used by api.cu after synchronising debug runs
int pcb_tc_read_abort_flag(int *value) {
    int *flag = abort_flag_ptr();
    PCB_CHECK(flag != nullptr, "no abort flag");
    PCB_CUDA(cudaMemcpy(value, flag, sizeof(int), cudaMemcpyDeviceToHost));
    if (*value != 0) cudaMemset(flag, 0, sizeof(int));
    return 0;
}

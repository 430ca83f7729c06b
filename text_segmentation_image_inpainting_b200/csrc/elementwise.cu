// elementwise.cu -- the HBM-bound companions of the convolution: BatchNorm statistics / apply (+activation,
// +residual), their backward, the renormalisation backward, nearest-upsample + channel concat, mask format
// conversion, weight re-layout, L1-mean loss and SGD.  All NHWC, 16/32-byte vector accesses, one pass each.
#include "pcb_common.cuh"

namespace {

constexpr int EW_THREADS = 256;

// activation as a template parameter of the hot kernels: the per-element switch on a runtime code was a third of their
// instruction count (they are issue-bound before they are bandwidth-bound)
#define PCB_ACT_SWITCH(act_code, ...)                                                  \
    switch (act_code) {                                                                \
        case PCB_ACT_RELU: { constexpr int ACT = PCB_ACT_RELU; __VA_ARGS__; } break;   \
        case PCB_ACT_LEAKY: { constexpr int ACT = PCB_ACT_LEAKY; __VA_ARGS__; } break; \
        case PCB_ACT_RELU6: { constexpr int ACT = PCB_ACT_RELU6; __VA_ARGS__; } break; \
        default: { constexpr int ACT = PCB_ACT_NONE; __VA_ARGS__; } break;             \
    }

inline int ew_grid(long long work_items, int per_block, int blocks_per_sm = 16) {
    long long b = (work_items + per_block - 1) / per_block;
    const long long cap = static_cast<long long>(blocks_per_sm) * pcb_num_sms();
    return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

// reductions end in one fp64 atomic per channel per block: a few blocks per SM keep the loads in flight, thousands of
// blocks would serialise thousands of atomics on the same c addresses
inline int ew_grid_red(long long work_items, int per_block) {
    long long b = (work_items + per_block - 1) / per_block;
    const long long cap = 3ll * pcb_num_sms();                  // launch bounds (256, 3): exactly one resident wave
    return static_cast<int>(b < 1 ? 1 : (b > cap ? cap : b));
}

// ---------------------------------------------------------------------------------------------
// per-channel reductions over an NHWC tensor viewed as [count][c]; c % 8 == 0, c <= 2048.
// Thread layout: tid -> (row-in-block r = tid / cv, channel vector v = tid % cv), cv = c / 8.
// F(row, v, vals...) is evaluated per 8-vector; NRED fp32 partials per channel are block-reduced through
// shared memory and flushed with fp64 atomics.
// ---------------------------------------------------------------------------------------------
// All NRED partial sets are staged in shared memory at once and the cv*8 channel columns are summed by cv*8 threads in
// parallel (letting only the cv threads of row 0 walk all rows serially, twice, makes the tail of a block as long as its
// whole streaming phase).
template <int NRED>
__device__ __forceinline__ void block_flush(float (&acc)[NRED][8], int cv, int rpb, int r, int v, double *const (&out)[NRED]) {
    __shared__ float s_red[NRED][EW_THREADS][8];
    if (r < rpb) {
#pragma unroll
        for (int q = 0; q < NRED; ++q)
#pragma unroll
            for (int j = 0; j < 8; ++j) s_red[q][threadIdx.x][j] = acc[q][j];
    }
    __syncthreads();
    const int ncol = cv * 8;                                     // = c, at most 2048
    for (int col = threadIdx.x; col < ncol; col += EW_THREADS) {
        const int vv = col >> 3, jj = col & 7;
#pragma unroll
        for (int q = 0; q < NRED; ++q) {
            float tot = 0.f;
            for (int rr = 0; rr < rpb; ++rr) tot += s_red[q][rr * cv + vv][jj];
            atomicAdd(out[q] + col, static_cast<double>(tot));
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(EW_THREADS) bn_stats_kernel(const T *__restrict__ x, long long count, int c, double *sum, double *sqsum) {
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    float acc[2][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
    if (r < rpb) {
#pragma unroll 4
        for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += static_cast<long long>(gridDim.x) * rpb) {
            float f[8];
            Vec8<T>::load(x + row * c + v * 8, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) { acc[0][j] += f[j]; acc[1][j] += f[j] * f[j]; }
        }
    }
    double *const outs[2] = {sum, sqsum};
    block_flush<2>(acc, cv, rpb, r, v, outs);
}

// scalar fallback (any c): one block-wide pass, smem float atomics per channel (tiny tensors only)
template <typename T>
__global__ void bn_stats_scalar_kernel(const T *__restrict__ x, long long count, int c, double *sum, double *sqsum) {
    for (int ch = blockIdx.x; ch < c; ch += gridDim.x) {
        float a = 0.f, b = 0.f;
        for (long long row = threadIdx.x; row < count; row += blockDim.x) {
            const float f = to_f32(x[row * c + ch]);
            a += f; b += f * f;
        }
        __shared__ float sa[32], sb[32];
        a = warp_sum(a); b = warp_sum(b);
        if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = a; sb[threadIdx.x >> 5] = b; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double ta = 0, tb = 0;
            for (int i = 0; i < (blockDim.x >> 5); ++i) { ta += sa[i]; tb += sb[i]; }
            atomicAdd(sum + ch, ta); atomicAdd(sqsum + ch, tb);
        }
        __syncthreads();
    }
}

__global__ void bn_finalize_kernel(const double *sum, const double *sqsum, long long count, int c, const float *gamma,
                                   const float *beta, float *running_mean, float *running_var, long long *nbt, float momentum,
                                   float eps, int training, float *scale, float *shift, float *save_mean, float *save_invstd) {
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch == 0 && training && nbt) *nbt += 1;
    if (ch >= c) return;
    float mean, invstd;
    if (training) {
        const double m = sum[ch] / static_cast<double>(count);
        double var = sqsum[ch] / static_cast<double>(count) - m * m;     // biased (normalisation)
        if (var < 0) var = 0;
        mean = static_cast<float>(m);
        invstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
        if (running_mean) {
            const double unbiased = count > 1 ? var * static_cast<double>(count) / static_cast<double>(count - 1) : var;
            running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
            running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * static_cast<float>(unbiased);
        }
    } else {
        mean = running_mean[ch];
        invstd = 1.0f / sqrtf(running_var[ch] + eps);
    }
    const float g = gamma ? gamma[ch] : 1.f, b = beta ? beta[ch] : 0.f;
    scale[ch] = g * invstd;
    shift[ch] = b - mean * g * invstd;
    if (save_mean) save_mean[ch] = mean;
    if (save_invstd) save_invstd[ch] = invstd;
}

// Thread layout as in the reductions: tid -> (row-in-block, channel vector), so the per-channel coefficients are loaded once
// into registers instead of once per element (the element-wise passes were load-instruction bound, not bandwidth bound).
template <typename T>
__global__ void __launch_bounds__(EW_THREADS) bn_act_fwd_kernel(const T *__restrict__ x, long long count, int c, const float *__restrict__ scale,
                                                                const float *__restrict__ shift, int act, float slope,
                                                                const T *__restrict__ residual, T *__restrict__ y) {
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    if (r >= rpb) return;
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = scale ? scale[v * 8 + j] : 1.f; sh[j] = scale ? shift[v * 8 + j] : 0.f; }
    const long long step = static_cast<long long>(gridDim.x) * rpb;
#pragma unroll 2
    for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += step) {
        float f[8], rres[8];
        Vec8<T>::load(x + row * c + v * 8, f);
        if (residual) Vec8<T>::load(residual + row * c + v * 8, rres);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float z = scale ? f[j] * sc[j] + sh[j] : f[j];
            z = apply_act(z, act, slope);
            if (residual) z += rres[j];
            f[j] = z;
        }
        Vec8<T>::store(y + row * c + v * 8, f);
    }
}

// BatchNorm (training mode) finalisation + apply + activation in ONE launch: every thread derives the scale / shift of its
// 8 channels from the complete fp64 sums (produced by the convolution epilogue or pcb_bn_stats_acc), block 0 additionally
// updates the running statistics and writes the per-channel coefficients the backward needs.
//   coef: [4][c] floats = scale (gamma * invstd) | shift (beta - mean * scale) | mean | invstd
// (fp64 arithmetic is much slower than fp32: the coefficient prologue is done ONCE per channel and block, cooperatively, and
// handed to the threads through shared memory instead of every thread finalising its own 8 channels in fp64.)
template <typename T, int ACT>
__global__ void __launch_bounds__(EW_THREADS) bn_fwd_fused_kernel(const T *__restrict__ x, long long count, int c, const double *__restrict__ sums,
                                                                  const float *__restrict__ gamma, const float *__restrict__ beta,
                                                                  float *running_mean, float *running_var, long long *nbt, float momentum, float eps,
                                                                  int act, float slope, const T *__restrict__ residual, T *__restrict__ y,
                                                                  float *__restrict__ coef) {
    extern __shared__ float s_coef[];                                 // [2][c]: scale | shift
    const double inv_n = 1.0 / static_cast<double>(count);
    const bool writer = blockIdx.x == 0;
    if (writer && threadIdx.x == 0 && nbt) *nbt += 1;
    for (int ch = threadIdx.x; ch < c; ch += EW_THREADS) {
        const double m = sums[ch] * inv_n;
        double var = sums[c + ch] * inv_n - m * m;                    // biased (normalisation)
        if (var < 0) var = 0;
        const float mean = static_cast<float>(m), fvar = static_cast<float>(var);
        const float invstd = 1.0f / sqrtf(fvar + eps);                // fp32 like torch's batch_norm kernels
        const float g = gamma ? gamma[ch] : 1.f, b = beta ? beta[ch] : 0.f;
        const float sc = g * invstd, sh = b - mean * g * invstd;
        s_coef[ch] = sc; s_coef[c + ch] = sh;
        if (writer) {
            coef[ch] = sc; coef[c + ch] = sh; coef[2 * c + ch] = mean; coef[3 * c + ch] = invstd;
            if (running_mean) {
                const float unbiased = count > 1 ? fvar * (static_cast<float>(count) / static_cast<float>(count - 1)) : fvar;
                running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
                running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * unbiased;
            }
        }
    }
    __syncthreads();
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    if (r >= rpb) return;
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = s_coef[v * 8 + j]; sh[j] = s_coef[c + v * 8 + j]; }
    const long long step = static_cast<long long>(gridDim.x) * rpb;
    const T *px = x + v * 8;
    const T *pr = residual ? residual + v * 8 : nullptr;
    T *py = y + v * 8;
#pragma unroll 4
    for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += step) {
        float f[8], rres[8];
        Vec8<T>::load(px + row * c, f);
        if (pr) Vec8<T>::load(pr + row * c, rres);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float z = apply_act(f[j] * sc[j] + sh[j], ACT, slope);
            if (pr) z += rres[j];
            f[j] = z;
        }
        Vec8<T>::store(py + row * c, f);
    }
}

template <typename T>
__global__ void bn_act_fwd_scalar_kernel(const T *x, long long numel, int c, const float *scale, const float *shift, int act,
                                         float slope, const T *residual, T *y) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % c);
        float z = to_f32(x[i]);
        if (scale) z = z * scale[ch] + shift[ch];
        z = apply_act(z, act, slope);
        if (residual) z += to_f32(residual[i]);
        y[i] = from_f32<T>(z);
    }
}

// sum_g = sum gz, sum_gx = sum gz * xhat with gz = gy * act'(BN(x)), xhat = (x - mean) * invstd.  The loop accumulates
// gz * (x - mean) and multiplies by invstd once at the end: three coefficient vectors live in registers instead of four.
template <typename T, int ACT>
__global__ void __launch_bounds__(EW_THREADS, 3) bn_bwd_reduce_kernel(const T *__restrict__ gy, const T *__restrict__ x, long long count, int c,
                                                                      const float *__restrict__ scale, const float *__restrict__ shift,
                                                                      const float *__restrict__ mean, const float *__restrict__ invstd,
                                                                      int act, float slope, double *sum_g, double *sum_gx) {
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    float acc[2][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[0][j] = acc[1][j] = 0.f;
    if (r < rpb) {
        float sc[8], sh[8], mu[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            sc[j] = scale ? scale[v * 8 + j] : 1.f; sh[j] = shift ? shift[v * 8 + j] : 0.f;
            mu[j] = mean ? mean[v * 8 + j] : 0.f;
        }
        const long long step = static_cast<long long>(gridDim.x) * rpb;
        const T *pg = gy + v * 8, *px = x + v * 8;
#pragma unroll 4
        for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += step) {
            float g[8], f[8];
            Vec8<T>::load(pg + row * c, g);
            Vec8<T>::load(px + row * c, f);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float gz = g[j] * act_grad(f[j] * sc[j] + sh[j], ACT, slope);
                acc[0][j] += gz;
                acc[1][j] += gz * (f[j] - mu[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[1][j] *= invstd ? invstd[v * 8 + j] : 1.f;
    }
    double *const outs[2] = {sum_g, sum_gx};
    block_flush<2>(acc, cv, rpb, r, v, outs);
}

// dx = scale * (gz - sum_g/count - xhat * sum_gx/count) [* 1/mask_sum] written as  A*gz + B*(x - mean) + C  with per-channel
// A = scale, B = -scale*invstd*sum_gx/count, C = -scale*sum_g/count: five coefficient vectors in registers.
template <typename T, int ACT>
__global__ void __launch_bounds__(EW_THREADS, 3) bn_bwd_apply_kernel(const T *__restrict__ gy, const T *__restrict__ x, long long count, int c,
                                                                     const float *__restrict__ scale, const float *__restrict__ shift,
                                                                     const float *__restrict__ mean, const float *__restrict__ invstd, int act,
                                                                     float slope, const double *__restrict__ sum_g, const double *__restrict__ sum_gx,
                                                                     int training, const float *__restrict__ msum, T *__restrict__ dx,
                                                                     float *__restrict__ dgamma, float *__restrict__ dbeta) {
    extern __shared__ float s_coef[];                                 // [5][c]: scale | shift | mean | B | C (see above)
    const float inv_count = 1.0f / static_cast<float>(count);
    const bool full = scale && training;
    const bool writer = full && blockIdx.x == 0;                      // parameter gradients: dgamma = sum gz*xhat, dbeta = sum gz
    for (int ch = threadIdx.x; ch < c; ch += EW_THREADS) {            // once per channel and block (fp64 -> fp32 conversions are slow)
        const float a = scale ? scale[ch] : 1.f;
        const float sg = full ? static_cast<float>(sum_g[ch]) : 0.f, sgx = full ? static_cast<float>(sum_gx[ch]) : 0.f;
        s_coef[ch] = a; s_coef[c + ch] = scale ? shift[ch] : 0.f; s_coef[2 * c + ch] = full ? mean[ch] : 0.f;
        s_coef[3 * c + ch] = full ? -a * invstd[ch] * sgx * inv_count : 0.f;
        s_coef[4 * c + ch] = full ? -a * sg * inv_count : 0.f;
        if (writer) {
            if (dgamma) dgamma[ch] = sgx;
            if (dbeta) dbeta[ch] = sg;
        }
    }
    __syncthreads();
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    if (r >= rpb) return;
    float sc[8], sh[8], mu[8], cb[8], cc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int ch = v * 8 + j;
        sc[j] = s_coef[ch]; sh[j] = s_coef[c + ch]; mu[j] = s_coef[2 * c + ch]; cb[j] = s_coef[3 * c + ch]; cc[j] = s_coef[4 * c + ch];
    }
    const float ca = (scale != nullptr) ? 1.f : 0.f;                  // no BN at all: d = gz
    const long long step = static_cast<long long>(gridDim.x) * rpb;
    const bool renorm = msum != nullptr;
    const T *pg = gy + v * 8, *px = x + v * 8;
    T *pd = dx + v * 8;
#pragma unroll 4
    for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += step) {
        float g[8], f[8];
        // optional fused renormalisation backward of the producing partial convolution: dc = d / s, 0 at holes
        const float s = renorm ? __ldg(msum + row) : 1.f;
        Vec8<T>::load(pg + row * c, g);
        Vec8<T>::load(px + row * c, f);
        const float rs = (s == 0.f) ? 0.f : __frcp_rn(s);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gz = g[j] * act_grad(f[j] * sc[j] + sh[j], ACT, slope);
            const float d = (ca != 0.f) ? fmaf(sc[j], gz, fmaf(cb[j], f[j] - mu[j], cc[j])) : gz;
            f[j] = renorm ? d * rs : d;
        }
        Vec8<T>::store(pd + row * c, f);
    }
}

// Small tensors (the bottom of the U: <= 16 K rows): reduction AND apply in one launch.  One CTA per 8-channel vector walks all
// rows twice (the second pass hits L2), so no grid-wide dependency exists: the whole BatchNorm backward of such a layer is one
// kernel instead of memset + reduce + apply + parameter-gradient.
constexpr int BN_SMALL_THREADS = 1024;
template <typename T, int ACT>
__global__ void __launch_bounds__(BN_SMALL_THREADS) bn_bwd_small_kernel(const T *__restrict__ gy, const T *__restrict__ x, int count, int c,
                                                                        const float *__restrict__ coef /* [4][c] scale|shift|mean|invstd */,
                                                                        int act, float slope, const float *__restrict__ msum, T *__restrict__ dx,
                                                                        float *__restrict__ dgamma, float *__restrict__ dbeta) {
    __shared__ float s_part[BN_SMALL_THREADS / 32][16];
    __shared__ float s_tot[16];
    const int v = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    float sc[8], sh[8], mu[8], is[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int ch = v * 8 + j;
        sc[j] = coef[ch]; sh[j] = coef[c + ch]; mu[j] = coef[2 * c + ch]; is[j] = coef[3 * c + ch];
    }
    const T *pg = gy + v * 8, *px = x + v * 8;
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
#pragma unroll 4
    for (int row = t; row < count; row += BN_SMALL_THREADS) {
        float g[8], f[8];
        Vec8<T>::load(pg + static_cast<long long>(row) * c, g);
        Vec8<T>::load(px + static_cast<long long>(row) * c, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gz = g[j] * act_grad(f[j] * sc[j] + sh[j], ACT, slope);
            acc[j] += gz;
            acc[8 + j] += gz * (f[j] - mu[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float w = warp_sum(acc[j]);
        if (lane == 0) s_part[warp][j] = w;
    }
    __syncthreads();
    if (t < 16) {
        float tot = 0.f;
        for (int w = 0; w < BN_SMALL_THREADS / 32; ++w) tot += s_part[w][t];
        const int ch = v * 8 + (t & 7);
        if (t >= 8) tot *= coef[3 * c + ch];                                  // invstd (read from memory: no dynamic register indexing)
        s_tot[t] = tot;
        if (t < 8 && dbeta) dbeta[ch] = tot;
        if (t >= 8 && dgamma) dgamma[ch] = tot;
    }
    __syncthreads();
    const float inv_count = 1.0f / static_cast<float>(count);
    float cb[8], cc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        cb[j] = -sc[j] * is[j] * s_tot[8 + j] * inv_count;
        cc[j] = -sc[j] * s_tot[j] * inv_count;
    }
    T *pd = dx + v * 8;
    const bool renorm = msum != nullptr;
#pragma unroll 4
    for (int row = t; row < count; row += BN_SMALL_THREADS) {
        float g[8], f[8];
        const float s = renorm ? __ldg(msum + row) : 1.f;
        Vec8<T>::load(pg + static_cast<long long>(row) * c, g);
        Vec8<T>::load(px + static_cast<long long>(row) * c, f);
        const float rs = (s == 0.f) ? 0.f : __frcp_rn(s);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gz = g[j] * act_grad(f[j] * sc[j] + sh[j], ACT, slope);
            const float d = fmaf(sc[j], gz, fmaf(cb[j], f[j] - mu[j], cc[j]));
            f[j] = renorm ? d * rs : d;
        }
        Vec8<T>::store(pd + static_cast<long long>(row) * c, f);
    }
}

// scalar fallbacks (any channel count; small tensors): one block per channel for the reductions
template <typename T>
__global__ void bn_bwd_reduce_scalar_kernel(const T *__restrict__ gy, const T *__restrict__ x, long long count, int c, const float *scale,
                                            const float *shift, const float *mean, const float *invstd, int act, float slope,
                                            double *sum_g, double *sum_gx) {
    for (int ch = blockIdx.x; ch < c; ch += gridDim.x) {
        const float sc = scale ? scale[ch] : 1.f, sh = shift ? shift[ch] : 0.f, mu = mean ? mean[ch] : 0.f, is = invstd ? invstd[ch] : 1.f;
        float a = 0.f, b = 0.f;
        for (long long row = threadIdx.x; row < count; row += blockDim.x) {
            const float f = to_f32(x[row * c + ch]);
            const float gz = to_f32(gy[row * c + ch]) * act_grad(f * sc + sh, act, slope);
            a += gz; b += gz * (f - mu) * is;
        }
        __shared__ float sa[32], sb[32];
        a = warp_sum(a); b = warp_sum(b);
        if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = a; sb[threadIdx.x >> 5] = b; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double ta = 0, tb = 0;
            for (int i = 0; i < (blockDim.x >> 5); ++i) { ta += sa[i]; tb += sb[i]; }
            sum_g[ch] = ta; sum_gx[ch] = tb;
        }
        __syncthreads();
    }
}

template <typename T>
__global__ void bn_bwd_apply_scalar_kernel(const T *__restrict__ gy, const T *__restrict__ x, long long numel, long long count, int c,
                                           const float *scale, const float *shift, const float *mean, const float *invstd, int act, float slope,
                                           const double *sum_g, const double *sum_gx, int training, T *__restrict__ dx) {
    const float inv_count = 1.0f / static_cast<float>(count);
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ch = static_cast<int>(i % c);
        const float f = to_f32(x[i]);
        const float sc = scale ? scale[ch] : 1.f, sh = shift ? shift[ch] : 0.f;
        const float gz = to_f32(gy[i]) * act_grad(f * sc + sh, act, slope);
        float d;
        if (!scale) d = gz;
        else if (!training) d = sc * gz;
        else {
            const float xhat = (f - mean[ch]) * invstd[ch];
            d = sc * (gz - static_cast<float>(sum_g[ch]) * inv_count - xhat * static_cast<float>(sum_gx[ch]) * inv_count);
        }
        dx[i] = from_f32<T>(d);
    }
}

__global__ void bn_param_grad_kernel(const double *sum_g, const double *sum_gx, int c, float *dgamma, float *dbeta) {
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= c) return;
    if (dgamma) dgamma[ch] = static_cast<float>(sum_gx[ch]);
    if (dbeta) dbeta[ch] = static_cast<float>(sum_g[ch]);
}

// dc = dy * [s>0]/s ; dbias += sum dy*[s>0].  msum is [mg][count]; group of channel ch = ch / (c/mg).
// dy rows have pitch dys, dc rows pitch dcs (>= c); dc channels [c, dcs) are zero-filled.
template <typename T>
__global__ void renorm_bwd_kernel(const T *__restrict__ dy, int dys, const float *__restrict__ msum, long long count, int c, int mg,
                                  int no_guard, T *__restrict__ dc, int dcs, float *dbias) {
    extern __shared__ float s_db[];
    for (int i = threadIdx.x; i < c; i += blockDim.x) s_db[i] = 0.f;
    __syncthreads();
    const int cog = c / mg;
    const long long numel = count * dcs;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long row = i / dcs;
        const int ch = static_cast<int>(i - row * dcs);
        if (ch >= c) { dc[i] = from_f32<T>(0.f); continue; }
        const float s = msum ? msum[(mg == 1 ? 0 : (ch / cog)) * count + row] : 1.f;     // null: plain convolution
        const float g = to_f32(dy[row * dys + ch]);
        float d, gb;
        if (no_guard) { d = g / s; gb = (d - d) + g; }      // reference: g/s - g/s + g  (NaN where s == 0, like autograd there)
        else { const bool hole = (s == 0.f); d = hole ? 0.f : g / s; gb = hole ? 0.f : g; }
        dc[i] = from_f32<T>(d);
        if (dbias) atomicAdd(&s_db[ch], gb);
    }
    __syncthreads();
    if (dbias)
        for (int i = threadIdx.x; i < c; i += blockDim.x) atomicAdd(dbias + i, s_db[i]);
}

// c <= 8 in an 8-channel-padded buffer (the RGB tail): one 16-byte pixel per thread and iteration, bias-gradient partials in
// registers -> warp shuffle -> one atomic per channel per warp (the scalar kernel above serialises on 3 shared atomics)
template <typename T>
__global__ void __launch_bounds__(EW_THREADS) renorm_bwd_pixel8_kernel(const T *__restrict__ dy, int dys, const float *__restrict__ msum, long long count, int c,
                                                                       int no_guard, T *__restrict__ dc, float *dbias) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll 4
    for (long long row = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; row < count; row += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float s = msum ? msum[row] : 1.f;
        const bool hole = (s == 0.f);
        const float inv = 1.0f / s;             // one reciprocal per pixel: an IEEE division per element made these kernels issue-bound
        float g[8], d[8];
        if (dys == 8) Vec8<T>::load(dy + row * 8, g);
        else {
#pragma unroll
            for (int j = 0; j < 8; ++j) g[j] = j < c ? to_f32(dy[row * dys + j]) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j >= c) { d[j] = 0.f; continue; }
            if (no_guard) { d[j] = g[j] * inv; acc[j] += (d[j] - d[j]) + g[j]; }
            else { d[j] = hole ? 0.f : g[j] * inv; acc[j] += hole ? 0.f : g[j]; }
        }
        Vec8<T>::store(dc + row * 8, d);
    }
    if (dbias) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float t = warp_sum(acc[j]);
            if ((threadIdx.x & 31) == 0 && j < c) atomicAdd(dbias + j, t);
        }
    }
}

// vector path of the renormalisation backward: 8 channels per thread, rows strided like bn_stats (one msum load per row,
// bias-gradient partials block-reduced through shared memory).  Requires c % 8 == 0, dense pitch multiple of 8, mg == 1.
template <typename T>
__global__ void __launch_bounds__(EW_THREADS) renorm_bwd_vec_kernel(const T *__restrict__ dy, int dys, const float *__restrict__ msum, long long count,
                                                                    int c, int no_guard, T *__restrict__ dc, int dcs, float *dbias) {
    __shared__ float s_red[EW_THREADS][8];
    const int cv = c >> 3, rpb = EW_THREADS / cv;
    const int r = threadIdx.x / cv, v = threadIdx.x - r * cv;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (r < rpb) {
#pragma unroll 8
        for (long long row = static_cast<long long>(blockIdx.x) * rpb + r; row < count; row += static_cast<long long>(gridDim.x) * rpb) {
            const float s = msum ? __ldg(msum + row) : 1.f;
            const bool hole = (s == 0.f);
            const float inv = 1.0f / s;         // one reciprocal per row instead of a division per element
            float g[8], d[8];
            Vec8<T>::load(dy + row * dys + v * 8, g);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (no_guard) { d[j] = g[j] * inv; acc[j] += (d[j] - d[j]) + g[j]; }        // NaN where s == 0, like autograd there
                else { d[j] = hole ? 0.f : g[j] * inv; acc[j] += hole ? 0.f : g[j]; }
            }
            Vec8<T>::store(dc + row * dcs + v * 8, d);
        }
    }
    if (dbias) {
        if (r < rpb) {
#pragma unroll
            for (int j = 0; j < 8; ++j) s_red[threadIdx.x][j] = acc[j];
        }
        __syncthreads();
        if (r == 0 && v < cv) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float tot = 0.f;
                for (int rr = 0; rr < rpb; ++rr) tot += s_red[rr * cv + v][j];
                atomicAdd(dbias + v * 8 + j, tot);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// concat (+ nearest 2x upsample) forward / backward
// ---------------------------------------------------------------------------------------------
struct CatPart { const void *x; int c, choff, cstride, up; };
struct CatParams { int n, h, w, ctot, nparts; CatPart parts[PCB_MAX_PARTS]; };

template <typename T, int VEC>
__global__ void concat_fwd_kernel(const CatParams P, T *__restrict__ y) {
    const long long cv = P.ctot / VEC;
    const long long total = static_cast<long long>(P.n) * P.h * P.w * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long pix = i / cv;
        const int ch = static_cast<int>(i - pix * cv) * VEC;
        int p = 0;
        while (p + 1 < P.nparts && ch >= P.parts[p].choff + P.parts[p].c) ++p;
        const CatPart &pt = P.parts[p];
        const int ww = static_cast<int>(pix % P.w);
        const long long t = pix / P.w;
        const int hh = static_cast<int>(t % P.h), nn = static_cast<int>(t / P.h);
        const T *src = static_cast<const T *>(pt.x) +
                       (static_cast<long long>(nn * (P.h >> pt.up) + (hh >> pt.up)) * (P.w >> pt.up) + (ww >> pt.up)) * pt.cstride + (ch - pt.choff);
        if (VEC == 8) {
            if (sizeof(T) == 2) *reinterpret_cast<uint4 *>(y + i * 8) = *reinterpret_cast<const uint4 *>(src);
            else { reinterpret_cast<float4 *>(y + i * 8)[0] = reinterpret_cast<const float4 *>(src)[0];
                   reinterpret_cast<float4 *>(y + i * 8)[1] = reinterpret_cast<const float4 *>(src)[1]; }
        } else {
            y[i] = src[0];
        }
    }
}

// gx[n, h>>up, w>>up, c] = sum over the up x up block of gy[..., choff + c]
template <typename T, int VEC>
__global__ void concat_bwd_kernel(const T *__restrict__ gy, int n, int h, int w, int ctot, int choff, int c, int up, T *__restrict__ gx) {
    const int hs = h >> up, ws = w >> up, f = 1 << up;
    const long long cv = c / VEC;
    const long long total = static_cast<long long>(n) * hs * ws * cv;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long pix = i / cv;
        const int ch = static_cast<int>(i - pix * cv) * VEC;
        const int ww = static_cast<int>(pix % ws);
        const long long t = pix / ws;
        const int hh = static_cast<int>(t % hs), nn = static_cast<int>(t / hs);
        float acc[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
        for (int dy = 0; dy < f; ++dy)
            for (int dx = 0; dx < f; ++dx) {
                const T *src = gy + (static_cast<long long>(nn * h + hh * f + dy) * w + ww * f + dx) * ctot + choff + ch;
                if (VEC == 8) {
                    float v[8];
                    Vec8<T>::load(src, v);
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] += v[j];
                } else acc[0] += to_f32(src[0]);
            }
        if (VEC == 8) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = acc[j];
            Vec8<T>::store(gx + i * 8, o);
        } else gx[i] = from_f32<T>(acc[0]);
    }
}

// ---------------------------------------------------------------------------------------------
// masks, weights, loss, optimiser
// ---------------------------------------------------------------------------------------------
__global__ void mask_from_dense_kernel(const float *__restrict__ m, int n, int c, long long hw, uint8_t *__restrict__ planes) {
    const long long total = static_cast<long long>(n) * c * hw;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long p = i % hw;
        const long long t = i / hw;
        const int ch = static_cast<int>(t % c), nn = static_cast<int>(t / c);
        planes[(static_cast<long long>(ch) * n + nn) * hw + p] = m[i] != 0.f ? 1 : 0;
    }
}

__global__ void mask_to_dense_kernel(const uint8_t *__restrict__ plane, int n, int h, int w, int up, float *__restrict__ dst, int ctot, int c0, int c) {
    const long long hw = static_cast<long long>(h) * w;
    const long long total = static_cast<long long>(n) * c * hw;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long p = i % hw;
        const long long t = i / hw;
        const int ch = static_cast<int>(t % c), nn = static_cast<int>(t / c);
        const int hh = static_cast<int>(p / w), ww = static_cast<int>(p - static_cast<long long>(hh) * w);
        const uint8_t v = plane[(static_cast<long long>(nn) * (h >> up) + (hh >> up)) * (w >> up) + (ww >> up)];
        dst[(static_cast<long long>(nn) * ctot + c0 + ch) * hw + p] = v ? 1.f : 0.f;
    }
}

template <typename T>
__global__ void weight_cast_kernel(const float *__restrict__ src, long long n, T *__restrict__ dst) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x)
        dst[i] = from_f32<T>(src[i]);
}

template <typename T>
__global__ void l1_sum_kernel(const T *__restrict__ x, long long numel, double *scratch) {
    float a = 0.f;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x)
        a += fabsf(to_f32(x[i]));
    a = warp_sum(a);
    __shared__ float s[32];
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < (blockDim.x >> 5); ++i) t += s[i];
        atomicAdd(scratch, t);
    }
}
__global__ void l1_finish_kernel(const double *scratch, long long numel, float *loss) { *loss = static_cast<float>(*scratch / static_cast<double>(numel)); }

template <typename T>
__global__ void l1_bwd_kernel(const T *__restrict__ x, long long numel, float gscale, T *__restrict__ gx) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float v = to_f32(x[i]);
        gx[i] = from_f32<T>(v > 0.f ? gscale : (v < 0.f ? -gscale : 0.f));
    }
}

__global__ void sgd_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ buf, long long numel, float lr, float mom,
                           float wd, int nesterov, int first, float gscale) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < numel; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float d = g[i] * gscale + wd * p[i];
        if (mom != 0.f) {
            const float b = first ? d : mom * buf[i] + d;
            buf[i] = b;
            d = nesterov ? d + mom * b : b;
        }
        p[i] -= lr * d;
    }
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
#define ST static_cast<cudaStream_t>(stream)

extern "C" __attribute__((visibility("default"))) int pcb_bn_stats(const void *x, int dtype, long long count, int c, double *sum, double *sqsum, pcb_stream_t stream) {
    PCB_CHECK(x && sum && sqsum && count > 0 && c > 0, "pcb_bn_stats: bad arguments");
    if (sqsum == sum + c) PCB_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * 2 * c, ST));       // one [2][c] buffer: one memset
    else {
        PCB_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * c, ST));
        PCB_CUDA(cudaMemsetAsync(sqsum, 0, sizeof(double) * c, ST));
    }
    if (c % 8 == 0 && c <= 2048) {
        const int rpb = EW_THREADS / (c / 8);
        const int grid = ew_grid_red(count, rpb * 16);
        if (dtype == PCB_BF16) bn_stats_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), count, c, sum, sqsum);
        else bn_stats_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), count, c, sum, sqsum);
    } else {
        if (dtype == PCB_BF16) bn_stats_scalar_kernel<bf16><<<min(c, 1024), 256, 0, ST>>>(static_cast<const bf16 *>(x), count, c, sum, sqsum);
        else bn_stats_scalar_kernel<float><<<min(c, 1024), 256, 0, ST>>>(static_cast<const float *>(x), count, c, sum, sqsum);
    }
    PCB_LAUNCH_CHECK();
    return 0;
}

// statistics WITHOUT the memset: `sums` = [2][c] doubles that the caller zeroed (e.g. a slice of a per-step zero arena)
extern "C" __attribute__((visibility("default"))) int pcb_bn_stats_acc(const void *x, int dtype, long long count, int c, double *sums, pcb_stream_t stream) {
    PCB_CHECK(x && sums && count > 0 && c > 0, "pcb_bn_stats_acc: bad arguments");
    if (c % 8 == 0 && c <= 2048) {
        const int rpb = EW_THREADS / (c / 8);
        const int grid = ew_grid_red(count, rpb * 8);
        if (dtype == PCB_BF16) bn_stats_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), count, c, sums, sums + c);
        else bn_stats_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), count, c, sums, sums + c);
    } else {
        if (dtype == PCB_BF16) bn_stats_scalar_kernel<bf16><<<min(c, 1024), 256, 0, ST>>>(static_cast<const bf16 *>(x), count, c, sums, sums + c);
        else bn_stats_scalar_kernel<float><<<min(c, 1024), 256, 0, ST>>>(static_cast<const float *>(x), count, c, sums, sums + c);
    }
    PCB_LAUNCH_CHECK();
    return 0;
}

// training-mode BatchNorm forward from COMPLETE sums: finalise (mean / invstd / running statistics) + apply + activation
// (+ residual) in one launch; `coef` receives [4][c] floats scale | shift | mean | invstd for the backward.
extern "C" __attribute__((visibility("default"))) int pcb_bn_forward_fused(const void *x, int dtype, long long count, int c, const double *sums, const float *gamma,
                                    const float *beta, float *running_mean, float *running_var, long long *num_batches_tracked,
                                    float momentum, float eps, int act, float slope, const void *residual, void *y, float *coef,
                                    pcb_stream_t stream) {
    PCB_CHECK(x && y && sums && coef && count > 0 && c > 0 && c % 8 == 0 && c <= 2048, "pcb_bn_forward_fused: bad arguments (c must be a multiple of 8, <= 2048)");
    PCB_CHECK((running_mean == nullptr) == (running_var == nullptr), "pcb_bn_forward_fused: running statistics come in pairs");
    const int grid = ew_grid(count, (EW_THREADS / (c / 8)) * 16, 8);      // >= 16 rows per thread: the block prologue is amortised
    PCB_ACT_SWITCH(act,
        if (dtype == PCB_BF16) bn_fwd_fused_kernel<bf16, ACT><<<grid, EW_THREADS, 2 * c * sizeof(float), ST>>>(static_cast<const bf16 *>(x), count, c, sums, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, act, slope, static_cast<const bf16 *>(residual), static_cast<bf16 *>(y), coef);
        else bn_fwd_fused_kernel<float, ACT><<<grid, EW_THREADS, 2 * c * sizeof(float), ST>>>(static_cast<const float *>(x), count, c, sums, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, act, slope, static_cast<const float *>(residual), static_cast<float *>(y), coef))
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_bn_finalize(const double *sum, const double *sqsum, long long count, int c, const float *gamma, const float *beta,
                               float *running_mean, float *running_var, long long *num_batches_tracked, float momentum, float eps,
                               int training, float *scale, float *shift, float *save_mean, float *save_invstd, pcb_stream_t stream) {
    PCB_CHECK(scale && shift && c > 0, "pcb_bn_finalize: bad arguments");
    PCB_CHECK(training ? (sum && sqsum && count > 0) : (running_mean && running_var), "pcb_bn_finalize: missing statistics");
    bn_finalize_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sum, sqsum, count, c, gamma, beta, running_mean, running_var, num_batches_tracked,
                                                       momentum, eps, training, scale, shift, save_mean, save_invstd);
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_bn_act_forward(const void *x, int dtype, long long count, int c, const float *scale, const float *shift, int act,
                                  float slope, const void *residual, void *y, pcb_stream_t stream) {
    PCB_CHECK(x && y && count > 0 && c > 0 && ((scale == nullptr) == (shift == nullptr)), "pcb_bn_act_forward: bad arguments");
    const long long numel = count * c;
    if (c % 8 == 0 && c <= 2048) {
        const int grid = ew_grid(count, (EW_THREADS / (c / 8)) * 4);
        if (dtype == PCB_BF16) bn_act_fwd_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), count, c, scale, shift, act, slope, static_cast<const bf16 *>(residual), static_cast<bf16 *>(y));
        else bn_act_fwd_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), count, c, scale, shift, act, slope, static_cast<const float *>(residual), static_cast<float *>(y));
    } else {
        const int grid = ew_grid(numel, EW_THREADS * 8);
        if (dtype == PCB_BF16) bn_act_fwd_scalar_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), numel, c, scale, shift, act, slope, static_cast<const bf16 *>(residual), static_cast<bf16 *>(y));
        else bn_act_fwd_scalar_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), numel, c, scale, shift, act, slope, static_cast<const float *>(residual), static_cast<float *>(y));
    }
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_bn_act_backward_reduce(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                          const float *shift, const float *mean, const float *invstd, int act, float slope,
                                          double *sum_g, double *sum_gx, pcb_stream_t stream) {
    PCB_CHECK(gy && x && sum_g && sum_gx && count > 0, "pcb_bn_act_backward_reduce: bad arguments");
    if (c % 8 != 0 || c > 2048) {
        if (dtype == PCB_BF16) bn_bwd_reduce_scalar_kernel<bf16><<<min(c, 1024), 256, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx);
        else bn_bwd_reduce_scalar_kernel<float><<<min(c, 1024), 256, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx);
        PCB_LAUNCH_CHECK();
        return 0;
    }
    if (sum_gx == sum_g + c) PCB_CUDA(cudaMemsetAsync(sum_g, 0, sizeof(double) * 2 * c, ST));
    else {
        PCB_CUDA(cudaMemsetAsync(sum_g, 0, sizeof(double) * c, ST));
        PCB_CUDA(cudaMemsetAsync(sum_gx, 0, sizeof(double) * c, ST));
    }
    const int rpb = EW_THREADS / (c / 8);
    const int grid = ew_grid_red(count, rpb * 16);
    PCB_ACT_SWITCH(act,
        if (dtype == PCB_BF16) bn_bwd_reduce_kernel<bf16, ACT><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx);
        else bn_bwd_reduce_kernel<float, ACT><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx))
    PCB_LAUNCH_CHECK();
    return 0;
}

// backward reduction WITHOUT the memset: `sums` = [2][c] doubles zeroed by the caller (sum gz | sum gz * xhat)
extern "C" __attribute__((visibility("default"))) int pcb_bn_act_backward_reduce_acc(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                          const float *shift, const float *mean, const float *invstd, int act, float slope,
                                          double *sums, pcb_stream_t stream) {
    PCB_CHECK(gy && x && sums && count > 0 && c % 8 == 0 && c <= 2048, "pcb_bn_act_backward_reduce_acc: bad arguments (c must be a multiple of 8, <= 2048)");
    const int rpb = EW_THREADS / (c / 8);
    const int grid = ew_grid_red(count, rpb * 8);
    PCB_ACT_SWITCH(act,
        if (dtype == PCB_BF16) bn_bwd_reduce_kernel<bf16, ACT><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), count, c, scale, shift, mean, invstd, act, slope, sums, sums + c);
        else bn_bwd_reduce_kernel<float, ACT><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), count, c, scale, shift, mean, invstd, act, slope, sums, sums + c))
    PCB_LAUNCH_CHECK();
    return 0;
}

// Whole training-mode BatchNorm(+act) backward of a SMALL tensor in one launch (reduction + apply + parameter gradients [+ the
// renormalisation backward of the producing partial convolution when msum != NULL]).  coef = the [4][c] block written by
// pcb_bn_forward_fused.  Intended for count <= 16384 rows (one CTA per 8 channels walks every row twice); c % 8 == 0.
extern "C" __attribute__((visibility("default"))) int pcb_bn_act_backward_small(const void *gy, const void *x, int dtype, long long count, int c, const float *coef,
                                         int act, float slope, const float *msum, void *dx, float *dgamma, float *dbeta, pcb_stream_t stream) {
    PCB_CHECK(gy && x && dx && coef && count > 0 && count <= (1 << 20) && c % 8 == 0, "pcb_bn_act_backward_small: bad arguments");
    PCB_ACT_SWITCH(act,
        if (dtype == PCB_BF16) bn_bwd_small_kernel<bf16, ACT><<<c / 8, BN_SMALL_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), static_cast<int>(count), c, coef, act, slope, msum, static_cast<bf16 *>(dx), dgamma, dbeta);
        else bn_bwd_small_kernel<float, ACT><<<c / 8, BN_SMALL_THREADS, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), static_cast<int>(count), c, coef, act, slope, msum, static_cast<float *>(dx), dgamma, dbeta))
    PCB_LAUNCH_CHECK();
    return 0;
}

static int bn_act_backward_apply_impl(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                      const float *shift, const float *mean, const float *invstd, int act, float slope,
                                      const double *sum_g, const double *sum_gx, int training, const float *msum, void *dx, float *dgamma,
                                      float *dbeta, pcb_stream_t stream) {
    PCB_CHECK(gy && x && dx && count > 0, "pcb_bn_act_backward_apply: bad arguments");
    PCB_CHECK(!msum || (c % 8 == 0 && c <= 2048), "pcb_bn_act_backward_apply_renorm: channel count must be a multiple of 8 (<= 2048)");
    PCB_CHECK(!(scale && training) || (mean && invstd && sum_g && sum_gx), "pcb_bn_act_backward_apply: training needs statistics");
    const bool vec = c % 8 == 0 && c <= 2048;
    const int grid = vec ? ew_grid(count, (EW_THREADS / (c / 8)) * 16, 6) : ew_grid(count * c, EW_THREADS * 4);
    if (!vec) {
        if (dtype == PCB_BF16) bn_bwd_apply_scalar_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), count * c, count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, static_cast<bf16 *>(dx));
        else bn_bwd_apply_scalar_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), count * c, count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, static_cast<float *>(dx));
        PCB_LAUNCH_CHECK();
        if ((dgamma || dbeta) && sum_g && sum_gx) {
            bn_param_grad_kernel<<<(c + 127) / 128, 128, 0, ST>>>(sum_g, sum_gx, c, dgamma, dbeta);
            PCB_LAUNCH_CHECK();
        }
        return 0;
    }
    // vector path: block 0 also writes the parameter gradients (dgamma = sum gz*xhat, dbeta = sum gz) -- no extra launch
    PCB_ACT_SWITCH(act,
        if (dtype == PCB_BF16) bn_bwd_apply_kernel<bf16, ACT><<<grid, EW_THREADS, 5 * c * sizeof(float), ST>>>(static_cast<const bf16 *>(gy), static_cast<const bf16 *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, msum, static_cast<bf16 *>(dx), dgamma, dbeta);
        else bn_bwd_apply_kernel<float, ACT><<<grid, EW_THREADS, 5 * c * sizeof(float), ST>>>(static_cast<const float *>(gy), static_cast<const float *>(x), count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, msum, static_cast<float *>(dx), dgamma, dbeta))
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_bn_act_backward_apply(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                         const float *shift, const float *mean, const float *invstd, int act, float slope,
                                         const double *sum_g, const double *sum_gx, int training, void *dx, float *dgamma, float *dbeta,
                                         pcb_stream_t stream) {
    return bn_act_backward_apply_impl(gy, x, dtype, count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, nullptr, dx, dgamma, dbeta, stream);
}

extern "C" __attribute__((visibility("default"))) int pcb_bn_act_backward_apply_renorm(const void *gy, const void *x, int dtype, long long count, int c, const float *scale,
                                         const float *shift, const float *mean, const float *invstd, int act, float slope,
                                         const double *sum_g, const double *sum_gx, int training, const float *msum, void *dc, float *dgamma,
                                         float *dbeta, pcb_stream_t stream) {
    PCB_CHECK(msum != nullptr, "pcb_bn_act_backward_apply_renorm: msum required");
    return bn_act_backward_apply_impl(gy, x, dtype, count, c, scale, shift, mean, invstd, act, slope, sum_g, sum_gx, training, msum, dc, dgamma, dbeta, stream);
}

extern "C" __attribute__((visibility("default"))) int pcb_pconv_renorm_backward(const pcb_conv *c, const void *dy, int dy_cstride, const float *msum, void *dc, int dc_cstride, float *dbias, pcb_stream_t stream) {
    PCB_CHECK(c && dy && (msum || c->plain) && dc && dy_cstride >= c->cout && dc_cstride >= c->cout, "pcb_pconv_renorm_backward: bad arguments");
    if (c->plain) msum = nullptr;                         // ordinary convolution: renormaliser 1 (the forward never wrote msum)
    const long long count = static_cast<long long>(c->n) * c->ho * c->wo;
    const int mg = (c->groups > 1 && !c->same_holes) ? c->groups : 1;
    if (dbias) PCB_CUDA(cudaMemsetAsync(dbias, 0, sizeof(float) * c->cout, ST));
    if (mg == 1 && c->cout % 8 == 0 && c->cout <= 2048 && dc_cstride == c->cout && dy_cstride % 8 == 0) {
        const int rpb = EW_THREADS / (c->cout / 8);
        // with a bias gradient the kernel ends in cout atomics per block on the same cout addresses: one resident wave keeps
        // the number of atomics per address small next to the streaming work
        const int vgrid = dbias ? ew_grid_red(count, rpb * 8) : ew_grid(count, rpb * 8);
        if (c->dtype == PCB_BF16) renorm_bwd_vec_kernel<bf16><<<vgrid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(dy), dy_cstride, msum, count, c->cout, c->no_guard, static_cast<bf16 *>(dc), dc_cstride, dbias);
        else renorm_bwd_vec_kernel<float><<<vgrid, EW_THREADS, 0, ST>>>(static_cast<const float *>(dy), dy_cstride, msum, count, c->cout, c->no_guard, static_cast<float *>(dc), dc_cstride, dbias);
        PCB_LAUNCH_CHECK();
        return 0;
    }
    if (mg == 1 && c->cout <= 8 && dc_cstride == 8 && (reinterpret_cast<uintptr_t>(dc) & 15) == 0 && (dy_cstride != 8 || (reinterpret_cast<uintptr_t>(dy) & 15) == 0)) {
        const int pgrid = ew_grid_red(count, EW_THREADS * 4);
        if (c->dtype == PCB_BF16) renorm_bwd_pixel8_kernel<bf16><<<pgrid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(dy), dy_cstride, msum, count, c->cout, c->no_guard, static_cast<bf16 *>(dc), dbias);
        else renorm_bwd_pixel8_kernel<float><<<pgrid, EW_THREADS, 0, ST>>>(static_cast<const float *>(dy), dy_cstride, msum, count, c->cout, c->no_guard, static_cast<float *>(dc), dbias);
        PCB_LAUNCH_CHECK();
        return 0;
    }
    const int grid = ew_grid(count * dc_cstride, EW_THREADS * 8);
    const size_t smem = sizeof(float) * c->cout;
    if (c->dtype == PCB_BF16) renorm_bwd_kernel<bf16><<<grid, EW_THREADS, smem, ST>>>(static_cast<const bf16 *>(dy), dy_cstride, msum, count, c->cout, mg, c->no_guard, static_cast<bf16 *>(dc), dc_cstride, dbias);
    else renorm_bwd_kernel<float><<<grid, EW_THREADS, smem, ST>>>(static_cast<const float *>(dy), dy_cstride, msum, count, c->cout, mg, c->no_guard, static_cast<float *>(dc), dc_cstride, dbias);
    PCB_LAUNCH_CHECK();
    return 0;
}

int pcb_cast_weights(const float *src, void *dst, long long n, int dtype, cudaStream_t st) {
    const int grid = ew_grid(n, EW_THREADS * 4);
    if (dtype == PCB_BF16) weight_cast_kernel<bf16><<<grid, EW_THREADS, 0, st>>>(src, n, static_cast<bf16 *>(dst));
    else weight_cast_kernel<float><<<grid, EW_THREADS, 0, st>>>(src, n, static_cast<float *>(dst));
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_concat_forward(const pcb_part *parts, int nparts, int dtype, int n, int h, int w, void *y, pcb_stream_t stream) {
    PCB_CHECK(parts && y && nparts >= 1 && nparts <= PCB_MAX_PARTS, "pcb_concat_forward: bad arguments");
    CatParams P;
    P.n = n; P.h = h; P.w = w; P.nparts = nparts;
    int off = 0;
    bool vec = true;
    for (int p = 0; p < nparts; ++p) {
        P.parts[p].x = parts[p].x; P.parts[p].c = parts[p].c; P.parts[p].choff = off; P.parts[p].cstride = parts[p].x_cstride;
        P.parts[p].up = parts[p].x_up;
        PCB_CHECK(parts[p].x != nullptr, "pcb_concat_forward: null part");
        PCB_CHECK(parts[p].x_up == 0 || (h % 2 == 0 && w % 2 == 0), "pcb_concat_forward: upsampled part needs even h, w");
        if (parts[p].c % 8 || off % 8 || parts[p].x_cstride % 8 || (reinterpret_cast<uintptr_t>(parts[p].x) & (dtype == PCB_BF16 ? 15 : 31))) vec = false;
        off += parts[p].c;
    }
    P.ctot = off;
    const long long numel = static_cast<long long>(n) * h * w * off;
    if (vec) {
        const int grid = ew_grid(numel / 8, EW_THREADS * 4);
        if (dtype == PCB_BF16) concat_fwd_kernel<bf16, 8><<<grid, EW_THREADS, 0, ST>>>(P, static_cast<bf16 *>(y));
        else concat_fwd_kernel<float, 8><<<grid, EW_THREADS, 0, ST>>>(P, static_cast<float *>(y));
    } else {
        const int grid = ew_grid(numel, EW_THREADS * 8);
        if (dtype == PCB_BF16) concat_fwd_kernel<bf16, 1><<<grid, EW_THREADS, 0, ST>>>(P, static_cast<bf16 *>(y));
        else concat_fwd_kernel<float, 1><<<grid, EW_THREADS, 0, ST>>>(P, static_cast<float *>(y));
    }
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_concat_backward(const void *gy, const int32_t *c, const int32_t *up, int nparts, int dtype, int n, int h, int w,
                                   void *const *gx, pcb_stream_t stream) {
    PCB_CHECK(gy && c && up && gx && nparts >= 1 && nparts <= PCB_MAX_PARTS, "pcb_concat_backward: bad arguments");
    int ctot = 0;
    for (int p = 0; p < nparts; ++p) ctot += c[p];
    int off = 0;
    for (int p = 0; p < nparts; ++p) {
        if (gx[p]) {
            const bool vec = (c[p] % 8 == 0) && (off % 8 == 0) && (ctot % 8 == 0);
            const long long numel = static_cast<long long>(n) * (h >> up[p]) * (w >> up[p]) * c[p];
            if (vec) {
                const int grid = ew_grid(numel / 8, EW_THREADS * 4);
                if (dtype == PCB_BF16) concat_bwd_kernel<bf16, 8><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), n, h, w, ctot, off, c[p], up[p], static_cast<bf16 *>(gx[p]));
                else concat_bwd_kernel<float, 8><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(gy), n, h, w, ctot, off, c[p], up[p], static_cast<float *>(gx[p]));
            } else {
                const int grid = ew_grid(numel, EW_THREADS * 8);
                if (dtype == PCB_BF16) concat_bwd_kernel<bf16, 1><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(gy), n, h, w, ctot, off, c[p], up[p], static_cast<bf16 *>(gx[p]));
                else concat_bwd_kernel<float, 1><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(gy), n, h, w, ctot, off, c[p], up[p], static_cast<float *>(gx[p]));
            }
            PCB_LAUNCH_CHECK();
        }
        off += c[p];
    }
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_upsample2x_forward(const void *x, int dtype, int n, int h, int w, int c, void *y, pcb_stream_t stream) {
    pcb_part p;
    p.x = x; p.mask = nullptr; p.c = c; p.x_cstride = c; p.x_up = 1; p.mask_up = 0;
    return pcb_concat_forward(&p, 1, dtype, n, 2 * h, 2 * w, y, stream);
}

extern "C" __attribute__((visibility("default"))) int pcb_upsample2x_backward(const void *gy, int dtype, int n, int h, int w, int c, void *gx, pcb_stream_t stream) {
    const int32_t cc = c, up = 1;
    void *g = gx;
    return pcb_concat_backward(gy, &cc, &up, 1, dtype, n, 2 * h, 2 * w, &g, stream);
}

extern "C" __attribute__((visibility("default"))) int pcb_mask_planes_from_dense(const float *mask_nchw, int n, int c, int h, int w, uint8_t *planes, pcb_stream_t stream) {
    PCB_CHECK(mask_nchw && planes && n > 0 && c > 0, "pcb_mask_planes_from_dense: bad arguments");
    const long long total = static_cast<long long>(n) * c * h * w;
    mask_from_dense_kernel<<<ew_grid(total, EW_THREADS * 4), EW_THREADS, 0, ST>>>(mask_nchw, n, c, static_cast<long long>(h) * w, planes);
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_mask_plane_to_dense(const uint8_t *plane, int n, int h, int w, int up, float *dst_nchw, int ctot, int c0, int c,
                                       pcb_stream_t stream) {
    PCB_CHECK(plane && dst_nchw && c0 >= 0 && c0 + c <= ctot, "pcb_mask_plane_to_dense: bad arguments");
    const long long total = static_cast<long long>(n) * c * h * w;
    mask_to_dense_kernel<<<ew_grid(total, EW_THREADS * 4), EW_THREADS, 0, ST>>>(plane, n, h, w, up, dst_nchw, ctot, c0, c);
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_l1_mean_forward(const void *x, int dtype, long long numel, float *loss, double *scratch, pcb_stream_t stream) {
    PCB_CHECK(x && loss && scratch && numel > 0, "pcb_l1_mean_forward: bad arguments");
    PCB_CUDA(cudaMemsetAsync(scratch, 0, sizeof(double), ST));
    const int grid = ew_grid(numel, EW_THREADS * 16);
    if (dtype == PCB_BF16) l1_sum_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), numel, scratch);
    else l1_sum_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), numel, scratch);
    PCB_LAUNCH_CHECK();
    l1_finish_kernel<<<1, 1, 0, ST>>>(scratch, numel, loss);
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_l1_mean_backward(const void *x, int dtype, long long numel, float gscale, void *gx, pcb_stream_t stream) {
    PCB_CHECK(x && gx && numel > 0, "pcb_l1_mean_backward: bad arguments");
    const int grid = ew_grid(numel, EW_THREADS * 8);
    if (dtype == PCB_BF16) l1_bwd_kernel<bf16><<<grid, EW_THREADS, 0, ST>>>(static_cast<const bf16 *>(x), numel, gscale, static_cast<bf16 *>(gx));
    else l1_bwd_kernel<float><<<grid, EW_THREADS, 0, ST>>>(static_cast<const float *>(x), numel, gscale, static_cast<float *>(gx));
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_sgd_step_scaled(float *param, const float *grad, float *momentum_buf, long long numel, float lr, float momentum,
                            float weight_decay, int nesterov, int first_step, float grad_scale, pcb_stream_t stream) {
    PCB_CHECK(param && grad && numel > 0 && (momentum == 0.f || momentum_buf), "pcb_sgd_step: bad arguments");
    sgd_kernel<<<ew_grid(numel, EW_THREADS * 8), EW_THREADS, 0, ST>>>(param, grad, momentum_buf, numel, lr, momentum, weight_decay, nesterov, first_step, grad_scale);
    PCB_LAUNCH_CHECK();
    return 0;
}

extern "C" __attribute__((visibility("default"))) int pcb_sgd_step(float *param, const float *grad, float *momentum_buf, long long numel, float lr, float momentum,
                            float weight_decay, int nesterov, int first_step, pcb_stream_t stream) {
    return pcb_sgd_step_scaled(param, grad, momentum_buf, numel, lr, momentum, weight_decay, nesterov, first_step, 1.0f, stream);
}

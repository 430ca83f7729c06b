// seg_data.cu -- the segmentation data path (TextSegmentationData.process_images, Dataloader.py:66-74) for a batch of gray
// pages and text masks, in four launches:
//   1. seg_sample_kernel: one thread per image draws the crop box (RandomResizedCrop.get_params(scale=(0.1, 2))), whether
//      brightness comes before contrast (ColorJitter's torch.randperm(4)) and the two factors from Philox4x32-10; seed and step
//      counter live in device memory and the kernel advances the counter, so every graph replay draws fresh parameters.
//      Skipped when the caller supplies parameters.  Saturation and hue are not drawn: on an `L` image they are the identity.
//   2. seg_hpass_kernel: Pillow's horizontal bicubic pass over every row of each image's crop box, page and mask together.
//   3. seg_vpass_kernel: Pillow's vertical pass into uint8 page and mask planes, and the 256-bin histogram of each page.
//   4. seg_store_kernel: the contrast mean from the histogram (through the brightness blend when brightness goes first), the
//      two Pillow blends in the drawn order, ToTensor, the optional Normalize, the 3-channel replication and the stores.
// Grids are sized from the batcher's capacity (largest source), so one captured graph serves any mix of source sizes.
#include "pil_data.cuh"

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))

namespace {

using pil::KMAX;
using pil::PB;
using pil::clip8;
using pil::pil_coeffs;

constexpr int HX = 128;       // horizontal pass: output columns per block (one per thread)
constexpr int HROWS = 16;     // horizontal pass: box rows per block
constexpr int T = 32;         // vertical pass: output tile edge
constexpr int SPB = 4096;     // store kernel: pixels per block

__device__ __forceinline__ bool source_ok(const pcb_seg_src &s, const pcb_seg_params &p, int cap_h, int cap_w) {
    return s.h >= 1 && s.w >= 1 && s.h <= cap_h && s.w <= cap_w && p.top >= 0 && p.left >= 0 && p.height >= 1 && p.width >= 1 &&
           p.top + p.height <= s.h && p.left + p.width <= s.w;
}

// Pillow's Image.blend(d, x, f) of one 8-bit value: float32 d + f * (x - d), two roundings, truncated and clipped to [0, 255]
__device__ __forceinline__ int blend(int d, int x, float f) {
    const float t = __fadd_rn(static_cast<float>(d), __fmul_rn(f, static_cast<float>(x - d)));
    return t <= 0.f ? 0 : (t >= 255.f ? 255 : static_cast<int>(t));
}

// ------------------------------------------------------------------------------------------------ 1. parameter sampler
__global__ void __launch_bounds__(1024) seg_sample_kernel(const pcb_seg_src *__restrict__ srcs, int n, unsigned long long *rng,
                                                          pcb_seg_params *__restrict__ params) {
    const int t = threadIdx.x;
    const unsigned long long seed = rng[0], step = rng[1];
    __syncthreads();
    if (t == 0) rng[1] = step + 1;
    if (t >= n) return;
    const pil::Draws d(static_cast<uint32_t>(t), step, seed);
    // RandomResizedCrop.get_params(scale=(0.1, 2)): torch's uniform_ works with float32 0.1 and float32 2 - float32 0.1
    const pil::Box box = pil::crop_box(d, srcs[t].h, srcs[t].w, 0.1f, __fsub_rn(2.0f, 0.1f));
    pcb_seg_params p{};
    p.top = box.top;
    p.left = box.left;
    p.height = box.height;
    p.width = box.width;
    // ColorJitter(brightness=0.2, contrast=0.2): the relative order of the two in randperm(4), then both factors on [0.8, 1.2]
    p.brightness_first = d.u(40) < 0.5f ? 1 : 0;
    p.brightness = __fadd_rn(0.8f, __fmul_rn(__fsub_rn(1.2f, 0.8f), d.u(41)));
    p.contrast = __fadd_rn(0.8f, __fmul_rn(__fsub_rn(1.2f, 0.8f), d.u(42)));
    params[t] = p;
}

// ------------------------------------------------------------------------------------------------ 2. horizontal pass
__global__ void __launch_bounds__(HX) seg_hpass_kernel(const pcb_seg_src *__restrict__ srcs, const pcb_seg_params *__restrict__ params,
                                                       int cap_h, int cap_w, int out, uchar2 *__restrict__ tmp, int *__restrict__ hist) {
    __shared__ int kk[KMAX * HX];
    const int n = blockIdx.z, x = blockIdx.x * HX + threadIdx.x, row0 = blockIdx.y * HROWS;
    if (blockIdx.x == 0 && blockIdx.y == 0)
        for (int v = threadIdx.x; v < 256; v += HX) hist[n * 256 + v] = 0;        // the vertical pass adds into it
    const pcb_seg_src s = srcs[n];
    const pcb_seg_params &p = params[n];
    const int top = p.top, left = p.left, bh = p.height, bw = p.width;
    if (row0 >= bh || x >= out || !source_ok(s, p, cap_h, cap_w)) return;
    int nt;
    const int xmin = pil_coeffs(x, bw, out, kk + threadIdx.x, HX, &nt);     // this thread's column only: no barrier
    const int rows = min(HROWS, bh - row0);
    for (int r = row0; r < row0 + rows; ++r) {
        const uint8_t *pp = s.page + static_cast<size_t>(top + r) * s.page_stride + left + xmin;
        const uint8_t *pm = s.mask + static_cast<size_t>(top + r) * s.mask_stride + left + xmin;
        int a0 = 1 << (PB - 1), a1 = a0;
        for (int t = 0; t < nt; ++t) {
            const int k = kk[t * HX + threadIdx.x];
            a0 += static_cast<int>(__ldg(pp + t)) * k;
            a1 += static_cast<int>(__ldg(pm + t)) * k;
        }
        tmp[(static_cast<size_t>(n) * cap_h + r) * out + x] = make_uchar2(clip8(a0), clip8(a1));
    }
}

// ------------------------------------------------------------------------------------------------ 3. vertical pass + histogram
__global__ void __launch_bounds__(256) seg_vpass_kernel(const pcb_seg_src *__restrict__ srcs, const pcb_seg_params *__restrict__ params,
                                                        int cap_h, int cap_w, int out, const uchar2 *__restrict__ tmp,
                                                        uint8_t *__restrict__ page, uint8_t *__restrict__ mask, int *__restrict__ hist) {
    __shared__ int vk[T * KMAX];
    __shared__ int vmin[T], vcnt[T];
    __shared__ int h[256];
    const int n = blockIdx.z, y0 = blockIdx.y * T, x0 = blockIdx.x * T, tid = threadIdx.x;
    const pcb_seg_params &p = params[n];
    const bool ok = source_ok(srcs[n], p, cap_h, cap_w);
    h[tid] = 0;
    if (tid < T) {
        int cnt = 0, m = 0;
        if (ok && y0 + tid < out) m = pil_coeffs(y0 + tid, p.height, out, vk + tid * KMAX, 1, &cnt);
        vmin[tid] = m;
        vcnt[tid] = cnt;
    }
    __syncthreads();
    const uchar2 *img = tmp + static_cast<size_t>(n) * cap_h * out;
    const size_t plane = static_cast<size_t>(n) * out * out;
    for (int q = tid; q < T * T; q += blockDim.x) {
        const int ly = q / T, lx = q - ly * T, gy = y0 + ly, gx = x0 + lx;
        if (gy >= out || gx >= out) continue;
        int a0 = 1 << (PB - 1), a1 = a0;
        const uchar2 *col = img + static_cast<size_t>(vmin[ly]) * out + gx;
        const int *k = vk + ly * KMAX;
        for (int t = 0; t < vcnt[ly]; ++t) {
            const uchar2 v = col[static_cast<size_t>(t) * out];
            a0 += v.x * k[t];
            a1 += v.y * k[t];
        }
        const int pv = ok ? clip8(a0) : 0, mv = ok ? clip8(a1) : 0;
        page[plane + static_cast<size_t>(gy) * out + gx] = static_cast<uint8_t>(pv);
        mask[plane + static_cast<size_t>(gy) * out + gx] = static_cast<uint8_t>(mv);
        atomicAdd(&h[pv], 1);
    }
    __syncthreads();
    if (h[tid]) atomicAdd(&hist[n * 256 + tid], h[tid]);
}

// ------------------------------------------------------------------------------------------------ 4. jitter + store
template <typename TO>
__global__ void __launch_bounds__(256) seg_store_kernel(const pcb_seg_params *__restrict__ params, const int *__restrict__ hist, int out,
                                                        const uint8_t *__restrict__ page, const uint8_t *__restrict__ mask,
                                                        const float4 norm_mean, const float4 norm_std, int normalize, TO *__restrict__ x,
                                                        float *__restrict__ target) {
    __shared__ long long part[8];
    const int n = blockIdx.y, tid = threadIdx.x;
    const pcb_seg_params p = params[n];
    // ImageEnhance.Contrast's mean of the image it is applied to: sum_v h[v] g(v) exactly, g = the brightness blend if that ran
    // first; ImageStat's sum / count in double, then int(mean + 0.5)
    long long s = static_cast<long long>(hist[n * 256 + tid]) * (p.brightness_first ? blend(0, tid, p.brightness) : tid);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((tid & 31) == 0) part[tid >> 5] = s;
    __syncthreads();
    long long sum = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += part[w];
    const int m = static_cast<int>(__dadd_rn(__ddiv_rn(static_cast<double>(sum), static_cast<double>(out) * out), 0.5));
    const size_t px = static_cast<size_t>(out) * out, base = static_cast<size_t>(n) * px;
    const float mean[3] = {norm_mean.x, norm_mean.y, norm_mean.z}, std[3] = {norm_std.x, norm_std.y, norm_std.z};
    const size_t end = min(px, static_cast<size_t>(blockIdx.x + 1) * SPB);
    for (size_t q = static_cast<size_t>(blockIdx.x) * SPB + tid; q < end; q += blockDim.x) {
        int v = page[base + q];
        if (p.brightness_first) v = blend(m, blend(0, v, p.brightness), p.contrast);
        else v = blend(0, blend(m, v, p.contrast), p.brightness);
        const float f = __fdiv_rn(static_cast<float>(v), 255.f);                  // to_tensor
        float o[8] = {f, f, f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (normalize) {
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c] = __fdiv_rn(__fsub_rn(f, mean[c]), std[c]);
        }
        Vec8<TO>::store(x + (base + q) * 8, o);
        target[base + q] = __fdiv_rn(static_cast<float>(mask[base + q]), 255.f);
    }
}

int validate(const pcb_seg_src *h_srcs, const pcb_seg_params *h_params, int n, int cap_n, int cap_h, int cap_w, int out) {
    PCB_CHECK(h_srcs && n >= 1 && n <= cap_n, "pcb_seg_validate: %d images for a batch of %d", n, cap_n);
    for (int i = 0; i < n; ++i) {
        const pcb_seg_src &s = h_srcs[i];
        PCB_CHECK(s.page && s.mask, "pcb_seg_validate: image %d has a null source", i);
        PCB_CHECK(s.h >= 1 && s.w >= 1 && s.h <= cap_h && s.w <= cap_w, "pcb_seg_validate: image %d is %dx%d, capacity %dx%d", i, s.h, s.w,
                  cap_h, cap_w);
        PCB_CHECK(s.page_stride >= s.w && s.mask_stride >= s.w, "pcb_seg_validate: image %d row strides %d / %d too small", i,
                  s.page_stride, s.mask_stride);
        if (!h_params) continue;
        const pcb_seg_params &p = h_params[i];
        PCB_CHECK(p.top >= 0 && p.left >= 0 && p.height >= 1 && p.width >= 1 && p.top + p.height <= s.h && p.left + p.width <= s.w,
                  "pcb_seg_validate: image %d crop box (%d, %d, %d, %d) is not inside its %dx%d source", i, p.top, p.left, p.height,
                  p.width, s.h, s.w);
        PCB_CHECK(p.height <= 8 * out && p.width <= 8 * out, "pcb_seg_validate: image %d crop box downscales more than 8x", i);
        PCB_CHECK((p.brightness_first == 0 || p.brightness_first == 1) && isfinite(p.brightness) && isfinite(p.contrast) &&
                      p.brightness >= 0.f && p.contrast >= 0.f,
                  "pcb_seg_validate: image %d has a bad order flag or jitter factor", i);
    }
    return 0;
}

}  // namespace

PCB_API int pcb_seg_validate(const pcb_seg_src *h_srcs, const pcb_seg_params *h_params, int n, int cap_n, int cap_h, int cap_w, int out) {
    PCB_CHECK(out >= 16 && out <= 4096 && cap_h <= 8 * out && cap_w <= 8 * out,
              "pcb_seg_validate: output %d and capacity %dx%d (at most 8x the output)", out, cap_h, cap_w);
    return validate(h_srcs, h_params, n, cap_n, cap_h, cap_w, out);
}

PCB_API int pcb_seg_sample(const pcb_seg_src *srcs, int n, uint64_t *rng, pcb_seg_params *params, pcb_stream_t stream) {
    PCB_CHECK(srcs && rng && params && n >= 1 && n <= 1024, "pcb_seg_sample: bad arguments (1..1024 images)");
    seg_sample_kernel<<<1, (n + 31) / 32 * 32, 0, ST>>>(srcs, n, reinterpret_cast<unsigned long long *>(rng), params);
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_seg_prepare(const pcb_seg_src *srcs, const pcb_seg_params *params, int n, int cap_h, int cap_w, int out, uint8_t *tmp,
                            uint8_t *planes, int *hist, const float *h_norm, void *x, int dtype, float *target, pcb_stream_t stream) {
    PCB_CHECK(srcs && params && tmp && planes && hist && x && target && (dtype == PCB_F32 || dtype == PCB_BF16),
              "pcb_seg_prepare: bad arguments");
    PCB_CHECK(n >= 1 && n <= 65535 && out >= 16 && out <= 4096 && cap_h >= 1 && cap_w >= 1 && cap_h <= 8 * out && cap_w <= 8 * out,
              "pcb_seg_prepare: %d images, output %d, capacity %dx%d (at most 8x the output)", n, out, cap_h, cap_w);
    const dim3 hgrid((out + HX - 1) / HX, (cap_h + HROWS - 1) / HROWS, n);
    seg_hpass_kernel<<<hgrid, HX, 0, ST>>>(srcs, params, cap_h, cap_w, out, reinterpret_cast<uchar2 *>(tmp), hist);
    PCB_LAUNCH_CHECK();
    const size_t px = static_cast<size_t>(out) * out;
    uint8_t *page = planes, *mask = planes + static_cast<size_t>(n) * px;
    const dim3 vgrid((out + T - 1) / T, (out + T - 1) / T, n);
    seg_vpass_kernel<<<vgrid, 256, 0, ST>>>(srcs, params, cap_h, cap_w, out, reinterpret_cast<const uchar2 *>(tmp), page, mask, hist);
    PCB_LAUNCH_CHECK();
    const float4 nm = h_norm ? make_float4(h_norm[0], h_norm[1], h_norm[2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 ns = h_norm ? make_float4(h_norm[3], h_norm[4], h_norm[5], 1.f) : make_float4(1.f, 1.f, 1.f, 1.f);
    const dim3 sgrid(static_cast<unsigned>((px + SPB - 1) / SPB), n);
    if (dtype == PCB_BF16)
        seg_store_kernel<bf16><<<sgrid, 256, 0, ST>>>(params, hist, out, page, mask, nm, ns, h_norm != nullptr, static_cast<bf16 *>(x), target);
    else
        seg_store_kernel<float><<<sgrid, 256, 0, ST>>>(params, hist, out, page, mask, nm, ns, h_norm != nullptr, static_cast<float *>(x), target);
    PCB_LAUNCH_CHECK();
    return 0;
}

// text_removal.cu -- the glue of the text-removal pipeline (engine.TextRemovalStep, DESIGN 5.2) between the segmentation
// network, the demo's mask post-processing (seg_ops.cu) and the inpainting U-Net:
//   1. removal_seg_input_kernel: the page's Normalize (EvaluateSet, Dataloader.py:271-273) and zero padding to the
//      segmentation grid (:296-303), stored as the network's 8-channel-padded NHWC input;
//   2. removal_holes_kernel: the text mask as the demo's {0, 255} image, > 0.4 * 255, cv2.dilate(10x10) (Dataloader.py:120-121),
//      then the valid plane and page * valid (:128-131) on the U-Net's grid, whose padding is hole;
//   3. removal_composite_kernel: valid ? page : fill (loss.py:196, comp_img), cropped to the page, fp32 NCHW.
// The page is fp32 NCHW [n, 3, h, w], contiguous.
#include "pcb_common.cuh"
#include "pcb_dilate.cuh"

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int LT = 256;       // threads per block of the per-pixel kernels
constexpr int T = 32;         // removal_holes_kernel: output tile edge
constexpr int HT = dil::Tile<T>::HT;

struct Norm { float mean[3], std[3]; int on; };

// ------------------------------------------------------------------------------------------------ 1. segmentation input
// One thread per pixel of the [n, hs, ws] grid; (x - mean) / std in torchvision's order (sub_ then div_, both rounded), then
// one rounding to the compute dtype.  Padding pixels and channels 3..7 are written as zero.
template <typename TO>
__global__ void __launch_bounds__(LT) removal_seg_input_kernel(const float *__restrict__ page, int n, int h, int w, int hs, int ws, Norm nm,
                                                               TO *__restrict__ out) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x, total = static_cast<long long>(n) * hs * ws;
    if (i >= total) return;
    const int x = static_cast<int>(i % ws);
    const long long r = i / ws;
    const int y = static_cast<int>(r % hs), b = static_cast<int>(r / hs);
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (y < h && x < w) {
        const size_t plane = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float p = __ldg(page + (static_cast<size_t>(b) * 3 + c) * plane + pix);
            v[c] = nm.on ? __fdiv_rn(__fsub_rn(p, nm.mean[c]), nm.std[c]) : p;
        }
    }
    Vec8<TO>::store(out + i * 8, v);
}

// ------------------------------------------------------------------------------------------------ 2. holes
// Per 32 x 32 tile of the U-Net grid [hu, wu]: the text mask over the tile and its 5 / 4 halo (pixels outside the page do not
// take part), dilated in shared memory, then per pixel the valid plane (0 = hole) and the 8-channel corrupted image.  Inside
// the page valid = !dilated and corrupted = page * valid in fp32, rounded once; the padding is hole and zero.
template <typename TO>
__global__ void __launch_bounds__(LT) removal_holes_kernel(const uint8_t *__restrict__ text_mask, const float *__restrict__ page, int h, int w,
                                                           int hu, int wu, uint8_t *__restrict__ valid, TO *__restrict__ corrupted) {
    __shared__ dil::Tile<T> dt;
    const int b = blockIdx.z, y0 = blockIdx.y * T, x0 = blockIdx.x * T, tid = threadIdx.x;
    const size_t plane = static_cast<size_t>(h) * w;
    const uint8_t *tm = text_mask + static_cast<size_t>(b) * plane;
    for (int q = tid; q < HT * HT; q += LT) {
        const int ly = q / HT, lx = q - ly * HT, gy = y0 - dil::BEFORE + ly, gx = x0 - dil::BEFORE + lx;
        // the demo's mask image holds 255 where the text mask is set (to_pil_image(mask).convert("L")), so the threshold
        // > 0.4 * 255 keeps exactly the set pixels
        dt.hole[ly][lx] = (gy >= 0 && gy < h && gx >= 0 && gx < w) ? (__ldg(tm + static_cast<size_t>(gy) * w + gx) != 0) : 0;
    }
    __syncthreads();
    dil::row_max(dt, tid, LT);
    __syncthreads();
    const size_t uplane = static_cast<size_t>(hu) * wu;
    for (int q = tid; q < T * T; q += LT) {
        const int ly = q / T, lx = q - ly * T, gy = y0 + ly, gx = x0 + lx;
        if (gy >= hu || gx >= wu) continue;
        const bool inside = gy < h && gx < w;
        const bool hole = inside ? dil::col_max(dt, ly, lx) != 0 : true;
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (inside) {
            const float keep = hole ? 0.f : 1.f;                             // binary_mask = 1 - ToTensor(mask)
            const size_t pix = static_cast<size_t>(gy) * w + gx;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = __fmul_rn(__ldg(page + (static_cast<size_t>(b) * 3 + c) * plane + pix), keep);
        }
        const size_t upix = static_cast<size_t>(b) * uplane + static_cast<size_t>(gy) * wu + gx;
        Vec8<TO>::store(corrupted + upix * 8, v);
        valid[upix] = hole ? 0 : 1;
    }
}

// ------------------------------------------------------------------------------------------------ 3. composite
// One thread per page pixel: the page where valid, the U-Net output (NHWC, pixel stride `cs`, on the [hu, wu] grid) elsewhere.
template <typename TI>
__global__ void __launch_bounds__(LT) removal_composite_kernel(const TI *__restrict__ fill, int cs, const float *__restrict__ page,
                                                               const uint8_t *__restrict__ valid, int n, int h, int w, int hu, int wu,
                                                               float *__restrict__ out) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x, total = static_cast<long long>(n) * h * w;
    if (i >= total) return;
    const int x = static_cast<int>(i % w);
    const long long r = i / w;
    const int y = static_cast<int>(r % h), b = static_cast<int>(r / h);
    const size_t plane = static_cast<size_t>(h) * w, pix = static_cast<size_t>(y) * w + x;
    const size_t upix = (static_cast<size_t>(b) * hu + y) * wu + x;
    const bool keep = __ldg(valid + upix) != 0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t o = (static_cast<size_t>(b) * 3 + c) * plane + pix;
        out[o] = keep ? __ldg(page + o) : to_f32<TI>(fill[upix * cs + c]);
    }
}

unsigned blocks(long long total) { return static_cast<unsigned>((total + LT - 1) / LT); }

}  // namespace

PCB_API int pcb_removal_seg_input(const float *page, int n, int h, int w, const float *norm, int hs, int ws, void *out, int dtype,
                                  pcb_stream_t stream) {
    const char *fn = "pcb_removal_seg_input";
    PCB_CHECK(page && out, "%s: null pointer", fn);
    PCB_CHECK(dtype == PCB_F32 || dtype == PCB_BF16, "%s: bad dtype code %d", fn, dtype);
    PCB_CHECK(n >= 1 && h >= 1 && w >= 1, "%s: empty page %dx3x%dx%d", fn, n, h, w);
    PCB_CHECK(hs >= h && ws >= w, "%s: padded size %dx%d smaller than the %dx%d page", fn, hs, ws, h, w);
    const long long total = static_cast<long long>(n) * hs * ws;
    PCB_CHECK(total <= (1ll << 38), "%s: %lld pixels", fn, total);
    PCB_CHECK(reinterpret_cast<uintptr_t>(out) % (8 * pcb_dtype_size(dtype)) == 0, "%s: output not aligned to its 8-channel pixels", fn);
    Norm nm{};
    if (norm) {
        for (int c = 0; c < 3; ++c) {
            nm.mean[c] = norm[c];
            nm.std[c] = norm[3 + c];
        }
        nm.on = 1;
    }
    if (dtype == PCB_BF16)
        removal_seg_input_kernel<bf16><<<blocks(total), LT, 0, ST>>>(page, n, h, w, hs, ws, nm, static_cast<bf16 *>(out));
    else
        removal_seg_input_kernel<float><<<blocks(total), LT, 0, ST>>>(page, n, h, w, hs, ws, nm, static_cast<float *>(out));
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_removal_holes(const uint8_t *text_mask, const float *page, int n, int h, int w, int hu, int wu, uint8_t *valid,
                              void *corrupted, int dtype, pcb_stream_t stream) {
    const char *fn = "pcb_removal_holes";
    PCB_CHECK(text_mask && page && valid && corrupted, "%s: null pointer", fn);
    PCB_CHECK(dtype == PCB_F32 || dtype == PCB_BF16, "%s: bad dtype code %d", fn, dtype);
    PCB_CHECK(n >= 1 && n <= 65535 && h >= 1 && w >= 1, "%s: page %dx3x%dx%d (1..65535 pages)", fn, n, h, w);
    PCB_CHECK(hu >= h && wu >= w, "%s: padded size %dx%d smaller than the %dx%d page", fn, hu, wu, h, w);
    PCB_CHECK((hu + T - 1) / T <= 65535, "%s: padded height %d too large", fn, hu);
    PCB_CHECK(reinterpret_cast<uintptr_t>(corrupted) % (8 * pcb_dtype_size(dtype)) == 0, "%s: corrupted buffer not aligned to its 8-channel pixels",
              fn);
    const dim3 grid((wu + T - 1) / T, (hu + T - 1) / T, n);
    if (dtype == PCB_BF16)
        removal_holes_kernel<bf16><<<grid, LT, 0, ST>>>(text_mask, page, h, w, hu, wu, valid, static_cast<bf16 *>(corrupted));
    else
        removal_holes_kernel<float><<<grid, LT, 0, ST>>>(text_mask, page, h, w, hu, wu, valid, static_cast<float *>(corrupted));
    PCB_LAUNCH_CHECK();
    return 0;
}

PCB_API int pcb_removal_composite(const void *fill, int dtype, int cstride, const float *page, const uint8_t *valid, int n, int h, int w,
                                  int hu, int wu, float *out, pcb_stream_t stream) {
    const char *fn = "pcb_removal_composite";
    PCB_CHECK(fill && page && valid && out, "%s: null pointer", fn);
    PCB_CHECK(dtype == PCB_F32 || dtype == PCB_BF16, "%s: bad dtype code %d", fn, dtype);
    PCB_CHECK(cstride >= 3, "%s: channel stride %d of a 3-channel output", fn, cstride);
    PCB_CHECK(n >= 1 && h >= 1 && w >= 1, "%s: empty page %dx3x%dx%d", fn, n, h, w);
    PCB_CHECK(hu >= h && wu >= w, "%s: padded size %dx%d smaller than the %dx%d page", fn, hu, wu, h, w);
    const long long total = static_cast<long long>(n) * h * w;
    PCB_CHECK(total <= (1ll << 38), "%s: %lld pixels", fn, total);
    if (dtype == PCB_BF16)
        removal_composite_kernel<bf16><<<blocks(total), LT, 0, ST>>>(static_cast<const bf16 *>(fill), cstride, page, valid, n, h, w, hu, wu, out);
    else
        removal_composite_kernel<float><<<blocks(total), LT, 0, ST>>>(static_cast<const float *>(fill), cstride, page, valid, n, h, w, hu, wu,
                                                                      out);
    PCB_LAUNCH_CHECK();
    return 0;
}

// text_removal.cu -- the glue of the text-removal pipeline (engine.TextRemovalStep, DESIGN 5.2) between the segmentation
// network, the demo's mask post-processing (seg_ops.cu) and the inpainting U-Net:
//   0. page_coeffs_kernel, page_hpass_kernel, page_vpass_kernel: EvaluateSet's page resize (Dataloader.py:290-291),
//      to_tensor(to_pil_image(page).resize((rw, rh), Image.BICUBIC)) with Pillow's integer resampler bit for bit;
//   1. removal_seg_input_kernel: the page's Normalize (EvaluateSet, Dataloader.py:271-273) and zero padding to the
//      segmentation grid (:296-303), stored as the network's 8-channel-padded NHWC input;
//   2. removal_holes_kernel: the text mask as the demo's {0, 255} image, > 0.4 * 255, cv2.dilate(10x10) (Dataloader.py:120-121),
//      then the valid plane and page * valid (:128-131) on the U-Net's grid, whose padding is hole;
//   3. removal_composite_kernel: valid ? page : fill (loss.py:196, comp_img), cropped to the page, fp32 NCHW.
// The page is fp32 NCHW [n, 3, h, w], contiguous.
#include "pcb_dilate.cuh"
#include "pil_data.cuh"

#define ST static_cast<cudaStream_t>(stream)
#define PCB_API extern "C" __attribute__((visibility("default")))

namespace {

constexpr int LT = 256;       // threads per block of the per-pixel kernels
constexpr int T = 32;         // removal_holes_kernel: output tile edge
constexpr int HT = dil::Tile<T>::HT;

struct Norm { float mean[3], std[3]; int on; };

// ------------------------------------------------------------------------------------------------ 0. page resize
// Pillow's ImagingResample of an RGB image: a horizontal pass into a clipped uint8 image, then a vertical pass.  Both passes
// always run: at scale 1 the bicubic weights are exactly {0, 1 << 22, 0, 0}, the identity that Pillow's skipped pass gives.
constexpr int RED = 16;                        // the largest reduction per axis (in / out)
constexpr int KP = pil::taps_for(RED);         // 65 taps
constexpr int HX = 128;                        // horizontal pass: output columns per block (one per thread)
constexpr int HROWS = 16;                      // horizontal pass: input rows per block

struct ResizeWs {                              // the caller's workspace: weights [KP][rw + rh], bounds, the uint8 image
    int *k;
    int2 *bounds;                              // (first tap, taps) per output column, then per output row
    uchar4 *tmp;                               // [n, h, rw], RGB + an unused byte
};

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

ResizeWs resize_ws(void *base, int rh, int rw) {
    char *p = static_cast<char *>(base);
    const size_t ks = static_cast<size_t>(rw) + rh, kb = align256(ks * KP * sizeof(int)), bb = align256(ks * sizeof(int2));
    return ResizeWs{reinterpret_cast<int *>(p), reinterpret_cast<int2 *>(p + kb), reinterpret_cast<uchar4 *>(p + kb + bb)};
}

size_t resize_ws_bytes(int n, int h, int rh, int rw) {
    const size_t ks = static_cast<size_t>(rw) + rh;
    return align256(ks * KP * sizeof(int)) + align256(ks * sizeof(int2)) + static_cast<size_t>(n) * h * rw * sizeof(uchar4);
}

// One thread per output column (i < rw, over the page width) or output row (i >= rw, over its height).
__global__ void __launch_bounds__(HX) page_coeffs_kernel(int h, int w, int rh, int rw, int *__restrict__ k, int2 *__restrict__ bounds) {
    const int i = blockIdx.x * HX + threadIdx.x, ks = rw + rh;
    if (i >= ks) return;
    int cnt;
    const int first = i < rw ? pil::pil_coeffs<KP>(i, w, rw, k + i, ks, &cnt) : pil::pil_coeffs<KP>(i - rw, h, rh, k + i, ks, &cnt);
    bounds[i] = make_int2(first, cnt);
}

// Output column x of HROWS input rows of one image: the three channels' bytes, weighted and clipped as Pillow's
// ImagingResampleHorizontal_8bpc does.  The column's weights go to shared memory (this thread's column only: no barrier).
__global__ void __launch_bounds__(HX) page_hpass_kernel(const float *__restrict__ page, int h, int w, int rh, int rw, const int *__restrict__ k,
                                                        const int2 *__restrict__ bounds, uchar4 *__restrict__ tmp) {
    __shared__ int kk[KP * HX];
    const int b = blockIdx.z, x = blockIdx.x * HX + threadIdx.x, row0 = blockIdx.y * HROWS;
    if (x >= rw) return;
    const int2 bd = __ldg(bounds + x);
    const int ks = rw + rh;
    for (int t = 0; t < bd.y; ++t) kk[t * HX + threadIdx.x] = __ldg(k + static_cast<size_t>(t) * ks + x);
    const size_t plane = static_cast<size_t>(h) * w;
    const float *src = page + static_cast<size_t>(b) * 3 * plane + bd.x;
    const int rows = min(HROWS, h - row0);
    for (int r = row0; r < row0 + rows; ++r) {
        const float *p = src + static_cast<size_t>(r) * w;
        int a0 = 1 << (pil::PB - 1), a1 = a0, a2 = a0;
        for (int t = 0; t < bd.y; ++t) {
            const int kt = kk[t * HX + threadIdx.x];
            a0 += pil::page_byte(__ldg(p + t)) * kt;
            a1 += pil::page_byte(__ldg(p + plane + t)) * kt;
            a2 += pil::page_byte(__ldg(p + 2 * plane + t)) * kt;
        }
        tmp[(static_cast<size_t>(b) * h + r) * rw + x] =
            make_uchar4(static_cast<uint8_t>(pil::clip8(a0)), static_cast<uint8_t>(pil::clip8(a1)), static_cast<uint8_t>(pil::clip8(a2)), 0);
    }
}

// One thread per output pixel: Pillow's vertical pass over the uint8 image, then to_tensor's / 255 into fp32 NCHW.
__global__ void __launch_bounds__(LT) page_vpass_kernel(const uchar4 *__restrict__ tmp, int n, int h, int rh, int rw, const int *__restrict__ k,
                                                        const int2 *__restrict__ bounds, float *__restrict__ out) {
    const long long i = static_cast<long long>(blockIdx.x) * LT + threadIdx.x, total = static_cast<long long>(n) * rh * rw;
    if (i >= total) return;
    const int x = static_cast<int>(i % rw);
    const long long r = i / rw;
    const int y = static_cast<int>(r % rh), b = static_cast<int>(r / rh);
    const int ks = rw + rh;
    const int2 bd = __ldg(bounds + rw + y);
    const uchar4 *col = tmp + (static_cast<size_t>(b) * h + bd.x) * rw + x;
    const int *ky = k + rw + y;
    int a0 = 1 << (pil::PB - 1), a1 = a0, a2 = a0;
    for (int t = 0; t < bd.y; ++t) {
        const int kt = __ldg(ky + static_cast<size_t>(t) * ks);
        const uchar4 v = col[static_cast<size_t>(t) * rw];
        a0 += v.x * kt;
        a1 += v.y * kt;
        a2 += v.z * kt;
    }
    const size_t plane = static_cast<size_t>(rh) * rw, o = static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(y) * rw + x;
    out[o] = __fdiv_rn(static_cast<float>(pil::clip8(a0)), 255.f);
    out[o + plane] = __fdiv_rn(static_cast<float>(pil::clip8(a1)), 255.f);
    out[o + 2 * plane] = __fdiv_rn(static_cast<float>(pil::clip8(a2)), 255.f);
}

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

// zero when the sizes are out of range (pcb_page_resize_bicubic says why)
PCB_API size_t pcb_page_resize_workspace(int n, int h, int w, int rh, int rw) {
    if (n < 1 || h < 1 || w < 1 || rh < 1 || rw < 1) return 0;
    return resize_ws_bytes(n, h, rh, rw);
}

PCB_API int pcb_page_resize_bicubic(const float *page, int n, int h, int w, int rh, int rw, void *workspace, float *out, pcb_stream_t stream) {
    const char *fn = "pcb_page_resize_bicubic";
    PCB_CHECK(page && workspace && out, "%s: null pointer", fn);
    PCB_CHECK(n >= 1 && n <= 65535 && h >= 1 && w >= 1 && rh >= 1 && rw >= 1, "%s: page %dx3x%dx%d to %dx%d (1..65535 pages, no empty side)",
              fn, n, h, w, rh, rw);
    PCB_CHECK(h <= static_cast<long long>(RED) * rh && w <= static_cast<long long>(RED) * rw,
              "%s: %dx%d to %dx%d reduces more than %dx on an axis", fn, h, w, rh, rw, RED);
    PCB_CHECK((h + HROWS - 1) / HROWS <= 65535, "%s: page height %d too large", fn, h);
    const long long total = static_cast<long long>(n) * rh * rw;
    PCB_CHECK(total <= (1ll << 38) && static_cast<long long>(n) * h * w <= (1ll << 38), "%s: too many pixels", fn);
    PCB_CHECK(reinterpret_cast<uintptr_t>(workspace) % 256 == 0, "%s: workspace not aligned to 256 bytes", fn);
    const ResizeWs ws = resize_ws(workspace, rh, rw);
    page_coeffs_kernel<<<(rw + rh + HX - 1) / HX, HX, 0, ST>>>(h, w, rh, rw, ws.k, ws.bounds);
    PCB_LAUNCH_CHECK();
    page_hpass_kernel<<<dim3((rw + HX - 1) / HX, (h + HROWS - 1) / HROWS, n), HX, 0, ST>>>(page, h, w, rh, rw, ws.k, ws.bounds, ws.tmp);
    PCB_LAUNCH_CHECK();
    page_vpass_kernel<<<blocks(total), LT, 0, ST>>>(ws.tmp, n, h, rh, rw, ws.k, ws.bounds, out);
    PCB_LAUNCH_CHECK();
    return 0;
}

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

// inpaint_data.cu -- the inpainting data paths for a batch, in three launches, for two source kinds:
//   * mask file (ImageInpaintingData.process_images, Dataloader.py:110-132): an RGB page and its text mask;
//   * raw/clean pair (TestDataset.process_images, Dataloader.py:201-222): a raw RGB page and its text-cleaned copy, the mask
//     being the thresholded |L(raw) - L(clean)| (get_mask) and no grayscale draw.
//   1. inpaint_sample_kernel: one thread per image draws the crop box (RandomResizedCrop.get_params), the grayscale flag and
//      the strokes (random_masks) from Philox4x32-10; seed and step counter live in device memory and the kernel advances the
//      counter, so every graph replay draws fresh parameters.  Skipped when the caller supplies parameters.
//   2. inpaint_hpass_kernel: Pillow's horizontal bicubic pass over every row of each image's crop box, both sources together,
//      into a uint8 intermediate (mask file: RGBM, 4 bytes per pixel; pair: raw RGB0 | clean RGB0, 8 bytes per pixel).
//   3. inpaint_fused_kernel: per 32x32 output tile, the vertical pass over the tile plus the 9-pixel dilation halo, the mask
//      value (the resized text mask, or the L difference of the pair), the strokes, the threshold, the 10x10 dilation
//      (separable max in shared memory), grayscale, /255, x mask and the three stores.
// Grids are sized from the batcher's capacity (largest source), so one captured graph serves any mix of source sizes.
// The resampler follows Pillow's fixed-point 8-bit path bit for bit (pil_data.cuh, shared with seg_data.cu).
#include "pcb_dilate.cuh"
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
constexpr int T = 32;         // fused kernel: output tile edge
constexpr int HT = dil::Tile<T>::HT;   // tile + dilation halo (5 rows / columns before, 4 after: cv2's anchor of a 10x10 kernel)

// What the kernels need to know about a source kind: its descriptor, the intermediate pixel, the horizontal pass of one box row
// at one output column (taps k[0], k[HX], ...), and the vertical pass of one output pixel (taps k[0], k[1], ...; rows `step`
// pixels apart), which yields the clean RGB and the mask value the threshold sees.
struct MaskFile {
    using Src = pcb_inpaint_src;
    using Px = uchar4;
    static __device__ __forceinline__ Px hrow(const Src &s, int y, int x, const int *k, int nt) {
        const uint8_t *pr = s.rgb + static_cast<size_t>(y) * s.rgb_stride + static_cast<size_t>(x) * 3;
        const uint8_t *pm = s.mask + static_cast<size_t>(y) * s.mask_stride + x;
        int a0 = 1 << (PB - 1), a1 = a0, a2 = a0, a3 = a0;
        for (int t = 0; t < nt; ++t) {
            const int kt = k[t * HX];
            a0 += static_cast<int>(__ldg(pr + 3 * t)) * kt;
            a1 += static_cast<int>(__ldg(pr + 3 * t + 1)) * kt;
            a2 += static_cast<int>(__ldg(pr + 3 * t + 2)) * kt;
            a3 += static_cast<int>(__ldg(pm + t)) * kt;
        }
        return make_uchar4(clip8(a0), clip8(a1), clip8(a2), clip8(a3));
    }
    static __device__ __forceinline__ int vcol(const Px *col, size_t step, const int *k, int nt, uchar4 &rgb) {
        int a0 = 1 << (PB - 1), a1 = a0, a2 = a0, a3 = a0;
        for (int t = 0; t < nt; ++t) {
            const uchar4 v = col[static_cast<size_t>(t) * step];
            a0 += v.x * k[t];
            a1 += v.y * k[t];
            a2 += v.z * k[t];
            a3 += v.w * k[t];
        }
        rgb = make_uchar4(clip8(a0), clip8(a1), clip8(a2), 0);
        return clip8(a3);
    }
};

__device__ __forceinline__ unsigned pil_l(unsigned r, unsigned g, unsigned b) {        // Image.convert("L")
    return (19595u * r + 38470u * g + 7471u * b + 0x8000u) >> 16;
}

struct Pair {
    using Src = pcb_inpaint_pair_src;
    using Px = uint2;                      // .x: raw R | G << 8 | B << 16, .y: clean, the same
    static __device__ __forceinline__ Px hrow(const Src &s, int y, int x, const int *k, int nt) {
        const uint8_t *pa = s.raw + static_cast<size_t>(y) * s.raw_stride + static_cast<size_t>(x) * 3;
        const uint8_t *pb = s.clean + static_cast<size_t>(y) * s.clean_stride + static_cast<size_t>(x) * 3;
        int a[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) a[c] = 1 << (PB - 1);
        for (int t = 0; t < nt; ++t) {
            const int kt = k[t * HX];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                a[c] += static_cast<int>(__ldg(pa + 3 * t + c)) * kt;
                a[3 + c] += static_cast<int>(__ldg(pb + 3 * t + c)) * kt;
            }
        }
        return make_uint2(clip8(a[0]) | clip8(a[1]) << 8 | clip8(a[2]) << 16, clip8(a[3]) | clip8(a[4]) << 8 | clip8(a[5]) << 16);
    }
    static __device__ __forceinline__ int vcol(const Px *col, size_t step, const int *k, int nt, uchar4 &rgb) {
        int a[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) a[c] = 1 << (PB - 1);
        for (int t = 0; t < nt; ++t) {
            const uint2 v = col[static_cast<size_t>(t) * step];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                a[c] += static_cast<int>((v.x >> (8 * c)) & 0xff) * k[t];
                a[3 + c] += static_cast<int>((v.y >> (8 * c)) & 0xff) * k[t];
            }
        }
        rgb = make_uchar4(clip8(a[3]), clip8(a[4]), clip8(a[5]), 0);
        const int lr = pil_l(clip8(a[0]), clip8(a[1]), clip8(a[2])), lc = pil_l(rgb.x, rgb.y, rgb.z);
        return lr > lc ? lr - lc : lc - lr;                                   // ImageChops.difference
    }
};

template <typename S>
__device__ __forceinline__ bool source_ok(const S &s, const pcb_inpaint_params &p, int cap_h, int cap_w) {
    return s.h >= 1 && s.w >= 1 && s.h <= cap_h && s.w <= cap_w && p.top >= 0 && p.left >= 0 && p.height >= 1 && p.width >= 1 &&
           p.top + p.height <= s.h && p.left + p.width <= s.w;
}

// ------------------------------------------------------------------------------------------------ 1. parameter sampler
// `gray`: draw RandomGrayscale(0.4) (mask file) or leave the flag 0 (pair: TestDataset's transformer has none); the slot is
// skipped either way, so both kinds draw the same boxes and strokes from the same (seed, counter, sizes).
template <typename S>
__global__ void __launch_bounds__(1024) inpaint_sample_kernel(const S *__restrict__ srcs, int n, int out, int strokes, int gray,
                                                              unsigned long long *rng, pcb_inpaint_params *__restrict__ params) {
    const int t = threadIdx.x;
    const unsigned long long seed = rng[0], step = rng[1];
    __syncthreads();
    if (t == 0) rng[1] = step + 1;
    if (t >= n) return;
    const pil::Draws d(static_cast<uint32_t>(t), step, seed);
    const int H = srcs[t].h, W = srcs[t].w;
    pcb_inpaint_params &p = params[t];
    p = pcb_inpaint_params{};
    const pil::Box box = pil::crop_box(d, H, W, 0.5f, 1.5f);        // RandomResizedCrop.get_params(scale=(0.5, 2.0))
    p.top = box.top;
    p.left = box.left;
    p.height = box.height;
    p.width = box.width;
    p.gray = gray && static_cast<double>(d.u(40)) < 0.4 ? 1 : 0;    // RandomGrayscale(p=0.4)
    if (strokes) {                                                   // random_masks(size=out, offset=10)
        const int off = 10;
        p.nlines = d.randint(41, 1, 5);
        for (int k = 0; k < p.nlines; ++k) {
            const int b = 42 + 5 * k;
            const int x0 = d.randint(b, off, out - 1), y0 = d.randint(b + 1, off, out - 1);
            const int x1 = min(max(d.randint(b + 2, off, out - 1), x0 - 75), x0 + 75);
            const int y1 = min(max(d.randint(b + 3, off, out - 1), y0 - 75), y0 + 75);
            p.lines[k][0] = x0; p.lines[k][1] = y0; p.lines[k][2] = x1; p.lines[k][3] = y1;
            p.lines[k][4] = d.randint(b + 4, 15, 20);
        }
        p.nellipses = d.randint(67, 1, 5);
        for (int k = 0; k < p.nellipses; ++k) {
            const int b = 68 + 4 * k;
            int c0 = d.randint(b, off, out - off - 1), c1 = d.randint(b + 1, off, out - off - 1);
            if (c1 < c0) { const int tmp = c0; c0 = c1; c1 = tmp; }                // cords.sort(): x0 <= y0
            p.ellipses[k][0] = c0; p.ellipses[k][1] = c1;
            p.ellipses[k][2] = min(max(c0 + d.randint(b + 2, 20, 69), off), out - off);
            p.ellipses[k][3] = min(max(c1 + d.randint(b + 3, 20, 69), off), out - off);
        }
    }
}

// ------------------------------------------------------------------------------------------------ 2. horizontal pass
template <typename K>
__global__ void __launch_bounds__(HX) inpaint_hpass_kernel(const typename K::Src *__restrict__ srcs, const pcb_inpaint_params *__restrict__ params,
                                                           int cap_h, int cap_w, int out, typename K::Px *__restrict__ tmp) {
    __shared__ int kk[KMAX * HX];
    const int n = blockIdx.z, x = blockIdx.x * HX + threadIdx.x, row0 = blockIdx.y * HROWS;
    const typename K::Src s = srcs[n];
    const pcb_inpaint_params &p = params[n];
    const int top = p.top, left = p.left, bh = p.height, bw = p.width;
    if (row0 >= bh || x >= out || !source_ok(s, p, cap_h, cap_w)) return;
    int nt;
    const int xmin = pil_coeffs(x, bw, out, kk + threadIdx.x, HX, &nt);     // this thread's column only: no barrier
    const int rows = min(HROWS, bh - row0);
    for (int r = row0; r < row0 + rows; ++r)
        tmp[(static_cast<size_t>(n) * cap_h + r) * out + x] = K::hrow(s, top + r, left + xmin, kk + threadIdx.x, nt);
}

// ------------------------------------------------------------------------------------------------ 3. fused tail
// Stroke rules (documented in DESIGN 4.8; numpy restatement in oracle/inpaint_data.py), exact integer arithmetic:
//   line (x0, y0, x1, y1, w): 0 <= <p - p0, d> <= |d|^2 and 4 cross(p - p0, d)^2 <= w^2 |d|^2; zero length: the pixel (x0, y0)
//   ellipse (x0, y0, x1, y1): (2x - x0 - x1)^2 B^2 + (2y - y0 - y1)^2 A^2 <= A^2 B^2, A = x1 - x0 + 1, B = y1 - y0 + 1
__device__ bool in_stroke(const pcb_inpaint_params &p, int x, int y) {
    for (int k = 0; k < p.nlines; ++k) {
        const long long x0 = p.lines[k][0], y0 = p.lines[k][1], dx = p.lines[k][2] - x0, dy = p.lines[k][3] - y0, w = p.lines[k][4];
        const long long px = x - x0, py = y - y0;
        if (dx == 0 && dy == 0) {
            if (px == 0 && py == 0) return true;
            continue;
        }
        const long long l2 = dx * dx + dy * dy, dot = px * dx + py * dy, cr = px * dy - py * dx;
        if (dot >= 0 && dot <= l2 && 4 * cr * cr <= w * w * l2) return true;
    }
    for (int k = 0; k < p.nellipses; ++k) {
        const long long x0 = p.ellipses[k][0], y0 = p.ellipses[k][1], x1 = p.ellipses[k][2], y1 = p.ellipses[k][3];
        const long long A = x1 - x0 + 1, B = y1 - y0 + 1, ex = 2ll * x - x0 - x1, ey = 2ll * y - y0 - y1;
        if (ex * ex * B * B + ey * ey * A * A <= A * A * B * B) return true;
    }
    return false;
}

template <typename K, typename TO>
__global__ void __launch_bounds__(256) inpaint_fused_kernel(const typename K::Src *__restrict__ srcs, const pcb_inpaint_params *__restrict__ params,
                                                            int cap_h, int cap_w, int out, int strokes, const typename K::Px *__restrict__ tmp,
                                                            TO *__restrict__ corrupted, uint8_t *__restrict__ plane, float *__restrict__ clean) {
    __shared__ int vk[HT * KMAX];
    __shared__ int vmin[HT], vcnt[HT];
    __shared__ dil::Tile<T> dt;
    __shared__ uchar4 rgb[T][T];
    const int n = blockIdx.z, y0 = blockIdx.y * T, x0 = blockIdx.x * T, tid = threadIdx.x;
    const pcb_inpaint_params &p = params[n];
    const bool ok = source_ok(srcs[n], p, cap_h, cap_w);
    const int bh = p.height;
    if (tid < HT) {
        const int yy = y0 - 5 + tid;
        int cnt = 0, m = 0;
        if (ok && yy >= 0 && yy < out) m = pil_coeffs(yy, bh, out, vk + tid * KMAX, 1, &cnt);
        vmin[tid] = m;
        vcnt[tid] = cnt;
    }
    __syncthreads();
    // vertical pass over the tile + halo; the mask value is thresholded (and stroked), RGB kept for the tile itself
    const typename K::Px *img = tmp + static_cast<size_t>(n) * cap_h * out;
    for (int q = tid; q < HT * HT; q += blockDim.x) {
        const int ly = q / HT, lx = q - ly * HT, gy = y0 - 5 + ly, gx = x0 - 5 + lx;
        uint8_t h = 0;
        if (ok && gy >= 0 && gy < out && gx >= 0 && gx < out) {
            uchar4 c;
            const int mv = K::vcol(img + static_cast<size_t>(vmin[ly]) * out + gx, out, vk + ly * KMAX, vcnt[ly], c);
            h = mv >= 103 || (strokes && in_stroke(p, gx, gy));                // mask > 0.4 * 255; strokes are drawn at 255
            if (ly >= 5 && ly < 5 + T && lx >= 5 && lx < 5 + T) rgb[ly - 5][lx - 5] = c;
        }
        dt.hole[ly][lx] = h;
    }
    __syncthreads();
    dil::row_max(dt, tid, blockDim.x);                                   // 10-wide row max: columns x-5 .. x+4
    __syncthreads();
    const size_t plane_px = static_cast<size_t>(out) * out;
    for (int q = tid; q < T * T; q += blockDim.x) {                       // 10-high column max, then the per-pixel tail
        const int ly = q / T, lx = q - ly * T, gy = y0 + ly, gx = x0 + lx;
        if (gy >= out || gx >= out) continue;
        const uint8_t m = ok ? dil::col_max(dt, ly, lx) : 1;
        uchar4 c = ok ? rgb[ly][lx] : make_uchar4(0, 0, 0, 0);
        if (p.gray) {
            const unsigned l = (19595u * c.x + 38470u * c.y + 7471u * c.z + 0x8000u) >> 16;
            c.x = c.y = c.z = static_cast<unsigned char>(l);
        }
        const float binary = __fsub_rn(1.f, __fdiv_rn(m ? 255.f : 0.f, 255.f));   // 1 - ToTensor(mask)
        const float f[3] = {__fdiv_rn(static_cast<float>(c.x), 255.f), __fdiv_rn(static_cast<float>(c.y), 255.f),
                            __fdiv_rn(static_cast<float>(c.z), 255.f)};
        const size_t pix = static_cast<size_t>(gy) * out + gx;
        float v[8] = {__fmul_rn(f[0], binary), __fmul_rn(f[1], binary), __fmul_rn(f[2], binary), 0.f, 0.f, 0.f, 0.f, 0.f};
        Vec8<TO>::store(corrupted + (static_cast<size_t>(n) * plane_px + pix) * 8, v);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) clean[(static_cast<size_t>(n) * 3 + ch) * plane_px + pix] = f[ch];
        plane[static_cast<size_t>(n) * plane_px + pix] = m ? 0 : 1;
    }
}

// The checks both source kinds share: image i's size against the capacity and, with parameters, its crop box and strokes.
// `fn` names the entry point in the messages.
int validate_image(const char *fn, int i, int h, int w, const pcb_inpaint_params *hp, int cap_h, int cap_w, int out) {
    PCB_CHECK(h >= 1 && w >= 1 && h <= cap_h && w <= cap_w, "%s: image %d is %dx%d, capacity %dx%d", fn, i, h, w, cap_h, cap_w);
    if (!hp) return 0;
    const pcb_inpaint_params &p = hp[i];
    PCB_CHECK(p.top >= 0 && p.left >= 0 && p.height >= 1 && p.width >= 1 && p.top + p.height <= h && p.left + p.width <= w,
              "%s: image %d crop box (%d, %d, %d, %d) is not inside its %dx%d source", fn, i, p.top, p.left, p.height, p.width, h, w);
    PCB_CHECK(p.height <= 8 * out && p.width <= 8 * out, "%s: image %d crop box downscales more than 8x", fn, i);
    PCB_CHECK((p.gray == 0 || p.gray == 1) && p.nlines >= 0 && p.nlines <= 5 && p.nellipses >= 0 && p.nellipses <= 5,
              "%s: image %d has a bad grayscale flag or stroke count", fn, i);
    for (int k = 0; k < 5; ++k) {
        for (int c = 0; c < 5; ++c)
            PCB_CHECK(p.lines[k][c] >= -4 * out && p.lines[k][c] <= 4 * out, "%s: image %d line %d out of range", fn, i, k);
        for (int c = 0; c < 4; ++c)
            PCB_CHECK(p.ellipses[k][c] >= -4 * out && p.ellipses[k][c] <= 4 * out, "%s: image %d ellipse %d out of range", fn, i, k);
    }
    return 0;
}

int check_batch(const char *fn, const void *h_srcs, int n, int cap_n, int cap_h, int cap_w, int out) {
    PCB_CHECK(out >= 16 && out <= 4096 && cap_h <= 8 * out && cap_w <= 8 * out, "%s: output %d and capacity %dx%d (at most 8x the output)",
              fn, out, cap_h, cap_w);
    PCB_CHECK(h_srcs && n >= 1 && n <= cap_n, "%s: %d images for a batch of %d", fn, n, cap_n);
    return 0;
}

template <typename K>
int launch_prepare(const char *fn, const typename K::Src *srcs, const pcb_inpaint_params *params, int n, int cap_h, int cap_w, int out,
                   int strokes, uint8_t *tmp, void *corrupted, int dtype, uint8_t *mask_plane, float *clean, pcb_stream_t stream) {
    PCB_CHECK(srcs && params && tmp && corrupted && mask_plane && clean && (dtype == PCB_F32 || dtype == PCB_BF16), "%s: bad arguments", fn);
    PCB_CHECK(n >= 1 && n <= 65535 && out >= 16 && out <= 4096 && cap_h >= 1 && cap_w >= 1 && cap_h <= 8 * out && cap_w <= 8 * out,
              "%s: %d images, output %d, capacity %dx%d (at most 8x the output)", fn, n, out, cap_h, cap_w);
    using Px = typename K::Px;
    const dim3 hgrid((out + HX - 1) / HX, (cap_h + HROWS - 1) / HROWS, n);
    inpaint_hpass_kernel<K><<<hgrid, HX, 0, ST>>>(srcs, params, cap_h, cap_w, out, reinterpret_cast<Px *>(tmp));
    PCB_LAUNCH_CHECK();
    const dim3 fgrid((out + T - 1) / T, (out + T - 1) / T, n);
    if (dtype == PCB_BF16)
        inpaint_fused_kernel<K, bf16><<<fgrid, 256, 0, ST>>>(srcs, params, cap_h, cap_w, out, strokes, reinterpret_cast<const Px *>(tmp),
                                                             static_cast<bf16 *>(corrupted), mask_plane, clean);
    else
        inpaint_fused_kernel<K, float><<<fgrid, 256, 0, ST>>>(srcs, params, cap_h, cap_w, out, strokes, reinterpret_cast<const Px *>(tmp),
                                                              static_cast<float *>(corrupted), mask_plane, clean);
    PCB_LAUNCH_CHECK();
    return 0;
}

template <typename S>
int launch_sample(const char *fn, const S *srcs, int n, int out, int strokes, int gray, uint64_t *rng, pcb_inpaint_params *params,
                  pcb_stream_t stream) {
    PCB_CHECK(srcs && rng && params && n >= 1 && n <= 1024 && out >= 32, "%s: bad arguments (1..1024 images, out >= 32)", fn);
    inpaint_sample_kernel<S><<<1, (n + 31) / 32 * 32, 0, ST>>>(srcs, n, out, strokes, gray, reinterpret_cast<unsigned long long *>(rng),
                                                               params);
    PCB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

PCB_API int pcb_inpaint_validate(const pcb_inpaint_src *h_srcs, const pcb_inpaint_params *h_params, int n, int cap_n, int cap_h, int cap_w,
                                 int out) {
    const char *fn = "pcb_inpaint_validate";
    if (const int e = check_batch(fn, h_srcs, n, cap_n, cap_h, cap_w, out)) return e;
    for (int i = 0; i < n; ++i) {
        const pcb_inpaint_src &s = h_srcs[i];
        PCB_CHECK(s.rgb && s.mask, "%s: image %d has a null source", fn, i);
        PCB_CHECK(s.rgb_stride >= 3 * s.w && s.mask_stride >= s.w, "%s: image %d row strides %d / %d too small", fn, i, s.rgb_stride,
                  s.mask_stride);
        if (const int e = validate_image(fn, i, s.h, s.w, h_params, cap_h, cap_w, out)) return e;
    }
    return 0;
}

PCB_API int pcb_inpaint_pair_validate(const pcb_inpaint_pair_src *h_srcs, const pcb_inpaint_params *h_params, int n, int cap_n, int cap_h,
                                      int cap_w, int out) {
    const char *fn = "pcb_inpaint_pair_validate";
    if (const int e = check_batch(fn, h_srcs, n, cap_n, cap_h, cap_w, out)) return e;
    for (int i = 0; i < n; ++i) {
        const pcb_inpaint_pair_src &s = h_srcs[i];
        PCB_CHECK(s.raw && s.clean, "%s: image %d has a null source", fn, i);
        PCB_CHECK(s.raw_stride >= 3 * s.w && s.clean_stride >= 3 * s.w, "%s: image %d row strides %d / %d too small", fn, i, s.raw_stride,
                  s.clean_stride);
        if (const int e = validate_image(fn, i, s.h, s.w, h_params, cap_h, cap_w, out)) return e;
        PCB_CHECK(!h_params || h_params[i].gray == 0, "%s: image %d asks for grayscale, which the pair path does not draw", fn, i);
    }
    return 0;
}

PCB_API int pcb_inpaint_sample(const pcb_inpaint_src *srcs, int n, int out, int strokes, uint64_t *rng, pcb_inpaint_params *params,
                               pcb_stream_t stream) {
    return launch_sample("pcb_inpaint_sample", srcs, n, out, strokes, 1, rng, params, stream);
}

PCB_API int pcb_inpaint_pair_sample(const pcb_inpaint_pair_src *srcs, int n, int out, int strokes, uint64_t *rng, pcb_inpaint_params *params,
                                    pcb_stream_t stream) {
    return launch_sample("pcb_inpaint_pair_sample", srcs, n, out, strokes, 0, rng, params, stream);
}

PCB_API int pcb_inpaint_prepare(const pcb_inpaint_src *srcs, const pcb_inpaint_params *params, int n, int cap_h, int cap_w, int out,
                                int strokes, uint8_t *tmp, void *corrupted, int dtype, uint8_t *mask_plane, float *clean, pcb_stream_t stream) {
    return launch_prepare<MaskFile>("pcb_inpaint_prepare", srcs, params, n, cap_h, cap_w, out, strokes, tmp, corrupted, dtype, mask_plane,
                                    clean, stream);
}

PCB_API int pcb_inpaint_pair_prepare(const pcb_inpaint_pair_src *srcs, const pcb_inpaint_params *params, int n, int cap_h, int cap_w,
                                     int out, int strokes, uint8_t *tmp, void *corrupted, int dtype, uint8_t *mask_plane, float *clean,
                                     pcb_stream_t stream) {
    return launch_prepare<Pair>("pcb_inpaint_pair_prepare", srcs, params, n, cap_h, cap_w, out, strokes, tmp, corrupted, dtype, mask_plane,
                                clean, stream);
}

// pil_data.cuh -- pieces shared by the GPU data paths (inpaint_data.cu, seg_data.cu):
//   * to_pil_image's byte of a fp32 page value (text_removal.cu, text_regions.cu);
//   * Pillow's bicubic resampling coefficients (precompute_coeffs + normalize_coeffs_8bpc) and its 8-bit clip, bit for bit:
//     the weights are computed in double with explicitly rounded operations (no FMA contraction, which Pillow's x86-64 build
//     does not do either);
//   * the Philox4x32-10 uniform stream the parameter samplers draw from;
//   * RandomResizedCrop.get_params(scale, ratio=(3/4, 4/3)) on that stream.
#pragma once
#include "pcb_common.cuh"

namespace pil {

constexpr int KMAX = 33;      // taps of a bicubic window at scale 8 (2 * ceil(2 * 8) + 1): box / out <= 8
constexpr int taps_for(int reduction) { return 4 * reduction + 1; }   // the window of a reduction of at most `reduction`
constexpr int PB = 22;        // Pillow's PRECISION_BITS for 8-bit images

__device__ __forceinline__ double bicubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(a + 2.0, x), a + 3.0), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), a);
    return 0.0;
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for output index xx of a box of `insize` input pixels resampled to
// `outsize`: writes the integer weights to k[0], k[stride], ... and returns the first tap; *count = number of taps.  KM bounds
// the window (taps_for(insize / outsize)), and with it the registers of the weights in double.
template <int KM = KMAX>
__device__ inline int pil_coeffs(int xx, int insize, int outsize, int *k, int stride, int *count) {
    const double scale = __ddiv_rn(static_cast<double>(insize), static_cast<double>(outsize));
    const double fs = scale < 1.0 ? 1.0 : scale;
    const double support = __dmul_rn(2.0, fs), ss = __ddiv_rn(1.0, fs);
    const double center = __dmul_rn(static_cast<double>(xx) + 0.5, scale);
    int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, support), 0.5));
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, support), 0.5));
    if (xmax > insize) xmax = insize;
    xmax -= xmin;
    if (xmax > KM) xmax = KM;                        // unreachable within the reduction KM was chosen for (checked on the host)
    double w[KM];
    double ww = 0.0;
#pragma unroll
    for (int x = 0; x < KM; ++x) {
        if (x < xmax) {
            w[x] = bicubic(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
            ww = __dadd_rn(ww, w[x]);
        }
    }
#pragma unroll
    for (int x = 0; x < KM; ++x) {
        if (x < xmax) {
            const double v = ww != 0.0 ? __ddiv_rn(w[x], ww) : w[x];
            const double s = __dmul_rn(v, static_cast<double>(1 << PB));
            k[x * stride] = v < 0 ? static_cast<int>(__dadd_rn(-0.5, s)) : static_cast<int>(__dadd_rn(0.5, s));
        }
    }
    *count = xmax;
    return xmin;
}

__device__ __forceinline__ int clip8(int acc) {
    acc >>= PB;
    return acc < 0 ? 0 : (acc > 255 ? 255 : acc);
}

// torchvision's to_pil_image byte of a fp32 page value: pic.mul(255).byte(), clamped to [0, 255], NaN to 0
__device__ __forceinline__ int page_byte(float p) {
    const float v = __fmul_rn(p, 255.f);
    return v >= 255.f ? 255 : (v > 0.f ? static_cast<int>(v) : 0);
}

__device__ __forceinline__ uint4 philox(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

struct Draws {
    uint32_t img, c_lo, c_hi, k0, k1;
    __device__ Draws(uint32_t image, unsigned long long step, unsigned long long seed)
        : img(image), c_lo(static_cast<uint32_t>(step)), c_hi(static_cast<uint32_t>(step >> 32)), k0(static_cast<uint32_t>(seed)),
          k1(static_cast<uint32_t>(seed >> 32)) {}
    // uniform of slot s in [0, 1), 24 bits: word s % 4 of philox(counter = (s / 4, image, step lo, step hi), key = seed)
    __device__ float u(int s) const {
        const uint4 r = philox(make_uint4(static_cast<uint32_t>(s >> 2), img, c_lo, c_hi), k0, k1);
        const int l = s & 3;
        const uint32_t w = l == 0 ? r.x : (l == 1 ? r.y : (l == 2 ? r.z : r.w));
        return static_cast<float>(w >> 8) * 5.9604644775390625e-8f;
    }
    __device__ int randint(int s, int lo, int hi) const {   // lo..hi inclusive
        return lo + static_cast<int>(__dmul_rn(static_cast<double>(u(s)), static_cast<double>(hi - lo + 1)));
    }
};

// RandomResizedCrop.get_params(scale=(scale_lo, scale_lo + scale_span), ratio=(3/4, 4/3)) for an H x W source; slots 4a..4a+3
// of attempt a: scale, log-aspect, top, left.  scale_lo and scale_span are the float32 values torch's uniform_ works with.
struct Box {
    int top, left, height, width;
};

__device__ inline Box crop_box(const Draws &d, int H, int W, float scale_lo, float scale_span) {
    const float lr0 = -0.28768208622932434f, span = 0.5753642320632935f;    // float32 log(3/4), log(4/3) - log(3/4) as torch has them
    const double area = static_cast<double>(H) * static_cast<double>(W);
    for (int a = 0; a < 10; ++a) {
        const float s = __fadd_rn(scale_lo, __fmul_rn(scale_span, d.u(4 * a)));
        const float r = __fadd_rn(lr0, __fmul_rn(span, d.u(4 * a + 1)));
        const double target = __dmul_rn(area, static_cast<double>(s));
        const double aspect = static_cast<double>(static_cast<float>(exp(static_cast<double>(r))));
        const int w = static_cast<int>(rint(__dsqrt_rn(__dmul_rn(target, aspect))));
        const int h = static_cast<int>(rint(__dsqrt_rn(__ddiv_rn(target, aspect))));
        if (0 < w && w <= W && 0 < h && h <= H) return Box{d.randint(4 * a + 2, 0, H - h), d.randint(4 * a + 3, 0, W - w), h, w};
    }
    // the centre-crop fallback
    const double in_ratio = __ddiv_rn(static_cast<double>(W), static_cast<double>(H));
    int w = W, h = H;
    if (in_ratio < 0.75) h = static_cast<int>(rint(__ddiv_rn(static_cast<double>(W), 0.75)));
    else if (in_ratio > 4.0 / 3.0) w = static_cast<int>(rint(__dmul_rn(static_cast<double>(H), 4.0 / 3.0)));
    return Box{(H - h) / 2, (W - w) / 2, h, w};
}

}  // namespace pil

"""Dense (non-depthwise) convolution kernels through the C ABI, every element against an fp64 reference of the same operands
computed on the device (F.conv2d / torch.nn.grad.conv2d_input / conv2d_weight, cuDNN off so that every reference is a direct
sum), on every route the plan of a problem can take: the TMA-fed and cp.async-gather wgmma kernels (conv_tc.cu), the stride-2
data gradient as four parity classes, the sub-pixel data gradient of a 2x-upsampled part, the space-to-depth stem
(conv_stem.cu), the kernel-to-row RGB tail (conv_k2r.cu), the mma.sync small-Cout kernels (conv_smallco.cu) and the
shape-general kernels (conv_generic.cu).  Three sets of cases:

  * one per dense descriptor of tests/golden/conv_dispatch.json (the layers the workloads run), batch capped at 2 -- or the
    smallest batch above that whose routes (pcb_debug_conv_routes) equal those of the uncapped descriptor.  A descriptor
    only inference reaches ("forward_only": TextRemovalStep and InferStep at page sizes, up to the 3584 x 2560 U-Net grid) is
    checked in the forward alone: the forward route of the trace, the forward and its mask pass, the two-call forward, the
    weight refresh, the fused BatchNorm sums and the eval epilogue; its fp64 references and comparisons run in bands of
    output rows (input halos included) of at most BAND_BYTES, and its peak device memory must stay below MEMORY_BUDGET;
  * hand cases for what production reaches rarely or never: a stride-1 gather layer, ragged M, two parts (one 2x-upsampled) on
    a non-power-of-two grid, dilation; row-packed layers with cin 1 / 3 / 8 and kw 3 / 5 / 7; stems with holes, no_guard, cout
    32 / 40 and a grid that is not a whole number of tiles; RGB tails with 1 / 3 / 4 image channels, 32 / 64 upsampled channels
    and holes in both parts; small-Cout layers at 80 packed channels, ragged h and w, 1x1, an upsampled part; the stride-2 data
    gradient with and without its four-stream fork; grouped, many-part, kh != kw and fp32 no_guard generic layers;
  * tile cases (TILE_CASES, at their own batch), one per tile configuration of the TMA-fed kernels, each asserting the tiles it
    is named for (TILE_KERNELS) from the template arguments of its kernels: 256-wide forward and data-gradient tiles and the
    eval epilogue at 256; cout 320 and 384 on 64- and 128-wide forward tiles; the sub-pixel data gradient of a 2x-upsampled
    part; row-halo forward and data-gradient tiles at dilation 48 (halo rows up to 224, past the fixers' third row at 192);
    no_guard on the row-halo forward; the stride-2 data gradient as four parity classes.  Weight gradient: 128-wide
    output-channel tiles with and without row-halo A blocks, ragged (cout 192, 320), an input-channel tile straddling two
    parts, a 2x-upsampled part; one 64-channel input block shared by both consumer warpgroups at N = 128 (each takes 64 output
    channels) and alone at N = 64 (the second warpgroup idles: DESIGN 4.1); 64-wide tiles for a short reduction (fewer than
    8192 output pixels); row-halo A blocks taller than 128 rows (dilation 48).

Each case asserts that the routes the query reports are the routes its kernels take: the kernel names of a torch.profiler
trace of the forward, data gradient and both weight gradients (kernel_harness.traced) are mapped back to a route per
direction.  A row-packed layer has no data-gradient route (the query says none); its callers run that gradient on the generic
kernels with force_generic and KRSC weights (ops.py), and so does this test.

Integer regime (every case, bit-exact).  x, w and dc are small integers (|x|, |w|, |dc| <= 4; <= 2 where noted below) and the bias a
multiple of 1/8, all exact in bf16.  Each case asserts that every partial sum stays below 2^24 (max|x| max|w| times the number of
terms, per element), so fp32 accumulation is exact in any order, tensor cores and atomics included, and the fp64 reference is
the exact sum S.  The kernels are built without fast math, so what they store must be BIT-IDENTICAL to the last fp32
operations each route applies to S, then one rounding to the storage type (bf16: round to nearest even):
  * tensor-core epilogues (TMA, gather, stem): inv = fl(1 / s), then fmaf(S, inv, b) = fl(S inv + b): S inv is exact in fp64
    (24 + 24 bits), the sum is rounded to fp32 once; the fp64 sum and its exact error (Knuth's two-sum) decide the fp32 ties an
    fp64 rounding could hide;
  * generic: fl(fl(S / s) + b): the fp64 quotient rounded to fp32 is the correctly rounded fp32 quotient (double rounding is
    innocuous for division when 53 >= 2 * 24 + 2), and adding b to it is exact in fp64;
  * small-Cout and kernel-to-row: the source writes a * inv + b, which nvcc contracts to an fma by default but the language does
    not promise: the fused value above or fl(fl(S inv) + b), nothing else;
  * plain convolutions have s = 1 on every route: fl(S + b).  Empty boxes (s = 0) store 0; under no_guard S = 0 there too
    (every tap is a hole), and 0 * inf = 0 / 0 = NaN, so NaN exactly where s = 0;
  * data gradient m * S, at source resolution (the 2x2 sum of the children) where pcb_conv_dgrad_at_source_resolution says so;
    weight gradient S, or fl(dw0 + S) accumulating onto an integer dw0;
  * renormalisation backward: dc = fl(dy / s) on the scalar kernel, fl(dy * fl(1 / s)) on the 8-channel kernels, 0 where s = 0
    (NaN or inf under no_guard), dbias the exact sum of dy over s > 0.
Intermediates that a route rounds to bf16 must stay exact: the kernel-to-row tail stores Z = sum_c u w (cu terms) and
D = the sum of four dc in bf16, so its ranges keep cu max|x| max|w| <= 256, where every integer is exact in bf16; sub-pixel
weights are sums of at most four taps, <= 16.  Outputs are prefilled with NaN and, past rup(c, 8), with a sentinel: y must
hold zeros in channels [cout, rup(cout, 8)) and may only zero the channels past them.  Weight refresh: pcb_conv_weight_refresh(W2) over buffers prepared from W1 must
leave them bitwise equal to pcb_conv_weight_prepare(W2) -- including the extra operands the stem, the tail and the sub-pixel
kernels keep behind the layer's own.

Gaussian regime (every case, error bounds).  Every product of two bf16 values is exact in fp32, so a kernel differs from the
exact sum only in how it adds the products of an element: fp32 tensor-core accumulation, plus fp32 red.global.add of the
split-K partials in the weight gradient, in an order the test does not know.  Adding an exact zero is exact, so only the n
nonzero products count.  Any order of n - 1 additions with unit roundoff u is off by at most (n - 1) u / (1 - (n - 1) u) * M,
M = the sum of |products| (Higham, Accuracy and Stability of Numerical Algorithms, 4.2).  The tensor cores' fp32 adder is
not guaranteed to round to nearest, so u = 2^-23 (one ulp) instead of 2^-24, and 1 / (1 - (n - 1) u) < 2 here: the
accumulation is off by at most n * 2^-22 * M (fp32 storage: each product and its add round once each, the same bound).
The renormalisation and the bias add two roundings (2^-22 of
|acc| / s and of the result), the eval epilogue's fma one (2^-23 of |z| + |shift|), LeakyReLU's multiply one (2^-23 of the
result); activations are 1-Lipschitz; a bf16 store adds half an ulp (2^-8 relative is used).  Rounding an intermediate to bf16
adds half an ulp of it, at most 2^-9 of the sum of the |products| it holds, bounded by 2^-8 M: the tail's Z (forward) and D
(both gradients), and the sub-pixel tap sums (data gradient).  The fused BatchNorm sums are checked against the stored values:
M fp32 additions of terms bounded by |y| are off by at most M * 2^-23 * sum |y|.  Where pcb_conv_fuses_bn_stats is 0 both fused
calls must be refused and write nothing.
"""
import collections
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from kernel_harness import (HOLE_VALUE, SENTINEL, act_ref, assert_bitwise, assert_within, conv_dispatch_cases, holes, nchw,
                            sentinel_kept, strided, traced)
from text_segmentation_image_inpainting_b200 import _lib

pytestmark = pytest.mark.gpu

SLOPE = 0.2
ACTS = (_lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_LEAKY, _lib.ACT_RELU6)
DTYPES = {"bf16": (torch.bfloat16, _lib.PCB_BF16), "f32": (torch.float32, _lib.PCB_F32)}
TC_ROUTES = {"stem", "k2r", "smallco", "tma", "tma_s2", "gather"}
BAND_BYTES = 2 ** 29         # fp64 working set of one band of output rows (forward-only cases)
MEMORY_BUDGET = 12 * 2 ** 30  # peak device memory of a forward-only case: page-size cases run on shared GPUs


def accumulation_bound(nz, mag, rounds_bf16_intermediate):
    """the Gaussian-regime bound of one convolution direction (module docstring): n nonzero products added in any order with
    one-ulp fp32 additions, n 2^-22 M, plus 2^-8 M where the route rounds an intermediate sum to bf16"""
    return nz * 2.0 ** -22 * mag + (2.0 ** -8 * mag if rounds_bf16_intermediate else 0.0)


def _rup8(v):
    return (v + 7) // 8 * 8


def _part(c, up=0, mask=False, mup=None, xcs=None):
    return dict(c=c, up=up, mask=bool(mask), mup=up if mup is None else mup, xcs=_rup8(c) if xcs is None else xcs)


def _case(n, h, w, parts, cout, k=3, s=1, pad=None, dil=1, dtype="bf16", groups=1, same_holes=False, no_guard=False,
          plain=False, force_generic=False, ycs=None, dcs=None, dxcs=None, route=None, ix=4, iw=4):
    """parts: list of _part.  route: the (forward, data gradient, weight gradient) route names the case covers.  ycs / dcs /
    dxcs: channel strides of y, dc and each dx (default: rup(c, 8)).  ix / iw: integer ranges of x and w."""
    kh, kw = (k, k) if isinstance(k, int) else k
    ph, pw = (dil * (kh - 1) // 2, dil * (kw - 1) // 2) if pad is None else ((pad, pad) if isinstance(pad, int) else pad)
    return dict(n=n, h=h, w=w, parts=parts, cin=sum(p["c"] for p in parts), cout=cout, kh=kh, kw=kw, s=s, ph=ph, pw=pw, dil=dil,
                dtype=dtype, groups=groups, same_holes=same_holes, no_guard=no_guard, plain=plain, force_generic=force_generic,
                ycs=ycs or _rup8(cout), dcs=dcs or _rup8(cout), dxcs=dxcs or [_rup8(p["c"]) for p in parts], route=route,
                ix=ix, iw=iw)


def _conv_struct(sp, n=None, masks=None, xs=None):
    cv = _lib.Conv()
    cv.n = sp["n"] if n is None else n
    cv.h, cv.w, cv.cin, cv.cout, cv.kh, cv.kw = sp["h"], sp["w"], sp["cin"], sp["cout"], sp["kh"], sp["kw"]
    cv.stride, cv.pad_h, cv.pad_w, cv.dil, cv.groups = sp["s"], sp["ph"], sp["pw"], sp["dil"], sp["groups"]
    cv.ho = (sp["h"] + 2 * sp["ph"] - sp["dil"] * (sp["kh"] - 1) - 1) // sp["s"] + 1
    cv.wo = (sp["w"] + 2 * sp["pw"] - sp["dil"] * (sp["kw"] - 1) - 1) // sp["s"] + 1
    cv.dtype = DTYPES[sp["dtype"]][1]
    cv.same_holes, cv.no_guard, cv.plain, cv.force_generic = (int(sp[k]) for k in ("same_holes", "no_guard", "plain", "force_generic"))
    cv.nparts = len(sp["parts"])
    for i, p in enumerate(sp["parts"]):
        cp = cv.parts[i]
        cp.c, cp.x_cstride, cp.x_up, cp.mask_up = p["c"], p["xcs"], p["up"], p["mup"]
        cp.mask = (masks[i] if masks else (1 << 12)) if p["mask"] else None   # the host queries only test the pointer for null
        cp.x = xs[i] if xs else None
    return cv


def _routes(lib, cv):
    r = (ctypes.c_int32 * 3)()
    _lib.check(lib.pcb_debug_conv_routes(ctypes.byref(cv), r))
    return tuple(_lib.ROUTES[v] for v in r)


def _fixture_cases():
    """one case per distinct dense descriptor of the dispatch fixture, at the smallest batch >= min(n, 2) whose routes equal those
    of the uncapped descriptor"""
    lib = _lib.load()
    out = {}
    for case in conv_dispatch_cases():
        d = case["conv"]
        if case["expect"]["routes"][0] == "depthwise":
            continue
        parts = [_part(p["c"], p["x_up"], p["mask"], p["mask_up"], p["x_cstride"]) for p in d["parts"]]
        dt = "bf16" if d["dtype"] == _lib.PCB_BF16 else "f32"
        sp = _case(d["n"], d["h"], d["w"], parts, d["cout"], (d["kh"], d["kw"]), d["stride"], (d["pad_h"], d["pad_w"]), d["dil"], dt,
                   d["groups"], bool(d["same_holes"]), bool(d["no_guard"]), bool(d["plain"]), bool(d["force_generic"]))
        full = _routes(lib, _conv_struct(sp))
        assert list(full) == case["expect"]["routes"], "the fixture's routes are stale: regenerate it (make_golden_conv_dispatch.py)"
        if full[0] == "k2r":                 # the tail's bf16 Z rows: cu max|x| max|w| <= 256
            sp["ix"], sp["iw"] = 2, min(4, 128 // max(p["c"] for p in parts if p["up"]))
        n = min(d["n"], 2)
        while _routes(lib, _conv_struct(sp, n)) != full:
            n += 1
        sp["n"], sp["route"], sp["forward_only"] = n, full, bool(case.get("forward_only"))
        pstr = "_".join(f"c{p['c']}" + (f"cs{p['xcs']}" if p["xcs"] != p["c"] else "") + ("u" if p["up"] else "")
                        + ("m" + str(p["mup"]) if p["mask"] else "") for p in parts)
        name = (f"fx_{dt}_n{n}_{d['h']}x{d['w']}_{pstr}_o{d['cout']}_k{d['kh']}x{d['kw']}_s{d['stride']}_p{d['pad_h']}x{d['pad_w']}"
                f"_d{d['dil']}" + (f"_g{d['groups']}" if d["groups"] > 1 else "") + ("_plain" if d["plain"] else "")
                + ("_same" if d["same_holes"] else "") + ("_noguard" if d["no_guard"] else "")
                + ("_forcegen" if d["force_generic"] else ""))
        if sp["forward_only"] and name in out:   # an inference descriptor that caps to a case tested in every direction
            continue
        out[name] = sp
    return out


P_ = _part
HAND_CASES = {
    # cp.async gather kernels: stride 1 on a 24 x 40 grid (w a multiple of 8, not a power of two), ragged M (143 pixels), two
    # parts with the first 2x-upsampled on a 24 x 40 grid, dilation 2; all with holes, so the gather weight gradient reads tap masks
    "gather_s1_w40_holes": _case(2, 24, 40, [P_(64, mask=True)], 64, route=("gather", "gather", "gather")),
    "gather_ragged_m_cout96": _case(1, 13, 11, [P_(64, mask=True)], 96, route=("gather", "gather", "gather")),
    "gather_two_parts_up": _case(2, 24, 40, [P_(64, 1, True), P_(32, mask=True)], 64, route=("gather", "gather", "gather")),
    "gather_dil2": _case(2, 20, 28, [P_(64, mask=True)], 64, dil=2, route=("gather", "gather", "gather")),
    # row-packed cp.async kernels (cin <= 8 in an 8-channel pixel), their data gradient on the generic kernels
    "rowpack_c3_k3_s2_holes": _case(2, 40, 36, [P_(3, mask=True)], 32, 3, 2, route=("gather", "none", "gather")),
    "rowpack_c1_k5_holes": _case(2, 30, 26, [P_(1, mask=True)], 16, 5, route=("gather", "none", "gather")),
    "rowpack_c8_k7": _case(2, 22, 20, [P_(8)], 32, 7, route=("gather", "none", "gather")),
    # space-to-depth stems: holes, no_guard, cout 40, a 26 x 38 sub-grid (not a whole number of tiles)
    "stem_c3_holes_o32": _case(2, 64, 64, [P_(3, mask=True)], 32, 7, 2, route=("stem", "none", "stem")),
    "stem_c3_holes_o40_ragged": _case(2, 52, 76, [P_(3, mask=True)], 40, 7, 2, route=("stem", "none", "stem")),
    "stem_c8_noguard_holes": _case(2, 48, 64, [P_(8, mask=True)], 32, 7, 2, no_guard=True, route=("stem", "none", "stem")),
    # kernel-to-row RGB tails: image part of 1, 3 and 4 channels, cu 32 and 64, holes in both parts, no_guard, cout 1 and 3
    "k2r_cs3_cu32_o3_holes": _case(2, 32, 48, [P_(32, 1, True), P_(3, mask=True)], 3, route=("k2r", "k2r", "k2r"), ix=2),
    "k2r_cs1_cu64_o1_holes": _case(2, 24, 40, [P_(64, 1, True), P_(1, mask=True)], 1, route=("k2r", "k2r", "k2r"), ix=2, iw=2),
    "k2r_cs4_cu32_o3_noguard": _case(1, 20, 36, [P_(32, 1, True), P_(4, mask=True)], 3, no_guard=True, route=("k2r", "k2r", "k2r"),
                                     ix=2),
    "k2r_image_first_cs3": _case(2, 16, 32, [P_(3, mask=True), P_(32, 1, True)], 3, route=("k2r", "k2r", "k2r"), ix=2),
    # mma.sync small-Cout kernels: 80 packed channels, h not a multiple of 8 and w not of 32, odd cout, 1x1, an upsampled part
    "smallco_c80_o5_holes": _case(2, 13, 45, [P_(80, mask=True)], 5, route=("smallco", "smallco", "smallco")),
    "smallco_1x1_two_parts_o3": _case(2, 19, 37, [P_(64, mask=True), P_(16)], 3, 1, route=("smallco", "smallco", "smallco")),
    "smallco_up_o7": _case(2, 22, 34, [P_(32, 1, True), P_(16, mask=True)], 7, route=("smallco", "smallco", "smallco")),
    "smallco_o8_noguard": _case(1, 17, 70, [P_(48, mask=True)], 8, no_guard=True, route=("smallco", "smallco", "smallco")),
    # stride-2 data gradient as four parity classes: forked (one class does not fill the GPU) and not
    "tma_s2_forked": _case(2, 32, 32, [P_(64, mask=True)], 128, 3, 2, route=("tma", "tma_s2", "tma")),
    "tma_s2_not_forked": _case(2, 256, 256, [P_(64, mask=True)], 64, 3, 2, route=("tma", "tma_s2", "tma")),
    # TMA forward / weight gradient with a strided view of everything
    "tma_strided_views": _case(2, 32, 64, [P_(64, mask=True, xcs=80)], 64, ycs=72, dcs=88, dxcs=[96], route=("tma", "tma", "tma")),
    # shape-general kernels: groups with one mask plane per group, all PCB_MAX_PARTS parts (upsampled, masked, strided),
    # kh != kw, fp32 no_guard, a force_generic bf16 layer
    "generic_groups2_planes": _case(2, 18, 22, [P_(16, mask=True), P_(16, mask=True)], 16, groups=2, route=("generic",) * 3),
    "generic_groups4_same_holes": _case(2, 18, 22, [P_(32, mask=True)], 16, groups=4, same_holes=True, route=("generic",) * 3),
    "generic_8_parts": _case(2, 16, 20, [P_(3, mask=True), P_(5, 1, True), P_(8), P_(2, mask=True, mup=1), P_(4, 1),
                                         P_(1, mask=True, xcs=8), P_(6, 1, True, 0), P_(3)], 8, route=("generic",) * 3),
    "generic_k3x5_f32_holes": _case(2, 21, 19, [P_(6, mask=True, xcs=6)], 10, (3, 5), 1, (1, 2), dtype="f32", route=("generic",) * 3),
    "generic_f32_noguard": _case(2, 17, 23, [P_(12, mask=True, xcs=12)], 12, no_guard=True, dtype="f32", route=("generic",) * 3),
    "generic_force_bf16_s2": _case(2, 26, 30, [P_(64, mask=True)], 64, 3, 2, force_generic=True, route=("generic",) * 3),
    "generic_f32_plain_d3_s2": _case(2, 25, 27, [P_(16)], 24, 3, 2, dil=3, dtype="f32", plain=True, route=("generic",) * 3),
}

# name: (n, h, w, parts [(channels, upsampled, masked)], cout, k, stride, dilation[, mode]), "same" padding; an upsampled part
# is stored at (h/2, w/2) with its hole plane at that resolution; mode "no_guard": NaN at empty boxes (every case runs the
# fused BatchNorm sums and the eval epilogue).  tests/golden/make_golden_conv_dispatch.py records these descriptors too.
TILE_CASES = {
    "n256_two_parts_1024_512": (8, 32, 32, [(512, 0, 1), (512, 0, 1)], 512, 3, 1, 1, "bn"),
    "eval_affine_leaky_n256": (8, 32, 32, [(256, 0, 1)], 512, 3, 1, 1, "eval"),
    "ragged_cout320": (2, 32, 64, [(128, 0, 1)], 320, 3, 1, 1, "bn"),
    "ragged_cout384": (2, 32, 64, [(128, 0, 1)], 384, 3, 1, 1, "bn"),
    # batch 6, not 1: the sub-pixel data gradient runs where the source grid has at least a third of a wave of 128-pixel tiles
    # (44 on 132 SMs); at batches 1 to 5 (8 to 40 tiles) the plan keeps the regular kernel and pconv_tc_sp_kernel never launches
    "two_parts_one_upsampled": (6, 64, 64, [(128, 1, 1), (64, 0, 1)], 64, 3, 1, 1, "bn"),
    "holes_no_guard_nan": (2, 32, 128, [(128, 0, 1)], 128, 3, 1, 1, "no_guard"),
    "s2_parity_dgrad_cin256": (2, 64, 64, [(256, 0, 1)], 512, 3, 2, 1, "bn"),
    "halo_n64_d48_holes_over_large_x": (2, 64, 128, [(64, 0, 1)], 64, 3, 1, 48, "bn"),
    "halo_n128_holes": (2, 32, 128, [(128, 0, 1)], 128, 3, 1, 1),
    "decoder_upsampled_two_parts_n128": (1, 64, 128, [(128, 1, 1), (64, 0, 1)], 128, 3, 1, 1),
    "enc1_like_k5_s2_64_128_split_n": (2, 128, 128, [(64, 0, 1)], 128, 5, 2, 1),
    "k3_s2_256_512": (2, 128, 128, [(256, 0, 1)], 512, 3, 2, 1),
    # the input-channel tile holding only the 64 skip channels is one 64-channel block: at N = 64 the second consumer warpgroup
    # idles (DESIGN 4.1: splitting the K blocks between the warpgroups is not used)
    "dec7_like_192_64_one_block_n64": (1, 16, 128, [(128, 1, 1), (64, 0, 1)], 64, 3, 1, 1),
    "ragged_cout192_halo": (1, 64, 128, [(128, 0, 1)], 192, 3, 1, 1),
    "ragged_cout320_split_n": (8, 32, 32, [(64, 0, 1)], 320, 3, 1, 1),
    "ci_tile_straddles_parts": (1, 128, 64, [(64, 0, 1), (128, 0, 1)], 128, 3, 1, 1),
    "short_reduction_n64_tiles": (2, 8, 64, [(256, 0, 1)], 256, 3, 1, 1),
    "halo_d48_holes_over_large_x": (1, 64, 128, [(128, 0, 1)], 128, 3, 1, 48),
}


def _tma(bn, mode, halo):
    return ("pconv_tc_tma_kernel", (str(bn), str(mode), str(halo).lower()))


def _wg(bn, halo):
    return ("pconv_tc_wgrad_tma_kernel", (str(bn), "3", str(halo).lower()))


# the launches each tile case is named for, per trace (one forward, one data gradient, two weight gradients)
TILE_KERNELS = {
    "n256_two_parts_1024_512": {_tma(256, 0, False): 1, _tma(256, 1, False): 1},
    "eval_affine_leaky_n256": {_tma(256, 0, False): 1},
    "ragged_cout320": {_tma(64, 0, False): 1},
    "ragged_cout384": {_tma(128, 0, False): 1},
    # the upsampled part's gradient at source resolution, the other part's on the regular kernel
    "two_parts_one_upsampled": {("pconv_tc_sp_kernel", ("64",)): 1, _tma(64, 1, False): 1},
    "holes_no_guard_nan": {_tma(64, 0, True): 1},
    "s2_parity_dgrad_cin256": {_tma(32, 1, False): 4},
    "halo_n64_d48_holes_over_large_x": {_tma(64, 0, True): 1, _tma(64, 1, True): 1},
    "halo_n128_holes": {_wg(128, True): 2},
    "decoder_upsampled_two_parts_n128": {_wg(128, True): 2},
    "enc1_like_k5_s2_64_128_split_n": {_wg(128, False): 2},
    "k3_s2_256_512": {_wg(128, False): 2},
    "dec7_like_192_64_one_block_n64": {_wg(64, True): 2},
    "ragged_cout192_halo": {_wg(128, True): 2},
    "ragged_cout320_split_n": {_wg(128, False): 2},
    "ci_tile_straddles_parts": {_wg(128, True): 2},
    "short_reduction_n64_tiles": {_wg(64, True): 2},
    "halo_d48_holes_over_large_x": {_wg(128, True): 2},
}


def _tile_cases():
    """every tile case covers the TMA-fed kernels: the stride-2 data gradient as parity classes"""
    out = {}
    for name, case in TILE_CASES.items():
        n, h, w, parts, cout, k, s, d = case[:8]
        sp = _case(n, h, w, [_part(c, up, masked) for c, up, masked in parts], cout, k, s, dil=d, no_guard=case[8:] == ("no_guard",),
                   route=("tma", "tma_s2" if s == 2 else "tma", "tma"))
        sp["tiles"] = TILE_KERNELS[name]
        out["tile_" + name] = sp
    return out


CASES = {**_fixture_cases(), **HAND_CASES, **_tile_cases()}


# ------------------------------------------------------------------------------------------------------------------------
def _up2(t):
    return t.repeat_interleave(2, -2).repeat_interleave(2, -1)


def _fl32_sum(t, b):
    """fl32(t + b) for fp64 tensors t, b whose exact sum may not fit fp64: two-sum gives r = fl64(t + b) and its exact error e;
    r only lies on an fp32 rounding tie by accident of the fp64 rounding, and then the sign of e picks the neighbour"""
    r = t + b
    bb = r - t
    e = (t - (r - bb)) + (b - bb)
    f = r.float()
    inf = torch.full_like(f, float("inf"))
    other = torch.nextafter(f, torch.where(r > f.double(), inf, -inf))
    tie = (r == (f.double() + other.double()) / 2) & (e != 0) & (other.double() != f.double())
    toward_e = torch.where((e > 0) == (other.double() > f.double()), other, f)
    return torch.where(tie, toward_e, f)


def _int_forward_want(S, s, b, route0, no_guard, dt):
    """the integer regime's stored forward (module docstring) from the exact sums S, the box sums s and the bias b: (want, alt),
    alt the other rounding a small-Cout / kernel-to-row route may store (or None)"""
    empty = s == 0
    safe = torch.where(empty, torch.ones_like(s), s)
    inv = (1.0 / safe).float().double()
    if route0 == "generic":
        want = ((S / safe).float().double() + b).float()
        alt = None
    else:
        want = _fl32_sum(S * inv, b.expand_as(S))
        alt = ((S * inv).float().double() + b).float() if route0 in ("smallco", "k2r") else None
    hole = torch.full_like(want, float("nan") if no_guard else 0.0)
    want = torch.where(empty, hole, want).to(dt)
    alt = torch.where(empty, hole, alt).to(dt) if alt is not None else None
    return want, alt


def _gauss_forward_ref(acc, mag, nz, s, b, k2r):
    """the Gaussian regime's forward reference and its bound (module docstring) from the exact sum acc, the sum of |products|
    mag, the nonzero-term counts nz and the box sums s: 0 and 0 where s == 0"""
    empty = s == 0
    safe = torch.where(empty, torch.ones_like(s), s)
    e_acc = accumulation_bound(nz, mag, k2r)
    v_ref = torch.where(empty, torch.zeros_like(acc), acc / safe + b)
    e_ref = torch.where(empty, torch.zeros_like(acc), e_acc / safe + 2.0 ** -22 * (acc.abs() / safe + v_ref.abs()))
    return v_ref, e_ref


def _check_y_values(name, tag, no_guard, got, v, e, store, live, nan_at_empty=True):
    """got (fp64 NCHW of a stored forward) within e + the store's rounding of v; under no_guard NaN where the box is empty"""
    if no_guard:                       # (an activation of NaN is whatever fmaxf / fminf make of it)
        assert not nan_at_empty or bool(got[~live.expand_as(got)].isnan().all()), f"{name}: {tag}: NaN expected where the box is empty"
        got = torch.where(live, got, v)
    assert_within(f"{name}: {tag}", got, v, e + store * (v.abs() + e))


def _kernel_routes(records):
    """(forward, data gradient, weight gradient) route names from the kernel records of a trace holding one forward, one data
    gradient and two weight gradients: the route-specific kernels first (a stem or a tail also runs its sub-problem on the
    tensor-core kernels), then the tensor-core kernels by their MODE template argument (0 forward, 1 data gradient); the
    stride-2 data gradient launches the stride-1 TMA kernel once per parity class"""
    cnt = collections.Counter()
    for (k, args), launches in records.items():
        cnt[(k, args[1] if k in ("pconv_tc_tma_kernel", "pconv_tc_persistent_kernel") else
             args[0] if k == "k2r_dbuild_kernel" else "")] += launches

    def one(options):
        found = [r for r, k in options if cnt[k]]
        return found[0] if found else "?"
    fwd = one([("stem", ("s2d_kernel", "")), ("k2r", ("k2r_combine_kernel", "")), ("smallco", ("smallco_fwd_kernel", "")),
               ("generic", ("generic_fwd_kernel", "")), ("tma", ("pconv_tc_tma_kernel", "0")),
               ("gather", ("pconv_tc_persistent_kernel", "0"))])
    tma_dg = cnt[("pconv_tc_tma_kernel", "1")]
    dg = one([("k2r", ("k2r_dbuild_kernel", "false")), ("smallco", ("smallco_dgrad_kernel", "")),
              ("generic", ("generic_dgrad_kernel", "")), ("tma", ("pconv_tc_sp_kernel", "")),
              ("tma_s2" if tma_dg == 4 else "tma", ("pconv_tc_tma_kernel", "1")), ("gather", ("pconv_tc_persistent_kernel", "1"))])
    wg = one([("stem", ("stem_dw_gather_kernel", "")), ("k2r", ("k2r_dw_scatter_kernel", "")), ("smallco", ("smallco_wgrad_kernel", "")),
              ("generic", ("generic_wgrad_kernel", "")), ("tma", ("pconv_tc_wgrad_tma_kernel", "")), ("gather", ("pconv_tc_wgrad_kernel", ""))])
    return (fwd, dg, wg), cnt


class _Problem:
    """one dense problem: hole planes, the descriptor, the fp64 masks / box sums and the reference helpers"""

    def __init__(self, sp, dev, gen):
        self.sp, self.dev = sp, dev
        n, h, w = sp["n"], sp["h"], sp["w"]
        self.dtype = DTYPES[sp["dtype"]][0]
        self.masks, mfull = [], []
        for p in sp["parts"]:
            if p["mask"]:
                mu = p["mup"]
                mk = holes(n, h >> mu, w >> mu, gen).to(dev)
                self.masks.append(mk)
                m = mk.double()
                mfull.append(_up2(m) if mu else m)
            else:
                self.masks.append(None)
                mfull.append(torch.ones(n, h, w, dtype=torch.float64, device=dev))
        self.mfull = mfull                                                          # per part, [n, h, w]
        self.conv = _conv_struct(sp, masks=[m.data_ptr() if m is not None else 0 for m in self.masks])
        self.ho, self.wo = self.conv.ho, self.conv.wo
        self.geo = dict(stride=sp["s"], padding=(sp["ph"], sp["pw"]), dilation=sp["dil"])
        g, cin, cout = sp["groups"], sp["cin"], sp["cout"]
        self.cig, self.cog = cin // g, cout // g
        self.mg = g if (g > 1 and not sp["same_holes"]) else 1
        if sp.get("forward_only"):             # fp64 operands band by band (band())
            assert g == 1 and self.mg == 1
            return
        self.M = torch.cat([m[:, None].expand(n, p["c"], h, w) for m, p in zip(mfull, sp["parts"])], 1)   # [n, cin, h, w]
        kh, kw = sp["kh"], sp["kw"]
        with torch.backends.cudnn.flags(enabled=False):
            ones = torch.ones(g, self.cig, kh, kw, dtype=torch.float64, device=dev)
            self.nz = F.conv2d(self.M, ones, groups=g, **self.geo).round()         # [n, groups, ho, wo]: valid terms of a group
            if sp["same_holes"]:
                box = F.conv2d(mfull[0][:, None], ones[:1, :1], **self.geo).round() * cin
            else:
                box = self.nz if self.mg > 1 else self.nz[:, :1]
            self.box = box                                                         # [n, mg, ho, wo]: the mask sums s
            one_k = torch.ones(1, 1, kh, kw, dtype=torch.float64, device=dev)
            one_o = torch.ones(n, 1, self.ho, self.wo, dtype=torch.float64, device=dev)
            self.nz_dg = conv2d_input((n, 1, h, w), one_k, one_o, **self.geo).round() * self.cog          # [n, 1, h, w]
            nzw = conv2d_weight(self.M, (1, cin, kh, kw), one_o, **self.geo).round()                     # [1, cin, kh, kw]
            self.nz_wg = nzw.reshape(g, self.cig, kh, kw).repeat_interleave(self.cog, 0)                # [cout, cig, kh, kw]
        self.nz_fwd = self.nz.repeat_interleave(self.cog, 1)                                              # [n, cout, ho, wo]
        s = self.box.repeat_interleave(cout // self.mg, 1) if not sp["plain"] else torch.ones_like(self.nz_fwd)
        self.s = s                                                                                         # [n, cout, ho, wo]

    # ---- operands
    def set_x(self, vals):
        """vals: per part [n, h >> up, w >> up, c] fp32; HOLE_VALUE where a source pixel is a hole everywhere it lands, zeros in
        channels [c, rup(c, 8)), SENTINEL past that"""
        sp = self.sp
        self.xbufs, xm = [], []
        for p, v, m in zip(sp["parts"], vals, self.mfull):
            mx = F.max_pool2d(m[:, None], 2)[:, 0] if p["up"] else m
            v = torch.where(mx[..., None] == 0, torch.full_like(v, HOLE_VALUE), v)
            buf = self.operand(v, p["xcs"])
            self.xbufs.append(buf)
            if not sp.get("forward_only"):
                xv = nchw(buf, p["c"])
                xm.append((_up2(xv) if p["up"] else xv) * m[:, None])
        for i, b in enumerate(self.xbufs):
            self.conv.parts[i].x = b.data_ptr()
        self.XM = torch.cat(xm, 1) if xm else None

    def bands(self):
        """output row ranges whose fp64 working set stays within BAND_BYTES: the reference's im2col columns (cin kh kw values
        per output pixel), or the eight [n, cout, rows, wo] slabs the Gaussian checks hold at once"""
        sp = self.sp
        per_row = 8 * sp["n"] * self.wo * max(sp["cin"] * sp["kh"] * sp["kw"], 8 * sp["cout"])
        rows = max(1, min(self.ho, BAND_BYTES // per_row))
        return [(r, min(r + rows, self.ho)) for r in range(0, self.ho, rows)]

    def band(self, r0, r1):
        """fp64 operands of output rows [r0, r1): x * m over the input rows they read (their halo, zero rows past the image:
        the convolution then pads only in w), the valid-term counts nz [n, 1, rows, wo] and the box sums s (1 for a plain
        convolution), for groups == 1"""
        sp = self.sp
        a = r0 * sp["s"] - sp["ph"]
        b = (r1 - 1) * sp["s"] - sp["ph"] + sp["dil"] * (sp["kh"] - 1) + 1
        lo, hi = max(a, 0), min(b, sp["h"])
        pad = (0, 0, lo - a, b - hi)
        xm, boxes = [], []
        ones = torch.ones(1, 1, sp["kh"], sp["kw"], dtype=torch.float64, device=self.dev)
        for p, buf, m in zip(sp["parts"], self.xbufs, self.mfull):
            if p["up"]:
                xv = _up2(nchw(buf[:, lo // 2:(hi - 1) // 2 + 1], p["c"]))[:, :, lo % 2:lo % 2 + hi - lo]
            else:
                xv = nchw(buf[:, lo:hi], p["c"])
            mm = m[:, None, lo:hi]
            xm.append(xv * mm)
            with torch.backends.cudnn.flags(enabled=False):
                boxes.append(F.conv2d(F.pad(mm, pad), ones, stride=sp["s"], padding=(0, sp["pw"]), dilation=sp["dil"]).round())
        nz = sum(bx * p["c"] for bx, p in zip(boxes, sp["parts"]))
        if sp["plain"]:
            s = torch.ones_like(nz)
        else:
            s = boxes[0] * sp["cin"] if sp["same_holes"] else nz
        return F.pad(torch.cat(xm, 1), pad), nz, s

    def conv_band(self, a, b):
        """the reference convolution of a band's operands (band()): padding in w only"""
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            return F.conv2d(a, b, stride=sp["s"], padding=(0, sp["pw"]), dilation=sp["dil"])

    def operand(self, vals, cs):
        """vals [..., c] in the storage type, zeros in channels [c, rup(c, 8)), SENTINEL past that"""
        buf = strided((*vals.shape[:-1], _rup8(vals.shape[-1])), cs, 0, self.dtype)
        buf[..., :vals.shape[-1]] = vals.to(self.dtype)
        return buf

    def master(self, wm):
        """wm: fp32 [cout, kh, kw, cig] (KRSC) -> reference weight fp64 [cout, cig, kh, kw] of the storage type's values"""
        self.wm = wm.contiguous()
        self.W = wm.to(self.dtype).double().permute(0, 3, 1, 2).contiguous()

    def new_y(self):
        return strided((self.sp["n"], self.ho, self.wo, _rup8(self.sp["cout"])), self.sp["ycs"], float("nan"), self.dtype)

    def y_padding_ok(self, y):
        """zeros in channels [cout, rup(cout, 8)); past that, channels that are no output: the sentinel, or zeros"""
        c8 = _rup8(self.sp["cout"])
        past = y[..., c8:]
        return bool((y[..., self.sp["cout"]:c8] == 0).all()) and bool(((past == SENTINEL) | (past == 0)).all())

    def new_dx(self, at_src):
        sp, out = self.sp, []
        for p, cs in zip(sp["parts"], sp["dxcs"]):
            sh = p["up"] if at_src else 0
            out.append(strided((sp["n"], sp["h"] >> sh, sp["w"] >> sh, p["c"]), cs, float("nan"), self.dtype))
        return out

    # ---- fp64 references
    def conv_ref(self, a, b):
        with torch.backends.cudnn.flags(enabled=False):
            return F.conv2d(a, b, groups=self.sp["groups"], **self.geo)

    def dgrad_ref(self, g, b):
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            return conv2d_input((sp["n"], sp["cin"], sp["h"], sp["w"]), b, g, groups=sp["groups"], **self.geo)

    def wgrad_ref(self, a, g):
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            return conv2d_weight(a, (sp["cout"], self.cig, sp["kh"], sp["kw"]), g, groups=sp["groups"], **self.geo)

    def dx_parts(self, full, at_src):
        """split a full-resolution [n, cin, h, w] gradient into parts: 2x2 sums of the children for upsampled parts at source
        resolution"""
        out, off = [], 0
        for p in self.sp["parts"]:
            g = full[:, off:off + p["c"]]
            if at_src and p["up"]:
                g = F.avg_pool2d(g, 2) * 4
            out.append(g)
            off += p["c"]
        return out


def _ws(lib, cref, dev):
    return torch.zeros(max(16, int(lib.pcb_pconv_workspace(cref))), dtype=torch.uint8, device=dev)


@pytest.mark.parametrize("name", sorted(CASES))
def test_conv_route_vs_fp64(name):
    sp = CASES[name]
    dev = torch.device("cuda:0")
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    dgen = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    n, cin, cout, kh, kw = sp["n"], sp["cin"], sp["cout"], sp["kh"], sp["kw"]
    P = _Problem(sp, dev, gen)
    torch.cuda.reset_peak_memory_stats(dev)          # (the peak still counts what is allocated now)
    cref = ctypes.byref(P.conv)
    dt, ho, wo, ycs, dcs = P.dtype, P.ho, P.wo, sp["ycs"], sp["dcs"]
    route = _routes(lib, P.conv)
    assert route == tuple(sp["route"]), f"{name}: the plan routes {route}, the case covers {sp['route']}"
    is_tc = route[0] in TC_ROUTES
    assert lib.pcb_conv_uses_tensor_cores(cref) == int(is_tc)
    fuses = lib.pcb_conv_fuses_bn_stats(cref)
    assert fuses == lib.pcb_conv_fuses_affine_act(cref) == int(route[0] in ("tma", "gather", "stem")), f"{name}: fused-epilogue query"
    at_src = bool(lib.pcb_conv_dgrad_at_source_resolution(cref))
    assert not at_src or route[1] in ("k2r", "tma", "tma_s2"), f"{name}: only the tail and the sub-pixel kernels work at source resolution"
    fuses_relu = lib.pcb_conv_dgrad_fuses_relu(cref)
    fe, de = ctypes.c_size_t(), ctypes.c_size_t()
    lib.pcb_conv_weight_layout(cref, ctypes.byref(fe), ctypes.byref(de))
    wbuf_dt = torch.bfloat16 if is_tc else dt
    ws = _ws(lib, cref, dev)
    mg, N = P.mg, n * ho * wo
    # the data gradient of a row-packed layer runs like ops.py runs it: force_generic, KRSC weights in the storage type
    dg_conv = P.conv
    if route[1] == "none":
        dg_conv = _conv_struct(dict(sp, force_generic=True), masks=[m.data_ptr() if m is not None else 0 for m in P.masks])
        assert _routes(lib, dg_conv) == ("generic",) * 3
    dg_ref = ctypes.byref(dg_conv)

    def prepare(wm):
        wf = torch.full((fe.value,), float("nan"), dtype=wbuf_dt, device=dev)
        wd = torch.full((de.value,), float("nan"), dtype=wbuf_dt, device=dev) if de.value else None
        _lib.check(lib.pcb_conv_weight_prepare(cref, wm.data_ptr(), wf.data_ptr(), wd.data_ptr() if wd is not None else None, stream))
        return wf, wd

    def run_dgrad(dc, wf, wd, wk, dxs):
        """into the prefilled dxs; wk: the KRSC weights in the storage type (row-packed layers)"""
        ptrs = (ctypes.c_void_p * len(dxs))(*[b.data_ptr() for b in dxs])
        strides = (ctypes.c_int32 * len(dxs))(*sp["dxcs"])
        if route[1] == "none":
            _lib.check(lib.pcb_pconv_backward_data(dg_ref, dc.data_ptr(), dcs, wk.data_ptr(), None, ptrs, strides, stream))
        else:
            _lib.check(lib.pcb_pconv_backward_data(cref, dc.data_ptr(), dcs, wf.data_ptr(), wd.data_ptr() if wd is not None else None,
                                                   ptrs, strides, stream))

    def ints(r, *shape):
        return torch.randint(-r, r + 1, shape, generator=dgen, device=dev).to(torch.float32)

    def check_dx(tag, dxs, want_parts, alt_parts=None):
        for i, (p, buf, want) in enumerate(zip(sp["parts"], dxs, want_parts)):
            got = nchw(buf, p["c"]).float()
            if alt_parts is None:
                assert_bitwise(f"{name}: {tag}, part {i}", got, want, nan_equal=True)
            else:
                assert_within(f"{name}: {tag}, part {i}", got.double(), want, alt_parts[i])
            c8 = _rup8(p["c"])
            assert sentinel_kept(buf, c8), f"{name}: {tag} wrote past rup(c, 8) of part {i}"
            pad = buf[..., p["c"]:c8]
            assert bool(((pad == SENTINEL) | (pad == 0)).all()), f"{name}: {tag} wrote garbage into the channel padding of part {i}"

    if sp.get("forward_only"):
        _forward_only_checks(name, sp, P, lib, stream, prepare, ints, dgen, ws, route, fuses)
        return

    # ================= integer regime: bit-exact
    ix, iw = sp["ix"], sp["iw"]
    P.set_x([ints(ix, n, sp["h"] >> p["up"], sp["w"] >> p["up"], p["c"]) for p in sp["parts"]])
    P.master(ints(iw, cout, kh, kw, P.cig))
    bias = torch.randint(-16, 17, (cout,), generator=dgen, device=dev).to(torch.float32) / 8
    dcv = ints(4, n, ho, wo, cout)
    dc = P.operand(dcv, dcs)
    G = nchw(dc, cout)
    # every partial sum below 2^24: at most (number of valid terms) x max|a| x max|b|
    big = max(float(P.nz_fwd.max()) * ix * iw, float(P.nz_dg.max()) * 4 * iw, float(P.nz_wg.max()) * 4 * ix)
    assert big < 2 ** 24, f"{name}: partial sums could round ({big:.3g}): not an exact case"
    if route[0] == "k2r":
        cu = max(p["c"] for p in sp["parts"] if p["up"])
        assert cu * ix * iw <= 256, f"{name}: the tail's bf16 Z rows would round"
    wf, wd = prepare(P.wm)
    wk = P.wm.to(dt).contiguous()
    y, dxs = P.new_y(), P.new_dx(at_src)
    msum = torch.full((mg, N), float("nan"), device=dev)
    newmask = torch.full((mg, N), 77, dtype=torch.uint8, device=dev)
    dw = torch.full((cout, kh, kw, P.cig), float("nan"), device=dev)
    dw0 = ints(4, cout, kh, kw, P.cig)
    dw_acc = dw0.clone()
    state = [(y, y.clone()), (msum, float("nan")), (newmask, 77), (dw, float("nan")), (dw_acc, dw0)] + [(b, b.clone()) for b in dxs]

    def run():
        _lib.check(lib.pcb_pconv_forward(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(), newmask.data_ptr(),
                                         ws.data_ptr(), stream))
        run_dgrad(dc, wf, wd, wk, dxs)
        _lib.check(lib.pcb_pconv_backward_weight(cref, dc.data_ptr(), dcs, dw.data_ptr(), ws.data_ptr(), stream))
        _lib.check(lib.pcb_pconv_backward_weight_acc(cref, dc.data_ptr(), dcs, dw_acc.data_ptr(), ws.data_ptr(), stream))

    want_ran = tuple("generic" if r == "none" else r for r in route)

    def check(records):
        ran, cnt = _kernel_routes(records)
        assert ran == want_ran, f"{name}: the kernels ran {ran}, the plan says {route}; kernels: {dict(cnt)}"
        for (k, args), launches in sp.get("tiles", {}).items():
            assert records[(k, args)] == launches, (f"{name}: {k}<{', '.join(args)}> launched {records[(k, args)]} times, the case is "
                                                    f"named for {launches}; kernels: {dict(records)}")
    records = traced(name, run, check, state)
    print(f"{name}: kernels {sorted(records or {})}")

    # mask pass: the fp64 box sums; a plain convolution leaves msum / newmask alone
    s_ref = P.box.permute(1, 0, 2, 3).reshape(mg, N)
    nm_ref = torch.ones_like(newmask) if sp["no_guard"] else (s_ref != 0).to(torch.uint8)
    if sp["plain"]:
        assert bool(msum.isnan().all()) and bool((newmask == 77).all()), f"{name}: a plain convolution must not touch msum / newmask"
    else:
        assert_bitwise(f"{name}: msum", msum.double(), s_ref, nan_equal=True)
        assert_bitwise(f"{name}: newmask", newmask, nm_ref, nan_equal=True)
    # the two-call forward: mask pass, then the rest, bitwise equal to the one-call forward
    msum2 = torch.full((mg, N), float("nan"), device=dev)
    newmask2 = torch.full((mg, N), 77, dtype=torch.uint8, device=dev)
    ws2, y2 = _ws(lib, cref, dev), P.new_y()
    _lib.check(lib.pcb_pconv_mask_pass(cref, msum2.data_ptr(), newmask2.data_ptr(), ws2.data_ptr(), stream))
    _lib.check(lib.pcb_pconv_forward_premasked(cref, wf.data_ptr(), bias.data_ptr(), y2.data_ptr(), ycs, msum2.data_ptr(),
                                               newmask2.data_ptr(), ws2.data_ptr(), stream))
    torch.cuda.synchronize()
    if not sp["plain"]:
        assert_bitwise(f"{name}: mask pass msum", msum2.double(), s_ref, nan_equal=True)
        assert_bitwise(f"{name}: mask pass newmask", newmask2, nm_ref, nan_equal=True)
    assert_bitwise(f"{name}: mask pass + premasked forward vs one-call forward", y2, y, nan_equal=True)

    # forward
    S = P.conv_ref(P.XM, P.W).round()
    s, b = P.s, bias.double()[None, :, None, None]
    empty = s == 0
    want, alt = _int_forward_want(S, s, b, route[0], sp["no_guard"], dt)
    assert_bitwise(f"{name}: forward", nchw(y, cout), want, alt, nan_equal=True)
    assert P.y_padding_ok(y), f"{name}: forward must write zeros into channels [cout, rup(cout, 8)) and nothing past them"

    # renormalisation backward: which of the three kernels runs is decided by the layout, each has its own last operation
    dyv = ints(4, n, ho, wo, cout)
    dy = P.operand(dyv, ycs)
    dco = torch.full((n, ho, wo, dcs), float("nan"), dtype=dt, device=dev)
    dbias = torch.full((cout,), float("nan"), device=dev)
    _lib.check(lib.pcb_pconv_renorm_backward(cref, dy.data_ptr(), ycs, msum.data_ptr(), dco.data_ptr(), dcs, dbias.data_ptr(), stream))
    torch.cuda.synchronize()
    Y = nchw(dy, cout).float()
    sf = P.s.float()
    vec = mg == 1 and cout % 8 == 0 and cout <= 2048 and dcs == cout and ycs % 8 == 0
    pix8 = mg == 1 and cout <= 8 and dcs == 8
    d = Y * (1.0 / sf) if (vec or pix8) else Y / sf
    keep = ~empty if not sp["no_guard"] else torch.ones_like(empty)
    d = torch.where(keep, d, torch.zeros_like(d))
    assert_bitwise(f"{name}: renormalisation backward", nchw(dco, cout).float(), d.to(dt).float(), nan_equal=True)
    assert bool((dco[..., cout:] == 0).all()), f"{name}: renormalisation backward must zero channels [cout, dc_cstride)"
    dbias_want = (Y.double() * (~empty)).sum((0, 2, 3))
    if sp["no_guard"] and bool(empty.any()):
        dbias_want = torch.where(empty.any(3).any(2).any(0), torch.full_like(dbias_want, float("nan")), dbias_want)
    assert_bitwise(f"{name}: bias gradient", dbias.double(), dbias_want, nan_equal=True)

    # data gradient: m * S, zero under the holes, at source resolution where the query says so
    gfull = P.dgrad_ref(G, P.W).round() * P.M
    wants = [g.float().to(dt).float() for g in P.dx_parts(gfull, at_src)]
    check_dx("data gradient", dxs, wants)
    if fuses_relu:
        assert len(sp["parts"]) == 1
        rx = P.xbufs[0]
        dxr = P.new_dx(False)[0]
        _lib.check(lib.pcb_pconv_backward_data_relu(cref, dc.data_ptr(), dcs, wd.data_ptr(), dxr.data_ptr(), sp["dxcs"][0],
                                                    rx.data_ptr(), sp["parts"][0]["xcs"], stream))
        torch.cuda.synchronize()
        relu_keep = nchw(rx, cin).float() > 0
        check_dx("data gradient with the ReLU backward", [dxr], [torch.where(relu_keep, wants[0], torch.zeros_like(wants[0]))])

    # weight gradient: S, and fl(dw0 + S) accumulating
    gw = P.wgrad_ref(P.XM, G).round().permute(0, 2, 3, 1)
    assert_bitwise(f"{name}: weight gradient", dw, gw.float(), nan_equal=True)
    assert_bitwise(f"{name}: weight gradient (accumulating)", dw_acc, (dw0.double() + gw).float(), nan_equal=True)
    for i, (p, buf) in enumerate(zip(sp["parts"], P.xbufs)):
        assert sentinel_kept(buf, _rup8(p["c"])), f"{name}: x of part {i} was written"

    # weight refresh: refresh(W2) over prepare(W1) is bitwise prepare(W2), extra operands included
    wm2 = ints(iw, cout, kh, kw, P.cig)
    _lib.check(lib.pcb_conv_weight_refresh(cref, wm2.data_ptr(), wf.data_ptr(), wd.data_ptr() if wd is not None else None, stream))
    wf2, wd2 = prepare(wm2)
    torch.cuda.synchronize()
    ib = torch.int16 if wbuf_dt == torch.bfloat16 else torch.int32
    assert torch.equal(wf.view(ib), wf2.view(ib)), f"{name}: refreshed forward operands differ from freshly prepared ones"
    if wd is not None:
        assert torch.equal(wd.view(ib), wd2.view(ib)), f"{name}: refreshed data-gradient operands differ from freshly prepared ones"

    # ================= Gaussian regime: error bounds
    P.set_x([torch.randn(n, sp["h"] >> p["up"], sp["w"] >> p["up"], p["c"], generator=dgen, device=dev) for p in sp["parts"]])
    P.master(torch.randn(cout, kh, kw, P.cig, generator=dgen, device=dev).to(dt).float() / 2)
    wf, wd = prepare(P.wm)
    bias = torch.randn(cout, generator=dgen, device=dev) * 0.1
    b = bias.double()[None, :, None, None]
    v_ref, e_ref = _gauss_forward_ref(P.conv_ref(P.XM, P.W), P.conv_ref(P.XM.abs(), P.W.abs()), P.nz_fwd, P.s, b, route[0] == "k2r")
    store = 2.0 ** -8 if dt == torch.bfloat16 else 0.0
    live = ~empty if sp["no_guard"] else torch.ones_like(empty)

    def check_y(tag, y, v, e, nan_at_empty=True):
        assert P.y_padding_ok(y), f"{name}: {tag} must write zeros into channels [cout, rup(cout, 8)) and nothing past them"
        _check_y_values(name, tag, sp["no_guard"], nchw(y, cout), v, e, store, live, nan_at_empty)

    y = P.new_y()
    _lib.check(lib.pcb_pconv_forward(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(), newmask.data_ptr(),
                                     ws.data_ptr(), stream))
    torch.cuda.synchronize()
    check_y("forward", y, v_ref, e_ref)
    scale = torch.rand(cout, generator=dgen, device=dev) + 0.5
    shift = torch.randn(cout, generator=dgen, device=dev) * 0.1
    if fuses:
        y = P.new_y()
        sums = torch.zeros(2, cout, dtype=torch.float64, device=dev)
        _lib.check(lib.pcb_pconv_forward_bn(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                            newmask.data_ptr(), ws.data_ptr(), 0, sums.data_ptr(), stream))
        torch.cuda.synchronize()
        check_y("forward with BatchNorm sums", y, v_ref, e_ref)
        if not sp["no_guard"]:
            yv = y[..., :cout].double().reshape(-1, cout)
            for row, vals in ((0, yv), (1, yv * yv)):
                tol = yv.shape[0] * 2.0 ** -23 * vals.abs().sum(0)
                assert bool(((sums[row] - vals.sum(0)).abs() <= tol).all()), f"{name}: BatchNorm {'sums' if row == 0 else 'squares'}"
        sc, sh = scale.double()[None, :, None, None], shift.double()[None, :, None, None]
        z = v_ref * sc + sh
        ez = sc * e_ref + 2.0 ** -23 * (z.abs() + sh.abs())
        for act in ACTS:
            y = P.new_y()
            _lib.check(lib.pcb_pconv_forward_affine_act(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                                        newmask.data_ptr(), ws.data_ptr(), 0, scale.data_ptr(), shift.data_ptr(), act,
                                                        SLOPE, stream))
            torch.cuda.synchronize()
            va = act_ref(z, act, SLOPE)
            check_y(f"eval epilogue, activation {act}", y, va, ez + 2.0 ** -23 * va.abs(), act == _lib.ACT_NONE)
    else:
        y = P.new_y()
        sums = torch.zeros(2, cout, dtype=torch.float64, device=dev)
        rc = lib.pcb_pconv_forward_bn(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(), newmask.data_ptr(),
                                      ws.data_ptr(), 0, sums.data_ptr(), stream)
        assert rc != 0 and b"does not fuse" in lib.pcb_last_error(), f"{name}: fused BatchNorm sums must be refused"
        rc = lib.pcb_pconv_forward_affine_act(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                              newmask.data_ptr(), ws.data_ptr(), 0, scale.data_ptr(), shift.data_ptr(), _lib.ACT_RELU,
                                              SLOPE, stream)
        assert rc != 0 and b"does not apply" in lib.pcb_last_error(), f"{name}: fused affine + activation must be refused"
        torch.cuda.synchronize()
        assert bool(y[..., :_rup8(cout)].isnan().all()) and bool((sums == 0).all()), f"{name}: a refused call must not run"

    dc = P.operand(torch.randn(n, ho, wo, cout, generator=dgen, device=dev), dcs)
    G = nchw(dc, cout)
    dxs = P.new_dx(at_src)
    run_dgrad(dc, wf, wd, P.wm.to(dt).contiguous(), dxs)
    dw = torch.full((cout, kh, kw, P.cig), float("nan"), device=dev)
    _lib.check(lib.pcb_pconv_backward_weight(cref, dc.data_ptr(), dcs, dw.data_ptr(), ws.data_ptr(), stream))
    torch.cuda.synchronize()
    rounds_d = route[1] == "k2r" or (route[1] != "none" and at_src)
    gref = P.dgrad_ref(G, P.W) * P.M
    gmag = P.dgrad_ref(G.abs(), P.W.abs()) * P.M
    gerr = accumulation_bound(P.nz_dg, gmag, rounds_d)
    refs, errs = P.dx_parts(gref, at_src), P.dx_parts(gerr, at_src)
    check_dx("Gaussian data gradient", dxs, refs, [e + store * (r.abs() + e) for r, e in zip(refs, errs)])
    del gref, gmag, gerr
    wref = P.wgrad_ref(P.XM, G)
    wmag = P.wgrad_ref(P.XM.abs(), G.abs())
    werr = accumulation_bound(P.nz_wg, wmag, route[2] == "k2r")
    assert_within(f"{name}: Gaussian weight gradient", dw.double(), wref.permute(0, 2, 3, 1), werr.permute(0, 2, 3, 1))


def _forward_only_checks(name, sp, P, lib, stream, prepare, ints, dgen, ws, route, fuses):
    """the checks of a descriptor only inference reaches: the forward route in the trace; in the integer regime the one-call
    forward and its mask pass, the two-call forward (mask pass, premasked forward) and the weight refresh; in the Gaussian
    regime the forward, the fused BatchNorm sums and the eval epilogue at every activation.  Every fp64 reference and
    comparison runs band by band (P.bands), and nothing page-sized leaves the device."""
    dev, dt = P.dev, P.dtype
    n, cout, kh, kw = sp["n"], sp["cout"], sp["kh"], sp["kw"]
    ho, wo, ycs, N = P.ho, P.wo, sp["ycs"], sp["n"] * P.ho * P.wo
    cref = ctypes.byref(P.conv)
    bands = P.bands()
    ix, iw = sp["ix"], sp["iw"]
    P.set_x([ints(ix, n, sp["h"] >> p["up"], sp["w"] >> p["up"], p["c"]) for p in sp["parts"]])
    P.master(ints(iw, cout, kh, kw, P.cig))
    bias = torch.randint(-16, 17, (cout,), generator=dgen, device=dev).to(torch.float32) / 8
    b = bias.double()[None, :, None, None]
    if route[0] == "k2r":
        cu = max(p["c"] for p in sp["parts"] if p["up"])
        assert cu * ix * iw <= 256, f"{name}: the tail's bf16 Z rows would round"
    wf, wd = prepare(P.wm)
    y = P.new_y()
    msum = torch.full((1, N), float("nan"), device=dev)
    newmask = torch.full((1, N), 77, dtype=torch.uint8, device=dev)

    def run():
        _lib.check(lib.pcb_pconv_forward(cref, wf.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(), newmask.data_ptr(),
                                         ws.data_ptr(), stream))

    def check(records):
        ran, cnt = _kernel_routes(records)
        assert ran[0] == route[0], f"{name}: the forward ran {ran[0]}, the plan says {route[0]}; kernels: {dict(cnt)}"
    records = traced(name, run, check, [(y, y.clone()), (msum, float("nan")), (newmask, 77)])
    print(f"{name}: kernels {sorted(records or {})}")

    msum2 = torch.full((1, N), float("nan"), device=dev)
    newmask2 = torch.full((1, N), 77, dtype=torch.uint8, device=dev)
    ws2, y2 = _ws(lib, cref, dev), P.new_y()
    _lib.check(lib.pcb_pconv_mask_pass(cref, msum2.data_ptr(), newmask2.data_ptr(), ws2.data_ptr(), stream))
    _lib.check(lib.pcb_pconv_forward_premasked(cref, wf.data_ptr(), bias.data_ptr(), y2.data_ptr(), ycs, msum2.data_ptr(),
                                               newmask2.data_ptr(), ws2.data_ptr(), stream))
    torch.cuda.synchronize()
    assert_bitwise(f"{name}: mask pass + premasked forward vs one-call forward", y2, y, nan_equal=True)
    del y2, ws2
    if sp["plain"]:
        assert bool(msum.isnan().all()) and bool((newmask == 77).all()), f"{name}: a plain convolution must not touch msum / newmask"
    assert P.y_padding_ok(y), f"{name}: forward must write zeros into channels [cout, rup(cout, 8)) and nothing past them"
    for r0, r1 in bands:
        XM, nz, s = P.band(r0, r1)
        assert float(nz.max()) * ix * iw < 2 ** 24, f"{name}: partial sums could round: not an exact case"
        if not sp["plain"]:
            s_ref = s[:, 0].reshape(1, -1)
            nm_ref = torch.ones_like(s_ref, dtype=torch.uint8) if sp["no_guard"] else (s_ref != 0).to(torch.uint8)
            for tag, ms, nm in (("", msum, newmask), ("mask pass ", msum2, newmask2)):
                assert_bitwise(f"{name}: {tag}msum, rows {r0}:{r1}", ms.view(n, ho, wo)[:, r0:r1].reshape(1, -1).double(), s_ref)
                assert_bitwise(f"{name}: {tag}newmask, rows {r0}:{r1}", nm.view(n, ho, wo)[:, r0:r1].reshape(1, -1), nm_ref)
        want, alt = _int_forward_want(P.conv_band(XM, P.W).round(), s, b, route[0], sp["no_guard"], dt)
        assert_bitwise(f"{name}: forward, rows {r0}:{r1}", nchw(y[:, r0:r1], cout), want, alt, nan_equal=True)
        del XM, want, alt

    wm2 = ints(iw, cout, kh, kw, P.cig)
    _lib.check(lib.pcb_conv_weight_refresh(cref, wm2.data_ptr(), wf.data_ptr(), wd.data_ptr() if wd is not None else None, stream))
    wf2, wd2 = prepare(wm2)
    torch.cuda.synchronize()
    ib = torch.int16 if wf.dtype == torch.bfloat16 else torch.int32
    assert torch.equal(wf.view(ib), wf2.view(ib)), f"{name}: refreshed forward operands differ from freshly prepared ones"
    if wd is not None:
        assert torch.equal(wd.view(ib), wd2.view(ib)), f"{name}: refreshed data-gradient operands differ from freshly prepared ones"
    del wf2, wd2

    # Gaussian regime: every output first (forward, BatchNorm sums, eval epilogue per activation), then the bands
    P.set_x([torch.randn(n, sp["h"] >> p["up"], sp["w"] >> p["up"], p["c"], generator=dgen, device=dev) for p in sp["parts"]])
    P.master(torch.randn(cout, kh, kw, P.cig, generator=dgen, device=dev).to(dt).float() / 2)
    wf, wd = prepare(P.wm)
    bias = torch.randn(cout, generator=dgen, device=dev) * 0.1
    b = bias.double()[None, :, None, None]
    scale = torch.rand(cout, generator=dgen, device=dev) + 0.5
    shift = torch.randn(cout, generator=dgen, device=dev) * 0.1
    outs = {"forward": P.new_y()}
    _lib.check(lib.pcb_pconv_forward(cref, wf.data_ptr(), bias.data_ptr(), outs["forward"].data_ptr(), ycs, msum.data_ptr(),
                                     newmask.data_ptr(), ws.data_ptr(), stream))
    sums = torch.zeros(2, cout, dtype=torch.float64, device=dev)
    if fuses:
        outs["forward with BatchNorm sums"] = P.new_y()
        _lib.check(lib.pcb_pconv_forward_bn(cref, wf.data_ptr(), bias.data_ptr(), outs["forward with BatchNorm sums"].data_ptr(), ycs,
                                            msum.data_ptr(), newmask.data_ptr(), ws.data_ptr(), 0, sums.data_ptr(), stream))
        for act in ACTS:
            outs[act] = P.new_y()
            _lib.check(lib.pcb_pconv_forward_affine_act(cref, wf.data_ptr(), bias.data_ptr(), outs[act].data_ptr(), ycs,
                                                        msum.data_ptr(), newmask.data_ptr(), ws.data_ptr(), 0, scale.data_ptr(),
                                                        shift.data_ptr(), act, SLOPE, stream))
    else:
        yr = P.new_y()
        rc = lib.pcb_pconv_forward_bn(cref, wf.data_ptr(), bias.data_ptr(), yr.data_ptr(), ycs, msum.data_ptr(), newmask.data_ptr(),
                                      ws.data_ptr(), 0, sums.data_ptr(), stream)
        assert rc != 0 and b"does not fuse" in lib.pcb_last_error(), f"{name}: fused BatchNorm sums must be refused"
        rc = lib.pcb_pconv_forward_affine_act(cref, wf.data_ptr(), bias.data_ptr(), yr.data_ptr(), ycs, msum.data_ptr(),
                                              newmask.data_ptr(), ws.data_ptr(), 0, scale.data_ptr(), shift.data_ptr(), _lib.ACT_RELU,
                                              SLOPE, stream)
        assert rc != 0 and b"does not apply" in lib.pcb_last_error(), f"{name}: fused affine + activation must be refused"
        torch.cuda.synchronize()
        assert bool(yr[..., :_rup8(cout)].isnan().all()) and bool((sums == 0).all()), f"{name}: a refused call must not run"
        del yr
    torch.cuda.synchronize()
    for tag, yo in outs.items():
        assert P.y_padding_ok(yo), f"{name}: {tag} must write zeros into channels [cout, rup(cout, 8)) and nothing past them"
    store = 2.0 ** -8 if dt == torch.bfloat16 else 0.0
    sc, sh = scale.double()[None, :, None, None], shift.double()[None, :, None, None]
    tot = torch.zeros(4, cout, dtype=torch.float64, device=dev)     # sum y, sum y^2, sum |y|, sum y^2 of the stored values
    for r0, r1 in bands:
        XM, nz, s = P.band(r0, r1)
        v_ref, e_ref = _gauss_forward_ref(P.conv_band(XM, P.W), P.conv_band(XM.abs(), P.W.abs()), nz, s, b, route[0] == "k2r")
        del XM
        live = s != 0 if sp["no_guard"] else torch.ones_like(s, dtype=torch.bool)
        rows = f"rows {r0}:{r1}"
        for tag in ("forward", "forward with BatchNorm sums"):
            if tag in outs:
                _check_y_values(name, f"{tag}, {rows}", sp["no_guard"], nchw(outs[tag][:, r0:r1], cout), v_ref, e_ref, store, live)
        if not fuses:
            continue
        if not sp["no_guard"]:
            yv = outs["forward with BatchNorm sums"][:, r0:r1, :, :cout].double().reshape(-1, cout)
            tot += torch.stack([yv.sum(0), (yv * yv).sum(0), yv.abs().sum(0), (yv * yv).sum(0)])
            del yv
        z = v_ref * sc + sh
        ez = sc * e_ref + 2.0 ** -23 * (z.abs() + sh.abs())
        for act in ACTS:
            va = act_ref(z, act, SLOPE)
            _check_y_values(name, f"eval epilogue, activation {act}, {rows}", sp["no_guard"], nchw(outs[act][:, r0:r1], cout), va,
                            ez + 2.0 ** -23 * va.abs(), store, live, act == _lib.ACT_NONE)
    if fuses and not sp["no_guard"]:
        for row, what in ((0, "sums"), (1, "squares")):
            tol = N * 2.0 ** -23 * tot[2 + row]
            assert bool(((sums[row] - tot[row]).abs() <= tol).all()), f"{name}: BatchNorm {what}"
    peak = torch.cuda.max_memory_allocated(dev)
    print(f"{name}: peak device memory {peak / 2 ** 30:.2f} GiB over {len(bands)} band(s)")
    assert peak < MEMORY_BUDGET, f"{name}: peak device memory {peak / 2 ** 30:.2f} GiB"

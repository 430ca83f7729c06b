"""Depthwise convolution kernels (dwconv.cu) through the C ABI, every element against an fp64 reference of the same operands
computed on the device (F.conv2d / torch.nn.grad.conv2d_input / conv2d_weight with groups = c, cuDNN off so that every
reference is a direct sum).  Two sets of cases:

  * every depthwise descriptor of tests/golden/conv_dispatch.json that the depthwise family accepts (the layers the workloads
    run: dw4 at dilations up to 29, dw3 at stride 2, the small GPU test cases), batch capped at 2.  A descriptor only
    inference reaches ("forward_only": the segmentation networks at page sizes) is checked in the forward alone, its fp64
    references in bands of output rows of at most BAND_BYTES, its peak device memory below MEMORY_BUDGET;
  * hand cases for the paths production does not reach: holes on dw3 (one msum plane or c of them, a half-resolution hole
    plane, large values under the holes), strided channel views, awkward channel counts (8, 40, 296, 2048), dw4 segment,
    x-tile and dilation-phase edges in both storage types, a "valid" 3x3 on dw3, and the depthwise shapes the family leaves to
    the shape-general kernels of conv_generic.cu (k5, k7, kh != kw, stride 3).

Each case asserts the route it covers from the kernel names of a torch.profiler trace (kernel_harness.traced), then checks:

  * mask pass: msum and newmask equal the fp64 box sums exactly (times cin with same_holes); a plain convolution leaves both
    untouched;
  * forward, data gradient, weight gradient (zeroing and accumulating), all outputs prefilled with NaN and channels past c of
    a strided view prefilled with a sentinel that must survive -- except in y on the generic route, whose channels past
    rup(c, 8) are no outputs and may be zeroed (the header's contract; the generic forward zero-fills them);
  * the fused BatchNorm statistics and the eval-mode affine + activation epilogue where pcb_conv_fuses_bn_stats says the
    kernel fuses them, and their refusal where it does not (the generic route).

Integer regime (every case).  x, w, dc are integers of magnitude <= 4 and the bias a multiple of 1/8, all exact in bf16.  Every
partial sum stays below 2^24 (the largest is a weight gradient over 2 x 256 x 256 pixels: 2^17 * 16 = 2^21), so fp32
accumulation is exact in any order, atomics included, and the fp64 reference rounded to the nearest integer is that exact sum.
The kernels are built without fast math, so what they store must be BIT-IDENTICAL to the last float32 operations applied to
the exact sum S:  plain forward fl(S + b);  renormalised forward fl(fl(S / s) + b), 0 where s == 0;  data gradient m * S;
weight gradient S, or fl(dw0 + S) accumulating onto an integer dw0; each then stored in the case's type (bf16: round to nearest
even).  fl(S / s) is taken as the fp64 quotient rounded to fp32, which is the correctly rounded fp32 quotient (double rounding
is innocuous for division when 53 >= 2 * 24 + 2).  A dropped or repeated row, column or tap changes some element.

Gaussian regime (fp32 storage, the eval epilogue, the BatchNorm sums).  Each of the n nonzero terms of an element costs at most
two fp32 roundings (product, or the fma, and add; bf16 products are exact), so the accumulation is off by at most
n * 2^-22 * S, S = sum of |products| (Higham, Accuracy and Stability of Numerical Algorithms, 4.2; n u < 1/2 here).  The
division by s and the bias add round twice more (2^-22 relative of |acc| / s and the result), the eval epilogue's fma once
(2^-23 of |z| + |shift|) and LeakyReLU's multiply once (2^-23 of the result); every activation is 1-Lipschitz.  A bf16 store
adds half an ulp (2^-8 relative is used, as in test_gpu_conv_routes.py).  The BatchNorm sums are checked against the stored
values: M fp32 additions of terms bounded by |y| are off by at most M * 2^-23 * sum |y|.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from kernel_harness import (HOLE_VALUE, SENTINEL, act_ref, assert_bitwise, assert_within, conv_dispatch_cases, holes, nchw,
                            sentinel_kept, strided, traced)
from text_segmentation_image_inpainting_b200 import _lib

pytestmark = pytest.mark.gpu

INT_RANGE = 4                # |x|, |w|, |dc| <= 4 in the integer regime
SLOPE = 0.2
ACTS = (_lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_LEAKY, _lib.ACT_RELU6)
DTYPES = {"bf16": (torch.bfloat16, _lib.PCB_BF16), "f32": (torch.float32, _lib.PCB_F32)}
BAND_BYTES = 2 ** 29         # one fp64 [n, c, rows, wo] slab of a band of output rows (forward-only cases)
MEMORY_BUDGET = 12 * 2 ** 30  # peak device memory of a forward-only case: page-size cases run on shared GPUs

# the kernels of each route, per direction (forward, data gradient, weight gradient)
KERNELS = {"dw4": ("dw4_s1_kernel", "dw4_s1_kernel", "dw4_s1_wgrad_kernel"),
           "dw3": ("dw3_fwd_kernel", "dw3_dgrad_kernel", "dw3_wgrad_kernel"),
           "generic": ("generic_fwd_kernel", "generic_dgrad_kernel", "generic_wgrad_kernel")}


def _case(n, h, w, c, k=3, s=1, pad=None, dil=1, dtype="bf16", holes=False, mask_up=0, same_holes=False, plain=None,
          cs=None, route=None, forward_only=False):
    """cs: channel strides (x, y, dc, dx), default c.  route: the kernels of (forward, data gradient, weight gradient);
    default: what the depthwise dispatch documents (dw4 for plain 3x3 stride 1 with padding == dilation, dw3 for other 3x3 at
    a power-of-two stride, the generic kernels otherwise)."""
    kh, kw = (k, k) if isinstance(k, int) else k
    ph, pw = (dil * (kh - 1) // 2, dil * (kw - 1) // 2) if pad is None else ((pad, pad) if isinstance(pad, int) else pad)
    plain = (not holes) if plain is None else plain
    if route is None:
        if (kh, kw) != (3, 3) or s & (s - 1):
            route = ("generic",) * 3
        elif s == 1 and ph == pw == dil and plain and not holes:
            route = ("dw4",) * 3
        else:
            route = ("dw3",) * 3
    return dict(n=n, h=h, w=w, c=c, kh=kh, kw=kw, s=s, ph=ph, pw=pw, dil=dil, dtype=dtype, holes=holes, mask_up=mask_up,
                same_holes=same_holes, plain=plain, cs=tuple(cs) if cs else (c,) * 4, route=route, forward_only=forward_only)


def _fixture_cases():
    """one case per distinct depthwise descriptor of the dispatch fixture (the depthwise family's eligibility test, n <= 2)"""
    out = {}
    for case in conv_dispatch_cases():
        d, p = case["conv"], case["conv"]["parts"]
        if not (d["groups"] == d["cin"] == d["cout"] > 1 and len(p) == 1):
            continue
        p = p[0]
        if d["cin"] % 8 or d["cin"] > 2048 or p["x_cstride"] % 8 or p["x_up"]:
            continue
        dt = "bf16" if d["dtype"] == _lib.PCB_BF16 else "f32"
        n = min(d["n"], 2)
        spec = _case(n, d["h"], d["w"], d["cin"], (d["kh"], d["kw"]), d["stride"], (d["pad_h"], d["pad_w"]), d["dil"], dt,
                     holes=bool(p["mask"]), mask_up=p["mask_up"], same_holes=bool(d["same_holes"]), plain=bool(d["plain"]),
                     cs=(p["x_cstride"],) + (d["cin"],) * 3, forward_only=bool(case.get("forward_only")))
        name = (f"fx_{dt}_n{n}_{d['h']}x{d['w']}_c{d['cin']}_k{d['kh']}x{d['kw']}_s{d['stride']}_p{d['pad_h']}x{d['pad_w']}"
                f"_d{d['dil']}" + ("_plain" if d["plain"] else "_renorm") + ("_holes" if p["mask"] else "")
                + ("_up" if p["mask_up"] else "") + ("_same" if d["same_holes"] else "")
                + (f"_xcs{p['x_cstride']}" if p["x_cstride"] != d["cin"] else ""))
        if spec["forward_only"] and name in out:   # an inference descriptor that caps to a case tested in every direction
            continue
        out[name] = spec
    return out


HAND_CASES = {
    # dw3 with holes: one msum plane (same_holes) or c planes, stride 1 and 2, dilation 2, 5 x 1 row blocks
    **{f"dw3_holes_{dt}_{'same' if sh else 'perch'}_s{s}_d2": _case(2, 40, 36, 64, 3, s, 2, 2, dt, holes=True, same_holes=sh)
       for dt in ("bf16", "f32") for sh in (True, False) for s in (1, 2)},
    "dw3_holes_half_res_mask": _case(2, 40, 36, 64, 3, 1, 1, 1, "bf16", holes=True, mask_up=1),
    # strided channel views of x, y, dc and dx on every generation
    "dw4_strided_views": _case(2, 33, 45, 64, 3, 1, 2, 2, "bf16", cs=(80, 72, 96, 88)),
    "dw3_strided_views_holes_s2": _case(2, 26, 30, 48, 3, 2, 1, 1, "f32", holes=True, cs=(56, 64, 72, 80)),
    "generic_k5_strided_views": _case(1, 20, 22, 32, 5, 1, 2, 1, "bf16", holes=True, cs=(40, 48, 56, 64)),
    # awkward channel counts: c 296 (37 vectors: dw3 falls back to 32-wide chunks, the last with 5; dw4 cq 2),
    # c 40 (dw3 cvb 5 x pl 51; dw4 cq 10 x xt 25, three x tiles, two row segments), c 8, c 2048 (the largest eligible)
    "dw3_c296_s2": _case(2, 30, 34, 296, 3, 2, 1, 1, "bf16"),
    "dw4_c296": _case(1, 37, 41, 296, 3, 1, 1, 1, "bf16"),
    "dw3_c40_holes": _case(2, 29, 70, 40, 3, 1, 1, 1, "bf16", holes=True),
    "dw4_c40": _case(2, 45, 60, 40, 3, 1, 1, 1, "bf16"),
    "dw4_c8_w300": _case(2, 34, 300, 8, 3, 1, 1, 1, "bf16"),
    "dw3_c8_holes_s2": _case(2, 21, 23, 8, 3, 2, 1, 1, "f32", holes=True),
    "dw4_c2048": _case(2, 10, 12, 2048, 3, 1, 2, 2, "bf16"),
    "dw3_c2048_holes_s2": _case(1, 9, 11, 2048, 3, 2, 1, 1, "bf16", holes=True, same_holes=True),
    "generic_k5_c2048": _case(1, 7, 9, 2048, 5, 1, 2, 1, "bf16"),
    # dw4 edges: the fp32 template (3-row load queue) with three row segments (the last 6 rows) and a ragged x tile; phases
    # of unequal length with 4 phases per block; dilation >= h (phases of 0 or 1 rows); w < 256 / cq; h = 1; w = 1
    "dw4_f32_nseg3_ragged_x": _case(2, 70, 40, 64, 3, 1, 1, 1, "f32"),
    "dw4_f32_h60_d8_ppb4_ragged_x": _case(2, 60, 40, 64, 3, 1, 8, 8, "f32"),
    "dw4_h60_d8_ppb4": _case(2, 60, 40, 128, 3, 1, 8, 8, "bf16"),
    "dw4_12x12_d29": _case(2, 12, 12, 64, 3, 1, 29, 29, "bf16"),
    "dw4_f32_12x12_d16_ppb16": _case(2, 12, 12, 32, 3, 1, 16, 16, "f32"),
    "dw4_w5": _case(2, 40, 5, 64, 3, 1, 1, 1, "bf16"),
    "dw4_h1": _case(2, 1, 50, 64, 3, 1, 1, 1, "bf16"),
    "dw4_w1_d2": _case(2, 50, 1, 64, 3, 1, 2, 2, "bf16"),
    "dw4_f32_1x1": _case(2, 1, 1, 64, 3, 1, 1, 1, "f32"),
    # a "valid" 3x3 at stride 1 (padding != dilation) runs on dw3
    "dw3_valid_s1": _case(2, 20, 22, 64, 3, 1, 0, 1, "bf16"),
    # the generic kernels: 25 and 49 taps, kh != kw with pad_h != pad_w, and a 3x3 at stride 3
    "generic_k5_holes": _case(2, 23, 29, 48, 5, 1, 2, 1, "bf16", holes=True),
    "generic_k7_s2_f32": _case(2, 30, 26, 24, 7, 2, 3, 1, "f32"),
    "generic_k3x5_p1x2_holes_same": _case(2, 19, 21, 32, (3, 5), 1, (1, 2), 1, "bf16", holes=True, same_holes=True),
    "generic_k5x3_p4x2_d2_f32": _case(2, 24, 20, 16, (5, 3), 1, (4, 2), 2, "f32"),
    "s3_generic_holes": _case(2, 25, 28, 32, 3, 3, 1, 1, "bf16", holes=True),
}
CASES = {**_fixture_cases(), **HAND_CASES}


class _Problem:
    """one depthwise problem: the descriptor, the hole plane and the fp64 reference helpers"""

    def __init__(self, sp, dev, gen):
        self.sp, self.dev = sp, dev
        n, h, w, c = sp["n"], sp["h"], sp["w"], sp["c"]
        self.dtype, code = DTYPES[sp["dtype"]]
        self.ho = (h + 2 * sp["ph"] - sp["dil"] * (sp["kh"] - 1) - 1) // sp["s"] + 1
        self.wo = (w + 2 * sp["pw"] - sp["dil"] * (sp["kw"] - 1) - 1) // sp["s"] + 1
        self.taps = sp["kh"] * sp["kw"]
        self.mg = 1 if sp["same_holes"] else c
        if sp["holes"]:
            mu = sp["mask_up"]
            self.mask = holes(n, h >> mu, w >> mu, gen).to(dev)
            m = self.mask.double()
            if mu:
                m = m.repeat_interleave(2, 1).repeat_interleave(2, 2)
        else:
            self.mask = None
            m = torch.ones(n, h, w, dtype=torch.float64, device=dev)
        self.M = m[:, None]                                           # [n, 1, h, w]
        self.ones = torch.ones(1, 1, sp["kh"], sp["kw"], dtype=torch.float64, device=dev)
        cv = _lib.Conv()
        cv.n, cv.h, cv.w, cv.cin, cv.cout, cv.kh, cv.kw = n, h, w, c, c, sp["kh"], sp["kw"]
        cv.stride, cv.pad_h, cv.pad_w, cv.dil, cv.groups, cv.ho, cv.wo = sp["s"], sp["ph"], sp["pw"], sp["dil"], c, self.ho, self.wo
        cv.dtype, cv.same_holes, cv.no_guard, cv.plain, cv.force_generic, cv.nparts = code, int(sp["same_holes"]), 0, int(sp["plain"]), 0, 1
        cv.parts[0].mask = self.mask.data_ptr() if self.mask is not None else None
        cv.parts[0].c, cv.parts[0].x_cstride, cv.parts[0].x_up, cv.parts[0].mask_up = c, sp["cs"][0], 0, sp["mask_up"]
        self.conv = cv
        self.geo = dict(stride=sp["s"], padding=(sp["ph"], sp["pw"]), dilation=sp["dil"])
        with torch.backends.cudnn.flags(enabled=False):
            ones = torch.ones(1, 1, sp["kh"], sp["kw"], dtype=torch.float64, device=dev)
            box = F.conv2d(self.M, ones, **self.geo).round()          # [n, 1, ho, wo]
        self.msum = box * (c if sp["same_holes"] else 1)              # the renormaliser s of every channel

    def set_x(self, x):
        """x: [n, h, w, c] values; HOLE_VALUE under the holes, the sentinel past c"""
        if self.mask is not None:
            x = torch.where(self.M[:, 0, :, :, None] == 0, torch.full_like(x, HOLE_VALUE), x)
        self.x = strided(x.shape, self.sp["cs"][0], x.to(self.dtype), self.dtype)
        self.conv.parts[0].x = self.x.data_ptr()
        self.XM = None if self.sp["forward_only"] else nchw(self.x, self.sp["c"]) * self.M

    def bands(self):
        """output row ranges of at most BAND_BYTES in the eight fp64 [n, c, rows, wo] slabs the Gaussian checks hold at once"""
        rows = max(1, min(self.ho, BAND_BYTES // (8 * 8 * self.sp["n"] * self.wo * self.sp["c"])))
        return [(r, min(r + rows, self.ho)) for r in range(0, self.ho, rows)]

    def band(self, r0, r1):
        """x * m over the input rows that output rows [r0, r1) read, zero rows past the image (conv_band pads only in w)"""
        sp = self.sp
        a = r0 * sp["s"] - sp["ph"]
        b = (r1 - 1) * sp["s"] - sp["ph"] + sp["dil"] * (sp["kh"] - 1) + 1
        lo, hi = max(a, 0), min(b, sp["h"])
        return F.pad(nchw(self.x[:, lo:hi], sp["c"]) * self.M[:, :, lo:hi], (0, 0, lo - a, b - hi))

    def conv_band(self, a, b):
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            return F.conv2d(a, b, groups=sp["c"], stride=sp["s"], padding=(0, sp["pw"]), dilation=sp["dil"])

    def prepare_weights(self, wm, stream, lib):
        fe, de = ctypes.c_size_t(), ctypes.c_size_t()
        lib.pcb_conv_weight_layout(ctypes.byref(self.conv), ctypes.byref(fe), ctypes.byref(de))
        assert fe.value == self.sp["c"] * self.taps and de.value == 0
        self.w_t = torch.empty(fe.value, dtype=self.dtype, device=self.dev)
        _lib.check(lib.pcb_conv_weight_prepare(ctypes.byref(self.conv), wm.data_ptr(), self.w_t.data_ptr(), None, stream))
        self.W = wm.to(self.dtype).double().reshape(self.sp["c"], 1, self.sp["kh"], self.sp["kw"])

    def conv_ref(self, a, b):
        with torch.backends.cudnn.flags(enabled=False):
            return F.conv2d(a, b, groups=self.sp["c"], **self.geo)

    def dgrad_ref(self, g, b):
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            return conv2d_input((sp["n"], sp["c"], sp["h"], sp["w"]), b, g, groups=sp["c"], **self.geo)

    def wgrad_ref(self, a, g):
        sp = self.sp
        with torch.backends.cudnn.flags(enabled=False):
            r = conv2d_weight(a, (sp["c"], 1, sp["kh"], sp["kw"]), g, groups=sp["c"], **self.geo)
        return r.reshape(sp["c"], self.taps)

    def new_y(self):
        return strided((self.sp["n"], self.ho, self.wo, self.sp["c"]), self.sp["cs"][1], float("nan"), self.dtype)

    def new_dc(self, vals):
        return strided(vals.shape, self.sp["cs"][2], vals.to(self.dtype), self.dtype)

    def new_dx(self):
        return strided((self.sp["n"], self.sp["h"], self.sp["w"], self.sp["c"]), self.sp["cs"][3], float("nan"), self.dtype)


@pytest.mark.parametrize("name", sorted(CASES))
def test_dwconv_vs_fp64(name):
    sp = CASES[name]
    dev = torch.device("cuda:0")
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    dgen = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    n, h, w, c = sp["n"], sp["h"], sp["w"], sp["c"]
    P = _Problem(sp, dev, gen)
    torch.cuda.reset_peak_memory_stats(dev)          # (the peak still counts what is allocated now)
    cref = ctypes.byref(P.conv)
    ho, wo, N, dt = P.ho, P.wo, sp["n"] * P.ho * P.wo, P.dtype
    ycs, dcs, dxcs = sp["cs"][1:]
    assert lib.pcb_conv_uses_tensor_cores(cref) == 0 and lib.pcb_pconv_workspace(cref) == 0
    fuses = lib.pcb_conv_fuses_bn_stats(cref)
    assert fuses == lib.pcb_conv_fuses_affine_act(cref) == int(sp["route"][0] != "generic"), f"{name}: fused-epilogue query"

    def ints(*shape):
        return torch.randint(-INT_RANGE, INT_RANGE + 1, shape, generator=dgen, device=dev).to(torch.float32)

    if sp["forward_only"]:
        _forward_only_checks(name, sp, P, lib, stream, ints, dgen, fuses)
        return

    # ================= integer regime: bit-exact
    P.set_x(ints(n, h, w, c))
    P.prepare_weights(ints(c, P.taps), stream, lib)
    bias = torch.randint(-16, 17, (c,), generator=dgen, device=dev).to(torch.float32) / 8
    dcv = ints(n, ho, wo, c)
    dc = P.new_dc(dcv)
    y, dx = P.new_y(), P.new_dx()
    msum = torch.full((P.mg, N), float("nan"), device=dev)
    newmask = torch.full((P.mg, N), 77, dtype=torch.uint8, device=dev)
    dw = torch.full((c, P.taps), float("nan"), device=dev)
    dw0 = ints(c, P.taps)
    dw_acc = dw0.clone()
    state = [(y, y.clone()), (dx, dx.clone()), (msum, float("nan")), (newmask, 77), (dw, float("nan")), (dw_acc, dw0)]

    def run():
        _lib.check(lib.pcb_pconv_forward(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                         newmask.data_ptr(), None, stream))
        _lib.check(lib.pcb_pconv_backward_data(cref, dc.data_ptr(), dcs, P.w_t.data_ptr(), None, (ctypes.c_void_p * 1)(dx.data_ptr()),
                                               (ctypes.c_int32 * 1)(dxcs), stream))
        _lib.check(lib.pcb_pconv_backward_weight(cref, dc.data_ptr(), dcs, dw.data_ptr(), None, stream))
        _lib.check(lib.pcb_pconv_backward_weight_acc(cref, dc.data_ptr(), dcs, dw_acc.data_ptr(), None, stream))

    want = {KERNELS[r][i] for i, r in enumerate(sp["route"])}

    def y_tail_kept(y):
        """channels past c (a multiple of 8) keep the sentinel; the generic forward may zero them instead"""
        past = y[..., c:]
        return bool(((past == SENTINEL) | ((past == 0) & (sp["route"][0] == "generic"))).all())

    def check(records):
        ran = {k for k, _ in records if k.startswith(("dw", "generic"))}
        assert ran == want, f"{name}: ran {sorted(ran)}, the case covers {sorted(want)}"
    records = traced(name, run, check, state)
    print(f"{name}: kernels {sorted(records or {})}")

    # mask pass
    if sp["plain"]:
        assert bool(msum.isnan().all()) and bool((newmask == 77).all()), f"{name}: a plain convolution must not touch msum / newmask"
    else:
        s_ref = P.msum[:, 0].reshape(1, N).expand(P.mg, N)
        assert_bitwise(f"{name}: msum", msum.double(), s_ref)
        assert_bitwise(f"{name}: newmask", newmask, (s_ref != 0).to(torch.uint8))

    # forward: fl(S + b) or fl(fl(S / s) + b)
    S = P.conv_ref(P.XM, P.W).round()
    b = bias.double()[None, :, None, None]
    if sp["plain"]:
        v = (S + b).float()
    else:
        s = P.msum
        q = (S / torch.where(s == 0, torch.ones_like(s), s)).float().double()
        v = torch.where(s == 0, torch.zeros_like(S), q + b).float()
    assert_bitwise(f"{name}: forward", y[..., :c].permute(0, 3, 1, 2), v.to(dt))
    assert y_tail_kept(y), f"{name}: forward wrote past c"

    # data gradient: m * S, zero under the holes
    G = nchw(dc, c)
    gx = (P.dgrad_ref(G, P.W).round() * P.M).float()
    got = dx[..., :c].permute(0, 3, 1, 2)
    assert_bitwise(f"{name}: data gradient", got, gx.to(dt))
    assert bool((got.float() * (P.M == 0) == 0).all()), f"{name}: data gradient under the holes"
    assert sentinel_kept(dx, c), f"{name}: data gradient wrote past c"

    # weight gradient: S, and fl(dw0 + S) accumulating
    gw = P.wgrad_ref(P.XM, G).round()
    assert float(P.wgrad_ref(P.XM.abs(), G.abs()).max()) < 2 ** 24, f"{name}: partial sums could round: not an exact case"
    assert_bitwise(f"{name}: weight gradient", dw, gw.float())
    assert_bitwise(f"{name}: weight gradient (accumulating)", dw_acc, (dw0.double() + gw).float())
    assert sentinel_kept(P.x, c) and sentinel_kept(dc, c)

    # ================= Gaussian regime: error bounds
    P.set_x(torch.randn(n, h, w, c, generator=dgen, device=dev))
    P.prepare_weights(torch.randn(c, P.taps, generator=dgen, device=dev) / 3, stream, lib)
    bias = torch.randn(c, generator=dgen, device=dev) * 0.1
    b = bias.double()[None, :, None, None]
    acc = P.conv_ref(P.XM, P.W)
    e_acc = P.conv_ref((P.XM != 0).double(), (P.W != 0).double()) * 2.0 ** -22 * P.conv_ref(P.XM.abs(), P.W.abs())
    s = P.msum if not sp["plain"] else torch.ones_like(P.msum)
    empty = (s == 0).expand_as(acc)
    safe = torch.where(s == 0, torch.ones_like(s), s)
    v_ref = torch.where(empty, torch.zeros_like(acc), acc / safe + b)
    e_ref = torch.where(empty, torch.zeros_like(acc), e_acc / safe + 2.0 ** -22 * (acc.abs() / safe + v_ref.abs()))
    del acc, e_acc
    store = 2.0 ** -8 if dt == torch.bfloat16 else 0.0

    def check_y(tag, y, v, e):
        assert y_tail_kept(y), f"{name}: {tag} wrote past c"
        assert_within(f"{name}: {tag}", nchw(y, c), v, e + store * (v.abs() + e))

    scale = torch.rand(c, generator=dgen, device=dev) + 0.5
    shift = torch.randn(c, generator=dgen, device=dev) * 0.1
    if fuses:
        y = P.new_y()
        sums = torch.zeros(2, c, dtype=torch.float64, device=dev)
        _lib.check(lib.pcb_pconv_forward_bn(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                            newmask.data_ptr(), None, 0, sums.data_ptr(), stream))
        torch.cuda.synchronize()
        check_y("forward with BatchNorm sums", y, v_ref, e_ref)
        yv = y[..., :c].double().reshape(-1, c)
        for row, vals in ((0, yv), (1, yv * yv)):
            tol = yv.shape[0] * 2.0 ** -23 * vals.abs().sum(0)
            assert bool(((sums[row] - vals.sum(0)).abs() <= tol).all()), f"{name}: BatchNorm {'sums' if row == 0 else 'squares'}"
        sc, sh = scale.double()[None, :, None, None], shift.double()[None, :, None, None]
        z = v_ref * sc + sh
        ez = sc * e_ref + 2.0 ** -23 * (z.abs() + sh.abs())
        for act in ACTS:
            y = P.new_y()
            _lib.check(lib.pcb_pconv_forward_affine_act(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                                        newmask.data_ptr(), None, 0, scale.data_ptr(), shift.data_ptr(), act, SLOPE,
                                                        stream))
            torch.cuda.synchronize()
            va = act_ref(z, act, SLOPE)
            check_y(f"eval epilogue, activation {act}", y, va, ez + 2.0 ** -23 * va.abs())
    else:
        y = P.new_y()
        sums = torch.zeros(2, c, dtype=torch.float64, device=dev)
        rc = lib.pcb_pconv_forward_bn(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                      newmask.data_ptr(), None, 0, sums.data_ptr(), stream)
        assert rc != 0 and b"does not fuse" in lib.pcb_last_error(), f"{name}: fused BatchNorm sums must be refused"
        rc = lib.pcb_pconv_forward_affine_act(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                              newmask.data_ptr(), None, 0, scale.data_ptr(), shift.data_ptr(), _lib.ACT_RELU, SLOPE,
                                              stream)
        assert rc != 0 and b"does not apply" in lib.pcb_last_error(), f"{name}: fused affine + activation must be refused"
        torch.cuda.synchronize()
        assert bool(y[..., :c].isnan().all()) and bool((sums == 0).all()), f"{name}: a refused call must not run"

    if dt == torch.float32:                      # fp32 storage: products are rounded, the integer regime alone is not enough
        y = P.new_y()
        _lib.check(lib.pcb_pconv_forward(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                         newmask.data_ptr(), None, stream))
        dc = P.new_dc(torch.randn(n, ho, wo, c, generator=dgen, device=dev))
        dx = P.new_dx()
        _lib.check(lib.pcb_pconv_backward_data(cref, dc.data_ptr(), dcs, P.w_t.data_ptr(), None, (ctypes.c_void_p * 1)(dx.data_ptr()),
                                               (ctypes.c_int32 * 1)(dxcs), stream))
        dw = torch.full((c, P.taps), float("nan"), device=dev)
        _lib.check(lib.pcb_pconv_backward_weight(cref, dc.data_ptr(), dcs, dw.data_ptr(), None, stream))
        torch.cuda.synchronize()
        check_y("fp32 forward", y, v_ref, e_ref)
        G = nchw(dc, c)
        gref = P.dgrad_ref(G, P.W) * P.M
        gb = P.dgrad_ref((G != 0).double(), (P.W != 0).double()) * 2.0 ** -22 * P.dgrad_ref(G.abs(), P.W.abs()) * P.M
        assert_within(f"{name}: fp32 data gradient", nchw(dx, c), gref, gb)
        assert sentinel_kept(dx, c), f"{name}: data gradient wrote past c"
        wref = P.wgrad_ref(P.XM, G)
        wb = P.wgrad_ref((P.XM != 0).double(), (G != 0).double()) * 2.0 ** -22 * P.wgrad_ref(P.XM.abs(), G.abs())
        assert_within(f"{name}: fp32 weight gradient", dw.double(), wref, wb)


def _forward_only_checks(name, sp, P, lib, stream, ints, dgen, fuses):
    """the checks of a descriptor only inference reaches: the forward kernel in the trace, the mask pass and the forward in
    the integer regime, the fused BatchNorm sums and the eval epilogue at every activation (or their refusal) in the Gaussian
    regime, and the fp32 forward; every fp64 reference and comparison runs band by band (P.bands)"""
    dev, dt = P.dev, P.dtype
    n, c, ho, wo = sp["n"], sp["c"], P.ho, P.wo
    N, ycs = n * ho * wo, sp["cs"][1]
    cref = ctypes.byref(P.conv)
    bands = P.bands()
    P.set_x(ints(n, sp["h"], sp["w"], c))
    P.prepare_weights(ints(c, P.taps), stream, lib)
    bias = torch.randint(-16, 17, (c,), generator=dgen, device=dev).to(torch.float32) / 8
    b = bias.double()[None, :, None, None]
    y = P.new_y()
    msum = torch.full((P.mg, N), float("nan"), device=dev)
    newmask = torch.full((P.mg, N), 77, dtype=torch.uint8, device=dev)

    def run():
        _lib.check(lib.pcb_pconv_forward(cref, P.w_t.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                         newmask.data_ptr(), None, stream))

    def check(records):
        ran = {k for k, _ in records if k.startswith(("dw", "generic"))}
        assert ran == {KERNELS[sp["route"][0]][0]}, f"{name}: ran {sorted(ran)}, the case covers {KERNELS[sp['route'][0]][0]}"
    records = traced(name, run, check, [(y, y.clone()), (msum, float("nan")), (newmask, 77)])
    print(f"{name}: kernels {sorted(records or {})}")

    def y_tail_kept(y):
        past = y[..., c:]
        return bool(((past == SENTINEL) | ((past == 0) & (sp["route"][0] == "generic"))).all())

    if sp["plain"]:
        assert bool(msum.isnan().all()) and bool((newmask == 77).all()), f"{name}: a plain convolution must not touch msum / newmask"
    else:
        s_ref = P.msum[:, 0].reshape(1, N).expand(P.mg, N)
        assert_bitwise(f"{name}: msum", msum.double(), s_ref)
        assert_bitwise(f"{name}: newmask", newmask, (s_ref != 0).to(torch.uint8))
    assert y_tail_kept(y), f"{name}: forward wrote past c"
    for r0, r1 in bands:
        S = P.conv_band(P.band(r0, r1), P.W).round()
        if sp["plain"]:
            v = (S + b).float()
        else:
            s = P.msum[:, :, r0:r1]
            q = (S / torch.where(s == 0, torch.ones_like(s), s)).float().double()
            v = torch.where(s == 0, torch.zeros_like(S), q + b).float()
        assert_bitwise(f"{name}: forward, rows {r0}:{r1}", y[:, r0:r1, :, :c].permute(0, 3, 1, 2), v.to(dt))
        del S, v

    P.set_x(torch.randn(n, sp["h"], sp["w"], c, generator=dgen, device=dev))
    P.prepare_weights(torch.randn(c, P.taps, generator=dgen, device=dev) / 3, stream, lib)
    bias = torch.randn(c, generator=dgen, device=dev) * 0.1
    b = bias.double()[None, :, None, None]
    scale = torch.rand(c, generator=dgen, device=dev) + 0.5
    shift = torch.randn(c, generator=dgen, device=dev) * 0.1
    outs = {}
    sums = torch.zeros(2, c, dtype=torch.float64, device=dev)
    if dt == torch.float32:
        outs["fp32 forward"] = P.new_y()
        _lib.check(lib.pcb_pconv_forward(cref, P.w_t.data_ptr(), bias.data_ptr(), outs["fp32 forward"].data_ptr(), ycs, msum.data_ptr(),
                                         newmask.data_ptr(), None, stream))
    if fuses:
        outs["forward with BatchNorm sums"] = P.new_y()
        _lib.check(lib.pcb_pconv_forward_bn(cref, P.w_t.data_ptr(), bias.data_ptr(), outs["forward with BatchNorm sums"].data_ptr(), ycs,
                                            msum.data_ptr(), newmask.data_ptr(), None, 0, sums.data_ptr(), stream))
        for act in ACTS:
            outs[act] = P.new_y()
            _lib.check(lib.pcb_pconv_forward_affine_act(cref, P.w_t.data_ptr(), bias.data_ptr(), outs[act].data_ptr(), ycs,
                                                        msum.data_ptr(), newmask.data_ptr(), None, 0, scale.data_ptr(), shift.data_ptr(),
                                                        act, SLOPE, stream))
    else:
        yr = P.new_y()
        rc = lib.pcb_pconv_forward_bn(cref, P.w_t.data_ptr(), bias.data_ptr(), yr.data_ptr(), ycs, msum.data_ptr(),
                                      newmask.data_ptr(), None, 0, sums.data_ptr(), stream)
        assert rc != 0 and b"does not fuse" in lib.pcb_last_error(), f"{name}: fused BatchNorm sums must be refused"
        rc = lib.pcb_pconv_forward_affine_act(cref, P.w_t.data_ptr(), bias.data_ptr(), yr.data_ptr(), ycs, msum.data_ptr(),
                                              newmask.data_ptr(), None, 0, scale.data_ptr(), shift.data_ptr(), _lib.ACT_RELU, SLOPE,
                                              stream)
        assert rc != 0 and b"does not apply" in lib.pcb_last_error(), f"{name}: fused affine + activation must be refused"
        torch.cuda.synchronize()
        assert bool(yr[..., :c].isnan().all()) and bool((sums == 0).all()), f"{name}: a refused call must not run"
        del yr
    torch.cuda.synchronize()
    for tag, yo in outs.items():
        assert y_tail_kept(yo), f"{name}: {tag} wrote past c"
    store = 2.0 ** -8 if dt == torch.bfloat16 else 0.0
    sc, sh = scale.double()[None, :, None, None], shift.double()[None, :, None, None]
    tot = torch.zeros(3, c, dtype=torch.float64, device=dev)        # sum y, sum y^2, sum |y| of the stored values
    for r0, r1 in bands:
        XM = P.band(r0, r1)
        acc = P.conv_band(XM, P.W)
        e_acc = P.conv_band((XM != 0).double(), (P.W != 0).double()) * 2.0 ** -22 * P.conv_band(XM.abs(), P.W.abs())
        del XM
        s = P.msum[:, :, r0:r1] if not sp["plain"] else torch.ones_like(P.msum[:, :, r0:r1])
        empty = (s == 0).expand_as(acc)
        safe = torch.where(s == 0, torch.ones_like(s), s)
        v_ref = torch.where(empty, torch.zeros_like(acc), acc / safe + b)
        e_ref = torch.where(empty, torch.zeros_like(acc), e_acc / safe + 2.0 ** -22 * (acc.abs() / safe + v_ref.abs()))
        del acc, e_acc, empty
        rows = f"rows {r0}:{r1}"

        def check_y(tag, v, e):
            assert_within(f"{name}: {tag}, {rows}", nchw(outs[tag][:, r0:r1], c), v, e + store * (v.abs() + e))
        for tag in ("fp32 forward", "forward with BatchNorm sums"):
            if tag in outs:
                check_y(tag, v_ref, e_ref)
        if not fuses:
            continue
        yv = outs["forward with BatchNorm sums"][:, r0:r1, :, :c].double().reshape(-1, c)
        tot += torch.stack([yv.sum(0), (yv * yv).sum(0), yv.abs().sum(0)])
        del yv
        z = v_ref * sc + sh
        ez = sc * e_ref + 2.0 ** -23 * (z.abs() + sh.abs())
        for act in ACTS:
            va = act_ref(z, act, SLOPE)
            check_y(act, va, ez + 2.0 ** -23 * va.abs())
    if fuses:
        for row, what in ((0, "sums"), (1, "squares")):
            tol = N * 2.0 ** -23 * tot[2 if row == 0 else 1]
            assert bool(((sums[row] - tot[row]).abs() <= tol).all()), f"{name}: BatchNorm {what}"
    peak = torch.cuda.max_memory_allocated(dev)
    print(f"{name}: peak device memory {peak / 2 ** 30:.2f} GiB over {len(bands)} band(s)")
    assert peak < MEMORY_BUDGET, f"{name}: peak device memory {peak / 2 ** 30:.2f} GiB"

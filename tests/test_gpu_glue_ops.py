"""The glue kernels of the training step through the C ABI, every element against an fp64 reference of the same stored operands
computed on the device: average pooling, bilinear upsampling, GAP and the scSE gate (seg_ops.cu), channel concat with nearest
2x upsampling, mask-format conversion, the L1-mean loss and SGD (elementwise.cu).  Cases: one per distinct call site of
tests/golden/elementwise_sites.json (the layers of the three training workloads, the eval forward and one optimiser step, at
the recorded size), plus hand cases for the edges production does not reach.  Outputs are prefilled with NaN, and each case
asserts its route from the kernel names (and template arguments) of one complete torch.profiler trace (see
kernel_harness.traced):

    route                 kernel                                  cases
    avgpool fwd / bwd     avgpool_kernel<T, false / true>         avgpool_*, fx_avgpool_*
    bilinear fwd / bwd    bilinear_fwd_kernel, bilinear_bwd_kernel bilinear_*, fx_bilinear_*
    GAP fwd / bwd         gap_kernel, gap_bwd_kernel              gap_*, fx_gap_*
    scSE fwd              scse_fwd_kernel                         scse_*, fx_scse_*
    scSE bwd, 1/2/4 vec   scse_bwd_kernel<T, 1 / 2 / 4>           scse_c<=256 / c<=512 / c<=1024
    concat vector         concat_fwd_kernel<T, 8>, concat_bwd_kernel<T, 8>   concat_* with 8-aligned parts, fx_concat_*
    concat scalar         concat_fwd_kernel<T, 1>, concat_bwd_kernel<T, 1>   concat_scalar_*, concat_misaligned (forward)
    upsample2x            concat_fwd_kernel<T, 8>, concat_bwd_kernel<T, 8>   upsample_*, fx_upsample2x_*
    masks                 mask_from_dense_kernel, mask_to_dense_kernel       mask_*, fx_mask_*
    L1 mean               l1_sum_kernel + l1_finish_kernel, l1_bwd_kernel   l1_*, fx_l1_*
    SGD                   sgd_kernel                              sgd_*, fx_sgd_*

Integer regime: inputs are integers of magnitude <= 4 (exact in bf16), every partial sum far below 2^24, so sums are exact
in fp32 in any order and the kernels' outputs must be BIT-IDENTICAL to the exact result rounded like their last fp32
operations:
  * avgpool: fl(S * fl(1/k^2)) with S the exact window sum (fwd) or covering-output sum (bwd), count_include_pad=True;
  * bilinear at scale 1, 2, 4, 8: every weight is a multiple of 1/(2s), so the forward and the gathered backward are exact;
    at scale 3 the weights round: src = (d + 0.5) / s - 0.5 is off by 2u (|src| + 1), so each weight by as much in absolute
    terms, and each term carries the weights' products and its addition: 8u (max(h, w) + 2) max|x| per term, u = 2^-24;
  * GAP: per block fl(tot * fl(1/hw)), added with fp32 atomics: exact when hw is a power of two, otherwise within
    (chunks + 1) u sum |x| / hw + u |S / hw| (one rounding per block product and per atomic, plus fl(1/hw)); the backward
    (accumulate or not) is o + g * fl(1/hw), accepted in its fused or unfused rounding;
  * scSE backward from a given sse (quarters in (0, 1)) with dyadic cse and ws: dot, dpre = dot sse (1 - sse), dx, dcse and
    dws are all exact (the gradient rows are thinned, asserted, where dws's magnitudes would pass 2^24 units);
  * concat, upsample2x and mask planes are copies or sums of 1 or 4 integers: exact.
Bounds:
  * scSE forward: the dot product of c fp32 products is off by at most (c / gw + log2 gw + 1) u sum |x w|; __expf's maximum
    error is 2 + floor(|1.173 t|) ulp (CUDA C Programming Guide, intrinsic functions) and the sigmoid's add and division round
    once each, so |sse - sigmoid(dot)| <= d_dot / 4 + sse (1 - sse) (2 + |1.173 dot|) 2^-23 + 2u; y must then equal
    fl(x * fl(cse + sse)) of the kernel's own sse exactly;
  * L1 mean: per-thread chains of rows / (grid * 256) additions, a 5-level warp tree and 8 warp partials summed in fp32:
    (rows per thread + 14) u sum |x| / numel, and the final division u |loss|; the backward is exact: fl(sign(x) * gscale);
  * SGD (fp32 state) against torch.optim.SGD evaluated in fp64 on the same values: each product and sum rounds once (3u of
    |g gscale| + |wd p| for d, 2u of |mom buf| + |d| for the momentum buffer, 2u of |d| + |mom buf| for Nesterov, 2u of
    |p| + |lr d| for the update), propagated through the momentum and learning-rate factors.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_harness import assert_bitwise, assert_within, elementwise_sites, nan, nchw, traced
from text_segmentation_image_inpainting_b200 import _lib

U = 2.0 ** -24
BF, F32 = _lib.PCB_BF16, _lib.PCB_F32
DT = {BF: torch.bfloat16, F32: torch.float32}
NAN = float("nan")
FAMILIES = ("avgpool", "bilinear", "gap", "scse", "concat", "upsample2x", "mask", "l1", "sgd")


def _family(fn):
    for f in FAMILIES:
        if fn.startswith(f"pcb_{f}"):
            return f
    return None


def _site_case(s):
    """(family, case name, spec) of a fixture site"""
    fam = _family(s["fn"])
    keys = sorted(k for k in s if k not in ("fn", "parts"))
    if fam in ("avgpool", "bilinear", "upsample2x", "scse", "gap", "l1"):      # forward and backward sites share a case
        keys = [k for k in keys if k not in ("accumulate", "gscale")]
    name = f"fx_{fam}_" + "_".join(f"{k}{s[k]}" for k in keys)
    if "parts" in s:
        name += "_p" + "_".join("x".join(str(v) for v in p) for p in s["parts"])
    return fam, name, dict(s)


def _fixture(fam):
    return {name: sp for f, name, sp in map(_site_case, elementwise_sites()) if f == fam}


def test_fixture_sites_map_to_cases():
    """every non-BatchNorm site of the fixture names exactly one case of one family"""
    sites = [s for s in elementwise_sites() if not s["fn"].startswith("pcb_bn_")]
    assert sites
    for s in sites:
        fam, name, _ = _site_case(s)
        assert fam is not None, f"no test family for {s['fn']}"
        assert name in _fixture(fam) and name not in HAND[fam]


def _route(name, want):
    """the check of traced for want = {(kernel, last template argument or None)}: those kernels ran, and no other"""
    def check(records):
        for k, last in want:
            assert any(r == k and (last is None or args[-1:] == (last,)) for r, args in records), \
                f"{name}: {k}<...{last or ''}> did not run; ran {sorted(records)}"
        assert {r for r, _ in records} == {k for k, _ in want}, f"{name}: ran {sorted(records)}, the case covers {sorted(want)}"
    return check


def _gen(name):
    return torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))


def _ints(gen, *shape, lo=-4, hi=4):
    return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda").double()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ hand cases
def _pool(dt, n, h, w, c, k, s, p):
    return dict(dtype=dt, n=n, h=h, w=w, c=c, k=k, stride=s, pad=p)


def _bil(dt, n, h, w, c, s):
    return dict(dtype=dt, n=n, h=h, w=w, c=c, scale=s)


def _nhw(dt, n, hw, c):
    return dict(dtype=dt, n=n, hw=hw, c=c)


HAND = {
    "avgpool": {
        "avgpool_k3s2p1_odd": _pool(BF, 2, 37, 41, 64, 3, 2, 1), "avgpool_k3s2p1_f32_c8": _pool(F32, 3, 17, 9, 8, 3, 2, 1),
        **{f"avgpool_asp_r{r}": _pool(BF, 2, 23, 19, 32, r, 1, (r - 1) // 2) for r in (3, 5, 9)},
        "avgpool_h_lt_k": _pool(BF, 2, 3, 12, 16, 5, 1, 2), "avgpool_w_lt_k_s2": _pool(F32, 2, 11, 2, 8, 3, 2, 1),
        "avgpool_c2048": _pool(BF, 1, 9, 7, 2048, 3, 2, 1), "avgpool_k9_1x1": _pool(BF, 2, 1, 1, 24, 9, 1, 4),
    },
    "bilinear": {
        **{f"bilinear_s{s}": _bil(BF, 2, 13, 11, 16, s) for s in (1, 2, 4, 8)},
        "bilinear_s3": _bil(F32, 2, 9, 7, 8, 3), "bilinear_s4_h1": _bil(BF, 2, 1, 9, 8, 4), "bilinear_s2_w1": _bil(F32, 2, 7, 1, 8, 2),
        "bilinear_s4_1x1": _bil(BF, 3, 1, 1, 24, 4), "bilinear_s4_odd_f32": _bil(F32, 1, 15, 17, 32, 4),
        "bilinear_s8_c2048": _bil(BF, 1, 3, 5, 2048, 8),
    },
    "gap": {
        "gap_hw1": _nhw(BF, 5, 1, 64), "gap_hw4093_c8": _nhw(F32, 3, 4093, 8), "gap_hw1000_c2048": _nhw(BF, 2, 1000, 2048),
        "gap_hw4096_c24": _nhw(BF, 4, 4096, 24), "gap_n600_hw37": _nhw(BF, 600, 37, 128), "gap_hw65537_c16": _nhw(F32, 2, 65537, 16),
    },
    "scse": {
        **{f"scse_c{c}": _nhw(BF, 2, 999, c) for c in (8, 16, 24, 64, 256, 264, 512, 520, 1024)},
        "scse_f32_c40_hw1": _nhw(F32, 7, 1, 40), "scse_n600_bps1": _nhw(BF, 600, 50, 64), "scse_refuse_c1032": _nhw(BF, 2, 64, 1032),
    },
    "concat": {
        "concat_two_vec": dict(dtype=BF, n=2, h=12, w=10, parts=[[64, 64, 0], [32, 32, 0]]),
        "concat_8_parts_up": dict(dtype=BF, n=2, h=8, w=6, parts=[[8, 8, 0], [16, 24, 1], [8, 8, 0], [24, 32, 1], [8, 16, 0], [16, 16, 0],
                                                                   [32, 32, 1], [8, 8, 0]]),
        "concat_strided_f32": dict(dtype=F32, n=2, h=6, w=10, parts=[[16, 40, 0], [8, 16, 1]]),
        "concat_scalar_c3": dict(dtype=BF, n=2, h=6, w=8, parts=[[3, 3, 0], [5, 8, 1], [8, 8, 0]]),
        "concat_scalar_f32_c12": dict(dtype=F32, n=1, h=4, w=4, parts=[[12, 12, 0], [4, 4, 1]]),
        "concat_misaligned": dict(dtype=BF, n=2, h=6, w=6, parts=[[16, 16, 0], [8, 8, 0]], misalign=1),
        "concat_null_grad": dict(dtype=BF, n=2, h=8, w=8, parts=[[16, 16, 0], [32, 32, 1], [8, 8, 0]], null=[1]),
        "concat_null_grad_scalar": dict(dtype=F32, n=2, h=4, w=6, parts=[[3, 3, 0], [13, 13, 1]], null=[0]),
    },
    "upsample2x": {"upsample_c8": dict(dtype=BF, n=2, h=5, w=3, c=8), "upsample_f32_c64": dict(dtype=F32, n=1, h=7, w=9, c=64)},
    "mask": {"mask_up_c0": dict(n=2, h=12, w=10, c=3, up=1, ctot=7, c0=2), "mask_plain": dict(n=3, h=9, w=11, c=1, up=0, ctot=1, c0=0),
             "mask_from_dense_c3": dict(n=2, h=5, w=7, c=3)},
    "l1": {"l1_bf16_odd": dict(dtype=BF, numel=1000003), "l1_f32_small": dict(dtype=F32, numel=17)},
    "sgd": {
        "sgd_mom0": dict(numel=100003, lr=0.01, momentum=0.0, weight_decay=0.0, nesterov=0, first_step=1, grad_scale=1.0),
        "sgd_mom0_wd": dict(numel=1000, lr=0.1, momentum=0.0, weight_decay=1e-3, nesterov=0, first_step=0, grad_scale=0.5),
        "sgd_first_plain": dict(numel=5000, lr=0.02, momentum=0.9, weight_decay=0.0, nesterov=0, first_step=1, grad_scale=1.0),
        "sgd_later_plain": dict(numel=5000, lr=0.02, momentum=0.9, weight_decay=1e-4, nesterov=0, first_step=0, grad_scale=1.0),
        "sgd_later_nesterov_scaled": dict(numel=77777, lr=2e-4, momentum=0.9, weight_decay=1e-4, nesterov=1, first_step=0,
                                          grad_scale=0.25),
    },
}


def _cases(fam):
    return {**_fixture(fam), **HAND[fam]}


# ------------------------------------------------------------------------------------------------ avgpool
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("avgpool")))
def test_avgpool_vs_fp64(name):
    sp = _cases("avgpool")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    dt, n, h, w, c, k, s, p = DT[sp["dtype"]], sp["n"], sp["h"], sp["w"], sp["c"], sp["k"], sp["stride"], sp["pad"]
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    x = _ints(gen, n, h, w, c).to(dt)
    gy = _ints(gen, n, ho, wo, c).to(dt)
    y, gx = nan(n, ho, wo, c, dtype=dt), nan(n, h, w, c, dtype=dt)
    traced(name, lambda: (_lib.check(lib.pcb_avgpool_forward(x.data_ptr(), y.data_ptr(), sp["dtype"], n, h, w, c, k, s, p, st)),
                          _lib.check(lib.pcb_avgpool_backward(gy.data_ptr(), gx.data_ptr(), sp["dtype"], n, h, w, c, k, s, p, st))),
            _route(name, {("avgpool_kernel", "false"), ("avgpool_kernel", "true")}), [(y, NAN), (gx, NAN)])
    inv = torch.tensor(1.0 / (k * k), dtype=torch.float32).double().item()     # fl(1/k^2): 1.0f / (float)(k*k)
    S = F.avg_pool2d(nchw(x), k, s, p, count_include_pad=True, divisor_override=1)
    # backward: scatter every output's gradient over its window in padded coordinates (output o, tap a -> row o s + a)
    G = nchw(gy)
    hp, wp = max((ho - 1) * s + k, p + h), max((wo - 1) * s + k, p + w)
    acc = torch.zeros(n, c, hp, wp, dtype=torch.float64, device="cuda")
    for a in range(k):
        for b in range(k):
            acc[:, :, a:a + (ho - 1) * s + 1:s, b:b + (wo - 1) * s + 1:s] += G
    Sb = acc[:, :, p:p + h, p:p + w]
    assert_bitwise(f"{name}: forward", nchw(y), (S * inv).float().to(dt).double())
    assert_bitwise(f"{name}: backward", nchw(gx), (Sb * inv).float().to(dt).double())


# ------------------------------------------------------------------------------------------------ bilinear
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("bilinear")))
def test_bilinear_vs_fp64(name):
    sp = _cases("bilinear")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    dt, n, h, w, c, s = DT[sp["dtype"]], sp["n"], sp["h"], sp["w"], sp["c"], sp["scale"]
    x = _ints(gen, n, h, w, c).to(dt)
    gy = _ints(gen, n, h * s, w * s, c).to(dt)
    y, gx = nan(n, h * s, w * s, c, dtype=dt), nan(n, h, w, c, dtype=dt)
    traced(name, lambda: (_lib.check(lib.pcb_bilinear_forward(x.data_ptr(), y.data_ptr(), sp["dtype"], n, h, w, c, s, st)),
                          _lib.check(lib.pcb_bilinear_backward(gy.data_ptr(), gx.data_ptr(), sp["dtype"], n, h, w, c, s, st))),
            _route(name, {("bilinear_fwd_kernel", None), ("bilinear_bwd_kernel", None)}), [(y, NAN), (gx, NAN)])
    xr = nchw(x).requires_grad_(True)
    Y = F.interpolate(xr, scale_factor=s, mode="bilinear", align_corners=False)
    G, = torch.autograd.grad(Y, xr, nchw(gy))
    if s & (s - 1) == 0:
        assert_bitwise(f"{name}: forward", nchw(y), Y.detach().float().to(dt).double())
        assert_bitwise(f"{name}: backward", nchw(gx), G.float().to(dt).double())
    else:
        store = 2.0 ** -8 if dt == torch.bfloat16 else 0.0
        # a weight 1 - l or l is off by 2u (|src| + 1) in absolute terms, src < max(h, w), whatever its size; with the
        # products and the additions each term is off by at most 8u (max(h, w) + 2) |x|, |x| <= 4: 4 terms per output
        # forward, at most (2 s + 2)^2 per input backward
        wb = 8 * U * (max(h, w) + 2) * 4
        assert_within(f"{name}: forward", nchw(y), Y.detach(), 4 * wb + store * Y.detach().abs())
        assert_within(f"{name}: backward", nchw(gx), G, (2 * s + 2) ** 2 * wb + store * G.abs())


# ------------------------------------------------------------------------------------------------ GAP
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("gap")))
def test_gap_vs_fp64(name):
    sp = _cases("gap")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    dt, n, hw, c = DT[sp["dtype"]], sp["n"], sp["hw"], sp["c"]
    x = _ints(gen, n, hw, c).to(dt)
    g = _ints(gen, n, c).float()
    dx0 = _ints(gen, n, hw, c).to(dt)
    out, dx, dxa = nan(n, c), nan(n, hw, c, dtype=dt), dx0.clone()
    traced(name, lambda: (_lib.check(lib.pcb_gap_forward(x.data_ptr(), sp["dtype"], n, hw, c, out.data_ptr(), st)),
                          _lib.check(lib.pcb_gap_backward(g.data_ptr(), dx.data_ptr(), sp["dtype"], n, hw, c, 0, st)),
                          _lib.check(lib.pcb_gap_backward(g.data_ptr(), dxa.data_ptr(), sp["dtype"], n, hw, c, 1, st))),
            _route(name, {("gap_kernel", None), ("gap_bwd_kernel", None)}), [(out, NAN), (dx, NAN), (dxa, dx0)])
    inv32 = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(hw), dtype=torch.float32)
    inv = float(inv32)
    S = x.double().sum(1)
    if hw & (hw - 1) == 0:
        assert_bitwise(f"{name}: forward", out.double(), S * inv)
    else:
        rpb = 256 // (c // 8)
        nsm = torch.cuda.get_device_properties(0).multi_processor_count
        chunks = max(1, min(math.ceil(hw / (rpb * 8)), max(1, 4 * nsm // n)))
        assert_within(f"{name}: forward", out, S / hw, (chunks + 1) * U * x.double().abs().sum(1) / hw + 2 * U * (S / hw).abs())
    gi = (g.double() * inv)[:, None, :]
    assert_bitwise(f"{name}: backward", dx, gi.float().expand(n, hw, c).to(dt))
    unf = (dx0.float() + (g * inv32.cuda())[:, None, :])
    fus = (dx0.double() + gi).float()
    assert_bitwise(f"{name}: backward (accumulate)", dxa, unf.to(dt), fus.to(dt))


# ------------------------------------------------------------------------------------------------ scSE
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("scse")))
def test_scse_vs_fp64(name):
    sp = _cases("scse")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    dt, n, hw, c = DT[sp["dtype"]], sp["n"], sp["hw"], sp["c"]
    npix = n * hw
    x = _ints(gen, npix, c).to(dt)
    cse = (_ints(gen, n, c, lo=0, hi=8) / 8).float()
    ws = (_ints(gen, c) / 8).float()
    sse = (_ints(gen, npix, lo=1, hi=3) / 4).float()
    gy = _ints(gen, npix, c)
    x64 = x.double()
    dpre_w = (gy * x64).sum(1) * (sse.double() * (1 - sse.double()))
    tot = float((x64.abs() * dpre_w.abs()[:, None]).sum(0).max()) * 16
    if tot >= 2 ** 23:                                                  # thin the gradient rows: dws stays exact
        gy = gy * (torch.rand(npix, 1, generator=gen, device="cuda") < 2 ** 22 / tot)
    gy = gy.to(dt)
    g64 = gy.double()
    y, sse_out = nan(npix, c, dtype=dt), nan(npix)
    dx, dcse, dws = nan(npix, c, dtype=dt), nan(n, c), nan(c)
    if c > 1024:                                                        # refused before anything is written or launched
        before = _lib.launch_count()
        assert lib.pcb_scse_backward(gy.data_ptr(), x.data_ptr(), cse.data_ptr(), ws.data_ptr(), sse.data_ptr(), dx.data_ptr(),
                                     dcse.data_ptr(), dws.data_ptr(), sp["dtype"], n, hw, c, st) != 0
        torch.cuda.synchronize()
        assert _lib.launch_count() == before and b"at most 1024" in lib.pcb_last_error()
        assert bool(dcse.isnan().all()) and bool(dws.isnan().all()) and bool(dx.isnan().all()), f"{name}: a refused call wrote"
        return
    vm = 1 if c <= 256 else (2 if c <= 512 else 4)
    traced(name, lambda: (_lib.check(lib.pcb_scse_forward(x.data_ptr(), cse.data_ptr(), ws.data_ptr(), y.data_ptr(), sse_out.data_ptr(),
                                                          sp["dtype"], n, hw, c, st)),
                          _lib.check(lib.pcb_scse_backward(gy.data_ptr(), x.data_ptr(), cse.data_ptr(), ws.data_ptr(), sse.data_ptr(),
                                                           dx.data_ptr(), dcse.data_ptr(), dws.data_ptr(), sp["dtype"], n, hw, c, st))),
            _route(name, {("scse_fwd_kernel", None), ("scse_bwd_kernel", str(vm))}),
            [(y, NAN), (sse_out, NAN), (dx, NAN), (dcse, NAN), (dws, NAN)])
    # forward: sse within the __expf bound, y exact given the kernel's sse
    cse_p = cse.repeat_interleave(hw, 0)                                # [npix, c]
    dot = x64 @ ws.double()
    cv = c // 8
    gw = 1
    while gw < cv and gw < 32:
        gw *= 2
    d_dot = (c / gw + math.log2(gw) + 1) * U * (x64.abs() @ ws.double().abs())
    ref = torch.sigmoid(dot)
    bound = d_dot / 4 + ref * (1 - ref) * (2 + (1.173 * dot).abs().floor()) * 2.0 ** -23 + 2 * U
    assert_within(f"{name}: sse", sse_out, ref, bound)
    assert_bitwise(f"{name}: forward y", y, (x.float() * (cse_p + sse_out[:, None])).to(dt))
    # backward from the given sse: exact
    s64 = sse.double()[:, None]
    dpre = (g64 * x64).sum(1, keepdim=True) * s64 * (1 - s64)
    assert_bitwise(f"{name}: dx", dx, (g64 * (cse_p.double() + s64) + ws.double() * dpre).float().to(dt))
    assert_bitwise(f"{name}: dcse", dcse, (g64 * x64).reshape(n, hw, c).sum(1).float())
    assert_bitwise(f"{name}: dws", dws, (x64 * dpre).sum(0).float())


# ------------------------------------------------------------------------------------------------ concat / upsample2x
def _concat_case(sp, name, lib):
    gen, st = _gen(name), _st()
    code, dt, n, h, w = sp["dtype"], DT[sp["dtype"]], sp["n"], sp["h"], sp["w"]
    parts = sp["parts"]
    np_ = len(parts)
    ctot = sum(p[0] for p in parts)
    bufs, views, arr = [], [], (_lib.Part * np_)()
    off = 0
    for i, (c, cs, up) in enumerate(parts):
        cs = max(cs, c)
        mis = sp.get("misalign", 0) if i == np_ - 1 else 0
        buf = _ints(gen, n * (h >> up) * (w >> up) * cs + mis).to(dt)
        view = buf[mis:].reshape(n, h >> up, w >> up, cs)
        bufs.append(buf)
        views.append(view[..., :c])
        arr[i].x, arr[i].mask, arr[i].c, arr[i].x_cstride, arr[i].x_up, arr[i].mask_up = view.data_ptr(), None, c, cs, up, 0
        off += c
    null = set(sp.get("null", []))
    y = nan(n, h, w, ctot, dtype=dt)
    gy = _ints(gen, n, h, w, ctot).to(dt)
    gxs = [None if i in null else nan(n, h >> p[2], w >> p[2], p[0], dtype=dt) for i, p in enumerate(parts)]
    ptrs = (ctypes.c_void_p * np_)(*[None if g is None else g.data_ptr() for g in gxs])
    carr = (ctypes.c_int32 * np_)(*[p[0] for p in parts])
    uarr = (ctypes.c_int32 * np_)(*[p[2] for p in parts])
    vec_f = all(p[0] % 8 == 0 and max(p[1], p[0]) % 8 == 0 for p in parts) and not sp.get("misalign")
    vec_b = [(p[0] % 8 == 0 and sum(q[0] for q in parts[:i]) % 8 == 0 and ctot % 8 == 0) for i, p in enumerate(parts)]
    want = {("concat_fwd_kernel", "8" if vec_f else "1")}
    want |= {("concat_bwd_kernel", "8" if v else "1") for i, v in enumerate(vec_b) if i not in null}
    traced(name, lambda: (_lib.check(lib.pcb_concat_forward(arr, np_, code, n, h, w, y.data_ptr(), st)),
                          _lib.check(lib.pcb_concat_backward(gy.data_ptr(), carr, uarr, np_, code, n, h, w, ptrs, st))),
            _route(name, want), [(y, NAN)] + [(g, NAN) for g in gxs if g is not None])
    ref = torch.cat([v.repeat_interleave(1 << p[2], 1).repeat_interleave(1 << p[2], 2) for v, p in zip(views, parts)], dim=3)
    assert_bitwise(f"{name}: forward", y, ref)
    off = 0
    for i, (c, _, up) in enumerate(parts):
        if gxs[i] is not None:
            f = 1 << up
            g = gy[..., off:off + c].double().reshape(n, h >> up, f, w >> up, f, c).sum((2, 4))
            assert_bitwise(f"{name}: backward part {i}", gxs[i], g.to(dt))
        off += c


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("concat")))
def test_concat_vs_exact(name):
    _concat_case(_cases("concat")[name], name, _lib.load())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("upsample2x")))
def test_upsample2x_vs_exact(name):
    sp = _cases("upsample2x")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    code, dt, n, h, w, c = sp["dtype"], DT[sp["dtype"]], sp["n"], sp["h"], sp["w"], sp["c"]
    x = _ints(gen, n, h, w, c).to(dt)
    gy = _ints(gen, n, 2 * h, 2 * w, c).to(dt)
    y, gx = nan(n, 2 * h, 2 * w, c, dtype=dt), nan(n, h, w, c, dtype=dt)
    v = "8" if c % 8 == 0 else "1"
    traced(name, lambda: (_lib.check(lib.pcb_upsample2x_forward(x.data_ptr(), code, n, h, w, c, y.data_ptr(), st)),
                          _lib.check(lib.pcb_upsample2x_backward(gy.data_ptr(), code, n, h, w, c, gx.data_ptr(), st))),
            _route(name, {("concat_fwd_kernel", v), ("concat_bwd_kernel", v)}), [(y, NAN), (gx, NAN)])
    assert_bitwise(f"{name}: forward", y, x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    assert_bitwise(f"{name}: backward", gx, gy.double().reshape(n, h, 2, w, 2, c).sum((2, 4)).to(dt))


# ------------------------------------------------------------------------------------------------ mask planes
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("mask")))
def test_mask_planes_exact(name):
    sp = _cases("mask")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    n, h, w, c = sp["n"], sp["h"], sp["w"], sp["c"]
    if "up" not in sp:                                                  # planes from a dense NCHW mask
        m = _ints(gen, n, c, h, w, lo=-1, hi=1).float() * 0.5
        planes = torch.full((c, n, h, w), 77, dtype=torch.uint8, device="cuda")
        traced(name, lambda: _lib.check(lib.pcb_mask_planes_from_dense(m.data_ptr(), n, c, h, w, planes.data_ptr(), st)),
                _route(name, {("mask_from_dense_kernel", None)}), [(planes, 77)])
        assert_bitwise(f"{name}: planes", planes, (m != 0).to(torch.uint8).permute(1, 0, 2, 3))
        return
    up, ctot, c0 = sp["up"], sp["ctot"], sp["c0"]
    plane = (torch.rand(n, h >> up, w >> up, generator=gen, device="cuda") > 0.3).to(torch.uint8)
    dst = nan(n, ctot, h, w)
    traced(name, lambda: _lib.check(lib.pcb_mask_plane_to_dense(plane.data_ptr(), n, h, w, up, dst.data_ptr(), ctot, c0, c, st)),
            _route(name, {("mask_to_dense_kernel", None)}), [(dst, NAN)])
    full = plane.float().repeat_interleave(1 << up, 1).repeat_interleave(1 << up, 2)[:, None].expand(n, c, h, w)
    assert_bitwise(f"{name}: channels [c0, c0 + c)", dst[:, c0:c0 + c], full)
    rest = torch.cat([dst[:, :c0], dst[:, c0 + c:]], dim=1)
    assert bool(rest.isnan().all()), f"{name}: wrote outside its channels"


# ------------------------------------------------------------------------------------------------ L1 mean
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("l1")))
def test_l1_mean_vs_fp64(name):
    sp = _cases("l1")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    code, dt, numel = sp["dtype"], DT[sp["dtype"]], sp["numel"]
    x = torch.randn(numel, generator=gen, device="cuda").to(dt)
    x[::7] = 0                                                          # sign(0) = 0
    gscale = float(torch.tensor(1.0 / numel, dtype=torch.float32))
    loss, scratch, gx = nan(1), torch.zeros(1, dtype=torch.float64, device="cuda") + 5, nan(numel, dtype=dt)
    traced(name, lambda: (_lib.check(lib.pcb_l1_mean_forward(x.data_ptr(), code, numel, loss.data_ptr(), scratch.data_ptr(), st)),
                          _lib.check(lib.pcb_l1_mean_backward(x.data_ptr(), code, numel, gscale, gx.data_ptr(), st))),
            _route(name, {("l1_sum_kernel", None), ("l1_finish_kernel", None), ("l1_bwd_kernel", None)}),
            [(loss, NAN), (scratch, 5.0), (gx, NAN)])
    a = x.double().abs()
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(math.ceil(numel / (256 * 16)), 16 * nsm))
    L = math.ceil(numel / (grid * 256)) + 14
    ref = a.sum() / numel
    assert_within(f"{name}: loss", loss[0], ref, L * U * ref + U * ref)
    assert_bitwise(f"{name}: backward", gx, (torch.sign(x.double()) * gscale).float().to(dt))


# ------------------------------------------------------------------------------------------------ SGD
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("sgd")))
def test_sgd_vs_torch_fp64(name):
    sp = _cases("sgd")[name]
    lib, gen, st = _lib.load(), _gen(name), _st()
    numel = sp["numel"]
    lr, mom, wd, gs = (float(torch.tensor(sp[k], dtype=torch.float32)) for k in ("lr", "momentum", "weight_decay", "grad_scale"))
    nest, first = sp["nesterov"], sp["first_step"]
    p = torch.randn(numel, generator=gen, device="cuda")
    g = torch.randn(numel, generator=gen, device="cuda")
    buf = torch.randn(numel, generator=gen, device="cuda") if mom else None
    p0, b0 = p.clone(), (buf.clone() if buf is not None else None)
    traced(name, lambda: _lib.check(lib.pcb_sgd_step_scaled(p.data_ptr(), g.data_ptr(), None if buf is None else buf.data_ptr(), numel,
                                                            lr, mom, wd, nest, first, gs, st)),
            _route(name, {("sgd_kernel", None)}), [(p, p0)] + ([(buf, b0)] if buf is not None else []))
    # torch.optim.SGD in fp64 on the same values
    p64 = torch.nn.Parameter(p0.double())
    p64.grad = g.double() * gs
    opt = torch.optim.SGD([p64], lr=lr, momentum=mom, weight_decay=wd, nesterov=bool(nest))
    if mom and not first:
        opt.state[p64]["momentum_buffer"] = b0.double().clone()
    opt.step()
    P, G = p0.double(), g.double() * gs
    d = G + wd * P
    e_d = 3 * U * (G.abs() + wd * P.abs())
    if mom:
        b = d if first else mom * b0.double() + d
        e_b = e_d + (0 if first else 2 * U * (mom * b0.double().abs() + d.abs()))
        assert_within(f"{name}: momentum buffer", buf, opt.state[p64]["momentum_buffer"], e_b)
        dn = d + mom * b if nest else b
        e_dn = (e_d + mom * e_b + 2 * U * (d.abs() + mom * b.abs())) if nest else e_b
    else:
        dn, e_dn = d, e_d
    assert_within(f"{name}: parameters", p, p64.detach(), lr * e_dn + 2 * U * (P.abs() + lr * dn.abs()))

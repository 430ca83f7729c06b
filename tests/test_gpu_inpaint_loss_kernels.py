"""The kernels of the inpainting loss (csrc/inpaint_loss.cu) through the C ABI, every element against an fp64 reference of the
same stored operands computed on the device: the pixel terms forward and backward, max-pool forward and backward, the
perceptual L1 sums and their backward, the Gram L1 sums and the Gram sign, conv1_1's kernel-to-row weight and tap sum, and the
finalize step; then the whole loss with a zero-weight VGG, where every perceptual and style quantity is exactly 0 and the
loss is the pixel terms alone.  Cases: one per distinct call site of tests/golden/inpaint_loss_sites.json (the loss at 512^2
batch 8 bf16 NHWC-padded and 256^2 batch 2 fp32 NCHW, and total_variation_loss), at the recorded size with the batch cut to
keep every buffer within 2^27 elements, plus hand cases for the edges.  Outputs are prefilled with NaN (and channel padding
with a sentinel), every owned element must be written and nothing else, and each case asserts its kernels and their template
arguments from one complete torch.profiler trace (kernel_harness.traced):

    entry point                        kernel                                  cases
    pcb_inpaint_loss_pixel_forward     pixel_fwd_kernel<TO, TX>                pix_*, fx_pixel_fwd_*
    pcb_inpaint_loss_pixel_backward    pixel_bwd_kernel<TO, TX>                pix_*, fx_pixel_bwd_*
    pcb_maxpool2x2_forward / backward  maxpool_fwd_kernel<T>, maxpool_bwd_kernel<T>   pool_*, fx_maxpool_*
    pcb_feature_l1_forward             feature_l1_kernel<T>                    feat_*, fx_feature_l1_*
    pcb_feature_loss_backward          feature_bwd_kernel<T>                   feat_*, fx_feature_bwd_*
    pcb_gram_l1_forward / sign_sym     gram_l1_kernel, gram_sign_kernel        gram_*, fx_gram_*
    pcb_k2r_image_weight / dgrad       k2r_image_weight_kernel, k2r_image_dgrad_kernel<T>   k2r_*, fx_k2r_*
    pcb_inpaint_loss_finalize          loss_finalize_kernel                    fin_*, fx_finalize_*

Every case runs two regimes.  u = 2^-24 (fp32), N = the number of terms of a sum.

Integer regime: images, features, gradients and Gram products are small integers, the coefficients dyadic (the fixture's
recorded ones are replaced) and gscale a power of two.  Every fp32 difference, product and sum of the kernels is then exact,
so every output must EQUAL the exact result rounded once to its storage type, and the fp64 sums, which the reductions ADD to
a nonzero prefill, must equal prefill + exact sum bit for bit whatever the order of the atomics.

Gaussian regime (the recorded coefficients, Gaussian operands):
  * pixel and feature L1 sums: each |a - b| is one fp32 difference, off by u |a - b|; the per-thread fp64 chains, the warp
    trees and the fp64 atomics add at most (N - 1) 2^-53 of the sum of the N terms (any order), and the prefill P one more
    rounding of P + S.  Bound: (u + 2 N 2^-53) sum |a - b| + 2^-53 |P + S| (the 2 covers the reference's own fp64 sum);
  * pixel backward: per element at most 8 fp32 roundings (gs * coef, the three partial TV sums, gs * tv, + dX_comp, the add
    to g, + dX_output), each of at most u times M = |gs| (|c_valid or c_hole| + hole (2 |c_tv_h| + 2 |c_tv_v|)) + hole
    |dX_comp| + |dX_output|; the `a*b + c` lines may be fused or not, which only removes roundings.  Bound 9 u M (a margin for
    the growth of the intermediates), plus 2^-8 (|ref| + 9 u M) for a bf16 store;
  * feature backward: l1 * sign is exact; + gram * g_gram, * gs and + g_next round at most 4 times, each by u of
    M = |gs| (|l1| + |gram g_gram|) + |g_next|: bound 5 u M, plus 2^-8 (|ref| + 5 u M) for a bf16 store;
  * Gram L1 and sign: the kernel's quotients G / norm are correctly rounded fp32 divisions (no fast-math), and so is its fp32
    difference; the reference rounds the fp64 quotient and then the fp64 difference to fp32, which gives the same values
    (double rounding through 53 bits is innocuous for one fp32 division or subtraction, p = 53 >= 2 * 24 + 2).  The sign
    operand must therefore be bit-identical, exactly symmetric, and the L1 sums within 2 N 2^-53 sum |d| + 2^-53 |P + S| of
    the sum of those differences;
  * kernel-to-row tap sum: up to 9 terms added in fp32 (8 u sum |Z|), plus 2^-8 (|ref| + 8 u sum |Z|) for a bf16 store;
  * max-pool, the kernel-to-row weight and the Gram sign are selections: bit-identical in both regimes, ±0 included;
  * finalize: each term s * inv and the loss are evaluated in fp64 and rounded once to fp32, so each is within one fp32 ulp
    of its exact rational value (fractions.Fraction).
"""
import ctypes
import fractions
import importlib.util
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_harness import GOLDEN, SENTINEL, assert_bitwise, assert_within, holes, nan, traced
from text_segmentation_image_inpainting_b200 import _lib

U = 2.0 ** -24
E53 = 2.0 ** -53
BF, F32 = _lib.PCB_BF16, _lib.PCB_F32
DT = {BF: torch.bfloat16, F32: torch.float32}
TNAME = {BF: "__nv_bfloat16", F32: "float"}
SHORT = {BF: "bf16", F32: "f32"}
STORE = {BF: 2.0 ** -8, F32: 0.0}
MAX_ELEMS = 1 << 27
NAN = float("nan")
PREFILL = 1000.0                  # the reductions add to their sums: prefilled sums must keep it
REGIMES = ("int", "gauss")
LOSS_WEIGHTS = (1.0, 6.0, 0.1, 0.05, 120.0)
INT_COEF = (0.125, 0.75, 0.0625, 0.15625)     # dyadic {valid, hole, tv_h, tv_v} for the integer regime
INT_GS = 2.0


def _sites():
    with open(os.path.join(GOLDEN, "inpaint_loss_sites.json")) as f:
        return json.load(f)


def _gen(name, device="cuda"):
    return torch.Generator(device=device).manual_seed(sum(map(ord, name)))


def _ints(gen, *shape, lo=-3, hi=3):
    return torch.randint(lo, hi + 1, shape, generator=gen, device="cuda").double()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _route(name, want, only=True):
    """the check of traced: each (kernel, template arguments) of want ran, and (only) no other kernel"""
    want = set(want)

    def check(records):
        got = set(records)
        missing = want - got
        assert not missing, f"{name}: {sorted(missing)} did not run; ran {sorted(got)}"
        assert not only or got == want, f"{name}: ran {sorted(got)}, the case covers {sorted(want)}"
    return check


def assert_same(name, got, want):
    """bit-identical values: NaN where want is NaN, elsewhere equal with the same sign (so -0 and +0 differ)"""
    g, w = got.double(), want.double()
    ok = (g.isnan() & w.isnan()) | ((g == w) & (g.signbit() == w.signbit()))
    if not bool(ok.all()):
        bad = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements differ; first at {list(bad)}: got {float(g[bad])!r}, "
                             f"want {float(w[bad])!r}")


def _sum_check(name, regime, got, prefill, terms_abs_sum, exact_sum, nterms):
    """a reduction's fp64 sum against prefill + exact sum: equal (integer regime) or within the module docstring's bound"""
    if regime == "int":
        assert float(got) == prefill + float(exact_sum), f"{name}: {float(got)!r} != {prefill} + {float(exact_sum)!r}"
    else:
        bound = (U + 2 * nterms * E53) * float(terms_abs_sum) + E53 * abs(prefill + float(exact_sum))
        err = abs(float(got) - (prefill + float(exact_sum)))
        assert err <= bound, f"{name}: error {err:.3e} exceeds the bound {bound:.3e}"


def _f32(v):
    return float(np.float32(v))


# ================================================================================================ fixture sites
def _layout(strides, h, w):
    if list(strides) == [3 * h * w, h * w, w, 1]:
        return "nchw"
    if list(strides) == [8 * h * w, 1, 8 * w, 8]:
        return "nhwc"
    raise AssertionError(f"no layout has strides {strides} at {h}x{w}")


def _cap(n, per_item):
    """the largest batch <= n with n * per_item <= 2^27 (at least 1)"""
    return max(1, min(n, MAX_ELEMS // per_item))


def _site_case(s):
    """(family, case name, spec) of a fixture site"""
    fn = s["fn"]
    if fn.startswith("pcb_inpaint_loss_pixel"):
        fwd = fn.endswith("forward")
        n, h, w = s["n"], s["h"], s["w"]
        sp = dict(to=s["out_dtype"], tx=s["dtype"], n=n, h=h, w=w, out=_layout(s["out_strides"], h, w), plane="rand", fwd=fwd, bwd=not fwd)
        name = f"fx_pixel_{'fwd' if fwd else 'bwd'}_{SHORT[sp['to']]}_{SHORT[sp['tx']]}_n{n}_{h}x{w}_{sp['out']}"
        if not fwd:
            sp.update(grad=_layout(s["grad_strides"], h, w), dvgg=not s["null_dvgg_in"], coef=tuple(s["coef"]))
            name += f"_g{sp['grad']}_dvgg{int(sp['dvgg'])}"
        return "pixel", name, sp
    if fn.startswith("pcb_maxpool2x2"):
        fwd = fn.endswith("forward")
        n, h, w, c = _cap(s["n"], s["h"] * s["w"] * s["c"]), s["h"], s["w"], s["c"]
        sp = dict(dtype=s["dtype"], n=n, h=h, w=w, c=c, fwd=fwd, relu=() if fwd else (s["relu_mask"],))
        return "pool", f"fx_maxpool_{'fwd' if fwd else 'bwd'}_{SHORT[s['dtype']]}_n{s['n']}_{h}x{w}_c{c}" + ("" if fwd else f"_r{s['relu_mask']}"), sp
    if fn.startswith("pcb_feature"):
        fwd = fn == "pcb_feature_l1_forward"
        n, hw, c = _cap(s["n"], 3 * s["hw"] * s["c"]), s["hw"], s["c"]
        sp = dict(dtype=s["dtype"], n=n, hw=hw, c=c, fwd=fwd, bwd=not fwd)
        name = f"fx_feature_{'l1' if fwd else 'bwd'}_{SHORT[s['dtype']]}_n{s['n']}_hw{hw}_c{c}"
        if not fwd:
            sp.update(gnext=not s["null_g_next"], ggram=not s["null_g_gram"], l1=s["l1_coef"], gram=s["gram_coef"])
            name += f"_gn{int(sp['gnext'])}_gg{int(sp['ggram'])}"
        return "feature", name, sp
    if fn.startswith("pcb_gram"):
        l1 = fn == "pcb_gram_l1_forward"
        sp = dict(n=s["n"], c=s["c"], norm=s["norm"], l1=l1, sign=not l1)
        return "gram", f"fx_gram_{'l1' if l1 else 'sign'}_n{s['n']}_c{s['c']}_norm{int(s['norm'])}", sp
    if fn == "pcb_k2r_image_weight":
        return "k2r_weight", f"fx_k2r_weight_co{s['cout']}", dict(cout=s["cout"])
    if fn == "pcb_k2r_image_dgrad":
        n, h, w = _cap(s["n"], s["h"] * s["w"] * 32), s["h"], s["w"]
        return "k2r_dgrad", f"fx_k2r_dgrad_{SHORT[s['dtype']]}_n{s['n']}_{h}x{w}", dict(dtype=s["dtype"], n=n, h=h, w=w)
    if fn == "pcb_inpaint_loss_finalize":
        inv = s["inv"]
        return "finalize", f"fx_finalize_inv{round(1 / inv[0])}", dict(inv=tuple(inv))
    return None, None, None


def _fixture(fam):
    return {name: sp for f, name, sp in map(_site_case, _sites()) if f == fam}


# ================================================================================================ hand cases
def _pix(to, tx, n, h, w, out="nhwc", grad=None, plane="rand", equal=False, dvgg=True, gs=1.0):
    return dict(to=to, tx=tx, n=n, h=h, w=w, out=out, grad=grad or out, plane=plane, equal=equal, dvgg=dvgg, gs=gs, fwd=True, bwd=True)


def _feat(dt, n, hw, c, gnext=True, ggram=True, gs=1.0):
    return dict(dtype=dt, n=n, hw=hw, c=c, gnext=gnext, ggram=ggram, gs=gs, fwd=True, bwd=True)


HAND = {
    "pixel": {
        **{f"pix_{SHORT[to]}_{SHORT[tx]}_{lay}": _pix(to, tx, 2, 24, 40, out=lay) for to in (BF, F32) for tx in (BF, F32)
           for lay in ("nchw", "nhwc")},
        "pix_bf16_out_nhwc_grad_nchw": _pix(BF, BF, 2, 20, 36, out="nhwc", grad="nchw"),
        "pix_f32_out_nchw_grad_nhwc": _pix(F32, F32, 2, 20, 36, out="nchw", grad="nhwc"),
        "pix_all_valid": _pix(BF, BF, 2, 16, 24, plane="valid"), "pix_all_hole": _pix(F32, BF, 2, 16, 24, out="nchw", plane="hole"),
        "pix_border_holes": _pix(BF, F32, 3, 17, 29, plane="border"), "pix_border_holes_f32": _pix(F32, F32, 1, 30, 18, out="nchw", plane="border"),
        "pix_h2": _pix(BF, BF, 2, 2, 37), "pix_w2": _pix(F32, BF, 2, 41, 2, out="nchw"), "pix_2x2_one_block": _pix(BF, BF, 3, 2, 2),
        "pix_grid_below_block": _pix(F32, F32, 1, 9, 13, out="nchw"),
        "pix_output_equals_origin": _pix(BF, BF, 2, 16, 24, equal=True), "pix_output_equals_origin_f32": _pix(F32, F32, 2, 12, 20, out="nchw", equal=True),
        "pix_dvgg_null": _pix(BF, BF, 2, 16, 24, dvgg=False), "pix_dvgg_null_f32": _pix(F32, F32, 2, 16, 24, out="nchw", dvgg=False),
        "pix_gscale": _pix(BF, BF, 2, 16, 24, gs=0.7), "pix_n1": _pix(BF, BF, 1, 32, 48), "pix_n3": _pix(F32, BF, 3, 24, 16, out="nchw"),
        "pix_large_grid_stride": _pix(BF, BF, 4, 300, 700),
    },
    "pool": {
        **{f"pool_{SHORT[dt]}_c{c}": dict(dtype=dt, n=2, h=8, w=12, c=c, fwd=True, relu=(0, 1)) for dt in (BF, F32) for c in (8, 256)},
        "pool_specials_bf16": dict(dtype=BF, n=2, h=8, w=12, c=16, fwd=True, relu=(0, 1), specials=True),
        "pool_specials_f32": dict(dtype=F32, n=3, h=6, w=4, c=8, fwd=True, relu=(0, 1), specials=True),
        "pool_grid_stride": dict(dtype=BF, n=4, h=256, w=260, c=64, fwd=True, relu=(0, 1)),
    },
    "feature": {
        **{f"feat_gn{int(a)}_gg{int(b)}": _feat(BF, 2, 37, 16, a, b) for a in (False, True) for b in (False, True)},
        "feat_n1_f32": _feat(F32, 1, 5, 8), "feat_n3_gscale": _feat(BF, 3, 9, 24, gs=0.7), "feat_n3_f32_nulls": _feat(F32, 3, 7, 8, False, False),
        "feat_c256_ragged": _feat(BF, 2, 77, 256), "feat_grid_stride": _feat(BF, 2, 128 * 129, 128),
    },
    "gram": {
        **{f"gram_c{c}": dict(n=2, c=c, norm=float(c * 3 * 5), l1=True, sign=True) for c in (3, 64, 256)},
        "gram_n1_c8": dict(n=1, c=8, norm=float(8 * 7 * 3), l1=True, sign=True),
        "gram_n3_c64_pow2": dict(n=3, c=64, norm=float(64 * 16 * 16), l1=True, sign=True),
        "gram_round_equal": dict(n=2, c=64, norm=float(64 * 3 * 5), l1=True, sign=True, near=True),
    },
    "k2r_weight": {"k2r_weight_co64": dict(cout=64), "k2r_weight_co37": dict(cout=37)},
    "k2r_dgrad": {
        "k2r_dgrad_bf16_5x7": dict(dtype=BF, n=2, h=5, w=7), "k2r_dgrad_f32_1x1": dict(dtype=F32, n=3, h=1, w=1),
        "k2r_dgrad_bf16_1x9": dict(dtype=BF, n=1, h=1, w=9), "k2r_dgrad_f32_33x2": dict(dtype=F32, n=2, h=33, w=2),
    },
    "finalize": {f"fin_random_{i}": dict(seed=i) for i in range(4)},
}


def _cases(fam):
    return {**_fixture(fam), **HAND[fam]}


def test_fixture_sites_map_to_cases():
    """every site of the fixture names exactly one case, distinct from the hand cases"""
    sites = _sites()
    assert sites, "the fixture holds no site"
    fns = set()
    for s in sites:
        fam, name, _ = _site_case(s)
        assert fam is not None, f"no case family for {s['fn']}"
        assert name in _fixture(fam) and name not in HAND[fam]
        fns.add(s["fn"])
    assert len(fns) == 11, f"the fixture reaches {sorted(fns)}"


# ================================================================================================ pixel terms
def _image(n, h, w, dt, layout, fill):
    """(logical [n, 3, h, w] view, its whole buffer): dense NCHW, or the 8-channel-padded NHWC view with SENTINEL in 3..7"""
    if layout == "nchw":
        buf = torch.empty(n, 3, h, w, dtype=dt, device="cuda")
        view = buf
    else:
        buf = torch.full((n, h, w, 8), SENTINEL, dtype=dt, device="cuda")
        view = buf.permute(0, 3, 1, 2)[:, :3]
    view.copy_(fill) if isinstance(fill, torch.Tensor) else view.fill_(fill)
    return view, buf


def _plane(kind, n, h, w, name):
    if kind == "valid":
        return torch.ones(n, h, w, dtype=torch.uint8, device="cuda")
    if kind == "hole":
        return torch.zeros(n, h, w, dtype=torch.uint8, device="cuda")
    m = holes(n, h, w, _gen(name, "cpu"))
    if kind == "border":
        m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0
    return m.cuda()


def _strides(t):
    return (ctypes.c_longlong * 4)(*t.stride())


def _pixel_operands(sp, regime, name):
    gen = _gen(name + regime)
    n, h, w, to, tx = sp["n"], sp["h"], sp["w"], DT[sp["to"]], DT[sp["tx"]]
    if sp.get("equal"):                                  # output == origin == raw, few values: sign(0) everywhere, equal neighbours
        v = _ints(gen, n, 3, h, w, lo=0, hi=1).to(to).double()
        orig, raw = v.clone(), v.clone()
    elif regime == "int":
        raw, orig, v = _ints(gen, n, 3, h, w), _ints(gen, n, 3, h, w), _ints(gen, n, 3, h, w).to(to).double()
    else:
        raw = torch.randn(n, 3, h, w, generator=gen, device="cuda").double()
        orig = torch.randn(n, 3, h, w, generator=gen, device="cuda").double()
        v = torch.randn(n, 3, h, w, generator=gen, device="cuda").to(to).double()
    raw, orig = raw.float().double(), orig.float().double()
    scale = 1.0 if regime == "int" else 1e-3
    dX = (_ints(gen, 2 * n, h, w, 8, lo=-4, hi=4) if regime == "int" else torch.randn(2 * n, h, w, 8, generator=gen, device="cuda").double() * scale).to(tx)
    dX[..., 3:] = SENTINEL                               # channels 3..7 of the VGG input gradient are not part of the image
    if regime == "int":
        coef, gs = INT_COEF, INT_GS
    else:
        cnt = (n * 3 * h * w, n * 3 * h * w, n * 3 * h * (w - 1), n * 3 * (h - 1) * w)
        coef = sp.get("coef") or tuple(_f32(LOSS_WEIGHTS[min(k, 2)] / cnt[k]) for k in range(4))
        gs = sp.get("gs", 1.0)
    return raw, orig, v, dX, tuple(_f32(c) for c in coef), _f32(gs)


def _pixel_ref(raw, orig, v, m, dX, coef, gs, dvgg):
    """fp64: (comp, |d| per term family, gradient, M of the bound)"""
    n = v.shape[0]
    mm = m.bool()[:, None].expand_as(v)
    cp = torch.where(mm, raw, v)
    dh, dv = cp[..., :-1] - cp[..., 1:], cp[..., :-1, :] - cp[..., 1:, :]
    d = v - orig
    sh, sv = torch.sign(dh), torch.sign(dv)
    tv = torch.zeros_like(v)
    tv[..., :-1] += coef[2] * sh
    tv[..., 1:] -= coef[2] * sh
    tv[..., :-1, :] += coef[3] * sv
    tv[..., 1:, :] -= coef[3] * sv
    cm = torch.where(mm, torch.full_like(v, coef[0]), torch.full_like(v, coef[1]))
    if dvgg:
        dxc, dxo = dX[:n, ..., :3].double().permute(0, 3, 1, 2), dX[n:, ..., :3].double().permute(0, 3, 1, 2)
    else:
        dxc = dxo = torch.zeros_like(v)
    hole = (~mm).double()
    g = gs * cm * torch.sign(d) + hole * (gs * tv + dxc) + dxo
    M = abs(gs) * (cm.abs() + hole * 2 * (abs(coef[2]) + abs(coef[3]))) + hole * dxc.abs() + dxo.abs()
    return cp, (d.abs() * mm, d.abs() * (~mm), dh.abs(), dv.abs()), g, M


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("pixel")))
def test_pixel_terms_vs_fp64(name):
    sp = _cases("pixel")[name]
    lib, st = _lib.load(), _st()
    n, h, w, to, tx = sp["n"], sp["h"], sp["w"], DT[sp["to"]], DT[sp["tx"]]
    m = _plane(sp["plane"], n, h, w, name)
    for regime in REGIMES:
        raw, orig, v, dX, coef, gs = _pixel_operands(sp, regime, name)
        raw32, orig32 = raw.float().contiguous(), orig.float().contiguous()
        out, _ = _image(n, h, w, to, sp["out"], v)
        X = nan(3 * n, h, w, 8, dtype=tx)
        sums0 = PREFILL + torch.arange(16, dtype=torch.float64, device="cuda")
        sums = sums0.clone()
        grad, gbuf = _image(n, h, w, to, sp.get("grad", sp["out"]), NAN)
        gbuf0 = gbuf.clone()
        gsd = torch.tensor([gs], dtype=torch.float32, device="cuda")
        cf = (ctypes.c_float * 4)(*coef)
        dvgg = sp.get("dvgg", True)

        def run():
            if sp["fwd"]:
                _lib.check(lib.pcb_inpaint_loss_pixel_forward(raw32.data_ptr(), orig32.data_ptr(), out.data_ptr(), sp["to"], _strides(out),
                                                              m.data_ptr(), n, h, w, X.data_ptr(), sp["tx"], sums.data_ptr(), st))
            if sp["bwd"]:
                _lib.check(lib.pcb_inpaint_loss_pixel_backward(raw32.data_ptr(), orig32.data_ptr(), out.data_ptr(), sp["to"], _strides(out),
                                                               m.data_ptr(), n, h, w, dX.data_ptr() if dvgg else None, sp["tx"], cf,
                                                               gsd.data_ptr(), grad.data_ptr(), _strides(grad), st))
        want = {(k, (TNAME[sp["to"]], TNAME[sp["tx"]])) for k, on in (("pixel_fwd_kernel", sp["fwd"]), ("pixel_bwd_kernel", sp["bwd"])) if on}
        if regime == REGIMES[0]:
            traced(name, run, _route(name, want), [(X, NAN), (sums, sums0), (gbuf, gbuf0)])
        else:
            run()
        torch.cuda.synchronize()
        cp, terms, g, M = _pixel_ref(raw, orig, v, m, dX, coef, gs, dvgg)
        tag = f"{name} [{regime}]"
        if sp["fwd"]:
            for i, img in enumerate((cp, v, orig)):
                assert_same(f"{tag}: VGG input image {i}", X[i * n:(i + 1) * n, ..., :3], img.permute(0, 2, 3, 1).float().to(tx))
            assert bool((X[..., 3:] == 0).all()), f"{tag}: VGG input channels 3..7 are not zero"
            for k in range(4):
                _sum_check(f"{tag}: sum {k}", regime, sums[k], float(sums0[k]), terms[k].sum(), terms[k].sum(), terms[k].numel())
            assert torch.equal(sums[4:], sums0[4:]), f"{tag}: sums past the pixel terms changed"
        else:
            assert torch.equal(sums, sums0) and bool(X.isnan().all()), f"{tag}: the forward outputs were written"
        if sp["bwd"]:
            if sp.get("grad", sp["out"]) == "nhwc":
                assert bool((gbuf[..., 3:] == SENTINEL).all()), f"{tag}: gradient written past channel 3"
            if regime == "int":
                assert_same(f"{tag}: gradient", grad, g.float().to(to))
            else:
                e = 9 * U * M
                assert_within(f"{tag}: gradient", grad, g, e + STORE[sp["to"]] * (g.abs() + e))
        else:
            assert bool(grad.isnan().all()), f"{tag}: the gradient was written"


# ================================================================================================ max-pool
def _pool_input(sp, regime, name):
    gen = _gen(name + regime)
    n, h, w, c, dt = sp["n"], sp["h"], sp["w"], sp["c"], DT[sp["dtype"]]
    x = (_ints(gen, n, h, w, c, lo=-2, hi=2) if regime == "int" else torch.randn(n, h, w, c, generator=gen, device="cuda").double()).to(dt)
    if sp.get("specials"):
        x[0, 2:4, 2:4, :] = float("-inf")                          # whole windows of -inf: the first tap is the index
        x[0, 0, 0, 0] = NAN                                        # NaN first, later and last in its window
        x[0, 1, 3, 1] = NAN
        x[1, 4:6, 4:6, 2] = NAN                                    # all-NaN window: the last NaN is the index
        x[1, 0:2, 0:2, :] = 0.0                                    # ±0 ties: the first zero wins, whatever its sign
        x[1, 0, 0, ::2] = -0.0
        x[1, 1, 1, 1::2] = -0.0
        x[0, 4:6, 0:2, :] = -1.0                                   # maximum < 0 (and ties): the ReLU mask drops it
        x[0, 0:2, 4:6, 3] = -0.0                                   # maximum -0 <= 0: dropped too
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("pool")))
def test_maxpool_vs_torch(name):
    sp = _cases("pool")[name]
    lib, st = _lib.load(), _st()
    n, h, w, c, code = sp["n"], sp["h"], sp["w"], sp["c"], sp["dtype"]
    dt = DT[code]
    for regime in REGIMES:
        gen = _gen(name + regime + "gy")
        x = _pool_input(sp, regime, name)
        gy = (_ints(gen, n, h // 2, w // 2, c, lo=-4, hi=4) if regime == "int" else
              torch.randn(n, h // 2, w // 2, c, generator=gen, device="cuda").double()).to(dt)
        y = nan(n, h // 2, w // 2, c, dtype=dt)
        gxs = {r: nan(n, h, w, c, dtype=dt) for r in sp["relu"]}

        def run():
            if sp["fwd"]:
                _lib.check(lib.pcb_maxpool2x2_forward(x.data_ptr(), y.data_ptr(), code, n, h, w, c, st))
            for r, gx in gxs.items():
                _lib.check(lib.pcb_maxpool2x2_backward(gy.data_ptr(), x.data_ptr(), gx.data_ptr(), code, n, h, w, c, r, st))
        want = ({("maxpool_fwd_kernel", (TNAME[code],))} if sp["fwd"] else set()) | ({("maxpool_bwd_kernel", (TNAME[code],))} if gxs else set())
        if regime == REGIMES[0]:
            traced(name, run, _route(name, want), [(y, NAN)] + [(g, NAN) for g in gxs.values()])
        else:
            run()
        torch.cuda.synchronize()
        tag = f"{name} [{regime}]"
        xr = x.float().permute(0, 3, 1, 2).contiguous()
        yr, idx = F.max_pool2d(xr, 2, 2, return_indices=True)
        if sp["fwd"]:
            assert_same(f"{tag}: forward", y, yr.permute(0, 2, 3, 1).to(dt))
        else:
            assert bool(y.isnan().all())
        g = gy.float().permute(0, 3, 1, 2)
        for r, gx in gxs.items():
            gr = torch.where(yr <= 0, torch.zeros_like(g), g) if r else g
            ref = torch.zeros(n, c, h * w, device="cuda").scatter_(2, idx.flatten(2), gr.flatten(2)).view(n, c, h, w)
            assert_same(f"{tag}: backward relu_mask={r}", gx, ref.permute(0, 2, 3, 1).to(dt))


# ================================================================================================ perceptual L1
def _feature_operands(sp, regime, name):
    gen = _gen(name + regime)
    n, hw, c, dt = sp["n"], sp["hw"], sp["c"], DT[sp["dtype"]]
    if regime == "int":
        f = _ints(gen, 3 * n, hw, c)
        gg, gn = _ints(gen, 2 * n, hw, c, lo=-4, hi=4), _ints(gen, 2 * n, hw, c, lo=-4, hi=4)
        l1, gram, gs = 0.25, 0.375, INT_GS
    else:
        f = torch.relu(torch.randn(3 * n, hw, c, generator=gen, device="cuda").double())
        gg = torch.randn(2 * n, hw, c, generator=gen, device="cuda").double()
        gn = torch.randn(2 * n, hw, c, generator=gen, device="cuda").double() * 1e-3
        l1 = sp.get("l1", LOSS_WEIGHTS[3] / (n * c * hw))
        gram = sp.get("gram", LOSS_WEIGHTS[4] / (n * c * c) / (c * hw))
        gs = sp.get("gs", 1.0)
    f[:n, : hw // 2] = f[2 * n:, : hw // 2]             # comp equals origin on half of every image: sign(0)
    f[n:2 * n, hw // 3:] = f[2 * n:, hw // 3:]           # output equals origin on two thirds
    return f.to(dt), gg.to(dt), gn.to(dt), _f32(l1), _f32(gram), _f32(gs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("feature")))
def test_feature_l1_vs_fp64(name):
    sp = _cases("feature")[name]
    lib, st = _lib.load(), _st()
    n, hw, c, code = sp["n"], sp["hw"], sp["c"], sp["dtype"]
    dt = DT[code]
    gnext, ggram = sp.get("gnext", True), sp.get("ggram", True)
    for regime in REGIMES:
        f, gg, gn, l1, gram, gs = _feature_operands(sp, regime, name)
        sums0 = PREFILL + torch.arange(4, dtype=torch.float64, device="cuda")
        sums = sums0.clone()
        df = nan(2 * n, hw, c, dtype=dt)
        gsd = torch.tensor([gs], dtype=torch.float32, device="cuda")

        def run():
            if sp["fwd"]:
                _lib.check(lib.pcb_feature_l1_forward(f.data_ptr(), code, n, hw, c, sums.data_ptr(), st))
            if sp["bwd"]:
                _lib.check(lib.pcb_feature_loss_backward(f.data_ptr(), code, n, hw, c, gn.data_ptr() if gnext else None,
                                                         gg.data_ptr() if ggram else None, l1, gram, gsd.data_ptr(), df.data_ptr(), st))
        want = {(k, (TNAME[code],)) for k, on in (("feature_l1_kernel", sp["fwd"]), ("feature_bwd_kernel", sp["bwd"])) if on}
        if regime == REGIMES[0]:
            traced(name, run, _route(name, want), [(sums, sums0), (df, NAN)])
        else:
            run()
        torch.cuda.synchronize()
        tag = f"{name} [{regime}]"
        fd = f.double()
        o = fd[2 * n:]
        if sp["fwd"]:
            for k in range(2):
                d = (fd[k * n:(k + 1) * n] - o).abs()
                _sum_check(f"{tag}: sum {k}", regime, sums[k], float(sums0[k]), d.sum(), d.sum(), d.numel())
            assert torch.equal(sums[2:], sums0[2:]), f"{tag}: sums past the two L1 terms changed"
        else:
            assert torch.equal(sums, sums0)
        if sp["bwd"]:
            oo = torch.cat([o, o])                                          # origin of image im is 2n + im % n
            v = l1 * torch.sign(fd[:2 * n] - oo)
            M = abs(gs) * abs(l1) + torch.zeros_like(v)
            if ggram:
                v = v + gram * gg.double()
                M = M + abs(gs * gram) * gg.double().abs()
            ref = gs * v
            if gnext:
                ref = ref + gn.double()
                M = M + gn.double().abs()
            if regime == "int":
                assert_same(f"{tag}: backward", df, ref.float().to(dt))
            else:
                e = 5 * U * M
                assert_within(f"{tag}: backward", df, ref, e + STORE[code] * (ref.abs() + e))
        else:
            assert bool(df.isnan().all())


# ================================================================================================ Gram L1 and sign
def _q32(g, norm):
    """the correctly rounded fp32 quotient of fp32 g by fp32 norm"""
    return (g.double() / norm).float().double()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("gram")))
def test_gram_vs_fp64(name):
    sp = _cases("gram")[name]
    lib, st = _lib.load(), _st()
    n, c = sp["n"], sp["c"]
    for regime in REGIMES:
        gen = _gen(name + regime)
        if regime == "int":
            norm = 2.0 ** round(np.log2(sp["norm"]))                    # a power of two: every quotient exact
            g = _ints(gen, 3 * n, c, c, lo=-64, hi=64).float()
            g[:n, : c // 2] = g[2 * n:, : c // 2]                      # equal products: sign 0
        else:
            norm = _f32(sp["norm"])
            g = (torch.randn(3 * n, c, c, generator=gen, device="cuda") * norm).float()
            g[n:2 * n, :, : c // 3] = g[2 * n:, :, : c // 3]
            if sp.get("near"):                                         # products one ulp apart: their quotients often round equal
                g[:n] = torch.nextafter(g[2 * n:], torch.full_like(g[2 * n:], float("inf")))
        sums0 = PREFILL + torch.arange(4, dtype=torch.float64, device="cuda")
        sums = sums0.clone()
        t = nan(2 * n, c, c)

        def run():
            if sp["l1"]:
                _lib.check(lib.pcb_gram_l1_forward(g.data_ptr(), n, c, norm, sums.data_ptr(), st))
            if sp["sign"]:
                _lib.check(lib.pcb_gram_sign_sym(g.data_ptr(), n, c, norm, t.data_ptr(), st))
        want = {(k, ()) for k, on in (("gram_l1_kernel", sp["l1"]), ("gram_sign_kernel", sp["sign"])) if on}
        if regime == REGIMES[0]:
            traced(name, run, _route(name, want), [(sums, sums0), (t, NAN)])
        else:
            run()
        torch.cuda.synchronize()
        tag = f"{name} [{regime}]"
        q = _q32(g, norm)
        qo = q[2 * n:]
        d32 = (q[:2 * n] - torch.cat([qo, qo])).float().double()          # the kernel's fp32 differences
        if sp.get("near") and regime == "gauss":
            same_q = (q[:n] == qo) & (g[:n] != g[2 * n:])
            assert bool(same_q.any()), f"{tag}: no product pair whose quotients round equal"
        if sp["l1"]:
            for k in range(2):
                a = d32[k * n:(k + 1) * n].abs()
                _sum_check(f"{tag}: sum {k}", regime, sums[k], float(sums0[k]), a.sum(), a.sum(), a.numel())
            assert torch.equal(sums[2:], sums0[2:])
        if sp["sign"]:
            s = torch.sign(d32)
            assert_same(f"{tag}: sign operand", t, (s + s.transpose(1, 2)).float())
            assert torch.equal(t, t.transpose(1, 2)), f"{tag}: sign operand not exactly symmetric"
        else:
            assert bool(t.isnan().all())


# ================================================================================================ kernel-to-row (conv1_1)
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("k2r_weight")))
def test_k2r_image_weight_is_a_permutation(name):
    sp = _cases("k2r_weight")[name]
    lib, st, cout = _lib.load(), _st(), sp["cout"]
    wt = torch.randn(cout, 3, 3, 3, generator=_gen(name), device="cuda")
    wz = nan(32, cout)
    traced(name, lambda: _lib.check(lib.pcb_k2r_image_weight(wt.data_ptr(), cout, wz.data_ptr(), st)),
           _route(name, {("k2r_image_weight_kernel", ())}), [(wz, NAN)])
    torch.cuda.synchronize()
    ref = torch.zeros(32, cout, device="cuda")
    ref[:27] = wt.permute(2, 3, 1, 0).reshape(27, cout)                 # row (kh * 3 + kw) * 3 + ci, column co
    assert_same(name, wz, ref)


def _tap_sum_ref(z, n, h, w):
    """dx[q][ci] = sum over taps (tr, tc) of Z[q - (tr - 1, tc - 1)][(tr * 3 + tc) * 3 + ci], outside pixels contributing 0;
    also the sum of |terms|"""
    zp = F.pad(z.double(), (0, 0, 1, 1, 1, 1))
    ref, ab = torch.zeros(n, h, w, 3, dtype=torch.float64, device="cuda"), torch.zeros(n, h, w, 3, dtype=torch.float64, device="cuda")
    for tr in range(3):
        for tc in range(3):
            blk = zp[:, 2 - tr:2 - tr + h, 2 - tc:2 - tc + w, (tr * 3 + tc) * 3:(tr * 3 + tc) * 3 + 3]
            ref += blk
            ab += blk.abs()
    return ref, ab


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("k2r_dgrad")))
def test_k2r_image_dgrad_vs_fp64(name):
    sp = _cases("k2r_dgrad")[name]
    lib, st = _lib.load(), _st()
    n, h, w, code = sp["n"], sp["h"], sp["w"], sp["dtype"]
    dt = DT[code]
    for regime in REGIMES:
        gen = _gen(name + regime)
        z = (_ints(gen, n, h, w, 32, lo=-8, hi=8) if regime == "int" else torch.randn(n, h, w, 32, generator=gen, device="cuda").double()).to(dt)
        z[..., 27:] = SENTINEL                                          # columns past the 27 taps are never read
        dx = nan(n, h, w, 8, dtype=dt)
        run = lambda: _lib.check(lib.pcb_k2r_image_dgrad(z.data_ptr(), code, n, h, w, dx.data_ptr(), st))  # noqa: E731
        if regime == REGIMES[0]:
            traced(name, run, _route(name, {("k2r_image_dgrad_kernel", (TNAME[code],))}), [(dx, NAN)])
        else:
            run()
        torch.cuda.synchronize()
        tag = f"{name} [{regime}]"
        ref, ab = _tap_sum_ref(z, n, h, w)
        assert bool((dx[..., 3:] == 0).all()), f"{tag}: channels 3..7 are not zero"
        if regime == "int":
            assert_same(tag, dx[..., :3], ref.float().to(dt))
        else:
            e = 8 * U * ab
            assert_within(tag, dx[..., :3], ref, e + STORE[code] * (ref.abs() + e))


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_k2r_image_dgrad_composed_vs_conv2d_input(dtype, regime):
    """conv1_1's data gradient as _Vgg.dgrad_image composes it (weight layout, 1x1 problem dc -> Z on the convolution forward
    kernels, tap sum) against torch.nn.grad.conv2d_input in fp64 with cuDNN off.  Integer regime (dc in {-1, 0, 1}, weights
    in {-2, ..., 2}, so |Z| <= 128): bit-identical.  Gaussian: Z accumulates 64 products (64 u sum |dc W|), is stored in the
    compute dtype (2^-8 |Z| in bf16), summed over 9 taps (8 u) and stored (2^-8 |dx| in bf16)."""
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.loss import VggExtractor, _Vgg
    enc = VggExtractor(pretrained=False).cuda()
    conv = enc.stage_convs(0)[0]
    gen = _gen(f"composed{dtype}{regime}")
    m, h, w = 2, 40, 72
    with torch.no_grad():
        if regime == "int":
            conv.weight.copy_(_ints(gen, 64, 3, 3, 3, lo=-2, hi=2))
        else:
            conv.weight.copy_(torch.randn(64, 3, 3, 3, generator=gen, device="cuda") * 0.1)
    dc = (_ints(gen, m, 64, h, w, lo=-1, hi=1) if regime == "int" else torch.randn(m, 64, h, w, generator=gen, device="cuda").double())
    dc = dc.to(dtype).contiguous(memory_format=torch.channels_last)
    x = ops.padded_empty(m, 3, h, w, dtype, torch.device("cuda"))
    vgg = _Vgg(enc, 1)
    code = _lib.PCB_BF16 if dtype == torch.bfloat16 else _lib.PCB_F32
    got = {}
    traced(f"composed {dtype} {regime}", lambda: got.__setitem__("dx", vgg.dgrad_image(conv, x, dc)),
           _route("composed", {("k2r_image_dgrad_kernel", (TNAME[code],))}, only=False), [])
    torch.cuda.synchronize()
    dx = got["dx"]
    wq = conv.weight.detach().to(dtype).double()                        # the operand the kernels read: the weight in the compute dtype
    with torch.backends.cudnn.flags(enabled=False):
        ref = torch.nn.grad.conv2d_input((m, 3, h, w), wq, dc.double(), padding=1)
        ab = torch.nn.grad.conv2d_input((m, 3, h, w), wq.abs(), dc.double().abs(), padding=1)
    if regime == "int":
        assert_same("composed", dx, ref.float().to(dtype))
    else:
        st = STORE[code]
        e = (72 * U + st) * 1.01 * ab
        assert_within("composed", dx, ref, e + st * (ref.abs() + e))


# ================================================================================================ finalize
def _fin_operands(sp, name):
    rng = np.random.default_rng(sum(map(ord, name)))
    sums = rng.uniform(0, 1e6, 16) * rng.choice([1e-6, 1.0, 1e3], 16)
    inv = sp.get("inv") or tuple(1.0 / float(rng.integers(1, 1 << 40)) for _ in range(16))
    return sums, inv


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases("finalize")))
def test_finalize_within_one_ulp(name):
    sp = _cases("finalize")[name]
    lib, st = _lib.load(), _st()
    sums_h, inv = _fin_operands(sp, name)
    sums = torch.tensor(sums_h, dtype=torch.float64, device="cuda")
    loss, terms = nan(1), nan(8)
    traced(name, lambda: _lib.check(lib.pcb_inpaint_loss_finalize(sums.data_ptr(), (ctypes.c_double * 16)(*inv), loss.data_ptr(),
                                                                  terms.data_ptr(), st)),
           _route(name, {("loss_finalize_kernel", ())}), [(loss, NAN), (terms, NAN)])
    torch.cuda.synchronize()
    S = [fractions.Fraction(float(v)) for v in sums_h]
    I = [fractions.Fraction(float(v)) for v in inv]
    exact = [S[0] * I[0], S[1] * I[1], S[2] * I[2] + S[3] * I[3],
             sum((S[4 + 2 * k] + S[5 + 2 * k]) * I[4 + 2 * k] for k in range(3)),
             sum((S[10 + 2 * k] + S[11 + 2 * k]) * I[10 + 2 * k] for k in range(3))]
    total = sum(fractions.Fraction(wt) * t for wt, t in zip(LOSS_WEIGHTS, exact))
    got = terms.cpu().tolist()
    for k, (g, e) in enumerate(zip(got[:5] + [float(loss)], exact + [total])):
        ulp = float(np.spacing(np.float32(float(e))))
        assert abs(fractions.Fraction(g) - e) <= fractions.Fraction(ulp), f"{name}: output {k} = {g!r}, exact {float(e)!r}"
    assert all(np.isnan(got[5:])), f"{name}: terms written past the five"


# ================================================================================================ refusals
def _refusals():
    lib, st = _lib.load(), _st()
    f32 = lambda *s: torch.zeros(*s, device="cuda")          # noqa: E731
    img, plane, X = f32(1, 3, 8, 8), torch.ones(1, 8, 8, dtype=torch.uint8, device="cuda"), nan(3, 8, 8, 8)
    big = nan(4096)
    sums, gs, cf = torch.zeros(16, dtype=torch.float64, device="cuda"), torch.ones(1, device="cuda"), (ctypes.c_float * 4)(1, 1, 1, 1)
    img1 = f32(1, 3, 1, 8)
    p = lambda t, off=0: t.data_ptr() + off                     # noqa: E731
    return {
        "pixel_fwd_h1": (lambda: lib.pcb_inpaint_loss_pixel_forward(p(img1), p(img1), p(img1), F32, _strides(img1), p(plane), 1, 1, 8, p(X),
                                                                    F32, p(sums), st), [X, sums]),
        "pixel_bwd_h1": (lambda: lib.pcb_inpaint_loss_pixel_backward(p(img1), p(img1), p(img1), F32, _strides(img1), p(plane), 1, 1, 8, None,
                                                                     F32, cf, p(gs), p(big), _strides(img1), st), [big]),
        "pixel_fwd_misaligned_vgg_in": (lambda: lib.pcb_inpaint_loss_pixel_forward(p(img), p(img), p(img), F32, _strides(img), p(plane), 1, 8,
                                                                                   8, p(big, 4), F32, p(sums), st), [big, sums]),
        "maxpool_fwd_odd_h": (lambda: lib.pcb_maxpool2x2_forward(p(big), p(big, 2048), F32, 1, 7, 8, 8, st), [big]),
        "maxpool_bwd_odd_w": (lambda: lib.pcb_maxpool2x2_backward(p(big), p(big), p(big, 2048), F32, 1, 8, 5, 8, 1, st), [big]),
        "maxpool_fwd_c12": (lambda: lib.pcb_maxpool2x2_forward(p(big), p(big, 2048), F32, 1, 4, 4, 12, st), [big]),
        "maxpool_bwd_c12": (lambda: lib.pcb_maxpool2x2_backward(p(big), p(big), p(big, 2048), BF, 1, 4, 4, 12, 0, st), [big]),
        "feature_l1_c12": (lambda: lib.pcb_feature_l1_forward(p(big), F32, 1, 4, 12, p(sums), st), [sums]),
        "feature_bwd_c12": (lambda: lib.pcb_feature_loss_backward(p(big), F32, 1, 4, 12, None, None, 1.0, 1.0, p(gs), p(big, 2048), st), [big]),
        "gram_l1_norm0": (lambda: lib.pcb_gram_l1_forward(p(big), 1, 8, 0.0, p(sums), st), [sums]),
        "gram_l1_norm_negative": (lambda: lib.pcb_gram_l1_forward(p(big), 1, 8, -64.0, p(sums), st), [sums]),
        "gram_sign_norm0": (lambda: lib.pcb_gram_sign_sym(p(big), 1, 8, 0.0, p(big, 2048), st), [big]),
        "gram_sign_norm_negative": (lambda: lib.pcb_gram_sign_sym(p(big), 1, 8, -1.0, p(big, 2048), st), [big]),
    }


REFUSALS = ("pixel_fwd_h1", "pixel_bwd_h1", "pixel_fwd_misaligned_vgg_in", "maxpool_fwd_odd_h", "maxpool_bwd_odd_w", "maxpool_fwd_c12",
            "maxpool_bwd_c12", "feature_l1_c12", "feature_bwd_c12", "gram_l1_norm0", "gram_l1_norm_negative", "gram_sign_norm0",
            "gram_sign_norm_negative")


@pytest.mark.gpu
@pytest.mark.parametrize("name", REFUSALS)
def test_refusals_write_nothing(name):
    call, outs = _refusals()[name]
    before_vals = [t.clone() for t in outs]
    torch.cuda.synchronize()
    before = _lib.launch_count()
    assert call() != 0, f"{name}: accepted"
    torch.cuda.synchronize()
    assert _lib.launch_count() == before, f"{name}: a refused call launched a kernel"
    for t, b in zip(outs, before_vals):
        assert torch.equal(t.isnan(), b.isnan()) and torch.equal(t.nan_to_num(), b.nan_to_num()), f"{name}: a refused call wrote"


# ================================================================================================ the composed loss
def _zero_vgg_criterion(feature_range):
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor
    vgg = VggExtractor(pretrained=False)
    g = torch.Generator().manual_seed(feature_range)
    with torch.no_grad():
        for mod in vgg.modules():
            if isinstance(mod, torch.nn.Conv2d):
                mod.weight.zero_()
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g))    # features relu(bias): nonzero, equal in all images
    return InpaintingLoss(vgg.cuda(), feature_range)


def _loss_output(n, h, w, dtype, layout, gen):
    from text_segmentation_image_inpainting_b200 import ops
    out = ops.padded_empty(n, 3, h, w, dtype, torch.device("cuda")) if layout == "nhwc" else torch.empty(n, 3, h, w, dtype=dtype, device="cuda")
    with torch.no_grad():
        out.copy_(torch.rand(n, 3, h, w, generator=gen, device="cuda"))
    return out.requires_grad_(True)


@pytest.mark.gpu
@pytest.mark.parametrize("feature_range", [1, 2, 3])
@pytest.mark.parametrize("layout", ["nhwc", "nchw"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_zero_weight_vgg_loss_is_the_pixel_loss(dtype, layout, feature_range):
    """With every VGG weight zero, each feature is relu(bias), identical in comp, output and origin: the perceptual and style
    terms are exactly 0 and so is the gradient they send back (sign(0) through the feature L1 and the Gram sign).  The loss
    is then valid + 6 hole + 0.1 tv: each term within the bound of its fp64 value (u + 2 N 2^-53 of its sum of |terms|, times
    its inverse count, and one fp32 rounding), and the gradient EQUAL to the pixel backward called with no VGG gradient and
    the fp32 coefficients WEIGHTS[k] / count; that gradient within 10 u M (the 9 u M of the pixel backward and the rounding of
    each coefficient to fp32) and the bf16 store of the fp64 gradient."""
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    lib = _lib.load()
    crit = _zero_vgg_criterion(feature_range)
    n, h, w = 2, 48, 64
    gen = _gen(f"zero{dtype}{layout}{feature_range}")
    clean = torch.rand(n, 3, h, w, generator=gen, device="cuda")
    mask = torch.from_numpy(random_hole_masks(n, h, w, seed=feature_range)).cuda()
    out = _loss_output(n, h, w, dtype, layout, gen)
    loss = crit(clean * mask, mask, out, clean)
    loss.backward()
    torch.cuda.synchronize()
    terms = crit.last_terms.double()
    assert float(terms[3]) == 0.0 and float(terms[4]) == 0.0, f"perceptual / style terms {terms[3:].tolist()} are not 0"
    # fp64 pixel terms
    v, o = out.detach().double(), clean.double()
    mm = mask.bool()
    cp = torch.where(mm, clean.double() * mask.double(), v)
    d, dh, dv = (v - o).abs(), (cp[..., :-1] - cp[..., 1:]).abs(), (cp[..., :-1, :] - cp[..., 1:, :]).abs()
    cnt = (n * 3 * h * w, n * 3 * h * w, n * 3 * h * (w - 1), n * 3 * (h - 1) * w)
    parts = ((d * mm).sum(), (d * ~mm).sum(), dh.sum(), dv.sum())
    exact = [float(parts[0]) / cnt[0], float(parts[1]) / cnt[1], float(parts[2]) / cnt[2] + float(parts[3]) / cnt[3]]
    errs = [(U + 2 * d.numel() * E53) * float(parts[k]) / cnt[k] for k in range(4)]
    errs = [errs[0], errs[1], errs[2] + errs[3]]
    for k in range(3):
        assert abs(float(terms[k]) - exact[k]) <= errs[k] + 2 * U * exact[k], (k, float(terms[k]), exact[k])
    ref_loss = exact[0] + 6 * exact[1] + 0.1 * exact[2]
    bound = errs[0] + 6 * errs[1] + 0.1 * errs[2] + 2 * U * ref_loss
    lv = float(loss.detach())
    assert abs(lv - ref_loss) <= bound, (lv, ref_loss)
    # the gradient: exactly the direct pixel backward without a VGG gradient
    coef = tuple(_f32(LOSS_WEIGHTS[min(k, 2)] / cnt[k]) for k in range(4))
    plane = mask[:, 0].to(torch.uint8).contiguous()
    raw, orig = (clean * mask).contiguous(), clean.contiguous()
    direct = torch.full_like(out.grad, NAN)
    one = torch.ones(1, device="cuda")
    code = _lib.PCB_BF16 if dtype == torch.bfloat16 else _lib.PCB_F32
    _lib.check(lib.pcb_inpaint_loss_pixel_backward(raw.data_ptr(), orig.data_ptr(), out.data_ptr(), code, _strides(out), plane.data_ptr(),
                                                   n, h, w, None, code, (ctypes.c_float * 4)(*coef), one.data_ptr(), direct.data_ptr(),
                                                   _strides(direct), _st()))
    torch.cuda.synchronize()
    assert bool((out.grad == direct).all()), "the loss's gradient differs from the pixel backward without a VGG gradient"
    exact_coef = tuple(LOSS_WEIGHTS[min(k, 2)] / cnt[k] for k in range(4))
    _, _, g, M = _pixel_ref(raw.double(), orig.double(), v, plane, None, exact_coef, 1.0, False)
    e = 10 * U * M
    assert_within("gradient", out.grad, g, e + STORE[code] * (g.abs() + e))


# ================================================================================================ fixture staleness
def _site_key(s):
    dts = (s["out_dtype"], s["dtype"]) if "out_dtype" in s else ((s["dtype"],) if "dtype" in s else ())
    return (s["fn"], dts, tuple(sorted((k, v) for k, v in s.items() if k.startswith("null_"))))


@pytest.mark.gpu
def test_fixture_covers_the_loss():
    """the loss at 64^2, batch 2 (bf16 NHWC-padded and fp32 NCHW output) reaches no (entry point, dtype pair, null pattern) that
    the fixture lacks"""
    from oracle.inpaint_loss import vgg_state_dict
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor
    spec = importlib.util.spec_from_file_location("make_golden_inpaint_loss_sites", os.path.join(GOLDEN, "make_golden_inpaint_loss_sites.py"))
    gen_mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_mod)
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(vgg_state_dict(0))
    crit = InpaintingLoss(vgg.cuda())
    rec = []
    with gen_mod.recording(_lib.load(), rec):
        gen_mod.run_loss(crit, 2, 64, torch.bfloat16, True, 3)
        gen_mod.run_loss(crit, 2, 64, torch.float32, False, 4)
    assert len({s["fn"] for s in rec}) == 11
    missing = {_site_key(s) for s in rec} - {_site_key(s) for s in _sites()}
    assert not missing, f"the fixture lacks {sorted(missing)}: regenerate tests/golden/inpaint_loss_sites.json"

"""The segmentation-loss kernels (csrc/seg_loss.cu) and the text-mask post-processing kernel (csrc/seg_ops.cu) through the C ABI:

    entry point                  kernel                          cases
    pcb_seg_loss_forward         seg_loss_forward_kernel<DT>     fx_loss_*, geom_*, layout_*, values_*, coef_*
    pcb_seg_loss_backward        seg_loss_backward_kernel<DT>    the same
    pcb_seg_mask_postprocess     seg_mask_post_kernel<T>         post_*, fx_post_*

DT is PCB_F32 (0) or PCB_BF16 (1).  Each case asserts its kernels, their template argument and one launch per call from a
profiler trace (kernel_harness.traced).  One case per call site of tests/golden/seg_loss_sites.json, recorded from the two
training steps at 512^2 (batch 8 and 16, bf16, three losses), fp32 dense NCHW logits at 256^2 and the 600^2 inference with
the demo's post-processing, runs at the recorded size: the point is the production grid.

Loss, per element.  u = 2^-24.  The bound is a running error analysis of the kernel's own fp32 expression (class Ev): every
intermediate carries its exact value and a bound on the error of its fp32 evaluation, propagated first order and
conservatively:
  * a correctly rounded +, -, *, / (every fp32 operation, __fadd_rn and __fdiv_rn included) adds half an ulp of its result,
    at most u |r| + 2^-150; a contracted a*b + c only removes a rounding;
  * expf adds 2 ulp and log1pf 1 ulp of the result (CUDA Programming Guide, maximum ulp errors without fast-math); the error
    of an argument propagates through exp as exp(v + e) - exp(v) and through log1p as e / (1 + v - e);
  * the focal factor f = exp(gamma logsigmoid(-x s)) therefore carries the absolute error of its exponent, about gamma times
    that of logsigmoid, as a relative error: gamma |logsigmoid| u and more, large for |x| near 80 or 100;
  * at a branch on a computed value (the sign of -x s, of x s) the error of both branches is taken where the sign is in doubt.
The reference is oracle/seg_loss.py in fp64 on the same fp32 operands; its own fp64 error is covered by 2^-48 times the
magnitude of the expression (the same expression with every operand made non-negative).  A bf16 gradient is that value
rounded once (2^-8 relative, 2^-133 absolute).

The reduction is exact given the elements: every reduction calls the same element(), so with S the exact sum (math.fsum) of
the fp32 values of the `none` call, `sum` must be fl32 of a value within (count - 1) 2^-53 sum |v| of S (fp64 accumulation in
any order) and `mean` fl32(fl64(. / count)) of such a value: every fp32 value between the roundings of the interval's
endpoints is accepted, almost always exactly one.  Focal has only `mean`; its value is checked against the oracle within
sum(element bounds) / count, the fp64 accumulation and one fp32 rounding.

The gradient scale is exactly one fp32 multiply: focal with gout = count has gs = 1, so dx is the raw per-element g; bootstrap
`sum` with gout = 1 likewise.  Every other call must then give exactly fl32(g * gs) per element, gs = fl32(fl64(gout) / count)
for `mean`, gout for `sum` and gout_e per element for `none`, and a bf16 dx that product rounded once more.  The raw g comes
from an fp32 call on the fp32 values of the logits (for bf16 logits, their exact fp32 widening).

Post-processing is checked bit for bit against the demo's statements on CPU torch (sigmoid > 0.5, MaxPool2d(3, 1, 1) over the
full padded map, crop, bilinear resize with align_corners=False, > 0): the threshold on every bf16 value and every fp32 value
in [2^-25, 2^-23), the taps per axis for every (in, out) in 1..64 x 1..192, 2-D sweeps, the crop border and the production
calls.  Outputs are prefilled with 0x77.  Refused calls launch nothing and write nothing.
"""
import ctypes
import importlib.util
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_harness import GOLDEN, SENTINEL, assert_within, traced
from oracle import seg_loss as OL
from text_segmentation_image_inpainting_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
E53 = 2.0 ** -53
TINY = 2.0 ** -149
BF, F32 = _lib.PCB_BF16, _lib.PCB_F32
DT = {BF: torch.bfloat16, F32: torch.float32}
SHORT = {BF: "bf16", F32: "f32"}
POST_T = {BF: "__nv_bfloat16", F32: "float"}
FOCAL, BOOT = _lib.SEG_FOCAL, _lib.SEG_BOOTSTRAP
NONE, MEAN, SUM = _lib.SEG_NONE, _lib.SEG_MEAN, _lib.SEG_SUM
RED = {NONE: "none", MEAN: "mean", SUM: "sum"}
PER_BLOCK = 256 * 8                     # TPB * EPT of seg_loss.cu
MAX_BLOCKS = 1024
THRESHOLD = float(OL.BOOT_THRESHOLD)    # 1.5 * 2^-24
NAN = float("nan")
FILL = 0x77                             # post-processing prefill


def _sites():
    with open(os.path.join(GOLDEN, "seg_loss_sites.json")) as f:
        return json.load(f)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _strides(t):
    return (ctypes.c_longlong * 4)(*t.stride())


def _f32(v):
    return float(np.float32(v))


def _route(name, want, calls):
    """the check of traced: exactly the kernels of want, one launch per call"""
    def check(records):
        assert set(records) == set(want), f"{name}: ran {sorted(records)}, the case covers {sorted(want)}"
        for k in want:
            assert records[k] == calls[k], f"{name}: {k} launched {records[k]} times for {calls[k]} calls"
    return check


# ================================================================================================ running error analysis
class Ev:
    """a quantity the kernel computes in fp32: v its exact value (fp64), e a bound on the error of its fp32 evaluation, m its
    magnitude (the same expression over absolute values: fp64 evaluations of it are within a few 2^-53 m)"""

    def __init__(self, v, e=None, m=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e
        self.m = v.abs() if m is None else m


def _half_ulp(v):
    return U * v.abs() + TINY / 2


def _const(c, like):
    return Ev(torch.full_like(like, float(c)))


def _add(a, b, sign=1.0):
    v = a.v + sign * b.v
    return Ev(v, a.e + b.e + _half_ulp(v), a.m + b.m)


def _mul(a, b):
    v = a.v * b.v
    return Ev(v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e + _half_ulp(v), a.m * b.m)


def _div(a, b):
    v = a.v / b.v
    return Ev(v, (a.e + v.abs() * b.e) / (b.v.abs() - b.e) + _half_ulp(v), a.m / (b.v.abs() - b.e))


def _neg(a):
    return Ev(-a.v, a.e, a.m)


def _expf(a):
    v = torch.exp(a.v)
    hi = torch.exp(a.v + a.e)
    return Ev(v, (hi - v) + 4 * _half_ulp(hi), v * (1 + a.m))


def _log1pf(a):
    v = torch.log1p(a.v)
    return Ev(v, a.e / (1 + (a.v - a.e).clamp(min=-0.5)) + 2 * _half_ulp(v), torch.log1p(a.m) + a.m)


def _where(cond, a, b):
    return Ev(torch.where(cond, a.v, b.v), torch.where(cond, a.e, b.e), torch.where(cond, a.m, b.m))


def _branch(y, a, b):
    """a where y >= 0 else b, for a branch the kernel takes on the computed sign of y: both errors where that sign is in doubt"""
    r = _where(y.v >= 0, a, b)
    doubt = y.v.abs() <= y.e
    both = torch.maximum(a.e.nan_to_num(posinf=0), b.e.nan_to_num(posinf=0)) + (a.v - b.v).abs().nan_to_num(posinf=0)
    return Ev(r.v, torch.where(doubt, both, r.e), r.m)


def _sigmoid(y):
    one = _const(1, y.v)
    pos = _div(one, _add(one, _expf(_neg(y))))
    e = _expf(y)
    neg = _div(e, _add(one, e))
    return _branch(y, pos, neg)


def _log_sigmoid(z):
    nonneg = _neg(_log1pf(_expf(_neg(z))))
    neg = _add(z, _log1pf(_expf(z)), -1.0)
    return _branch(z, nonneg, neg)


def _bce(x, y):
    one = _const(1, x.v)
    p = _where(x.v >= 0, _mul(x, _add(one, y, -1.0)), _mul(_neg(x), y))
    return _add(p, _log1pf(_expf(_neg(Ev(x.v.abs())))))


def element(x, t, loss, p0, omb, bg, words):
    """(loss, d loss / d x) of seg_loss.cu's element() on fp32 operands x, t (fp64 CUDA tensors), as Ev"""
    X, T = Ev(x), Ev(t)
    W = Ev(torch.where(t > 0, torch.full_like(t, words), torch.full_like(t, bg)))
    if loss == FOCAL:
        s = _add(Ev(2 * t), _const(1, t), -1.0)
        b = _bce(X, T)
        f = _expf(_mul(_const(p0, t), _log_sigmoid(_mul(_neg(X), s))))
        q = _mul(_mul(_mul(_const(-p0, t), s), _sigmoid(_mul(X, s))), b)
        g = _mul(_mul(W, f), _add(_add(q, _sigmoid(X)), T, -1.0))
        return _mul(_mul(f, W), b), g
    tb = _add(_mul(_const(p0, t), T), Ev(torch.where(x > THRESHOLD, torch.full_like(x, omb), torch.zeros_like(x))))
    return _mul(W, _bce(X, tb)), _mul(W, _add(_sigmoid(X), tb, -1.0))


def oracle(x, t, loss, p0, omb, bg, words):
    """oracle/seg_loss.py in fp64: (per-element loss, per-element gradient of the summed loss), numpy"""
    if loss == FOCAL:
        _, g = OL.focal(x, t, gamma=p0, background_weights=bg, words_weights=words)
        tt = np.asarray(t, np.float64)
        w, s = np.where(tt > 0, words, bg), 2 * tt - 1
        le = np.exp(p0 * OL.log_sigmoid(-x * s)) * w * OL.bce(x, tt)
        return le, g * x.size
    # OL.bootstrap with the two fp32 coefficients the kernel receives (it would take 1 - beta in fp64)
    w, tb = np.where(t > 0, words, bg), p0 * t + omb * OL.indicator(x.astype(np.float32))
    return w * OL.bce(x, tb), w * (OL.sigmoid(x) - tb)


# ================================================================================================ operands and layouts
def _layout(kind, n, h, w, dtype, fill):
    """(logical [n, 1, h, w] view, whole buffer, the view of a buffer): nchw dense; nhwcC the [:, :1] view of a C-channel NHWC
    buffer (SENTINEL elsewhere); swap a dense [n, 1, w, h] buffer transposed; col2 every second column of [n, 1, h, 2w] (to
    ops.nhwc_layout an NHWC view with channel stride 2); sub2 every second row and column of [n, 1, 2h, 2w] (no NHWC view)"""
    if kind == "nchw":
        buf = torch.empty(n, 1, h, w, dtype=dtype, device="cuda")
        of = lambda b: b                                                   # noqa: E731
    elif kind.startswith("nhwc"):
        buf = torch.full((n, h, w, int(kind[4:])), SENTINEL, dtype=dtype, device="cuda")
        of = lambda b: b.permute(0, 3, 1, 2)[:, :1]                        # noqa: E731
    elif kind == "swap":
        buf = torch.empty(n, 1, w, h, dtype=dtype, device="cuda")
        of = lambda b: b.transpose(2, 3)                                   # noqa: E731
    elif kind == "col2":
        buf = torch.full((n, 1, h, 2 * w), SENTINEL, dtype=dtype, device="cuda")
        of = lambda b: b[..., ::2]                                         # noqa: E731
    elif kind == "sub2":
        buf = torch.full((n, 1, 2 * h, 2 * w), SENTINEL, dtype=dtype, device="cuda")
        of = lambda b: b[..., ::2, ::2]                                    # noqa: E731
    else:
        raise AssertionError(kind)
    view = of(buf)
    view.copy_(fill) if isinstance(fill, torch.Tensor) else view.fill_(fill)
    return view, buf, of


def _outside_kept(buf, of, name):
    rest = buf.clone()
    of(rest).fill_(SENTINEL)
    assert bool((rest == SENTINEL).all()), f"{name}: written outside the [:, :1] view"


SPECIAL_X = [0.0, -0.0, TINY, -TINY, 2.0 ** -130, -(2.0 ** -130), 2.0 ** -126, THRESHOLD, np.nextafter(np.float32(THRESHOLD), np.float32(1)),
             np.nextafter(np.float32(THRESHOLD), np.float32(0)), -THRESHOLD, 2.0 ** -24, 2.0 ** -23, 1.0, -1.0, 20.0, -20.0, 88.0, -88.0,
             100.0, -100.0]
HUGE_X = [1e30, -1e30]
SPECIAL_T = [0.0, TINY, 2.0 ** -126, 0.5, 1.0, 1.0 - U, U]


def operands(n, h, w, seed, dtype=torch.float32, hard=False, specials=True):
    """(x as stored in dtype, widened to fp32, dense [n, 1, h, w] on the device; t fp32 dense): Gaussian logits times 4 with the
    special values spread through them, hard {0, 1} or soft targets with 0, the smallest subnormal and 1 spread through"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    cnt = n * h * w
    x = torch.randn(cnt, generator=g, device="cuda") * 4
    t = (torch.rand(cnt, generator=g, device="cuda") < 0.3).float() if hard else torch.rand(cnt, generator=g, device="cuda")
    if specials and cnt > 1:
        sx = torch.tensor(SPECIAL_X + (HUGE_X if dtype == torch.float32 else []), dtype=torch.float32, device="cuda")
        idx = torch.randperm(cnt, generator=g, device="cuda")[: min(cnt // 2, 64 * sx.numel())]
        x[idx] = sx.repeat(len(idx) // sx.numel() + 1)[: len(idx)]
        st = torch.tensor([0.0, 1.0, TINY] if hard else SPECIAL_T, dtype=torch.float32, device="cuda")
        jdx = torch.randperm(cnt, generator=g, device="cuda")[: min(cnt // 2, 64 * st.numel())]
        t[jdx] = st.repeat(len(jdx) // st.numel() + 1)[: len(jdx)]
    x = x.to(dtype).float()
    return x.view(n, 1, h, w), t.view(n, 1, h, w)


# ================================================================================================ calling the kernels
class Workspace:
    """fp64 partials (NaN-prefilled) for MAX_BLOCKS blocks and the uint32 counter"""

    def __init__(self):
        self.partials = torch.full((MAX_BLOCKS,), NAN, dtype=torch.float64, device="cuda")
        self.counter = torch.zeros(1, dtype=torch.int32, device="cuda")


def forward(x, code, t, loss, red, coefs, ws, out=None):
    lib = _lib.load()
    n, _, h, w = x.shape
    if out is None:
        out = torch.full((n * h * w,) if red == NONE else (1,), NAN, device="cuda")
    _lib.check(lib.pcb_seg_loss_forward(x.data_ptr(), code, _strides(x), t.data_ptr(), n, h, w, loss, red, *coefs,
                                        ws.partials.data_ptr(), ws.counter.data_ptr(), out.data_ptr(), _st()))
    return out


def backward(x, code, t, loss, red, coefs, gout, dx):
    lib = _lib.load()
    n, _, h, w = x.shape
    _lib.check(lib.pcb_seg_loss_backward(x.data_ptr(), code, _strides(x), t.data_ptr(), n, h, w, loss, red, *coefs, gout.data_ptr(),
                                         dx.data_ptr(), _strides(dx), _st()))


def _accepted(lo, hi, count, red):
    """the fp32 values an fp64 total in [lo, hi] becomes: fl32(total) for sum, fl32(fl64(total / count)) for mean"""
    if red == MEAN:
        lo, hi = lo / count, hi / count
    return float(np.float32(lo)), float(np.float32(hi))


def _reference(x32, t, loss, coefs):
    """(oracle loss elements, oracle gradient, Ev of the loss, Ev of the gradient), all fp64 CUDA, flat in element order"""
    xd, td = x32.double().flatten(), t.double().flatten()
    le, ge = oracle(xd.cpu().numpy(), td.cpu().numpy(), loss, *coefs)
    lv, gv = element(xd, td, loss, *coefs)
    return torch.from_numpy(le).cuda(), torch.from_numpy(ge).cuda(), lv, gv


def _bound(ev):
    """the error bound of ev, the fp64 error of the reference and one subnormal ulp (results below 2^-150 round either way)"""
    return ev.e + 2.0 ** -48 * ev.m + TINY


def check_loss(name, x32, t, code, layout, dx_layout, loss, red, coefs, ws, ref=None, trace=True):
    """Every check of the module docstring for one (loss, reduction) on x32 (fp32 values of the logits, dense), read as dtype
    `code` in `layout`, with dx written in `dx_layout`.  Returns the reference for reuse."""
    n, _, h, w = x32.shape
    count = n * h * w
    dt = DT[code]
    tag = f"{name} [{'focal' if loss == FOCAL else 'bootstrap'} {RED[red]}]"
    if ref is None:
        ref = _reference(x32, t, loss, coefs)
    le, ge, lv, gv = ref
    x, xbuf, xof = _layout(layout, n, h, w, dt, x32.to(dt))
    assert torch.equal(x.float(), x32), f"{tag}: the logits are not representable in {dt}"
    # ---------------------------------------------------------------- raw gradient: fp32, dense, gs = 1
    raw_red, raw_gout = (MEAN, float(count)) if loss == FOCAL else (SUM, 1.0)
    g32 = torch.full((n, 1, h, w), NAN, device="cuda")
    backward(x32, F32, t, loss, raw_red, coefs, torch.tensor([raw_gout], device="cuda"), g32)
    torch.cuda.synchronize()
    gflat = g32.flatten().double()
    assert_within(f"{tag}: raw gradient vs the fp64 oracle", gflat, ge, _bound(gv))
    # ---------------------------------------------------------------- the case's own call pair
    if red == NONE:
        gout = (torch.rand(count, 1, generator=torch.Generator(device="cuda").manual_seed(count), device="cuda") * 3 - 1).float()
        scale = gout.flatten().double()
    else:
        gval = 0.7 if red == MEAN else 1.7
        gout = torch.tensor([gval], device="cuda")
        scale = _f32(_f32(gval) / count) if red == MEAN else _f32(gval)
    out = torch.full((count,) if red == NONE else (1,), NAN, device="cuda")
    dx, dxbuf, dxof = _layout(dx_layout, n, h, w, dt, NAN)
    dxbuf0 = dxbuf.clone()
    assert int(ws.counter.item()) == 0, f"{tag}: the counter is not 0 before the call"

    def run():
        forward(x, code, t, loss, red, coefs, ws, out)
        backward(x, code, t, loss, red, coefs, gout, dx)
    calls = {("seg_loss_forward_kernel", (str(code),)): 1, ("seg_loss_backward_kernel", (str(code),)): 1}
    if trace:
        traced(tag, run, _route(tag, calls, calls), [(out, NAN), (dxbuf, dxbuf0)])
    else:
        run()
    torch.cuda.synchronize()
    assert int(ws.counter.item()) == 0, f"{tag}: the counter is not 0 after the call"
    # gradient: exactly one fp32 multiply of the raw g, then the store in dtype, in dx's layout, and nothing else written
    want = (gflat * scale).float().to(dt)
    got = dx.reshape(-1)
    bad = ~((got == want) | (got.isnan() & want.isnan()))
    assert not bool(bad.any()), (f"{tag}: {int(bad.sum())} of {count} gradient elements are not fl32(g * gs); first at "
                                 f"{int(bad.nonzero()[0])}: got {float(got[bad][0])!r}, want {float(want[bad][0])!r}")
    assert not bool(got.isnan().any()), f"{tag}: gradient left unwritten"
    if dx_layout != "nchw" and dx_layout != "swap":
        _outside_kept(dxbuf, dxof, f"{tag}: dx")
    if layout != "nchw" and layout != "swap":
        _outside_kept(xbuf, xof, f"{tag}: x")
    # ---------------------------------------------------------------- forward
    if loss == BOOT:
        elems = out if red == NONE else forward(x, code, t, BOOT, NONE, coefs, ws)
        torch.cuda.synchronize()
        assert int(ws.counter.item()) == 0
        assert_within(f"{tag}: loss elements vs the fp64 oracle", elems.double(), le, _bound(lv))
        if red != NONE:
            vals = elems.double().cpu().numpy()
            S = math.fsum(vals.tolist())
            E = (count - 1) * E53 * float(np.abs(vals).sum()) * (1 + 1e-6) + 4 * E53 * abs(S)
            lo, hi = _accepted(S - E, S + E, count, red)
            got1 = float(out[0])
            assert lo <= got1 <= hi, f"{tag}: {got1!r} is not the fp32 rounding of a total within {E:.3e} of {S!r} (accepted [{lo!r}, {hi!r}])"
    if red != NONE:
        total_ref = float(le.sum())
        err = float(_bound(lv).sum()) + count * E53 * float(le.abs().sum())
        if red == MEAN:
            total_ref, err = total_ref / count, err / count
        assert abs(float(out[0]) - total_ref) <= err + U * abs(total_ref) + TINY, f"{tag}: {float(out[0])!r} vs the oracle's {total_ref!r}"
    # repeated calls are bit-identical
    again = forward(x, code, t, loss, red, coefs, ws)
    dx2 = torch.full_like(dx, NAN)
    backward(x, code, t, loss, red, coefs, gout, dx2)
    torch.cuda.synchronize()
    assert torch.equal(again, out) and torch.equal(dx2, dx), f"{tag}: a repeated call differs"
    assert int(ws.counter.item()) == 0
    return ref


def _boot(beta, bg=1.0, words=2.0):
    """the coefficients loss.SoftBootstrapCrossEntropy passes: fp32(beta), fp32(1 - beta) and the weights"""
    return (_f32(beta), _f32(1 - beta), _f32(bg), _f32(words))


def _focal(gamma, bg=1.0, words=2.0):
    return (_f32(gamma), 0.0, _f32(bg), _f32(words))


ALL = ((FOCAL, MEAN), (BOOT, NONE), (BOOT, MEAN), (BOOT, SUM))


def run_all(name, sp, ws=None):
    n, h, w = sp["shape"]
    ws = ws or Workspace()
    x32, t = operands(n, h, w, sp.get("seed", n * 7919 + h * 31 + w), DT[sp["dtype"]], sp.get("hard", False), sp.get("specials", True))
    for loss, red in sp.get("pairs", ALL):
        coefs = sp.get("coefs", {}).get(loss) or (_focal(2.0) if loss == FOCAL else _boot(0.95))
        check_loss(name, x32, t, sp["dtype"], sp.get("layout", "nchw"), sp.get("dx", "nchw"), loss, red, coefs, ws)


# ================================================================================================ fixture sites
def _kind(strides, h, w):
    s = list(strides)
    if s == [h * w, h * w, w, 1]:
        return "nchw"
    c = s[3]
    if s == [c * h * w, 1, c * w, c]:
        return f"nhwc{c}"
    raise AssertionError(f"no layout has strides {strides} at {h}x{w}")


def _site_case(s):
    """(family, case name, spec) of a fixture site"""
    if s["fn"] == "pcb_seg_mask_postprocess":
        name = f"fx_post_{SHORT[s['dtype']]}_n{s['n']}_{s['h']}x{s['w']}_c{s['cstride']}_crop{s['h_valid']}x{s['w_valid']}_to{s['oh']}x{s['ow']}"
        return "post", name, dict(s)
    n, h, w = s["n"], s["h"], s["w"]
    loss, red = s["loss"], s["reduction"]
    coefs = (s["p0"], s["one_minus_beta"], s["background_weight"], s["words_weight"])
    lay = _kind(s["x_strides"], h, w)
    dxl = _kind(s["dx_strides"], h, w) if "dx_strides" in s else lay
    fwd = s["fn"].endswith("forward")
    name = (f"fx_loss_{'fwd' if fwd else 'bwd'}_{SHORT[s['dtype']]}_n{n}_{h}x{w}_{lay}_{'focal' if loss == FOCAL else 'boot'}{RED[red]}"
            f"_p{coefs[0]:g}" + ("" if fwd else f"_dx{dxl}"))
    return "loss", name, dict(shape=(n, h, w), dtype=s["dtype"], layout=lay, dx=dxl if not fwd else ("nhwc8" if lay != "nchw" else "nchw"),
                              pairs=((loss, red),), coefs={loss: coefs}, hard=True)


def _fixture(fam):
    return {name: sp for f, name, sp in map(_site_case, _sites()) if f == fam}


def test_fixture_sites_map_to_cases():
    sites = _sites()
    fns = {s["fn"] for s in sites}
    assert fns == {"pcb_seg_loss_forward", "pcb_seg_loss_backward", "pcb_seg_mask_postprocess"}, fns
    names = [_site_case(s)[1] for s in sites]
    assert len(set(names)) == len(names), "two sites map to one case"
    counts = {s["n"] * s["h"] * s["w"] for s in sites if s["fn"] != "pcb_seg_mask_postprocess"}
    assert 8 * 512 * 512 in counts and 16 * 512 * 512 in counts, counts


@pytest.mark.parametrize("name", sorted(_fixture("loss")))
def test_fixture_loss_sites(name):
    run_all(name, _fixture("loss")[name])


# ================================================================================================ hand cases
def _geom_shape(count):
    return {1: (1, 1, 1), 2047: (1, 23, 89), 2048: (2, 32, 32), 2049: (3, 1, 683), 524288: (2, 512, 512), 524289: (3, 1, 174763),
            2097152: (8, 512, 512), 2097153: (3, 3, 233017), 4194304: (16, 512, 512)}[count]


GEOM = {f"geom_{c}": dict(shape=_geom_shape(c), dtype=F32 if i % 2 else BF, layout=("nchw", "nhwc8", "nhwc16")[i % 3],
                          dx=("nhwc8", "nchw", "swap")[i % 3])
        for i, c in enumerate((1, 2047, 2048, 2049, 524288, 524289, 2097152, 2097153, 4194304))}
SHAPES = {"shape_n1_h1_w1": (1, 1, 1), "shape_h1": (2, 1, 301), "shape_w1": (3, 97, 1), "shape_odd": (2, 37, 53), "shape_n1_odd": (1, 129, 65)}
LAYOUTS = ("nchw", "nhwc8", "nhwc16", "swap", "col2")
HAND = {
    **GEOM,
    **{name: dict(shape=s, dtype=BF if i % 2 else F32, layout=LAYOUTS[i % 5], dx=LAYOUTS[(i + 2) % 5]) for i, (name, s) in enumerate(SHAPES.items())},
    **{f"layout_{SHORT[code]}_{a}_dx_{b}": dict(shape=(3, 19, 41), dtype=code, layout=a, dx=b, seed=17)
       for code in (F32, BF) for a in LAYOUTS for b in LAYOUTS if a == b or (code == F32) == (LAYOUTS.index(a) % 2 == 0)},
    **{f"values_{SHORT[code]}_{'hard' if hard else 'soft'}": dict(shape=(2, 48, 80), dtype=code, hard=hard, layout="nhwc8" if code == BF else "nchw",
                                                                  dx="nchw" if code == BF else "col2")
       for code in (F32, BF) for hard in (False, True)},
}


@pytest.mark.parametrize("name", sorted(HAND))
def test_loss_case(name):
    run_all(name, HAND[name])


COEFS = [(g, b, wt) for g in (0.0, 0.5, 1.0, 2.0) for b in (0.0, 0.95, 1.0) for wt in ((1.0, 2.0), (0.25, 3.0))]


@pytest.mark.parametrize("gamma,beta,weights", COEFS, ids=[f"g{g}_b{b}_w{wt[0]}-{wt[1]}" for g, b, wt in COEFS])
def test_loss_coefficients(gamma, beta, weights):
    name = f"coef_g{gamma}_b{beta}_w{weights}"
    sp = dict(shape=(2, 33, 47), dtype=F32 if beta != 0.95 else BF, layout="nhwc8", dx="nchw",
              coefs={FOCAL: _focal(gamma, *weights), BOOT: _boot(beta, *weights)},
              pairs=((FOCAL, MEAN), (BOOT, NONE), (BOOT, MEAN if gamma in (0.0, 1.0) else SUM)))
    run_all(name, sp)


def test_subnormal_target_takes_the_words_weight():
    """t = 0 takes the background weight and the smallest positive subnormal t the words weight (the switch is t > 0)"""
    ws = Workspace()
    x = torch.tensor([2.0, 2.0, -3.0, -3.0], device="cuda").view(1, 1, 1, 4)
    t = torch.tensor([0.0, TINY, 0.0, TINY], device="cuda").view(1, 1, 1, 4)
    for coefs in (_boot(0.95, 0.25, 3.0), _boot(0.0, 1.0, 2.0)):
        out = forward(x, F32, t, BOOT, NONE, coefs, ws)
        torch.cuda.synchronize()
        le, _, lv, _ = _reference(x, t, BOOT, coefs)
        assert_within("subnormal target", out.double(), le, _bound(lv))
        r = out.cpu()
        assert abs(float(r[1] / r[0]) - coefs[3] / coefs[2]) < 1e-5 and abs(float(r[3] / r[2]) - coefs[3] / coefs[2]) < 1e-5, r


def test_workspace_reused_across_counts():
    """one workspace through counts of the same block count (2049, 4096: 2 blocks), then other block counts: the counter is 0
    after every call and every sum follows from its elements"""
    ws = Workspace()
    for i, shape in enumerate([(3, 1, 683), (2, 32, 64), (1, 23, 89), (3, 1, 174763), (2, 32, 64), (1, 1, 1)]):
        x32, t = operands(*shape, seed=100 + i)
        check_loss(f"workspace_{i}", x32, t, F32, "nchw", "nchw", BOOT, SUM, _boot(0.95), ws, trace=False)
        check_loss(f"workspace_{i}", x32, t, F32, "nchw", "nchw", FOCAL, MEAN, _focal(2.0), ws, trace=False)


def test_loss_module_gradient_layouts():
    """through loss.py: an NHWC view x (channel-padded, or every second column, an NHWC view with channel stride 2) gets a
    channel-padded dx, a dense x with other strides a dx of its own strides, and a strided x that is no NHWC view a contiguous
    one, both from empty_like; either way dx is exactly fl32(g * fl32(1 / count)) of the raw gradient"""
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss, SoftBootstrapCrossEntropy
    n, h, w = 2, 24, 40
    for code in (F32, BF):
        x32, t = operands(n, h, w, seed=7, dtype=DT[code])
        for layout in LAYOUTS + ("sub2",):
            for crit, loss, coefs in ((BinaryFocalLoss(gamma=2), FOCAL, _focal(2.0)), (SoftBootstrapCrossEntropy(), BOOT, _boot(0.95))):
                x, _, _ = _layout(layout, n, h, w, DT[code], x32.to(DT[code]))
                x.requires_grad_(True)
                raw = []
                x.register_hook(lambda g: raw.append(g))
                crit(x, t).backward()
                g32 = torch.full((n, 1, h, w), NAN, device="cuda")
                backward(x32, F32, t, loss, SUM if loss == BOOT else MEAN, coefs,
                         torch.tensor([1.0 if loss == BOOT else float(n * h * w)], device="cuda"), g32)
                torch.cuda.synchronize()
                d = raw[0]
                if layout.startswith("nhwc") or layout == "col2":
                    assert ops.nhwc_layout(d) == 8 and not d.is_contiguous(), (layout, d.stride())
                elif layout == "swap":
                    assert d.stride() == x.stride()
                else:
                    assert d.is_contiguous() and (layout == "nchw" or not x.is_contiguous()), (layout, d.stride())
                want = (g32.double() * _f32(1.0 / (n * h * w))).float().to(DT[code])
                assert torch.equal(d, want), f"{layout} {SHORT[code]}: the module's gradient is not fl32(g * gs)"


# ================================================================================================ refusals
def _loss_refusals():
    lib, st = _lib.load(), _st()
    x = torch.zeros(1, 1, 4, 8, device="cuda")
    t = torch.zeros(1, 1, 4, 8, device="cuda")
    xs = _strides(x)
    ws = Workspace()
    out = torch.full((32,), NAN, device="cuda")
    dx = torch.full((1, 1, 4, 8), NAN, device="cuda")
    gout = torch.ones(32, device="cuda")
    outs = [out, dx, ws.partials, ws.counter]
    P = lambda v: None if v is None else v.data_ptr()                                       # noqa: E731

    def fwd(xp=x, dtype=F32, tp=t, n=1, h=4, w=8, loss=BOOT, red=MEAN, partials=ws.partials, counter=ws.counter, o=out):
        return lambda: lib.pcb_seg_loss_forward(P(xp), dtype, xs, P(tp), n, h, w, loss, red, 0.95, _f32(0.05), 1.0, 2.0, P(partials),
                                                P(counter), P(o), st)

    def bwd(xp=x, dtype=F32, tp=t, n=1, h=4, w=8, loss=BOOT, red=MEAN, g=gout, d=dx):
        return lambda: lib.pcb_seg_loss_backward(P(xp), dtype, xs, P(tp), n, h, w, loss, red, 0.95, _f32(0.05), 1.0, 2.0, P(g), P(d),
                                                 _strides(dx), st)
    r = {}
    for k, f in (("fwd", fwd), ("bwd", bwd)):
        r[f"{k}_null_x"] = f(xp=None)
        r[f"{k}_null_target"] = f(tp=None)
        r[f"{k}_dtype_2"] = f(dtype=2)
        r[f"{k}_dtype_neg"] = f(dtype=-1)
        r[f"{k}_loss_2"] = f(loss=2)
        r[f"{k}_reduction_3"] = f(red=3)
        r[f"{k}_reduction_neg"] = f(red=-1)
        r[f"{k}_n0"] = f(n=0)
        r[f"{k}_h0"] = f(h=0)
        r[f"{k}_w_neg"] = f(w=-4)
        r[f"{k}_focal_sum"] = f(loss=FOCAL, red=SUM)
        r[f"{k}_focal_none"] = f(loss=FOCAL, red=NONE)
    r["fwd_mean_null_partials"] = fwd(partials=None)
    r["fwd_mean_null_counter"] = fwd(counter=None)
    r["fwd_sum_null_partials"] = fwd(red=SUM, partials=None)
    r["fwd_sum_null_counter"] = fwd(red=SUM, counter=None)
    r["fwd_null_out"] = fwd(o=None)
    r["bwd_null_gout"] = bwd(g=None)
    r["bwd_null_dx"] = bwd(d=None)
    return r, outs


def _post_refusals():
    lib, st = _lib.load(), _st()
    x = torch.zeros(2, 8, 8, 8, device="cuda")
    out = torch.full((2 * 16 * 16,), FILL, dtype=torch.uint8, device="cuda")

    def f(xp=True, dtype=F32, n=2, h=8, w=8, cs=8, hv=8, wv=8, oh=16, ow=16, o=True):
        return lambda: lib.pcb_seg_mask_postprocess(x.data_ptr() if xp else None, dtype, n, h, w, cs, hv, wv, oh, ow,
                                                    out.data_ptr() if o else None, st)
    r = {"post_null_logits": f(xp=False), "post_null_out": f(o=False), "post_dtype_2": f(dtype=2), "post_dtype_neg": f(dtype=-1),
         "post_h_valid_0": f(hv=0), "post_h_valid_past": f(hv=9), "post_w_valid_0": f(wv=0), "post_w_valid_past": f(wv=9),
         "post_oh_0": f(oh=0), "post_ow_neg": f(ow=-1), "post_cstride_0": f(cs=0), "post_cstride_neg": f(cs=-8), "post_n0": f(n=0),
         "post_h0": f(h=0, hv=0), "post_w_neg": f(w=-8, wv=-8)}
    return r, [out]


def _refusal_names():
    # the names only; building the calls needs the device
    names = [f"{k}_{s}" for k in ("fwd", "bwd") for s in ("null_x", "null_target", "dtype_2", "dtype_neg", "loss_2", "reduction_3",
                                                           "reduction_neg", "n0", "h0", "w_neg", "focal_sum", "focal_none")]
    names += ["fwd_mean_null_partials", "fwd_mean_null_counter", "fwd_sum_null_partials", "fwd_sum_null_counter", "fwd_null_out",
              "bwd_null_gout", "bwd_null_dx"]
    names += ["post_null_logits", "post_null_out", "post_dtype_2", "post_dtype_neg", "post_h_valid_0", "post_h_valid_past",
              "post_w_valid_0", "post_w_valid_past", "post_oh_0", "post_ow_neg", "post_cstride_0", "post_cstride_neg", "post_n0", "post_h0",
              "post_w_neg"]
    return names


@pytest.mark.parametrize("name", _refusal_names())
def test_refusals_launch_and_write_nothing(name):
    calls, outs = _post_refusals() if name.startswith("post_") else _loss_refusals()
    call = calls[name]
    before_vals = [t.clone() for t in outs]
    torch.cuda.synchronize()
    before = _lib.launch_count()
    assert call() != 0, f"{name}: accepted"
    torch.cuda.synchronize()
    assert _lib.launch_count() == before, f"{name}: a refused call launched a kernel"
    for t, b in zip(outs, before_vals):
        assert torch.equal(t.isnan(), b.isnan()) and torch.equal(t.nan_to_num(), b.nan_to_num()), f"{name}: a refused call wrote"


# ================================================================================================ post-processing
def post_ref(x, hv, wv, oh, ow):
    """the demo's statements on CPU torch: x fp32 [n, 1, h, w] (CPU) -> uint8 [n, 1, oh, ow]"""
    m = (torch.sigmoid(x.float()) > 0.5).float()
    m = torch.nn.MaxPool2d(kernel_size=(3, 3), padding=(1, 1), stride=1)(m).byte()
    m = m[:, :, :hv, :wv]
    return (F.interpolate(m.float(), size=(oh, ow), mode="bilinear", align_corners=False) > 0).to(torch.uint8)


def post_gpu(x32, code, cs, hv, wv, oh, ow, name=None):
    """pcb_seg_mask_postprocess of x32 (fp32 CPU [n, 1, h, w]) stored in dtype code as the [:, :1] view of a cs-channel NHWC
    buffer (SENTINEL elsewhere); traced when name is given"""
    n, _, h, w = x32.shape
    buf = torch.full((n, h, w, cs), SENTINEL, dtype=DT[code], device="cuda")
    buf[..., 0] = x32[:, 0].to(DT[code]).cuda()
    out = torch.full((n, 1, oh, ow), FILL, dtype=torch.uint8, device="cuda")
    lib = _lib.load()
    run = lambda: _lib.check(lib.pcb_seg_mask_postprocess(buf.data_ptr(), code, n, h, w, cs, hv, wv, oh, ow, out.data_ptr(), _st()))  # noqa: E731
    if name is not None:
        k = {("seg_mask_post_kernel", (POST_T[code],)): 1}
        traced(name, run, _route(name, k, k), [(out, FILL)])
    else:
        run()
    return out


def assert_post(name, got, want):
    got = got.cpu()
    assert bool(((got == 0) | (got == 1)).all()), f"{name}: bytes other than 0 and 1 (0x77: unwritten)"
    bad = got != want
    if bool(bad.any()):
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} mask pixels differ; first at {bad.nonzero()[0].tolist()}")


def _threshold_values():
    bf = torch.arange(0, 65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    bits = np.arange(0x33000000, 0x34000000, dtype=np.int64).astype(np.int32).view(np.float32)
    th = np.float32(THRESHOLD)
    near = [th, np.nextafter(th, np.float32(1)), np.nextafter(th, np.float32(0)), np.nextafter(np.nextafter(th, np.float32(1)), np.float32(1))]
    f = np.concatenate([bits, -bits, near, [-v for v in near]]).astype(np.float32)
    return bf, torch.from_numpy(f)


@pytest.mark.parametrize("code", [BF, F32], ids=["bf16_every_value", "f32_near_zero"])
def test_post_threshold_sweep(code):
    """1x1 images, out 1x1: the mask is the threshold of one logit, with nothing pooled or resized"""
    bf, f = _threshold_values()
    vals = bf.float() if code == BF else f
    x = vals.view(-1, 1, 1, 1)
    got = post_gpu(x, code, 1, 1, 1, 1, 1, name=f"threshold {SHORT[code]}")
    torch.cuda.synchronize()
    want = (torch.sigmoid(vals) > 0.5).to(torch.uint8).view(-1, 1, 1, 1)
    assert torch.equal(want.view(-1), (vals > THRESHOLD).to(torch.uint8)), "torch's CPU sigmoid threshold moved"
    bad = (got.cpu() != want).view(-1)
    assert not bool(bad.any()), (f"threshold {SHORT[code]}: {int(bad.sum())} values disagree with torch.sigmoid(x) > 0.5, e.g. "
                                 f"{vals[bad][:8].tolist()}")


@pytest.mark.parametrize("axis", ["h", "w"])
def test_post_taps_per_axis(axis):
    """maps of one row (or column) for every in in 1..64 and out in 1..192, one image per positive position plus two random
    sparse ones"""
    g = torch.Generator().manual_seed(1 if axis == "h" else 2)
    for size in range(1, 65):
        imgs = torch.full((size + 2, size), -2.0)
        imgs[torch.arange(size), torch.arange(size)] = 2.0
        imgs[size:] = torch.where(torch.rand(2, size, generator=g) < 0.15, 2.0, -2.0)
        x = imgs.view(size + 2, 1, 1, size) if axis == "w" else imgs.view(size + 2, 1, size, 1)
        outs = []
        for out in range(1, 193):
            oh, ow = (1, out) if axis == "w" else (out, 1)
            h, w = x.shape[2:]
            outs.append((out, post_gpu(x, F32, 1, h, w, oh, ow)))
        torch.cuda.synchronize()
        for out, got in outs:
            oh, ow = (1, out) if axis == "w" else (out, 1)
            assert_post(f"taps {axis} in {size} out {out}", got, post_ref(x, x.shape[2], x.shape[3], oh, ow))


SWEEPS = [(n, h, w, hv, wv, oh, ow) for n, h, w, hv, wv, oh, ow in
          ((1, 40, 40, 40, 40, 40, 40), (2, 37, 53, 31, 50, 45, 70), (3, 64, 64, 60, 48, 23, 17), (4, 29, 31, 29, 20, 100, 61),
           (2, 48, 48, 48, 36, 75, 100), (4, 17, 96, 11, 96, 11, 300))]


@pytest.mark.parametrize("cs", [1, 8, 16])
@pytest.mark.parametrize("code", [F32, BF], ids=["f32", "bf16"])
def test_post_2d_sweeps(code, cs):
    for i, (n, h, w, hv, wv, oh, ow) in enumerate(SWEEPS):
        for density in (0.003, 0.05, 0.3, 0.7):
            g = torch.Generator().manual_seed(1000 * i + int(density * 1000) + cs)
            x = torch.randn(n, 1, h, w, generator=g) * 4
            x = torch.where(torch.rand(n, 1, h, w, generator=g) < density, x.abs() + 0.01, -x.abs() - 0.01).to(DT[code]).float()
            name = f"sweep {SHORT[code]} c{cs} {n}x{h}x{w} crop {hv}x{wv} to {oh}x{ow} density {density}"
            got = post_gpu(x, code, cs, hv, wv, oh, ow, name=name if density == 0.05 else None)
            torch.cuda.synchronize()
            assert_post(name, got, post_ref(x, hv, wv, oh, ow))


@pytest.mark.parametrize("code", [F32, BF], ids=["f32", "bf16"])
def test_post_crop_border(code):
    """positives only in the cropped-away rows and columns [h_valid, h), [w_valid, w): pooling runs before the crop, so they
    reach row h_valid - 1 (column w_valid - 1) and nothing else"""
    n, h, w, hv, wv = 2, 40, 48, 32, 36
    x = torch.full((n, 1, h, w), -3.0)
    x[0, 0, hv, ::5] = 3.0
    x[0, 0, ::7, wv] = 3.0
    x[1, 0, hv + 1:, :] = 3.0                       # beyond reach of the pool: nothing
    x[1, 0, 5, wv + 2] = 3.0
    for oh, ow in ((hv, wv), (48, 54), (16, 18)):
        want = post_ref(x, hv, wv, oh, ow)
        assert int(want[0].sum()) > 0 and int(want[1].sum()) == 0
        got = post_gpu(x, code, 8, hv, wv, oh, ow, name=f"crop border {SHORT[code]} to {oh}x{ow}")
        torch.cuda.synchronize()
        assert_post(f"crop border {SHORT[code]} to {oh}x{ow}", got, want)


def _blobs(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    x = torch.full((n, 1, h, w), -2.0)
    for i in range(n):
        for _ in range(12):
            cy, cx, r = float(torch.rand(1, generator=g)) * h, float(torch.rand(1, generator=g)) * w, 2 + float(torch.rand(1, generator=g)) * h / 20
            x[i, 0] += 5.0 * torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))
    return x + torch.randn(n, 1, h, w, generator=g) * 0.8


PRODUCTION_POST = {"post_bf16_b16_512_padded": dict(dtype=BF, n=16, h=512, w=512, cstride=8, h_valid=448, w_valid=512, oh=896, ow=1024)}


@pytest.mark.parametrize("name", sorted({**_fixture("post"), **PRODUCTION_POST}))
def test_post_production_calls(name):
    sp = {**_fixture("post"), **PRODUCTION_POST}[name]
    x = _blobs(sp["n"], sp["h"], sp["w"], sp["n"] + sp["h"]).to(DT[sp["dtype"]]).float()
    got = post_gpu(x, sp["dtype"], sp["cstride"], sp["h_valid"], sp["w_valid"], sp["oh"], sp["ow"], name=name)
    torch.cuda.synchronize()
    want = post_ref(x, sp["h_valid"], sp["w_valid"], sp["oh"], sp["ow"])
    assert 0.005 < float(want.float().mean()) < 0.9
    assert_post(name, got, want)


# ================================================================================================ fixture staleness
def _site_key(s):
    if s["fn"] == "pcb_seg_mask_postprocess":
        return (s["fn"], s["dtype"], s["cstride"])
    return (s["fn"], s["dtype"], _kind(s["x_strides"], s["h"], s["w"]),
            _kind(s["dx_strides"], s["h"], s["w"]) if "dx_strides" in s else None, s["loss"], s["reduction"])


def test_fixture_covers_training_and_inference():
    """both training steps with the three losses, the dense fp32 call and the inference with post-processing, at a small size,
    reach no (entry point, dtype, layout kinds, loss, reduction) that the fixture lacks"""
    spec = importlib.util.spec_from_file_location("make_golden_seg_loss_sites", os.path.join(GOLDEN, "make_golden_seg_loss_sites.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    rec = []
    with gen.recording(_lib.load(), rec):
        for name in ("TextSegament", "XceptionTextSegment"):
            for k, crit in enumerate(gen.criteria()):
                gen.run_train(name, 2, 128, crit, 30 + k)
        for k, crit in enumerate(gen.criteria()):
            gen.run_dense(2, 64, crit, 40 + k)
        gen.run_infer("XceptionTextSegment", 160, (0, 0, 0, 40), (160, 213))
    assert {s["fn"] for s in rec} == {"pcb_seg_loss_forward", "pcb_seg_loss_backward", "pcb_seg_mask_postprocess"}
    missing = {_site_key(s) for s in rec} - {_site_key(s) for s in _sites()}
    assert not missing, f"the fixture lacks {sorted(missing)}: regenerate tests/golden/seg_loss_sites.json"

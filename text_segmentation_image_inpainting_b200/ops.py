"""autograd Functions over the C ABI (include/pconv_b200.h).  Tensors are NHWC in memory
(``torch.channels_last``) with the usual logical NCHW shape; dtype fp32 (exact mode) or bf16
(tensor-core mode).  There is no CPU / eager fallback: non-CUDA input raises."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import ACT_LEAKY, ACT_NONE, ACT_RELU, ACT_RELU6, PCB_BF16, PCB_F32, Conv, Part
from .masks import HoleMask, as_hole_mask

CL = torch.channels_last


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dtype_code(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return PCB_F32
    if t.dtype == torch.bfloat16:
        return PCB_BF16
    raise _lib.PcbError(f"unsupported dtype {t.dtype}: the GPU path computes in float32 or bfloat16")


def as_feature(x: torch.Tensor) -> torch.Tensor:
    """CUDA + NHWC-contiguous view/copy of a 4-D activation (no dtype change)."""
    if not x.is_cuda:
        raise _lib.PcbError("text_segmentation_image_inpainting_b200 ops need CUDA tensors: there is no CPU fallback")
    if x.dim() != 4:
        raise _lib.PcbError(f"expected a 4-D NCHW activation, got shape {tuple(x.shape)}")
    _dtype_code(x)
    return x if x.is_contiguous(memory_format=CL) else x.contiguous(memory_format=CL)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def act_code(act) -> Tuple[int, float]:
    """nn.Module activation instance (or None/False) -> (code, negative slope)."""
    import torch.nn as nn
    if act is None or act is False:
        return ACT_NONE, 0.0
    if isinstance(act, nn.LeakyReLU):
        return ACT_LEAKY, float(act.negative_slope)
    if isinstance(act, nn.ReLU6):
        return ACT_RELU6, 0.0
    if isinstance(act, nn.ReLU):
        return ACT_RELU, 0.0
    raise NotImplementedError(f"activation {type(act).__name__} has no fused GPU kernel (supported: ReLU, ReLU6, LeakyReLU)")


# ------------------------------------------------------------------------------------------------
# partial convolution
# ------------------------------------------------------------------------------------------------
def nhwc_layout(x: torch.Tensor):
    """(channel stride) of a logical-NCHW tensor whose memory is NHWC with an optionally PADDED pixel stride
    (e.g. ``buf8[:, :3]`` of a channels_last [N,8,H,W] buffer), or None if it is not such a layout."""
    n, c, h, w = x.shape
    if x.is_contiguous(memory_format=CL):
        return c
    sn, sc, sh, sw = x.stride()
    cs = sw if w > 1 else (sh if h > 1 else (sn if n > 1 else c))
    if sc != 1 and c > 1:
        return None
    if cs < c or (w > 1 and sw != cs) or (h > 1 and sh != w * cs) or (n > 1 and sn != h * w * cs):
        return None
    return cs


def as_feature_padded(x: torch.Tensor) -> torch.Tensor:
    """Like as_feature but keeps channel-padded NHWC views as they are."""
    if not x.is_cuda:
        raise _lib.PcbError("text_segmentation_image_inpainting_b200 ops need CUDA tensors: there is no CPU fallback")
    if x.dim() != 4:
        raise _lib.PcbError(f"expected a 4-D NCHW activation, got shape {tuple(x.shape)}")
    _dtype_code(x)
    # Kernel family and weight layout are chosen from the problem geometry alone (ConvGeom.signature); the families test
    # 16/32-byte alignment of the source pointers, so a channel-sliced view with a misaligned first element is copied to an
    # aligned buffer here instead of silently changing family after the weights were laid out.
    if nhwc_layout(x) is None:
        return x.contiguous(memory_format=CL)
    if x.data_ptr() % 32:
        return _aligned_copy(x)
    return x


def _aligned_copy(x: torch.Tensor) -> torch.Tensor:
    """Copy of an NHWC (possibly channel-padded) view into a fresh, allocator-aligned buffer with the same logical shape."""
    buf = padded_empty(*x.shape, x.dtype, x.device)
    buf.copy_(x)
    return buf


def padded_empty(n, c, h, w, dtype, device):
    """NHWC buffer whose channel stride is rounded up to 8 (zero-filled padding); returns the logical view."""
    c8 = (c + 7) // 8 * 8
    if c8 == c:
        return torch.empty((n, c, h, w), dtype=dtype, device=device, memory_format=CL)
    return torch.empty((n, c8, h, w), dtype=dtype, device=device, memory_format=CL).zero_()[:, :c]


_LAZY_META = {"shape", "size", "dim", "ndim", "device", "dtype", "is_cuda", "requires_grad", "numel", "ndimension", "layout",
              "is_floating_point", "__len__", "grad_fn", "is_leaf", "names", "grad", "_version", "is_sparse", "is_quantized", "is_meta",
              "is_complex"}
_LAZY_CAT_FUNCS = {torch.cat, getattr(torch, "concat", torch.cat), getattr(torch, "concatenate", torch.cat)}
LAZYCAT_MATERIALIZED = 0          # how many times a LazyCat had to be turned into a dense tensor (tests assert the fast path)


class LazyCat(torch.Tensor):
    """cat([up2x?(x_i)], dim=1) that is never materialised: a partial convolution consumes the parts directly
    (image_inpainting.py:183-185 folded into the operand loads of the next layer).

    A ``torch.Tensor`` wrapper subclass with the logical shape / dtype / device of the concatenation, so that the REFERENCE's
    own network files run unchanged on top of this layer library and still get the fast path:
      * ``DoubleUpSample`` returns ``LazyCat([x], ups=(1,))`` -- a nearest-x2 view that moves no data,
      * ``torch.cat([x_up, skip], dim=1)`` (image_inpainting.py:184) concatenates part lists,
      * the next partial convolution reads ``.xs`` / ``.ups``,
      * any other torch function first materialises the dense tensor (one fused upsample + concat pass, differentiable).
    Autograd flows through the constituent tensors ``xs``; the wrapper itself is not part of the graph."""

    @staticmethod
    def __new__(cls, xs: Sequence[torch.Tensor], ups: Sequence[int]):
        xs = [as_feature_padded(x) for x in xs]
        ups = [int(u) for u in ups]
        n = xs[0].shape[0]
        h, w = xs[0].shape[2] << ups[0], xs[0].shape[3] << ups[0]
        for x, u in zip(xs, ups):
            if (x.shape[0], x.shape[2] << u, x.shape[3] << u) != (n, h, w) or x.dtype != xs[0].dtype:
                raise _lib.PcbError("LazyCat: mismatched batch / spatial size / dtype")
        r = torch.Tensor._make_wrapper_subclass(cls, (n, sum(x.shape[1] for x in xs), h, w), dtype=xs[0].dtype, device=xs[0].device,
                                                requires_grad=False)
        r.xs, r.ups = xs, ups
        return r

    def materialize(self) -> torch.Tensor:
        global LAZYCAT_MATERIALIZED
        LAZYCAT_MATERIALIZED += 1
        return concat_features([x if nhwc_layout(x) == x.shape[1] else x.contiguous(memory_format=CL) for x in self.xs], self.ups)

    def __repr__(self):  # noqa: D105
        with torch._C.DisableTorchFunctionSubclass():
            shp = tuple(self.shape)
        return f"LazyCat(shape={shp}, parts={[(tuple(x.shape), u) for x, u in zip(self.xs, self.ups)]})"

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, "__name__", "")
        if name in _LAZY_META or (name == "__get__" and getattr(getattr(func, "__self__", None), "__name__", "") in _LAZY_META):
            with torch._C.DisableTorchFunctionSubclass():
                return func(*args, **kwargs)
        if func in _LAZY_CAT_FUNCS:
            tensors = args[0]
            dim = kwargs.get("dim", args[1] if len(args) > 1 else 0)
            if dim in (1, -3) and all(isinstance(t, torch.Tensor) and t.dim() == 4 for t in tensors):
                xs, ups = [], []
                for t in tensors:
                    if isinstance(t, LazyCat):
                        xs += t.xs; ups += t.ups
                    else:
                        xs.append(t); ups.append(0)
                if len({x.dtype for x in xs}) == 1 and all(x.is_cuda for x in xs):
                    return LazyCat(xs, ups)

        def conv(a):
            if isinstance(a, LazyCat):
                return a.materialize()
            if isinstance(a, (list, tuple)):
                return type(a)(conv(b) for b in a)
            return a
        with torch._C.DisableTorchFunctionSubclass():
            return func(*conv(args), **{k: conv(v) for k, v in kwargs.items()})

    __torch_dispatch__ = None  # all handling happens at the torch-function level


def upsample2x_lazy(x: torch.Tensor) -> "LazyCat":
    """nearest x2 of a feature map as a LazyCat (no data movement); an already lazily-upsampled source is materialised first."""
    if isinstance(x, LazyCat):
        x = x.materialize()
    return LazyCat([as_feature_padded(x)], [1])


class TooManyParts(Exception):
    """The (source, mask-plane) partition of a convolution does not fit the kernels' part table: ops.partial_conv falls back to
    the general dense-mask formulation."""


class ConvGeom:
    """One partial-convolution problem: geometry + the channel partition (x source, mask plane) per part."""

    def __init__(self, xs: Sequence[torch.Tensor], ups: Sequence[int], cout, k, stride, padding, dilation, groups, same_holes,
                 no_guard, mask_parts: Sequence[Tuple[Optional[torch.Tensor], int, int]], plain=False):
        n = xs[0].shape[0]
        h, w = xs[0].shape[2] << ups[0], xs[0].shape[3] << ups[0]
        cin = sum(x.shape[1] for x in xs)
        kh, kw = (k, k) if isinstance(k, int) else k
        ph, pw = (padding, padding) if isinstance(padding, int) else padding
        s = stride if isinstance(stride, int) else stride[0]
        d = dilation if isinstance(dilation, int) else dilation[0]
        if (not isinstance(stride, int) and stride[0] != stride[1]) or (not isinstance(dilation, int) and dilation[0] != dilation[1]):
            raise NotImplementedError("anisotropic stride / dilation")
        self.n, self.cin, self.h, self.w = n, cin, h, w
        self.cout, self.kh, self.kw, self.stride, self.ph, self.pw, self.dil, self.groups = cout, kh, kw, s, ph, pw, d, groups
        self.ho = (h + 2 * ph - d * (kh - 1) - 1) // s + 1
        self.wo = (w + 2 * pw - d * (kw - 1) - 1) // s + 1
        self.same_holes, self.no_guard, self.plain = int(same_holes), int(no_guard), int(plain)
        self.dtype = _dtype_code(xs[0])
        self.esz = 2 if self.dtype == PCB_BF16 else 4
        self.mg = groups if (groups > 1 and not same_holes) else 1
        if self.ho <= 0 or self.wo <= 0:
            raise _lib.PcbError(f"convolution output would be empty ({self.ho}x{self.wo})")
        self.x_channels = [x.shape[1] for x in xs]
        self.x_cstrides = [nhwc_layout(x) for x in xs]
        self.x_ups = list(ups)
        # common refinement of the x partition and the mask partition
        xb, off = [], 0
        for i, c in enumerate(self.x_channels):
            xb.append((off, off + c, i)); off += c
        mb, off = [], 0
        for plane, c, up in mask_parts:
            mb.append((off, off + c, plane, up)); off += c
        if off != cin:
            raise _lib.PcbError(f"mask covers {off} channels but the input has {cin}")
        self.parts = []            # (x index, channel offset inside that x, channels, plane, mask_up)
        for lo, hi, xi in xb:
            for mlo, mhi, plane, mup in mb:
                a, b_ = max(lo, mlo), min(hi, mhi)
                if a < b_:
                    self.parts.append((xi, a - lo, b_ - a, plane, mup))
        if len(self.parts) > _lib.MAX_PARTS:
            raise TooManyParts(f"more than {_lib.MAX_PARTS} (source, mask-plane) parts in one convolution")
        self.signature = (self.dtype, cin, cout, kh, kw, groups, tuple(p[2] for p in self.parts), tuple(self.x_cstrides),
                          tuple(self.x_ups), tuple(p[4] for p in self.parts), tuple(p[3] is not None for p in self.parts), s, d,
                          ph, pw, h & 1, w & 1)
        # the sub-pixel path (conv over a 2x-upsampled source) carries extra operand matrices: its eligibility depends on the
        # spatial size, so it is part of the operand-cache key
        self.subpixel = bool(_lib.load().pcb_conv_dgrad_at_source_resolution(ctypes.byref(self.struct(None)))) if any(self.x_ups) else False
        self.signature = self.signature + (self.subpixel,)

    def struct(self, xs: Optional[Sequence[torch.Tensor]], force_generic=False) -> Conv:
        c = Conv()
        c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw = self.n, self.h, self.w, self.cin, self.cout, self.kh, self.kw
        c.stride, c.pad_h, c.pad_w, c.dil, c.groups, c.ho, c.wo = self.stride, self.ph, self.pw, self.dil, self.groups, self.ho, self.wo
        c.dtype, c.same_holes, c.no_guard, c.plain, c.force_generic = self.dtype, self.same_holes, self.no_guard, self.plain, int(force_generic)
        c.nparts = len(self.parts)
        for i, (xi, choff, ch, plane, mup) in enumerate(self.parts):
            c.parts[i].x = (xs[xi].data_ptr() + choff * self.esz) if xs is not None else None
            c.parts[i].mask = plane.data_ptr() if plane is not None else None
            c.parts[i].c, c.parts[i].x_cstride, c.parts[i].x_up, c.parts[i].mask_up = ch, self.x_cstrides[xi], self.x_ups[xi], mup
        return c


# ------------------------------------------------------------------------------------------------
# per-step zero arena: reduction targets (BatchNorm sums) are slices of ONE buffer that the training engine zeroes once per
# step, instead of one cudaMemsetAsync per reduction (the step had 106 of them)
# ------------------------------------------------------------------------------------------------
class _ZeroArena:
    def __init__(self):
        self.buf, self.off, self.active = None, 0, False


_ARENAS = {}


def begin_step_arena(device, nbytes=1 << 20):
    """Zero the arena of `device` on the current stream and hand out slices of it until end_step_arena()."""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    a = _ARENAS.setdefault(key, _ZeroArena())
    if a.buf is None or a.buf.numel() < nbytes:
        a.buf = torch.empty((nbytes,), dtype=torch.uint8, device=device)
    a.buf.zero_()
    a.off, a.active = 0, True


def end_step_arena(device):
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    if key in _ARENAS:
        _ARENAS[key].active = False


def zeros_f64(n, device):
    """n zeroed doubles: a slice of the step arena when one is active (and has room), else a fresh zero tensor."""
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    a = _ARENAS.get(key)
    nbytes = (n * 8 + 255) // 256 * 256
    if a is not None and a.active and a.off + nbytes <= a.buf.numel():
        view = a.buf[a.off:a.off + n * 8].view(torch.float64)
        a.off += nbytes
        return view
    return torch.zeros((n,), dtype=torch.float64, device=device)


_PROFILE = None     # optional list: (kind, geom, start_event, end_event) appended per conv kernel call


def set_profile(sink):
    """bench.py: pass a list to record CUDA-event-bracketed conv launches (eager mode only), or None to stop."""
    global _PROFILE
    _PROFILE = sink


class _Timed:
    def __init__(self, kind, geom):
        self.kind, self.geom = kind, geom

    def __enter__(self):
        if _PROFILE is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *exc):
        if _PROFILE is not None:
            self.e.record()
            _PROFILE.append((self.kind, self.geom, self.s, self.e))
        return False


def _workspace(lib, c, device):
    nbytes = lib.pcb_pconv_workspace(ctypes.byref(c))
    return torch.empty((max(nbytes, 16),), dtype=torch.uint8, device=device)


class PartialConvFn(torch.autograd.Function):
    """y, msum, newmask = pconv(cat(up?(x_i)), W, b | mask)   (models/partial_convolution.py:49-80 / :121-137)."""

    @staticmethod
    def forward(ctx, geom: ConvGeom, wprep, weight, bias, handoff, *xs):
        lib = _lib.load()
        w_fwd, w_dg = wprep
        c = geom.struct(xs)
        dev = xs[0].device
        if geom.dtype == PCB_BF16:
            y = padded_empty(geom.n, geom.cout, geom.ho, geom.wo, xs[0].dtype, dev)
        else:
            y = torch.empty((geom.n, geom.cout, geom.ho, geom.wo), dtype=xs[0].dtype, device=dev, memory_format=CL)
        b32 = bias.detach().float().contiguous() if bias is not None else None
        # BatchNorm statistics of y in the convolution epilogue when the consumer announced itself (RenormHandoff.want_stats)
        bn_sums = None
        if handoff is not None and handoff.want_stats and _FUSED_BN_STATS and lib.pcb_conv_fuses_bn_stats(ctypes.byref(c)) \
                and nhwc_layout(y) == geom.cout:
            bn_sums = zeros_f64(2 * geom.cout, dev)
            handoff.bn_sums = bn_sums
        global _LAST_MASK_EVENT
        _LAST_MASK_EVENT = None
        if _MASK_CHAIN_STREAM and _PROFILE is None and not geom.plain:
            # Mask updates never depend on features (partial_convolution.py:59-77): the mask pass of this layer runs on the
            # mask stream, ordered only after the passes that produced its input planes, i.e. ahead of the feature path.
            # Its buffers are allocated on that stream and kept alive until join_side_streams() (engine, once per step).
            main, ms = torch.cuda.current_stream(), _mask_stream(dev)
            for (_, _, _, pl, _) in geom.parts:
                if pl is None:
                    continue
                ev_in = getattr(pl, "_pcb_ev", None)
                if ev_in is None:                        # a plane written on the main stream (the network's input mask): mark it
                    ev_in = torch.cuda.Event()           # ready from here on, so later consumers (the tail) need not wait for main
                    ev_in.record(main)
                    pl._pcb_ev = ev_in
                ms.wait_event(ev_in)
            with torch.cuda.stream(ms):
                msum = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.float32, device=dev)
                newmask = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.uint8, device=dev)
                ws = _workspace(lib, c, dev)
                _lib.check(lib.pcb_pconv_mask_pass(ctypes.byref(c), msum.data_ptr(), newmask.data_ptr(), ws.data_ptr(), _stream()))
                ev = torch.cuda.Event()
                ev.record()
            main.wait_event(ev)
            _DEFERRED.append((msum, newmask, ws))
            _LAST_MASK_EVENT = ev
            _lib.check(lib.pcb_pconv_forward_bn(ctypes.byref(c), w_fwd.data_ptr(), _ptr(b32), y.data_ptr(), nhwc_layout(y),
                                                msum.data_ptr(), newmask.data_ptr(), ws.data_ptr(), 1, _ptr(bn_sums), _stream()))
        else:
            msum = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.float32, device=dev)
            newmask = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.uint8, device=dev)
            ws = _workspace(lib, c, dev)
            with _Timed("fwd", geom):
                _lib.check(lib.pcb_pconv_forward_bn(ctypes.byref(c), w_fwd.data_ptr(), _ptr(b32), y.data_ptr(), nhwc_layout(y), msum.data_ptr(),
                                                    newmask.data_ptr(), ws.data_ptr(), 0, _ptr(bn_sums), _stream()))
        ctx.geom, ctx.wprep, ctx.has_bias, ctx.weight_ref, ctx.bias_ref = geom, wprep, bias is not None, weight, bias
        ctx.handoff = handoff
        if handoff is not None:
            handoff.msum = msum
            handoff.eligible = (geom.mg == 1 and not geom.no_guard and not geom.plain and bias is None and geom.cout % 8 == 0
                                and geom.dtype == PCB_BF16)
        ctx.save_for_backward(msum, *xs)
        ctx.mark_non_differentiable(msum, newmask)
        # without this autograd zero-fills a gradient tensor for msum and newmask on every backward (two fill kernels per layer)
        ctx.set_materialize_grads(False)
        return y, msum, newmask

    @staticmethod
    def backward(ctx, gy, _gmsum, _gnewmask):
        if gy is None:
            return (None,) * (5 + len(ctx.saved_tensors) - 1)
        lib = _lib.load()
        msum, *xs = ctx.saved_tensors
        geom: ConvGeom = ctx.geom
        w_fwd, w_dg = ctx.wprep
        dev, tdtype = xs[0].device, xs[0].dtype
        gy = as_feature_padded(gy if gy.dtype == tdtype else gy.to(tdtype))
        c = geom.struct(xs)
        dbias = None
        if ctx.handoff is not None and ctx.handoff.fused:
            # the BatchNorm backward of the block already divided by the mask sums (RenormHandoff): gy IS dc
            dc = gy
            dcs = nhwc_layout(dc)
        elif geom.plain and not ctx.has_bias and geom.cout % 8 == 0 and nhwc_layout(gy) == geom.cout and gy.data_ptr() % 16 == 0:
            # ordinary convolution without bias: the renormaliser is 1 and there is no bias gradient -- the "renormalisation
            # backward" would be a copy of gy
            dc = gy
            dcs = geom.cout
        else:
            dc = padded_empty(geom.n, geom.cout, geom.ho, geom.wo, tdtype, dev) if geom.dtype == PCB_BF16 else \
                torch.empty((geom.n, geom.cout, geom.ho, geom.wo), dtype=tdtype, device=dev, memory_format=CL)
            dcs = nhwc_layout(dc)
            dbias = bsink = None
            if ctx.has_bias:
                bsink = getattr(ctx.bias_ref, "_pcb_grad_sink", None)
                if bsink is not None and not bsink.used and bsink.view.dtype == torch.float32 and bsink.view.numel() == geom.cout \
                        and bsink.view.is_contiguous():
                    bsink.used = True                     # the kernel overwrites the arena slice: no gradient tensor for autograd
                else:
                    bsink = None
                    dbias = torch.empty((geom.cout,), dtype=torch.float32, device=dev)
            _lib.check(lib.pcb_pconv_renorm_backward(ctypes.byref(c), gy.data_ptr(), nhwc_layout(gy), msum.data_ptr(), dc.data_ptr(), dcs,
                                                     _ptr(bsink.view if bsink is not None else dbias), _stream()))
            if bsink is not None and bsink.on_written is not None:
                bsink.on_written()
        dw = None
        need = [ctx.needs_input_grad[5 + i] for i in range(len(xs))]
        side = None
        deferred = False
        if ctx.needs_input_grad[2]:
            # A training engine may register a gradient sink on the parameter (engine.FlatParams: a view of its flat fp32
            # gradient arena with the weight's physical layout).  The kernel then writes the gradient in place (it overwrites:
            # no accumulation pass) and autograd gets no tensor; with the side stream below the join can then wait until
            # the engine calls join_side_streams(), so the weight gradient also overlaps the element-wise backward kernels
            # of the layers that follow.  A second use of the same weight in one pass falls back to autograd accumulation.
            sink = getattr(ctx.weight_ref, "_pcb_grad_sink", None)
            wgrad_fn = lib.pcb_pconv_backward_weight
            shape = (geom.cout, geom.cin // geom.groups, geom.kh, geom.kw)
            if sink is not None and not sink.used and tuple(sink.view.shape) == shape and sink.view.dtype == torch.float32 \
                    and sink.view.is_contiguous(memory_format=CL):
                dw_buf, sink.used = sink.view, True
                if sink.prezeroed:           # the owner zeroed the whole arena at the start of the step: accumulate, no memset
                    wgrad_fn = lib.pcb_pconv_backward_weight_acc
            else:
                sink = None
                dw_buf = dw = torch.empty(shape, dtype=torch.float32, device=dev, memory_format=CL)
            ws = _workspace(lib, c, dev)
            # weight and data gradient only share their input dc: run the weight gradient on a side stream so that the two
            # kernels of a low-resolution layer (far fewer tiles than SMs each) fill the GPU together.  Buffers are
            # allocated on the main stream before the fork and the streams re-join before this function returns.
            if _OVERLAP_WGRAD and (any(need) or sink is not None) and _PROFILE is None:
                side = _side_stream(dev)
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    _lib.check(wgrad_fn(ctypes.byref(c), dc.data_ptr(), dcs, dw_buf.data_ptr(), ws.data_ptr(), _stream()))
                if sink is not None:
                    deferred = True
                    _DEFERRED.append((dc, ws, xs))            # keep the side stream's operands alive until the join
                    if sink.on_written is not None:
                        sink.on_written()
            else:
                with _Timed("wgrad", geom):
                    _lib.check(wgrad_fn(ctypes.byref(c), dc.data_ptr(), dcs, dw_buf.data_ptr(), ws.data_ptr(), _stream()))
                if sink is not None and sink.on_written is not None:
                    sink.on_written()
        gxs: List[Optional[torch.Tensor]] = [None] * len(xs)
        if any(need):
            # gradient buffer per source tensor; parts write their channel slices.  Full resolution -- except on the sub-pixel
            # path, which computes the gradient of a 2x-upsampled source directly at that source's resolution
            at_src = bool(lib.pcb_conv_dgrad_at_source_resolution(ctypes.byref(c)))
            full = [padded_empty(geom.n, geom.x_channels[i], geom.h >> (geom.x_ups[i] if at_src else 0), geom.w >> (geom.x_ups[i] if at_src else 0),
                                 tdtype, dev) if need[i] else None for i in range(len(xs))]
            nparts = len(geom.parts)
            ptrs = (ctypes.c_void_p * nparts)()
            strides = (ctypes.c_int32 * nparts)()
            for pi, (xi, choff, ch, plane, mup) in enumerate(geom.parts):
                if full[xi] is not None:
                    ptrs[pi] = full[xi].data_ptr() + choff * geom.esz
                    strides[pi] = nhwc_layout(full[xi])
                else:
                    ptrs[pi], strides[pi] = None, 0
            cc, wf, wd = c, w_fwd, w_dg
            if lib.pcb_conv_uses_tensor_cores(ctypes.byref(c)) and w_dg is None:
                # row-packed (cin <= 8) tensor-core layer whose input wants a gradient: generic data-gradient kernel
                cc = geom.struct(xs, force_generic=True)
                wf = ctx.weight_ref.detach().float().contiguous(memory_format=CL).to(tdtype)
                wd = None
            with _Timed("dgrad", geom):
                _lib.check(lib.pcb_pconv_backward_data(ctypes.byref(cc), dc.data_ptr(), dcs, wf.data_ptr(), _ptr(wd), ptrs, strides, _stream()))
            for i in range(len(xs)):
                if full[i] is None:
                    continue
                if geom.x_ups[i] and not at_src:
                    g = padded_empty(geom.n, geom.x_channels[i], geom.h >> 1, geom.w >> 1, tdtype, dev)
                    src = full[i]
                    cs_src, cs_dst = nhwc_layout(src), nhwc_layout(g)
                    if cs_src != cs_dst or cs_src != geom.x_channels[i]:
                        raise NotImplementedError("upsampled conv source with padded channels")
                    _lib.check(lib.pcb_upsample2x_backward(src.data_ptr(), geom.dtype, geom.n, geom.h >> 1, geom.w >> 1, geom.x_channels[i],
                                                           g.data_ptr(), _stream()))
                    gxs[i] = g
                else:
                    gxs[i] = full[i]
        if side is not None and not deferred:
            torch.cuda.current_stream().wait_stream(side)
        return (None, None, dw, dbias, None, *gxs)


_WEIGHT_EPOCH = 0


def bump_weight_epoch():
    """Invalidate every cached compute-dtype weight copy (call after updating parameters through raw pointers,
    e.g. `sgd_step`, which does not bump tensor version counters)."""
    global _WEIGHT_EPOCH
    _WEIGHT_EPOCH += 1


_INPLACE_WEIGHT_REFRESH = False


def set_inplace_weight_refresh(enabled: bool):
    """Training engines that update the masters once per step (after every backward of that step has run) may let
    `prepare_weight` rewrite the cached operand buffers in place instead of allocating + zero-filling new ones each step.
    Off by default: a backward that runs after a later weight update would otherwise read the new weights."""
    global _INPLACE_WEIGHT_REFRESH
    _INPLACE_WEIGHT_REFRESH = bool(enabled)


def prepare_weight(weight: torch.Tensor, geom: ConvGeom, cache: dict):
    """fp32 master weight (OIHW logical, KRSC physical) -> the operand buffers the kernels want
    (pcb_conv_weight_layout / pcb_conv_weight_prepare), cached per parameter version and problem signature."""
    key = (weight.data_ptr(), weight._version, str(weight.device), _WEIGHT_EPOCH, geom.signature)
    if cache.get("key") == key:
        ev = cache.get("ready")
        if ev is not None:                                # refreshed ahead of time on the prefetch stream (prefetch_weights)
            torch.cuda.current_stream().wait_event(ev)
            cache["ready"] = None
        return cache["val"]
    lib = _lib.load()
    wm = weight.detach()
    if wm.dtype != torch.float32:
        wm = wm.float()
    wm = wm.contiguous(memory_format=CL)          # physical [cout][kh][kw][cig]
    c = geom.struct(None)
    fe, de = ctypes.c_size_t(0), ctypes.c_size_t(0)
    lib.pcb_conv_weight_layout(ctypes.byref(c), ctypes.byref(fe), ctypes.byref(de))
    tdt = torch.bfloat16 if geom.dtype == PCB_BF16 else torch.float32
    old = cache.get("val")
    if _INPLACE_WEIGHT_REFRESH and old is not None and cache.get("sig") == (geom.signature, str(wm.device), fe.value, de.value):
        w_fwd, w_dg = old
        _lib.check(lib.pcb_conv_weight_refresh(ctypes.byref(c), wm.data_ptr(), w_fwd.data_ptr(), _ptr(w_dg), _stream()))
    else:
        w_fwd = torch.empty((fe.value,), dtype=tdt, device=wm.device)
        w_dg = torch.empty((de.value,), dtype=tdt, device=wm.device) if de.value else None
        _lib.check(lib.pcb_conv_weight_prepare(ctypes.byref(c), wm.data_ptr(), w_fwd.data_ptr(), _ptr(w_dg), _stream()))
    cache["sig"] = (geom.signature, str(wm.device), fe.value, de.value)
    cache["key"], cache["val"] = key, (w_fwd, w_dg)
    cache["ready"] = None
    cache["geom"], cache["weight"] = geom, weight         # remembered for prefetch_weights()
    return cache["val"]


_PREFETCH_STREAMS = {}


def prefetch_weights(caches):
    """Re-lay-out the convolution weights behind `caches` (the per-module operand caches) on a prefetch stream, ahead of the layers' forward calls (training
    engines call this right after the optimiser step / epoch bump; requires the in-place refresh mode).  Each layer's
    forward then only waits on its own event, so the re-layout of layer k overlaps the forward of the layers before it."""
    caches = [c for c in caches if c.get("val") is not None and c.get("weight") is not None]
    if not _INPLACE_WEIGHT_REFRESH or not caches:
        return
    lib = _lib.load()
    dev = caches[0]["weight"].device
    key_dev = (dev.type, dev.index if dev.index is not None else torch.cuda.current_device())
    if key_dev not in _PREFETCH_STREAMS:
        _PREFETCH_STREAMS[key_dev] = torch.cuda.Stream(device=dev)
    ps = _PREFETCH_STREAMS[key_dev]
    ps.wait_stream(torch.cuda.current_stream())           # after the optimiser step, and after every reader of the old buffers
    with torch.cuda.stream(ps):
        for cache in caches:
            weight, geom = cache["weight"], cache["geom"]
            if weight.device != dev or weight.dtype != torch.float32:
                continue
            key = (weight.data_ptr(), weight._version, str(weight.device), _WEIGHT_EPOCH, geom.signature)
            if cache.get("key") == key:
                continue
            wm = weight.detach().contiguous(memory_format=CL)
            c = geom.struct(None)
            w_fwd, w_dg = cache["val"]
            _lib.check(lib.pcb_conv_weight_refresh(ctypes.byref(c), wm.data_ptr(), w_fwd.data_ptr(), _ptr(w_dg), _stream()))
            ev = torch.cuda.Event()
            ev.record()
            cache["key"], cache["ready"] = key, ev


_OVERLAP_WGRAD = True
_MASK_CHAIN_STREAM = False
_LAST_MASK_EVENT = None
_SIDE_STREAMS = {}
_MASK_STREAMS = {}
_DEFERRED = []


def set_mask_chain_stream(enabled: bool):
    """Run every layer's mask pass (mask box sums, new mask, tap-validity words) on a dedicated stream ahead of the feature
    path.  Only for callers that call join_side_streams() once per step (the buffers of the pass live until then)."""
    global _MASK_CHAIN_STREAM
    _MASK_CHAIN_STREAM = bool(enabled)


def _mask_stream(dev):
    key = (dev.type, dev.index if dev.index is not None else torch.cuda.current_device())
    if key not in _MASK_STREAMS:
        _MASK_STREAMS[key] = torch.cuda.Stream(device=dev)
    return _MASK_STREAMS[key]


class GradSink:
    """In-place destination for a convolution weight gradient (see PartialConvFn.backward).  The owner resets `used` before
    every backward pass and calls join_side_streams() after it."""

    def __init__(self, view: torch.Tensor):
        self.view, self.used = view, False
        self.prezeroed = False        # the owner guarantees `view` is zero when the backward pass starts (skip the kernel's memset)
        self.on_written = None        # optional callback: the kernel that writes `view` has just been launched


def side_streams():
    """The weight-gradient side streams created so far (a training engine orders its gradient exchange after them)."""
    return list(_SIDE_STREAMS.values())


def join_side_streams():
    """Make the current stream wait for every weight gradient still running on a side stream (gradient sinks only)."""
    for st in list(_SIDE_STREAMS.values()) + list(_MASK_STREAMS.values()) + list(_PREFETCH_STREAMS.values()):
        torch.cuda.current_stream().wait_stream(st)
    _DEFERRED.clear()


def set_overlap_wgrad(enabled: bool):
    global _OVERLAP_WGRAD
    _OVERLAP_WGRAD = bool(enabled)


def _side_stream(dev):
    key = (dev.type, dev.index if dev.index is not None else torch.cuda.current_device())
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=dev)
    return _SIDE_STREAMS[key]


class RenormHandoff:
    """Links a partial convolution to the BatchNorm(+activation) that is the ONLY consumer of its output (the blocks of
    models/partial_convolution.py): the BN backward then writes dc = dy / mask_sum directly (one pass less over every conv
    output) and the convolution's backward skips its renormalisation step.  Never use it when y has another consumer."""

    def __init__(self, want_stats=False):
        self.msum, self.eligible, self.fused = None, False, False
        # want_stats: the consumer is a training-mode BatchNorm -> the convolution accumulates the per-channel sum / sum of
        # squares of its output in its epilogue (`bn_sums`, [2][cout] doubles) and the statistics pass over y disappears
        self.want_stats, self.bn_sums = bool(want_stats), None


_FUSED_BN_STATS = True


def set_fused_bn_stats(enabled: bool):
    global _FUSED_BN_STATS
    _FUSED_BN_STATS = bool(enabled)


def partial_conv(x, mask, weight, bias, stride, padding, dilation, groups, same_holes=False, no_guard=False, cache=None,
                 plain=False, handoff=None):
    """Returns (y, new_mask: HoleMask).  `x` is a tensor or a LazyCat; `mask` a HoleMask or a dense tensor; with
    ``plain=True`` the mask is ignored and an ordinary convolution is computed (same kernels, renormaliser 1)."""
    if isinstance(x, LazyCat):
        xs, ups = x.xs, x.ups
    else:
        xs, ups = [as_feature_padded(x)], [0]
    n, h, w = xs[0].shape[0], xs[0].shape[2] << ups[0], xs[0].shape[3] << ups[0]
    cin = sum(t.shape[1] for t in xs)
    if plain:
        parts = [(None, cin, 0)]
    else:
        hm = as_hole_mask(mask)
        if tuple(hm.shape[2:]) != (h, w) or hm.shape[0] != n:
            raise _lib.PcbError(f"mask shape {tuple(hm.shape)} does not match input {(n, cin, h, w)}")
        parts = hm.parts
        if hm.shape[1] != cin:
            if hm.shape[1] == 1:                       # broadcast of a 1-channel mask over x (x * mask, :51)
                parts = [(parts[0][0], cin, parts[0][2])]
            else:
                raise _lib.PcbError(f"mask has {hm.shape[1]} channels, input has {cin}")
    cout = weight.shape[0]
    if weight.shape[1] * groups != cin:
        raise _lib.PcbError(f"weight expects {weight.shape[1] * groups} input channels, got {cin}")
    try:
        geom = ConvGeom(xs, ups, cout, tuple(weight.shape[2:]), stride, padding, dilation, groups, same_holes, no_guard, parts, plain=plain)
    except TooManyParts:
        return _partial_conv_dense_masks(x, hm, weight, bias, stride, padding, dilation, groups, same_holes, no_guard, cache)
    wprep = prepare_weight(weight, geom, cache if cache is not None else {})
    y, msum, newmask = PartialConvFn.apply(geom, wprep, weight, bias, handoff, *xs)
    planes = [newmask[g] for g in range(geom.mg)]
    if _LAST_MASK_EVENT is not None:                      # written on the mask stream: consumers there wait on this event
        for pl in planes:
            pl._pcb_ev = _LAST_MASK_EVENT
    if geom.mg == 1:
        new = HoleMask.from_plane(planes[0], cout, 0)
    else:
        cog = cout // groups
        new = HoleMask([(planes[g], cog, 0) for g in range(groups)], n, geom.ho, geom.wo)
    return y, new


def _partial_conv_dense_masks(x, hm: HoleMask, weight, bias, stride, padding, dilation, groups, same_holes, no_guard, cache):
    """General per-channel masks (partial_convolution.py:62-64 accepts ANY [N,C,H,W] mask): when the mask has more distinct
    (source, plane) parts than the kernels' part table holds (PCB_MAX_PARTS), the partial convolution is computed the way the
    reference states it, on the GPU, from this library's own kernels:
        c = conv(x * m; W)              -- the same convolution kernels in `plain` mode (tensor cores when eligible)
        s = conv(m; ones) per group     -- exact fp32 mode (mask sums reach cin*k*k: never in bf16)
        y = where(s == 0, 0, c / s + b) ; m' = (s != 0)
    Slower than the fused path (the dense mask is materialised); exact; differentiable through the same autograd Functions."""
    if isinstance(x, LazyCat):
        x = x.materialize()
    x = as_feature_padded(x)
    cin, cout = x.shape[1], weight.shape[0]
    m = hm.dense()                                                   # fp32 [N, C, H, W]
    if m.shape[1] != cin:
        m = m[:, :1].expand(-1, cin, -1, -1)
    xm = (x * m.to(x.dtype)).contiguous(memory_format=CL)
    c_raw, _ = partial_conv(xm, None, weight, None, stride, padding, dilation, groups, cache=cache, plain=True)
    kh, kw = weight.shape[2:]
    with torch.no_grad():
        if same_holes:
            ones = torch.ones((1, 1, kh, kw), dtype=torch.float32, device=x.device).contiguous(memory_format=CL)
            s, _ = partial_conv(m[:, :1].contiguous(memory_format=CL), None, ones, None, stride, padding, dilation, 1, plain=True)
            s = s * float(cin)                                       # :61 (total in_channels, also for depthwise)
            mg = 1
        else:
            ones = torch.ones((groups, cin // groups, kh, kw), dtype=torch.float32, device=x.device).contiguous(memory_format=CL)
            s, _ = partial_conv(m.contiguous(memory_format=CL), None, ones, None, stride, padding, dilation, groups, plain=True)
            mg = groups
        hole = s == 0
        rep = cout // mg
        s_full = s.repeat_interleave(rep, dim=1) if rep > 1 else s
        hole_full = s_full == 0
    b = bias.view(1, -1, 1, 1).to(torch.float32) if bias is not None else None
    y = c_raw.float() / (s_full if no_guard else s_full.masked_fill(hole_full, 1.0))
    if b is not None:
        y = y + b
    if not no_guard:
        y = y.masked_fill(hole_full, 0.0)
    y = y.to(x.dtype).contiguous(memory_format=CL)
    n, _, ho, wo = y.shape
    if no_guard:
        planes = [torch.ones((n, ho, wo), dtype=torch.uint8, device=x.device)]
        return y, HoleMask.from_plane(planes[0], cout, 0)
    newmask = (~hole).to(torch.uint8)                                # [N, mg, Ho, Wo]
    if mg == 1:
        return y, HoleMask.from_plane(newmask[:, 0].contiguous(), cout, 0)
    return y, HoleMask([(newmask[:, g].contiguous(), rep, 0) for g in range(mg)], n, ho, wo)


# ------------------------------------------------------------------------------------------------
# BatchNorm2d (+ activation, + residual)
# ------------------------------------------------------------------------------------------------
def _vec_bn(c):
    return c % 8 == 0 and c <= 2048


_BN_SMALL = True


def set_bn_small_kernel(enabled: bool):
    global _BN_SMALL
    _BN_SMALL = bool(enabled)


class BNActFn(torch.autograd.Function):
    """y = act(BN(x)) [+ residual]; BN optional (gamma None => plain activation).

    Training mode, channel count a multiple of 8: the statistics come either from the producing convolution's epilogue
    (`pre_sums`) or from one accumulate-only pass into a slice of the step's zero arena; finalisation (mean / invstd / running
    statistics), normalisation and activation are ONE launch (pcb_bn_forward_fused).  Backward = one reduction + one apply
    launch that also writes dgamma / dbeta -- straight into the training engine's gradient arena when the parameters carry
    gradient sinks (no autograd accumulation kernels)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, residual, running_mean, running_var, nbt, training, momentum, eps, act, slope, msum=None, pre_sums=None):
        lib = _lib.load()
        n, c, h, w = x.shape
        count = n * h * w
        code = _dtype_code(x)
        dev = x.device
        has_bn = gamma is not None
        scale = shift = mean = invstd = None
        y = torch.empty_like(x, memory_format=CL)
        use_batch = has_bn and (training or running_mean is None)
        if use_batch and count <= 1 and training:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size {tuple(x.shape)}")
        if use_batch and _vec_bn(c):
            sums = pre_sums
            if sums is None:
                sums = zeros_f64(2 * c, dev)
                _lib.check(lib.pcb_bn_stats_acc(x.data_ptr(), code, count, c, sums.data_ptr(), _stream()))
            coef = torch.empty((4, c), dtype=torch.float32, device=dev)
            _lib.check(lib.pcb_bn_forward_fused(x.data_ptr(), code, count, c, sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                _ptr(running_mean) if training else None, _ptr(running_var) if training else None,
                                                _ptr(nbt) if training else None, float(momentum), float(eps), act, float(slope),
                                                _ptr(residual), y.data_ptr(), coef.data_ptr(), _stream()))
            scale, shift, mean, invstd = coef[0], coef[1], coef[2], coef[3]
        else:
            if has_bn:
                scale = torch.empty((c,), dtype=torch.float32, device=dev)
                shift = torch.empty_like(scale)
                if use_batch:
                    sums = torch.empty((2, c), dtype=torch.float64, device=dev)
                    _lib.check(lib.pcb_bn_stats(x.data_ptr(), code, count, c, sums[0].data_ptr(), sums[1].data_ptr(), _stream()))
                    mean = torch.empty_like(scale)
                    invstd = torch.empty_like(scale)
                    _lib.check(lib.pcb_bn_finalize(sums[0].data_ptr(), sums[1].data_ptr(), count, c, gamma.data_ptr(), beta.data_ptr(),
                                                   _ptr(running_mean) if training else None, _ptr(running_var) if training else None,
                                                   _ptr(nbt) if training else None, float(momentum), float(eps), 1,
                                                   scale.data_ptr(), shift.data_ptr(), mean.data_ptr(), invstd.data_ptr(), _stream()))
                else:
                    _lib.check(lib.pcb_bn_finalize(None, None, count, c, gamma.data_ptr(), beta.data_ptr(), running_mean.data_ptr(),
                                                   running_var.data_ptr(), None, float(momentum), float(eps), 0,
                                                   scale.data_ptr(), shift.data_ptr(), None, None, _stream()))
            _lib.check(lib.pcb_bn_act_forward(x.data_ptr(), code, count, c, _ptr(scale), _ptr(shift), act, float(slope),
                                              _ptr(residual), y.data_ptr(), _stream()))
        ctx.cfg = (count, c, code, act, float(slope), has_bn, mean is not None, residual is not None)
        ctx.params = (gamma, beta)
        ctx.save_for_backward(x, scale, shift, mean, invstd, msum)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x, scale, shift, mean, invstd, msum = ctx.saved_tensors
        count, c, code, act, slope, has_bn, batch_stats, has_res = ctx.cfg
        gy = gy.contiguous(memory_format=CL)
        if gy.dtype != x.dtype:
            gy = gy.to(x.dtype)
        dx = torch.empty_like(x, memory_format=CL)
        dgamma = dbeta = None
        if has_bn and batch_stats:
            dev = x.device
            # parameter gradients: written in place into the engine's gradient arena when the parameters carry sinks
            gamma, beta = ctx.params
            sinks = []
            outs = []
            for p in (gamma, beta):
                sk = getattr(p, "_pcb_grad_sink", None)
                if sk is not None and not sk.used and sk.view.dtype == torch.float32 and sk.view.numel() == c and sk.view.is_contiguous() \
                        and p.requires_grad:
                    sk.used = True
                    sinks.append(sk); outs.append(sk.view)
                else:
                    sinks.append(None); outs.append(torch.empty((c,), dtype=torch.float32, device=dev))
            small = _vec_bn(c) and _BN_SMALL and count <= 16384 and c >= 256 and scale.data_ptr() + 4 * c == shift.data_ptr() \
                and shift.data_ptr() + 4 * c == mean.data_ptr() and mean.data_ptr() + 4 * c == invstd.data_ptr()
            if small:
                # the bottom of the U: one launch does reduction + apply + parameter gradients (scale|shift|mean|invstd are the
                # four rows of the [4][c] block pcb_bn_forward_fused wrote)
                _lib.check(lib.pcb_bn_act_backward_small(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), act, slope,
                                                         _ptr(msum), dx.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), _stream()))
                s0 = s1 = None
            elif _vec_bn(c):
                sums = zeros_f64(2 * c, dev)
                _lib.check(lib.pcb_bn_act_backward_reduce_acc(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), shift.data_ptr(),
                                                              mean.data_ptr(), invstd.data_ptr(), act, slope, sums.data_ptr(), _stream()))
                s0, s1 = sums.data_ptr(), sums.data_ptr() + 8 * c
            else:
                sums = torch.empty((2, c), dtype=torch.float64, device=dev)
                _lib.check(lib.pcb_bn_act_backward_reduce(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), shift.data_ptr(),
                                                          mean.data_ptr(), invstd.data_ptr(), act, slope, sums[0].data_ptr(),
                                                          sums[1].data_ptr(), _stream()))
                s0, s1 = sums[0].data_ptr(), sums[1].data_ptr()
            if small:
                pass
            elif msum is not None:
                _lib.check(lib.pcb_bn_act_backward_apply_renorm(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), shift.data_ptr(),
                                                                mean.data_ptr(), invstd.data_ptr(), act, slope, s0, s1, 1, msum.data_ptr(),
                                                                dx.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr(), _stream()))
            else:
                _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), shift.data_ptr(),
                                                         mean.data_ptr(), invstd.data_ptr(), act, slope, s0, s1, 1, dx.data_ptr(),
                                                         outs[0].data_ptr(), outs[1].data_ptr(), _stream()))
            dgamma = None if sinks[0] is not None else outs[0]
            dbeta = None if sinks[1] is not None else outs[1]
            for sk in sinks:
                if sk is not None and sk.on_written is not None:
                    sk.on_written()
        elif has_bn:   # eval-mode BN: a fixed affine map (parameter grads not produced in eval)
            _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), code, count, c, scale.data_ptr(), shift.data_ptr(),
                                                     None, None, act, slope, None, None, 0, dx.data_ptr(), None, None, _stream()))
        else:
            _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), code, count, c, None, None, None, None, act, slope,
                                                     None, None, 0, dx.data_ptr(), None, None, _stream()))
        return dx, dgamma, dbeta, (gy if has_res else None), None, None, None, None, None, None, None, None, None, None


def bn_act(x, bn, act, residual=None, handoff=None, pre_sums=None):
    """`bn`: nn.BatchNorm2d or None; `act`: nn activation module / None.  `handoff`: the RenormHandoff of the partial
    convolution whose output `x` is, when this call is that output's only consumer."""
    x = as_feature(x)
    code, slope = act_code(act)
    if residual is not None:
        residual = as_feature(residual)
    if bn is None:
        return BNActFn.apply(x, None, None, residual, None, None, None, False, 0.0, 0.0, code, slope)
    momentum = 0.1 if bn.momentum is None else bn.momentum
    msum = None
    if handoff is not None and handoff.eligible and bn.training and x.requires_grad and x.shape[1] % 8 == 0 and x.shape[1] <= 2048 \
            and x.is_contiguous(memory_format=CL):
        msum, handoff.fused = handoff.msum, True
    if pre_sums is None:
        pre_sums = handoff.bn_sums if (handoff is not None and bn.training and bn.weight is not None) else None
    if pre_sums is not None and not (bn.training and x.is_contiguous(memory_format=CL)):
        pre_sums = None
    return BNActFn.apply(x, bn.weight, bn.bias, residual, bn.running_mean, bn.running_var, bn.num_batches_tracked,
                         bn.training, momentum, bn.eps, code, slope, msum, pre_sums)


def activation_only(x, act, residual=None):
    x = as_feature(x)
    code, slope = act_code(act)
    return BNActFn.apply(x, None, None, residual, None, None, None, False, 0.0, 0.0, code, slope)


# ------------------------------------------------------------------------------------------------
# nearest upsample / channel concat
# ------------------------------------------------------------------------------------------------
class ConcatFn(torch.autograd.Function):
    """cat([up2x?(x_i)], dim=1) in one pass (image_inpainting.py:183-184)."""

    @staticmethod
    def forward(ctx, ups: Tuple[int, ...], *xs):
        lib = _lib.load()
        x0 = xs[0]
        n = x0.shape[0]
        h, w = x0.shape[2] << ups[0], x0.shape[3] << ups[0]
        code = _dtype_code(x0)
        parts = (Part * len(xs))()
        ctot = 0
        for i, (x, up) in enumerate(zip(xs, ups)):
            if (x.shape[2] << up, x.shape[3] << up) != (h, w) or x.dtype != x0.dtype:
                raise _lib.PcbError("concat: mismatched spatial size or dtype")
            parts[i].x, parts[i].mask, parts[i].c, parts[i].x_cstride, parts[i].x_up, parts[i].mask_up = x.data_ptr(), None, x.shape[1], x.shape[1], up, 0
            ctot += x.shape[1]
        y = torch.empty((n, ctot, h, w), dtype=x0.dtype, device=x0.device, memory_format=CL)
        _lib.check(lib.pcb_concat_forward(parts, len(xs), code, n, h, w, y.data_ptr(), _stream()))
        ctx.meta = (ups, [x.shape[1] for x in xs], code, n, h, w)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        ups, cs, code, n, h, w = ctx.meta
        gy = gy.contiguous(memory_format=CL)
        outs: List[Optional[torch.Tensor]] = []
        ptrs = (ctypes.c_void_p * len(cs))()
        for i, (c, up) in enumerate(zip(cs, ups)):
            if ctx.needs_input_grad[i + 1]:
                g = torch.empty((n, c, h >> up, w >> up), dtype=gy.dtype, device=gy.device, memory_format=CL)
                outs.append(g)
                ptrs[i] = g.data_ptr()
            else:
                outs.append(None)
                ptrs[i] = None
        carr = (ctypes.c_int32 * len(cs))(*cs)
        uarr = (ctypes.c_int32 * len(cs))(*ups)
        _lib.check(lib.pcb_concat_backward(gy.data_ptr(), carr, uarr, len(cs), code, n, h, w, ptrs, _stream()))
        return (None, *outs)


def concat_features(xs: Sequence[torch.Tensor], ups: Optional[Sequence[int]] = None) -> torch.Tensor:
    xs = [as_feature(x) for x in xs]
    ups = tuple(int(u) for u in (ups if ups is not None else [0] * len(xs)))
    dt = xs[0].dtype
    xs = [x if x.dtype == dt else x.to(dt) for x in xs]
    return ConcatFn.apply(ups, *xs)


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    return ConcatFn.apply((1,), as_feature(x))


# ------------------------------------------------------------------------------------------------
# benchmark-step helpers: L1-mean loss and fused SGD
# ------------------------------------------------------------------------------------------------
class L1MeanFn(torch.autograd.Function):
    """loss = x.abs().mean()  (SURVEY 8d benchmark loss)."""

    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        x = x.contiguous(memory_format=CL) if x.dim() == 4 else x.contiguous()
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        scratch = torch.empty((1,), dtype=torch.float64, device=x.device)
        _lib.check(lib.pcb_l1_mean_forward(x.data_ptr(), _dtype_code(x), x.numel(), loss.data_ptr(), scratch.data_ptr(), _stream()))
        ctx.save_for_backward(x)
        return loss

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        (x,) = ctx.saved_tensors
        gx = torch.empty_like(x)
        # the incoming gradient of a scalar loss is 1 in the benchmark; fold a general scale in on the host only
        # when it is a Python number -- otherwise multiply afterwards (keeps the kernel sync-free)
        _lib.check(lib.pcb_l1_mean_backward(x.data_ptr(), _dtype_code(x), x.numel(), 1.0 / x.numel(), gx.data_ptr(), _stream()))
        return gx * g.to(gx.dtype) if g is not None else gx


def l1_mean(x):
    return L1MeanFn.apply(as_feature(x) if x.dim() == 4 else x)


def sgd_step(param, grad, buf, lr, momentum=0.0, weight_decay=0.0, nesterov=False, first_step=False, grad_scale=1.0):
    """torch.optim.SGD semantics on flat buffers; `grad_scale` multiplies the gradient first (data parallel: 1 / world on the
    all-reduced SUM, so no separate scaling pass)."""
    lib = _lib.load()
    if not (param.is_contiguous() or param.is_contiguous(memory_format=CL)) or param.stride() != grad.stride():
        raise _lib.PcbError("sgd_step: param and grad must be dense with identical strides")
    _lib.check(lib.pcb_sgd_step_scaled(param.data_ptr(), grad.data_ptr(), _ptr(buf), param.numel(), float(lr), float(momentum),
                                       float(weight_decay), int(nesterov), int(first_step), float(grad_scale), _stream()))
    bump_weight_epoch()


# ------------------------------------------------------------------------------------------------
# dense (non-partial) building blocks of the segmentation networks
# ------------------------------------------------------------------------------------------------
def _dense8(x: torch.Tensor):
    """x as a dense NHWC tensor whose channel count is a multiple of 8 (zero-padded copy if needed).
    Returns (tensor with c8 channels, original channel count)."""
    x = as_feature_padded(x)
    n, c, h, w = x.shape
    c8 = (c + 7) // 8 * 8
    cs = nhwc_layout(x)
    if c8 == c and cs == c:
        return x, c
    if cs == c8:                       # a [:, :c] view of a padded buffer: use the buffer itself
        base = x.as_strided((n, c8, h, w), (h * w * c8, 1, w * c8, c8))
        return base, c
    buf = padded_empty(n, c, h, w, x.dtype, x.device)
    buf.copy_(x)
    return buf.as_strided((n, c8, h, w), (h * w * c8, 1, w * c8, c8)), c


def conv2d(x, weight, bias, stride, padding, dilation, groups, cache=None, handoff=None):
    """nn.Conv2d on the same kernels as the partial convolution (`plain`: mask ignored, renormaliser 1)."""
    x = as_feature_padded(x)
    if x.dtype == torch.bfloat16 and x.shape[1] < 8 and nhwc_layout(x) % 8 != 0 and groups == 1:
        buf = padded_empty(*x.shape, x.dtype, x.device)          # 16-byte pixels -> row-packed tensor-core path
        buf.copy_(x)
        x = buf
    y, _ = partial_conv(x, None, weight, bias, stride, padding, dilation, groups, cache=cache, plain=True, handoff=handoff)
    return y


class _Pool2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad):
        lib = _lib.load()
        n, c, h, w = x.shape
        ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
        y = torch.empty((n, c, ho, wo), dtype=x.dtype, device=x.device, memory_format=CL)
        _lib.check(lib.pcb_avgpool_forward(x.data_ptr(), y.data_ptr(), _dtype_code(x), n, h, w, c, k, stride, pad, _stream()))
        ctx.meta = (n, c, h, w, k, stride, pad)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        n, c, h, w, k, stride, pad = ctx.meta
        gy = gy.contiguous(memory_format=CL)
        gx = torch.empty((n, c, h, w), dtype=gy.dtype, device=gy.device, memory_format=CL)
        _lib.check(lib.pcb_avgpool_backward(gy.data_ptr(), gx.data_ptr(), _dtype_code(gy), n, h, w, c, k, stride, pad, _stream()))
        return gx, None, None, None


def avg_pool2d(x, k, stride, pad):
    """nn.AvgPool2d(k, stride, pad), count_include_pad=True."""
    xb, c = _dense8(x)
    y = _Pool2dFn.apply(xb, int(k), int(stride), int(pad))
    return y if y.shape[1] == c else y[:, :c]


class _BilinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, scale):
        lib = _lib.load()
        n, c, h, w = x.shape
        y = torch.empty((n, c, h * scale, w * scale), dtype=x.dtype, device=x.device, memory_format=CL)
        _lib.check(lib.pcb_bilinear_forward(x.data_ptr(), y.data_ptr(), _dtype_code(x), n, h, w, c, scale, _stream()))
        ctx.meta = (n, c, h, w, scale)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        n, c, h, w, scale = ctx.meta
        gy = gy.contiguous(memory_format=CL)
        gx = torch.empty((n, c, h, w), dtype=gy.dtype, device=gy.device, memory_format=CL)
        _lib.check(lib.pcb_bilinear_backward(gy.data_ptr(), gx.data_ptr(), _dtype_code(gy), n, h, w, c, scale, _stream()))
        return gx, None


def bilinear_upsample(x, scale):
    """F.interpolate(x, scale_factor=scale, mode='bilinear', align_corners=False) for integer scale."""
    if int(scale) != scale or scale < 1:
        raise NotImplementedError("bilinear upsampling: integer scale factors only")
    xb, c = _dense8(x)
    y = _BilinearFn.apply(xb, int(scale))
    return y if y.shape[1] == c else y[:, :c]


class _GapFn(torch.autograd.Function):
    """nn.AdaptiveAvgPool2d(1)(x).view(n, c) in fp32."""

    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        n, c, h, w = x.shape
        out = torch.empty((n, c), dtype=torch.float32, device=x.device)
        _lib.check(lib.pcb_gap_forward(x.data_ptr(), _dtype_code(x), n, h * w, c, out.data_ptr(), _stream()))
        ctx.meta = (n, c, h, w, x.dtype)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        n, c, h, w, dt = ctx.meta
        g = g.contiguous().float()
        dx = torch.empty((n, c, h, w), dtype=dt, device=g.device, memory_format=CL)
        _lib.check(lib.pcb_gap_backward(g.data_ptr(), dx.data_ptr(), PCB_BF16 if dt == torch.bfloat16 else PCB_F32, n, h * w, c, 0, _stream()))
        return dx


class _ScseFn(torch.autograd.Function):
    """y = x * cse[n, c] + x * sigmoid(<x[p, :], ws>)   (models/common.py:37-43)."""

    @staticmethod
    def forward(ctx, x, cse, ws):
        lib = _lib.load()
        n, c, h, w = x.shape
        cse32, ws32 = cse.contiguous().float(), ws.contiguous().float()
        y = torch.empty_like(x, memory_format=CL)
        sse = torch.empty((n * h * w,), dtype=torch.float32, device=x.device)
        _lib.check(lib.pcb_scse_forward(x.data_ptr(), cse32.data_ptr(), ws32.data_ptr(), y.data_ptr(), sse.data_ptr(), _dtype_code(x),
                                        n, h * w, c, _stream()))
        ctx.save_for_backward(x, cse32, ws32, sse)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x, cse, ws, sse = ctx.saved_tensors
        n, c, h, w = x.shape
        gy = gy.contiguous(memory_format=CL)
        if gy.dtype != x.dtype:
            gy = gy.to(x.dtype)
        dx = torch.empty_like(x, memory_format=CL)
        dcse = torch.empty_like(cse)
        dws = torch.empty_like(ws)
        _lib.check(lib.pcb_scse_backward(gy.data_ptr(), x.data_ptr(), cse.data_ptr(), ws.data_ptr(), sse.data_ptr(), dx.data_ptr(),
                                         dcse.data_ptr(), dws.data_ptr(), _dtype_code(x), n, h * w, c, _stream()))
        return dx, dcse, dws


def global_avg_pool(x):
    return _GapFn.apply(as_feature(x))


def scse_gate(x, cse, ws):
    return _ScseFn.apply(as_feature(x), cse, ws)

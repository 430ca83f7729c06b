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
# the execution mode of one engine step
# ------------------------------------------------------------------------------------------------
_SCOPE: Optional["StepScope"] = None


class StepScope:
    """The execution mode of one engine step, and the state that lives exactly as long as one entry.  An engine builds one and
    runs each step (training) or forward (inference) inside ``with scope:``; at most one scope is current at a time.

    Both kinds run every layer's mask pass on the mask stream, ahead of the feature path (its ready events are kept per entry,
    keyed by mask plane).  A training scope also owns a zero arena, so that reduction targets (BatchNorm sums) are slices of one
    buffer zeroed once on entry (`zeros_f64`) instead of one memset each.  It lets `OperandCache` rewrite operand buffers in
    place and `prefetch_weights` refresh them ahead, and lets weight-gradient sinks defer their side stream's join to the exit.  An
    inference scope applies eval-mode BatchNorm + activation in the convolution epilogues (`eval_epilogue`) and counts the
    sites: `fused_sites` in an epilogue, `unfused_sites` still run on their own.  Outside any scope every one of these is off.

    Leaving, on an exception too, joins the current stream to the auxiliary streams this entry put work on (`streams`, kept
    until the next entry) and drops the entry's keep-alive list and ready events."""

    ARENA_BYTES = 1 << 20

    def __init__(self, device, training: bool):
        self.training = bool(training)
        self._arena = torch.empty((self.ARENA_BYTES,), dtype=torch.uint8, device=device) if self.training else None
        self._off = 0
        self.fused_sites = self.unfused_sites = 0
        self.streams: List[torch.cuda.Stream] = []
        self._keep = []
        self._ready = {}            # mask plane -> the event it is ready at (tensors hash by identity)

    def __enter__(self):
        global _SCOPE
        if _SCOPE is not None:
            raise _lib.PcbError("a StepScope is already current: engine steps do not nest")
        self._off = self.fused_sites = self.unfused_sites = 0
        self.streams = []
        if self._arena is not None:
            self._arena.zero_()
        _SCOPE = self
        return self

    def __exit__(self, *exc):
        global _SCOPE
        try:
            cur = torch.cuda.current_stream()
            for st in self.streams:
                cur.wait_stream(st)
        finally:
            self._keep, self._ready = [], {}
            _SCOPE = None
        return False

    def _use(self, stream, keep=None):
        """`stream` carries work of this entry (that reads or writes `keep`): join it on exit, keep `keep` alive until then."""
        if stream not in self.streams:
            self.streams.append(stream)
        if keep is not None:
            self._keep.append(keep)


def current_scope() -> Optional[StepScope]:
    """The StepScope the current step runs in, or None."""
    return _SCOPE


def zeros_f64(n, device):
    """n zeroed doubles: a slice of the training scope's arena when it has room, else a fresh zero tensor."""
    s = _SCOPE
    nbytes = (n * 8 + 255) // 256 * 256
    if s is not None and s._arena is not None and device == s._arena.device and s._off + nbytes <= s._arena.numel():
        view = s._arena[s._off:s._off + n * 8].view(torch.float64)
        s._off += nbytes
        return view
    return torch.zeros((n,), dtype=torch.float64, device=device)


_AUX_STREAMS = {}


def _aux_stream(kind: str, device) -> torch.cuda.Stream:
    """The process-wide auxiliary stream `kind` ("mask", "side": weight gradients, "prefetch": operand refreshes) of `device`."""
    key = (kind, device.index if device.index is not None else torch.cuda.current_device())
    if key not in _AUX_STREAMS:
        _AUX_STREAMS[key] = torch.cuda.Stream(device=device)
    return _AUX_STREAMS[key]


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


def _pconv_launch(lib, geom: ConvGeom, c: Conv, w_fwd, b32, y, bn_sums, epi: Optional["EvalEpilogue"]):
    """Mask pass + forward of one partial convolution into `y`; returns (msum, newmask, the event newmask is ready at on the
    mask stream or None).  `bn_sums`: training statistics target (pcb_pconv_forward_bn); `epi`: eval-mode BatchNorm +
    activation applied in the epilogue (pcb_pconv_forward_affine_act)."""
    dev = y.device
    scope = _SCOPE

    def forward(mask_pass_done, msum, newmask, ws):
        if epi is None:
            return lib.pcb_pconv_forward_bn(ctypes.byref(c), w_fwd.data_ptr(), _ptr(b32), y.data_ptr(), nhwc_layout(y), msum.data_ptr(),
                                            newmask.data_ptr(), ws.data_ptr(), mask_pass_done, _ptr(bn_sums), _stream())
        scale, shift = epi.coefficients()
        return lib.pcb_pconv_forward_affine_act(ctypes.byref(c), w_fwd.data_ptr(), _ptr(b32), y.data_ptr(), nhwc_layout(y), msum.data_ptr(),
                                                newmask.data_ptr(), ws.data_ptr(), mask_pass_done, _ptr(scale), _ptr(shift), epi.code,
                                                epi.slope, _stream())

    if scope is not None and _PROFILE is None and not geom.plain:
        # Mask updates never depend on features (partial_convolution.py:59-77): the mask pass of this layer runs on the
        # mask stream, ordered only after the passes that produced its input planes, i.e. ahead of the feature path.
        # Its buffers are allocated on that stream and kept alive until the scope's exit joins it.
        main, ms = torch.cuda.current_stream(), _aux_stream("mask", dev)
        for (_, _, _, pl, _) in geom.parts:
            if pl is None:
                continue
            ev_in = scope._ready.get(pl)
            if ev_in is None:                        # a plane written on the main stream (the network's input mask): mark it
                ev_in = torch.cuda.Event()           # ready from here on, so later consumers (the tail) need not wait for main
                ev_in.record(main)
                scope._ready[pl] = ev_in
            ms.wait_event(ev_in)
        with torch.cuda.stream(ms):
            msum = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.float32, device=dev)
            newmask = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.uint8, device=dev)
            ws = _workspace(lib, c, dev)
            _lib.check(lib.pcb_pconv_mask_pass(ctypes.byref(c), msum.data_ptr(), newmask.data_ptr(), ws.data_ptr(), _stream()))
            ev = torch.cuda.Event()
            ev.record()
        main.wait_event(ev)
        scope._use(ms, (msum, newmask, ws))
        _lib.check(forward(1, msum, newmask, ws))
    else:
        msum = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.float32, device=dev)
        newmask = torch.empty((geom.mg, geom.n, geom.ho, geom.wo), dtype=torch.uint8, device=dev)
        ws = _workspace(lib, c, dev)
        ev = None
        with _Timed("fwd", geom):
            _lib.check(forward(0, msum, newmask, ws))
    return msum, newmask, ev


# ------------------------------------------------------------------------------------------------
# inference: eval-mode BatchNorm + activation fused into the convolution epilogue
# ------------------------------------------------------------------------------------------------
def _inference_scope() -> Optional[StepScope]:
    return _SCOPE if _SCOPE is not None and not _SCOPE.training else None


def bn_eval_coefficients(bn) -> Tuple[torch.Tensor, torch.Tensor]:
    """(scale, shift) fp32 [c] of an eval-mode nn.BatchNorm2d, from pcb_bn_finalize(training=0) -- the same coefficients the
    two-pass path computes.  Cached on the module; rewritten IN PLACE when the weight epoch or a parameter / buffer version
    changes, so a captured graph that reads them sees the new values.  Not recomputed during a graph capture."""
    key = (_WEIGHT_EPOCH, bn.weight._version, bn.bias._version, bn.running_mean._version, bn.running_var._version,
           bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr())
    cache = bn.__dict__.setdefault("_pcb_bn_coef", {})
    if cache.get("key") != key:
        if torch.cuda.is_current_stream_capturing():
            raise _lib.PcbError("BatchNorm eval coefficients are stale inside a graph capture: refresh them before capturing")
        c = bn.num_features
        buf = cache.get("buf")
        if buf is None or buf.device != bn.weight.device:
            buf = torch.empty((2, c), dtype=torch.float32, device=bn.weight.device)
        momentum = 0.1 if bn.momentum is None else bn.momentum
        lib = _lib.load()
        _lib.check(lib.pcb_bn_finalize(None, None, 1, c, bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(),
                                       bn.running_var.data_ptr(), None, float(momentum), float(bn.eps), 0,
                                       buf[0].data_ptr(), buf[1].data_ptr(), None, None, _stream()))
        cache["key"], cache["buf"] = key, buf
    return cache["buf"][0], cache["buf"][1]


class EvalEpilogue:
    """An eval-mode BatchNorm (or none) + activation that a convolution may apply in its epilogue.  `fused` tells the caller
    whether it did (pcb_conv_fuses_affine_act refused the problem otherwise: the caller then runs the BatchNorm pass itself)."""

    def __init__(self, bn, act):
        self.bn, self.act = bn, act
        self.code, self.slope = act_code(act)
        self.fused = False

    def coefficients(self):
        return bn_eval_coefficients(self.bn) if self.bn is not None else (None, None)


def eval_epilogue(bn, act) -> Optional[EvalEpilogue]:
    """The epilogue for a convolution whose ONLY consumer is `act(bn(.))`, or None outside an inference StepScope, when the
    BatchNorm is in training mode / has no running statistics or affine parameters, or when the activation has no kernel.
    A plain ``net.eval(); net(x)`` therefore runs the two-pass path."""
    if _inference_scope() is None:
        return None
    if bn is not None and (bn.training or bn.running_mean is None or bn.weight is None or bn.bias is None):
        return None
    try:
        return EvalEpilogue(bn, act)
    except NotImplementedError:
        return None


def _partial_conv_fused_eval(geom: ConvGeom, wprep, bias, xs, epi: EvalEpilogue):
    """Forward of a partial convolution with `epi` applied in its epilogue (inference only: no autograd), or None when the
    kernel this problem dispatches to cannot apply it."""
    lib = _lib.load()
    c = geom.struct(xs)
    if torch.is_grad_enabled() or not lib.pcb_conv_fuses_affine_act(ctypes.byref(c)):
        return None
    dev = xs[0].device
    if geom.dtype == PCB_BF16:
        y = padded_empty(geom.n, geom.cout, geom.ho, geom.wo, xs[0].dtype, dev)
    else:
        y = torch.empty((geom.n, geom.cout, geom.ho, geom.wo), dtype=xs[0].dtype, device=dev, memory_format=CL)
    b32 = bias.detach().float().contiguous() if bias is not None else None
    out = _pconv_launch(lib, geom, c, wprep.w_fwd, b32, y, None, epi)
    epi.fused = True
    if _SCOPE is not None:
        _SCOPE.fused_sites += 1
    return (y, *out)


class PartialConvFn(torch.autograd.Function):
    """y, msum, newmask = pconv(cat(up?(x_i)), W, b | mask)   (models/partial_convolution.py:49-80 / :121-137), and the event
    newmask is ready at when the mask pass ran on the mask stream (else None)."""

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
        if handoff is not None and handoff.want_stats and lib.pcb_conv_fuses_bn_stats(ctypes.byref(c)) \
                and nhwc_layout(y) == geom.cout:
            bn_sums = zeros_f64(2 * geom.cout, dev)
            handoff.bn_sums = bn_sums
        msum, newmask, mask_ready = _pconv_launch(lib, geom, c, w_fwd, b32, y, bn_sums, None)
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
        return y, msum, newmask, mask_ready

    @staticmethod
    def backward(ctx, gy, _gmsum, _gnewmask, _gready):
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
            # no accumulation pass) and autograd gets no tensor; inside a training StepScope the side stream below then joins
            # at the scope's exit, so the weight gradient also overlaps the element-wise backward kernels of the layers that
            # follow.  A second use of the same weight in one pass falls back to autograd accumulation.
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
            if (any(need) or sink is not None) and _PROFILE is None:
                side = _aux_stream("side", dev)
                side.wait_stream(torch.cuda.current_stream())
                deferred = sink is not None and _SCOPE is not None and _SCOPE.training
                if deferred:
                    _SCOPE._use(side, (dc, ws, xs))            # keep the side stream's operands alive until the join
                with torch.cuda.stream(side):
                    _lib.check(wgrad_fn(ctypes.byref(c), dc.data_ptr(), dcs, dw_buf.data_ptr(), ws.data_ptr(), _stream()))
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


def _inplace_weight_refresh() -> bool:
    """Inside a training StepScope an `OperandCache` may rewrite its operand buffers in place instead of allocating + zero-filling
    new ones: the engine updates the masters once per step, after every backward of that step has run.  Outside one, a backward
    that runs after a later weight update would read the new weights."""
    return _SCOPE is not None and _SCOPE.training


def _operand_key(weight: torch.Tensor, geom: ConvGeom, frozen: bool):
    """What operands laid out from `weight` for `geom` stay valid for: the weight's storage, version and device, the problem
    signature and, unless frozen, the weight epoch (updates through raw pointers do not bump the version)."""
    return (weight.data_ptr(), weight._version, str(weight.device), None if frozen else _WEIGHT_EPOCH, geom.signature)


class Operands:
    """One convolution weight as the compute-dtype operand buffers the kernels read for the problem `geom`: `w_fwd`, and `w_dg`
    (None when the problem has none); unpacks as the pair ``w_fwd, w_dg``.  The fp32 master laid out is `derive(weight)`, by
    default the weight itself (physically [cout][kh][kw][cin/groups])."""

    def __init__(self, weight: torch.Tensor, geom: ConvGeom, derive=None):
        self.weight, self.geom, self.derive = weight, geom, derive
        wm, c = self.master(), geom.struct(None)
        fe, de = self.sizes(c)
        tdt = torch.bfloat16 if geom.dtype == PCB_BF16 else torch.float32
        self.w_fwd = torch.empty((fe,), dtype=tdt, device=wm.device)
        self.w_dg = torch.empty((de,), dtype=tdt, device=wm.device) if de else None
        self.lay_out(c, wm, self.w_fwd, self.w_dg)

    @staticmethod
    def sizes(c: Conv) -> Tuple[int, int]:
        """Element counts of the forward and data-gradient operand buffers of problem `c` (0: none)."""
        fe, de = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.load().pcb_conv_weight_layout(ctypes.byref(c), ctypes.byref(fe), ctypes.byref(de))
        return fe.value, de.value

    @staticmethod
    def lay_out(c: Conv, master: torch.Tensor, w_fwd, w_dg, refresh=False):
        """Lay `master` out into the buffers of problem `c` on the current stream; `refresh`: buffers a prepare already filled."""
        lib = _lib.load()
        fn = lib.pcb_conv_weight_refresh if refresh else lib.pcb_conv_weight_prepare
        _lib.check(fn(ctypes.byref(c), master.data_ptr(), w_fwd.data_ptr(), _ptr(w_dg), _stream()))

    def __iter__(self):
        return iter((self.w_fwd, self.w_dg))

    def master(self) -> torch.Tensor:
        return self.derive(self.weight) if self.derive is not None else self.weight.detach().float().contiguous(memory_format=CL)

    def refresh(self):
        """Rewrite the buffers in place from the weight's current values, on the current stream."""
        self.lay_out(self.geom.struct(None), self.master(), self.w_fwd, self.w_dg, refresh=True)


class OperandCache:
    """A module's operands of one convolution weight, kept from one call to the next.  `get(weight, geom)` returns the current
    record while its key (`_operand_key`) matches, else the current record rewritten in place inside a training StepScope when
    the layout is unchanged, else a new record: the buffers of a record a captured graph keeps are never freed.

    `frozen` (weights no optimiser updates, the VGG loss): the key leaves out the weight epoch, so the operands are laid out again
    only when the weight itself changes, never in place and never inside a graph capture.  `derive`: see Operands."""

    def __init__(self, frozen=False, derive=None):
        self.frozen, self.derive = frozen, derive
        self.current: Optional[Operands] = None
        self.key, self.ready = None, None       # ready: event of a prefetch_weights() refresh not yet waited on

    def get(self, weight: torch.Tensor, geom: ConvGeom) -> Operands:
        key = _operand_key(weight, geom, self.frozen)
        rec = self.current
        if key == self.key:
            if self.ready is not None:
                torch.cuda.current_stream().wait_event(self.ready)
                self.ready = None
            return rec
        if self.frozen and torch.cuda.is_current_stream_capturing():
            raise _lib.PcbError("VGG operands are stale inside a graph capture: run the loss once before capturing")
        if (_inplace_weight_refresh() and not self.frozen and rec is not None and rec.geom.signature == geom.signature
                and rec.w_fwd.device == weight.device
                and Operands.sizes(geom.struct(None)) == (rec.w_fwd.numel(), rec.w_dg.numel() if rec.w_dg is not None else 0)):
            rec.weight, rec.geom = weight, geom
            rec.refresh()
        else:
            rec = Operands(weight, geom, self.derive)
        self.current, self.key, self.ready = rec, key, None
        return rec

    def refresh(self, rec: Operands):
        """Rewrite `rec`, a record this cache handed out, in place on the current stream; the next get() hits if it is current."""
        rec.refresh()
        if rec is self.current:
            self.key, self.ready = _operand_key(rec.weight, rec.geom, self.frozen), None


def operand_caches(*roots: torch.nn.Module):
    """(module, attribute name, cache) of every OperandCache that a module of these module trees holds."""
    return [(m, name, c) for r in roots for m in r.modules() for name, c in vars(m).items() if isinstance(c, OperandCache)]


def prefetch_weights(caches):
    """Re-lay-out the weights behind `caches` (OperandCache; frozen and empty ones are skipped) on a prefetch stream, ahead of the
    layers' forward calls (training engines call this right after the optimiser step / epoch bump; only inside a training
    StepScope).  Each layer's forward then only waits on its own event, so the re-layout of layer k overlaps the layers before it."""
    caches = [c for c in caches if c.current is not None and not c.frozen]
    if not _inplace_weight_refresh() or not caches:
        return
    dev = caches[0].current.weight.device
    ps = _aux_stream("prefetch", dev)
    ps.wait_stream(torch.cuda.current_stream())           # after the optimiser step, and after every reader of the old buffers
    _SCOPE._use(ps)
    with torch.cuda.stream(ps):
        for cache in caches:
            rec = cache.current
            if rec.weight.device != dev or rec.weight.dtype != torch.float32 or cache.key == _operand_key(rec.weight, rec.geom, False):
                continue
            cache.refresh(rec)
            cache.ready = torch.cuda.Event()
            cache.ready.record()


class GradSink:
    """In-place destination for a convolution weight gradient (see PartialConvFn.backward).  The owner resets `used` before
    every backward pass; inside a training StepScope the gradient is complete on the scope's exit, outside one when the
    backward returns."""

    def __init__(self, view: torch.Tensor):
        self.view, self.used = view, False
        self.prezeroed = False        # the owner guarantees `view` is zero when the backward pass starts (skip the kernel's memset)
        self.on_written = None        # optional callback: the kernel that writes `view` has just been launched


class RenormHandoff:
    """Links a partial convolution to the BatchNorm(+activation) that is the ONLY consumer of its output (the blocks of
    models/partial_convolution.py): the BN backward then writes dc = dy / mask_sum directly (one pass less over every conv
    output) and the convolution's backward skips its renormalisation step.  Never use it when y has another consumer."""

    def __init__(self, want_stats=False):
        self.msum, self.eligible, self.fused = None, False, False
        # want_stats: the consumer is a training-mode BatchNorm -> the convolution accumulates the per-channel sum / sum of
        # squares of its output in its epilogue (`bn_sums`, [2][cout] doubles) and the statistics pass over y disappears
        self.want_stats, self.bn_sums = bool(want_stats), None


def partial_conv(x, mask, weight, bias, stride, padding, dilation, groups, same_holes=False, no_guard=False, cache=None,
                 plain=False, handoff=None, epilogue: Optional[EvalEpilogue] = None):
    """Returns (y, new_mask: HoleMask).  `x` is a tensor or a LazyCat; `mask` a HoleMask or a dense tensor; with
    ``plain=True`` the mask is ignored and an ordinary convolution is computed (same kernels, renormaliser 1).
    `epilogue` (inference, no autograd): the eval-mode BatchNorm + activation that is y's only consumer, applied in the
    convolution epilogue when the kernel can (``epilogue.fused`` tells; otherwise y is the plain convolution output)."""
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
    wprep = (cache if cache is not None else OperandCache()).get(weight, geom)
    out = _partial_conv_fused_eval(geom, wprep, bias, xs, epilogue) if epilogue is not None else None
    y, msum, newmask, mask_ready = out if out is not None else PartialConvFn.apply(geom, wprep, weight, bias, handoff, *xs)
    planes = [newmask[g] for g in range(geom.mg)]
    if mask_ready is not None:                            # written on the mask stream: consumers there wait on this event
        for pl in planes:
            _SCOPE._ready[pl] = mask_ready
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
            small = _vec_bn(c) and count <= 16384 and c >= 256 and scale.data_ptr() + 4 * c == shift.data_ptr() \
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
    scope = _inference_scope()
    if scope is not None:
        scope.unfused_sites += 1
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
    scope = _inference_scope()
    if scope is not None:
        scope.unfused_sites += 1
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


def sgd_step_dev(param, grad, buf, lr, momentum=0.0, weight_decay=0.0, nesterov=False, grad_scale=1.0):
    """sgd_step with the learning rate read on the device from `lr` (fp32, one element) and no first-step flag: `buf` is always
    read, so it must start zeroed (momentum * 0 + d == d) and a restored buffer is never discarded."""
    lib = _lib.load()
    if not param.is_cuda or not (param.is_contiguous() or param.is_contiguous(memory_format=CL)) or param.stride() != grad.stride():
        raise _lib.PcbError("sgd_step_dev: param and grad must be dense CUDA tensors with identical strides")
    if lr.dtype != torch.float32 or lr.numel() != 1 or lr.device != param.device:
        raise _lib.PcbError("sgd_step_dev: lr must be one fp32 element on the parameters' device")
    _lib.check(lib.pcb_sgd_step_dev(param.data_ptr(), grad.data_ptr(), _ptr(buf), param.numel(), lr.data_ptr(), float(momentum),
                                    float(weight_decay), int(nesterov), float(grad_scale), _stream()))
    bump_weight_epoch()


def lr_cyclic(iteration, lr, lr64, base_lr, max_lr, step_size, mode, gamma=1.0):
    """The cyclical learning rate of device iteration counter `iteration` (int64, one element) into `lr` (fp32) and `lr64`
    (fp64), then iteration += 1 -- all on the device, so a captured graph advances the schedule on every replay.  `mode`:
    _lib.CLR_TRIANGULAR, CLR_TRIANGULAR2 or CLR_EXP_RANGE."""
    lib = _lib.load()
    if iteration.dtype != torch.int64 or lr.dtype != torch.float32 or lr64.dtype != torch.float64 or \
            not (iteration.device == lr.device == lr64.device) or not iteration.is_cuda:
        raise _lib.PcbError("lr_cyclic: iteration (int64), lr (fp32) and lr64 (fp64) must be CUDA tensors on one device")
    _lib.check(lib.pcb_lr_cyclic(iteration.data_ptr(), float(base_lr), float(max_lr), float(step_size), int(mode), float(gamma),
                                 lr.data_ptr(), lr64.data_ptr(), _stream()))


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


def conv2d(x, weight, bias, stride, padding, dilation, groups, cache=None, handoff=None, epilogue=None):
    """nn.Conv2d on the same kernels as the partial convolution (`plain`: mask ignored, renormaliser 1)."""
    x = as_feature_padded(x)
    if x.dtype == torch.bfloat16 and x.shape[1] < 8 and nhwc_layout(x) % 8 != 0 and groups == 1:
        buf = padded_empty(*x.shape, x.dtype, x.device)          # 16-byte pixels -> row-packed tensor-core path
        buf.copy_(x)
        x = buf
    y, _ = partial_conv(x, None, weight, bias, stride, padding, dilation, groups, cache=cache, plain=True, handoff=handoff,
                        epilogue=epilogue)
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


# ------------------------------------------------------------------------------------------------
# post-processing of the text-segmentation output
# ------------------------------------------------------------------------------------------------
def text_mask_postprocess(logits: torch.Tensor, border_pad, out_hw) -> torch.Tensor:
    """The demo's mask from the segmentation logits in one launch (Examples/demo_segmentation.py:33-36 with the resizer of
    Dataloader.py:308-316): ``upsample_bilinear(unpad(maxpool3x3(sigmoid(logits) > 0.5)), out_hw) > 0`` of channel 0.
    `border_pad`: the (left, right, top, bottom) padding EvaluateSet added (``boarder_pad``; it pads right or bottom only);
    `out_hw`: (height, width) of the original image.  Returns uint8 [n, 1, oh, ow] (1 = text); the reference's 3-channel
    boolean is ``out.expand(-1, 3, -1, -1).bool()``."""
    if logits.dim() != 4 or not logits.is_cuda:
        raise _lib.PcbError("text_mask_postprocess: expected 4-D CUDA logits [n, c, h, w]")
    left, right, top, bottom = (int(v) for v in border_pad)
    if left != 0 or top != 0 or right < 0 or bottom < 0:
        raise NotImplementedError("text_mask_postprocess: only non-negative right / bottom padding (the EvaluateSet layout)")
    x = logits if nhwc_layout(logits) is not None else as_feature(logits)
    n, _, h, w = x.shape
    oh, ow = (int(v) for v in out_hw)
    out = torch.empty((n, 1, oh, ow), dtype=torch.uint8, device=x.device)
    _lib.check(_lib.load().pcb_seg_mask_postprocess(x.data_ptr(), _dtype_code(x), n, h, w, nhwc_layout(x), h - bottom, w - right, oh, ow,
                                                    out.data_ptr(), _stream()))
    return out


# ------------------------------------------------------------------------------------------------
# text removal: the glue between segmentation, mask and inpainting (csrc/text_removal.cu, engine.TextRemovalStep)
# ------------------------------------------------------------------------------------------------
def _check_page(page: torch.Tensor, fn: str, contiguous: bool = True):
    if not isinstance(page, torch.Tensor) or not page.is_cuda or page.dtype != torch.float32 or page.dim() != 4 or page.shape[1] != 3:
        shape = tuple(page.shape) if isinstance(page, torch.Tensor) else type(page).__name__
        raise _lib.PcbError(f"{fn}: expected a 4-D CUDA fp32 page [n, 3, h, w], got {shape}"
                            + (f" {page.dtype} on {page.device}" if isinstance(page, torch.Tensor) else ""))
    if contiguous and not page.is_contiguous():
        raise _lib.PcbError(f"{fn}: the page must be contiguous NCHW")
    if min(page.shape) < 1:
        raise _lib.PcbError(f"{fn}: empty page {tuple(page.shape)}")


def _check_padded(fn, what, ph, pw, h, w):
    if int(ph) < h or int(pw) < w:
        raise _lib.PcbError(f"{fn}: {what} {int(ph)}x{int(pw)} is smaller than the {h}x{w} page")


def _compute_code(dtype) -> int:
    if dtype == torch.bfloat16:
        return PCB_BF16
    if dtype == torch.float32:
        return PCB_F32
    raise _lib.PcbError(f"unsupported compute dtype {dtype}: the GPU path computes in float32 or bfloat16")


PAGE_RESIZE_MAX_REDUCTION = 16            # page_resize_bicubic's largest reduction per axis (in / out)


def evaluate_set_geometry(h: int, w: int, resize: int):
    """EvaluateSet.resize_pad_tensor's geometry for an h x w page (Dataloader.py:287-303), in Python float arithmetic as written
    there: ``ratio = resize / max(w, h)``, each side ``int(side * ratio) // 8 * 8``, then the one-sided pad: on the right when the
    resized width is below `resize`, else at the bottom.  Returns ((rh, rw), border_pad) with border_pad the (left, right, top,
    bottom) padding, so the segmentation grid is (rh + bottom) x (rw + right).  Raises ValueError for a `resize` that is not a
    positive multiple of 8, an empty resized side, or a reduction beyond page_resize_bicubic's."""
    h, w, fix_len = int(h), int(w), int(resize)
    if fix_len <= 0 or fix_len % 8 != 0:
        raise ValueError(f"evaluate_set_geometry: resize {resize} is not a positive multiple of 8")
    if h < 1 or w < 1:
        raise ValueError(f"evaluate_set_geometry: empty page {h}x{w}")
    ratio = fix_len / max(w, h)
    rw, rh = (int(x * ratio) // 8 * 8 for x in (w, h))
    if rh == 0 or rw == 0:
        raise ValueError(f"evaluate_set_geometry: a {h}x{w} page resizes to {rh}x{rw} at resize {fix_len}")
    if h > PAGE_RESIZE_MAX_REDUCTION * rh or w > PAGE_RESIZE_MAX_REDUCTION * rw:
        raise ValueError(f"evaluate_set_geometry: a {h}x{w} page resizes to {rh}x{rw}, more than a "
                         f"{PAGE_RESIZE_MAX_REDUCTION}x reduction on an axis")
    pad = (0, fix_len - rw, 0, 0) if fix_len > rw else (0, 0, 0, fix_len - rh)
    return (rh, rw), pad


def page_resize_bicubic(page: torch.Tensor, rh: int, rw: int) -> torch.Tensor:
    """EvaluateSet's page resize (Dataloader.py:291) of fp32 NCHW pages [n, 3, h, w] in [0, 1]:
    ``to_tensor(to_pil_image(page[i]).resize((rw, rh), Image.BICUBIC))`` per image, with Pillow's integer resampler bit for bit.
    Bytes are recovered as to_pil_image does (``mul(255)``, truncated), clamped to [0, 255] with NaN as 0, so a page made by
    to_tensor gives back its own bytes.  At most a 16x reduction per axis.  Returns a new fp32 [n, 3, rh, rw] tensor."""
    fn = "page_resize_bicubic"
    _check_page(page, fn)
    n, _, h, w = page.shape
    rh, rw = int(rh), int(rw)
    if rh < 1 or rw < 1:
        raise _lib.PcbError(f"{fn}: empty output size {rh}x{rw}")
    if h > PAGE_RESIZE_MAX_REDUCTION * rh or w > PAGE_RESIZE_MAX_REDUCTION * rw:
        raise _lib.PcbError(f"{fn}: {h}x{w} to {rh}x{rw} reduces more than {PAGE_RESIZE_MAX_REDUCTION}x on an axis")
    lib = _lib.load()
    ws = torch.empty((lib.pcb_page_resize_workspace(n, h, w, rh, rw),), dtype=torch.uint8, device=page.device)
    out = torch.empty((n, 3, rh, rw), dtype=torch.float32, device=page.device)
    _lib.check(lib.pcb_page_resize_bicubic(page.data_ptr(), n, h, w, rh, rw, ws.data_ptr(), out.data_ptr(), _stream()))
    return out


def removal_seg_input(page: torch.Tensor, mean_std, hs: int, ws: int, dtype=torch.bfloat16) -> torch.Tensor:
    """The segmentation network's input in one launch (EvaluateSet, Dataloader.py:271-273, 296-303): ``Normalize(mean, std)``
    of the fp32 page in torchvision's order, zero padding on the right and bottom to `hs` x `ws`, rounded once to `dtype`.
    `mean_std`: (mean[3], std[3]), or None to skip the normalization.  Returns the [n, 3, hs, ws] view of a new 8-channel NHWC
    buffer whose padded pixels and channels are zero."""
    fn = "removal_seg_input"
    _check_page(page, fn)
    n, _, h, w = page.shape
    _check_padded(fn, "padded size", hs, ws, h, w)
    norm = None
    if mean_std is not None:
        mean, std = (tuple(float(v) for v in t) for t in mean_std)
        if len(mean) != 3 or len(std) != 3:
            raise ValueError(f"{fn}: mean_std takes (mean, std) with three values each")
        norm = (ctypes.c_float * 6)(*mean, *std)
    code = _compute_code(dtype)
    buf = torch.empty((n, 8, int(hs), int(ws)), dtype=dtype, device=page.device, memory_format=CL)
    _lib.check(_lib.load().pcb_removal_seg_input(page.data_ptr(), n, h, w, norm, int(hs), int(ws), buf.data_ptr(), code, _stream()))
    return buf[:, :3]


def removal_holes(text_mask: torch.Tensor, page: torch.Tensor, hu: int, wu: int, dtype=torch.bfloat16):
    """The inpainting U-Net's input from the demo's text mask in one launch (Dataloader.py:120-121, 128-131): the mask as the
    {0, 255} image, ``> 0.4 * 255``, ``cv2.dilate`` with a 10x10 kernel, then ``valid = 1 - hole`` and ``page * valid`` on the
    `hu` x `wu` grid, whose padding on the right and bottom is hole and zero.  `text_mask`: uint8 [n, 1, h, w] (nonzero = text,
    text_mask_postprocess's output).  Returns (corrupted, valid): the [n, 3, hu, wu] view of a new 8-channel NHWC buffer in
    `dtype`, and uint8 [n, hu, wu] (1 = valid)."""
    fn = "removal_holes"
    _check_page(page, fn)
    n, _, h, w = page.shape
    if not isinstance(text_mask, torch.Tensor) or text_mask.dtype != torch.uint8 or tuple(text_mask.shape) != (n, 1, h, w) \
            or text_mask.device != page.device or not text_mask.is_contiguous():
        got = (tuple(text_mask.shape), text_mask.dtype, str(text_mask.device)) if isinstance(text_mask, torch.Tensor) else text_mask
        raise _lib.PcbError(f"{fn}: expected a contiguous uint8 text mask [{n}, 1, {h}, {w}] on {page.device}, got {got}")
    _check_padded(fn, "padded size", hu, wu, h, w)
    code = _compute_code(dtype)
    buf = torch.empty((n, 8, int(hu), int(wu)), dtype=dtype, device=page.device, memory_format=CL)
    valid = torch.empty((n, int(hu), int(wu)), dtype=torch.uint8, device=page.device)
    _lib.check(_lib.load().pcb_removal_holes(text_mask.data_ptr(), page.data_ptr(), n, h, w, int(hu), int(wu), valid.data_ptr(),
                                             buf.data_ptr(), code, _stream()))
    return buf[:, :3], valid


def removal_composite(fill: torch.Tensor, page: torch.Tensor, valid: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The composite ``valid * page + (1 - valid) * fill`` (loss.py:196, comp_img) cropped to the page, as a select: the page
    where valid, the U-Net output elsewhere.  `fill`: the U-Net output [n, 3, hu, wu] (bf16 or fp32, NHWC, possibly
    channel-padded); `valid`: uint8 [n, hu, wu] (removal_holes).  Writes fp32 NCHW [n, 3, h, w] into `out` (a new tensor when
    None) and returns it."""
    fn = "removal_composite"
    _check_page(page, fn)
    n, _, h, w = page.shape
    if not isinstance(valid, torch.Tensor) or valid.dtype != torch.uint8 or valid.dim() != 3 or valid.shape[0] != n \
            or valid.device != page.device or not valid.is_contiguous():
        raise _lib.PcbError(f"{fn}: expected a contiguous uint8 valid plane [{n}, hu, wu] on {page.device}")
    hu, wu = valid.shape[1:]
    _check_padded(fn, "valid plane", hu, wu, h, w)
    if not isinstance(fill, torch.Tensor) or not fill.is_cuda or fill.dim() != 4 or tuple(fill.shape) != (n, 3, hu, wu) \
            or fill.device != page.device:
        raise _lib.PcbError(f"{fn}: expected a CUDA U-Net output [{n}, 3, {hu}, {wu}] on {page.device}")
    if nhwc_layout(fill) is None:
        fill = fill.contiguous(memory_format=CL)
    if out is None:
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=page.device)
    elif out.dtype != torch.float32 or tuple(out.shape) != (n, 3, h, w) or not out.is_contiguous() or out.device != page.device:
        raise _lib.PcbError(f"{fn}: out must be a contiguous fp32 [{n}, 3, {h}, {w}] tensor on {page.device}")
    _lib.check(_lib.load().pcb_removal_composite(fill.data_ptr(), _dtype_code(fill), nhwc_layout(fill), page.data_ptr(), valid.data_ptr(),
                                                 n, h, w, hu, wu, out.data_ptr(), _stream()))
    return out

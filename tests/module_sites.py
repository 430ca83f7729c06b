"""Per-module fp64 check of a live network: record what every module of a fixed type table received and produced inside the
network (forward pre-hooks with kwargs, forward hooks, tensor gradient hooks), then hold each module to an fp64 reference of its
own operation on exactly those operands.  Nothing propagates through the network, so every bound is one module deep and the
bf16 error that builds up through BatchNorm layers (DESIGN 2) never enters a bound.

Recording never allocates on the device during the recorded pass: each tensor is copied to the host synchronously through its
storage (one D2H copy of the bytes, no device temporary) and no device reference is kept.  Two markers of the library are
keyed by an output's address (the BatchNorm statistics of a convolution epilogue, the fused eval epilogue), and the caching
allocator's reuse of addresses is exactly what they must survive: a recorder that cloned tensors on the device or kept them
alive would change the addresses and so change what is tested.

Checks per leaf:
  * convolutions (PartialConv, PartialConvNoHoles, PartialConv1x1, B200Conv2d): y against fp64 on the recorded input and mask
    with the weight rounded to the compute type (the conv-route suite's bound n 2^-22 M / s plus the renormalisation, bias and
    storage roundings), zeros in the channel padding, the new mask bit-exact against the fp64 box sums, the weight and bias
    gradients from the recorded input and the recorded output gradient, and the data gradient delivered to each input part;
  * BatchNorm + activation (PartialActivatedBN, B200BNAct, PartialActivation): y against fp64 batch statistics within the
    BatchNorm suite's coefficient bounds (_coef_ref), running statistics (_check_running), num_batches_tracked + 1, dgamma,
    dbeta, dx and the residual gradient; an element whose pre-activation lies within its bound of a kink may take either
    derivative.  Where the renormalisation handoff fused, the gradient carried into the convolution output must be
    dL/dy / msum, and 0 at holes.
Composites (PartialBlock, DoublePartialResidual, PartialInvertedResidual, the U-Net heads) are checked on their own glue only:
the LazyCat parts and the HoleMask concatenation each decoder layer receives, and the residual each fold hands its BatchNorm.

Input gradients: for every recorded tensor, the gradient autograd delivered must equal the sum over its consumers of each
consumer's fp64 input gradient, within the sum of their bounds plus one storage rounding per autograd add.  This is what
catches a dropped residual gradient or a skip connection that lost its share.
"""
import ctypes
import math
from functools import partial

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.grad import conv2d_input, conv2d_weight

from kernel_harness import act_ref, assert_within
from test_gpu_batchnorm import U, _act_grad, _chain, _check_running, _coef_ref
from test_gpu_conv_routes import accumulation_bound
from text_segmentation_image_inpainting_b200 import _lib, ops
from text_segmentation_image_inpainting_b200.masks import HoleMask
from text_segmentation_image_inpainting_b200.models import BaseModels as MB
from text_segmentation_image_inpainting_b200.models import MobileNetV2 as MM
from text_segmentation_image_inpainting_b200.models import Xception as MX
from text_segmentation_image_inpainting_b200.models import common as MC
from text_segmentation_image_inpainting_b200.models import image_inpainting as MI
from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
from text_segmentation_image_inpainting_b200.models import text_segmentation as MT

CONV_LEAVES = (PC.PartialConv, PC.PartialConvNoHoles, PC.PartialConv1x1, MB.B200Conv2d)
BN_LEAVES = (PC.PartialActivatedBN, MB.B200BNAct, PC.PartialActivation)
OTHER_LEAVES = (MC.B200AvgPool2d, MT.B200Upsample, MC.SpatialChannelSqueezeExcitation, PC.DoubleUpSample)
COMPOSITES = (PC.PartialBlock, MI.DoublePartialResidual, MM.PartialInvertedResidual, MB.DSConvBlock, MM.InvertedResidual,
              MX.ResidualBlock, MC.RFB, MC.ASP, MI.ImageFillOrigin, MI.ImageFillOriginV2, MI.ImageFill, MT.TextSegament,
              MT.XceptionTextSegment)
TABLE = CONV_LEAVES + BN_LEAVES + OTHER_LEAVES + COMPOSITES
# modules whose forward only chains its children (nothing of their own to check)
CONTAINERS = (nn.Sequential, MM.MobileNetV2, MM.DilatedMobileNetV2, MX.Xception)
# modules owned by a table leaf and never called on their own: their parameters are the leaf's
LEAF_PARTS = (nn.BatchNorm2d, nn.ReLU, nn.ReLU6, nn.LeakyReLU, nn.Conv2d, nn.Upsample, nn.Linear, nn.Sigmoid, nn.AdaptiveAvgPool2d)
# table modules a network builds but its forward never calls (kept for the reference's state_dict keys)
NOT_CALLED = {"double_upscale"}

# glue branches of ops.py / models/ that the union of the runs must reach (see test_gpu_module_sites.BRANCHES_REACHED)
BRANCHES = {
    "handoff_fused": "PartialConvFn.backward skips its renormalisation: the BatchNorm backward wrote dc = dy / msum",
    "handoff_not_fused": "a PartialBlock handoff that was not eligible: PartialConvFn.backward renormalises itself",
    "bn_sums_from_conv_epilogue": "BatchNorm statistics accumulated in the convolution epilogue (handoff.bn_sums / _pending_stats)",
    "bn_stats_pass": "BatchNorm statistics from their own accumulate pass (pcb_bn_stats_acc)",
    "bn_nonvector": "BatchNorm on the non-vector path (c % 8 != 0 or c > 2048: pcb_bn_stats + pcb_bn_finalize)",
    "bn_bwd_small": "BatchNorm backward in one launch (pcb_bn_act_backward_small)",
    "bn_bwd_reduce_acc": "BatchNorm backward reduction into the step arena (pcb_bn_act_backward_reduce_acc)",
    "bn_bwd_reduce": "BatchNorm backward reduction on the non-vector path (pcb_bn_act_backward_reduce)",
    "bn_bwd_apply_renorm": "BatchNorm backward apply with the renormalisation (pcb_bn_act_backward_apply_renorm)",
    "bn_bwd_apply": "BatchNorm backward apply with batch statistics (pcb_bn_act_backward_apply)",
    "bn_bwd_eval": "BatchNorm backward in eval mode (apply with running-statistics coefficients)",
    "act_only_bwd": "activation-only backward (PartialActivation)",
    "residual_grad": "the residual gradient a BatchNorm pass returns as gy",
    "conv_plain_passthrough": "plain bias-free convolution backward: dc = gy, no renormalisation pass",
    "conv_renorm_backward": "pcb_pconv_renorm_backward (renormalisation and bias gradient)",
    "bias_grad_sink": "bias gradient written into a gradient sink",
    "weight_grad_sink_side_stream": "weight gradient written into a sink from the side stream, joined at the training scope's exit",
    "weight_grad_autograd": "weight gradient returned to autograd",
    "weight_used_twice": "a weight used twice in one pass: the second use falls back from the sink to autograd accumulation",
    "rowpacked_dgrad_generic": "row-packed layer whose input needs a gradient: generic data gradient with a per-backward weight cast",
    "upsampled_at_source": "data gradient of a 2x-upsampled part computed at source resolution",
    "upsampled_full_then_backward": "data gradient of a 2x-upsampled part at full resolution, then pcb_upsample2x_backward",
    "residual_folded_into_bn": "residual folded into the BatchNorm pass (DoublePartialResidual, PartialInvertedResidual)",
    "lazycat_input": "a decoder layer reading LazyCat parts",
    "holemask_cat": "a convolution reading a concatenation of HoleMasks",
    "dense_mask_fallback": "more (source, plane) parts than PCB_MAX_PARTS: the dense-mask formulation",
    "eval_epilogue_fused": "eval-mode BatchNorm + activation applied in the convolution epilogue (PartialBlock._eval_epilogue, "
                           "B200Conv2d's _pcb_fused_out marker)",
    "eval_epilogue_refused": "an eval epilogue offered to a convolution whose kernel refused it: the two-pass path",
    "bn_passthrough": "a B200BNAct passing through an output its convolution's epilogue already normalised",
}

CL = torch.channels_last


# ------------------------------------------------------------------------------------------------ recording
def host(t: torch.Tensor) -> torch.Tensor:
    """host copy of a device tensor with the same shape and strides, read through its storage: one synchronous D2H copy, no
    device allocation"""
    st = t.untyped_storage()
    buf = torch.empty(st.nbytes(), dtype=torch.uint8)
    buf.untyped_storage().copy_(st)
    return torch.empty(0, dtype=t.dtype).set_(buf.untyped_storage(), t.storage_offset(), t.shape, t.stride())


class Rec:
    """a recorded tensor: its tag (shared by every consumer of the same tensor), host copy and channel padding"""

    def __init__(self, tag, value, pad):
        self.tag, self.value, self.pad = tag, value, pad


class MaskRec:
    def __init__(self, parts, shape):
        self.parts, self.shape = parts, tuple(shape)     # [(host plane, channels, up)]


class LazyRec:
    def __init__(self, parts, ups, shape):
        self.parts, self.ups, self.shape = parts, list(ups), tuple(shape)


class Unit:
    def __init__(self, idx, name, module, parent):
        self.idx, self.name, self.module, self.parent = idx, name, module, parent
        self.children, self.inp, self.kw, self.out, self.facts = [], None, {}, None, {}
        self.live = {}


def _bn_of(m):
    if isinstance(m, PC.PartialActivatedBN):
        return m.bn_act[0], (m.bn_act[1] if len(m.bn_act) > 1 else None)
    if isinstance(m, MB.B200BNAct):
        return m[0], (m[1] if len(m) > 1 else None)
    return None, m.act_fn


class Recorder:
    """attach(net) hooks every module of TABLE; run the pass; detach(); then Checker(recorder) checks it"""

    COUNTED = ("pcb_bn_stats", "pcb_bn_stats_acc", "pcb_bn_forward_fused", "pcb_bn_finalize", "pcb_bn_act_forward",
               "pcb_bn_act_backward_small", "pcb_bn_act_backward_reduce_acc", "pcb_bn_act_backward_reduce",
               "pcb_bn_act_backward_apply_renorm", "pcb_bn_act_backward_apply", "pcb_pconv_renorm_backward",
               "pcb_pconv_backward_weight", "pcb_pconv_backward_weight_acc", "pcb_pconv_backward_data", "pcb_upsample2x_backward",
               "pcb_pconv_forward_bn", "pcb_pconv_forward_affine_act")
    WGRAD = ("pcb_pconv_backward_weight", "pcb_pconv_backward_weight_acc")

    def __init__(self):
        self.units, self.stack, self.values, self.grads, self.handles = [], [], {}, {}, []
        self.rg = {}
        self.attr = f"_ms_tag_{id(self)}"
        self.calls, self.features = {}, set()
        self.plain_renorm, self.with_sinks = 0, False
        self.names = {}

    # ---- library entry points: counting recorders
    def _wrap(self):
        lib = _lib.load()
        self._orig = {fn: getattr(lib, fn) for fn in self.COUNTED}

        def rec(fn, f):
            def call(*args):
                self.calls[fn] = self.calls.get(fn, 0) + 1
                self._feature(fn, args)
                return f(*args)
            return call
        for fn, f in self._orig.items():
            setattr(lib, fn, rec(fn, f))

    def _feature(self, fn, args):
        if fn in self.WGRAD:
            scope = ops.current_scope()
            side = scope is not None and torch.cuda.current_stream() in scope.streams
            if fn == "pcb_pconv_backward_weight_acc" and side:
                self.features.add("weight_grad_sink_side_stream")
            if fn == "pcb_pconv_backward_weight":
                self.features.add("weight_grad_autograd")
        elif fn == "pcb_pconv_renorm_backward":
            self.plain_renorm += int(args[0]._obj.plain)
        elif fn == "pcb_bn_act_backward_apply":
            if args[5] is None:
                self.features.add("act_only_bwd")
            elif args[7] is None:
                self.features.add("bn_bwd_eval")
            else:
                self.features.add("bn_bwd_apply")
        elif fn == "pcb_pconv_backward_data":
            c = args[0]._obj
            if c.force_generic:
                self.features.add("rowpacked_dgrad_generic")
            if any(c.parts[i].x_up for i in range(c.nparts)) and _lib.load().pcb_conv_dgrad_at_source_resolution(args[0]):
                self.features.add("upsampled_at_source")
        elif fn in ("pcb_pconv_forward_bn", "pcb_pconv_forward_affine_act") and self.stack:
            c = args[0]._obj
            r = (ctypes.c_int32 * 3)()
            _lib.check(_lib.load().pcb_debug_conv_routes(args[0], r))
            self.stack[-1].facts["routes"] = tuple(_lib.ROUTES[v] for v in r)
            self.stack[-1].facts["at_src"] = bool(any(c.parts[i].x_up for i in range(c.nparts))
                                                  and _lib.load().pcb_conv_dgrad_at_source_resolution(args[0]))

    def _unwrap(self):
        lib = _lib.load()
        for fn, f in self._orig.items():
            setattr(lib, fn, f)

    # ---- tensors
    def tensor(self, t):
        tag = t.__dict__.get(self.attr)
        if tag is None:
            tag = len(self.values)
            t.__dict__[self.attr] = tag
            pad = None
            cs = ops.nhwc_layout(t) if t.dim() == 4 else None
            if cs is not None and cs > t.shape[1] and t.is_contiguous(memory_format=CL) is False:
                n, c, h, w = t.shape
                full = t.as_strided((n, cs, h, w), t.stride()[:1] + (1,) + t.stride()[2:])
                pad = host(full)[:, c:]
            self.values[tag] = (host(t), pad)
            self.rg[tag] = t.requires_grad
            if t.requires_grad:
                t.register_hook(partial(self._on_grad, tag))
        v, pad = self.values[tag]
        return Rec(tag, v, pad)

    def _on_grad(self, tag, g):
        self.grads[tag] = host(g)

    def flat(self, obj):
        if isinstance(obj, ops.LazyCat):
            return LazyRec([self.tensor(x) for x in obj.xs], obj.ups, obj.shape)
        if isinstance(obj, HoleMask):
            return MaskRec([(host(p), c, up) for p, c, up in obj.parts], obj.shape)
        if isinstance(obj, torch.Tensor):
            return self.tensor(obj)
        if isinstance(obj, (tuple, list)):
            return [self.flat(o) for o in obj]
        return None

    # ---- hooks
    def _pre(self, mod, args, kwargs):
        u = Unit(len(self.units), self.names.get(mod, type(mod).__name__), mod, self.stack[-1] if self.stack else None)
        if u.parent is not None:
            u.parent.children.append(u)
        self.units.append(u)
        self.stack.append(u)
        u.inp = self.flat(list(args))
        if kwargs.get("residual") is not None:
            u.kw["residual"] = self.flat(kwargs["residual"])
        for k in ("handoff", "epilogue"):
            if kwargs.get(k) is not None:
                u.live[k] = kwargs[k]
        if isinstance(mod, BN_LEAVES):
            bn, _ = _bn_of(mod)
            if bn is not None:
                u.facts["bn0"] = (host(bn.running_mean), host(bn.running_var), int(bn.num_batches_tracked))
                u.facts["training"] = bn.training
            x = args[0][0] if isinstance(args[0], (tuple, list)) else args[0]
            if isinstance(mod, MB.B200BNAct):
                pend, fused = mod.__dict__.get("_pending_stats"), mod.__dict__.get("_pcb_fused_out")
                key = (x.data_ptr(), tuple(x.shape))
                u.facts["pre_sums"] = pend is not None and bn.training and (pend[0], pend[1]) == key
                u.facts["passthrough"] = fused == key
            elif "handoff" in u.live:
                u.facts["pre_sums"] = u.live["handoff"].bn_sums is not None and bn.training
        return None

    def _post(self, mod, args, kwargs, out):
        u = self.stack.pop()
        u.out = self.flat(out)
        if isinstance(mod, BN_LEAVES):
            bn, _ = _bn_of(mod)
            if bn is not None:
                u.facts["bn1"] = (host(bn.running_mean), host(bn.running_var), int(bn.num_batches_tracked))
        h = u.live.get("handoff")
        if h is not None and isinstance(mod, CONV_LEAVES):
            u.facts["msum"] = host(h.msum)
        e = u.live.get("epilogue")
        if e is not None:
            u.facts["epi_offered"], u.facts["epi_fused"] = True, e.fused
            if e.fused:
                u.facts["epi"] = (e.bn, e.act, self._coef(e.bn))
        if isinstance(mod, MB.B200Conv2d):
            hint = mod.__dict__.get("_bn_hint")
            y = out
            if hint is not None:
                pend = hint.__dict__.get("_pending_stats")
                u.facts["bn_sums"] = pend is not None and pend[0] == y.data_ptr()
                scope = ops.current_scope()
                if scope is not None and not scope.training and not hint[0].training and not hint.__dict__.get("_pcb_residual_site"):
                    fused = hint.__dict__.get("_pcb_fused_out") == (y.data_ptr(), tuple(y.shape))
                    u.facts["epi_offered"], u.facts["epi_fused"] = True, fused
                    if fused:
                        u.facts["epi"] = (hint[0], hint[1] if len(hint) > 1 else None, self._coef(hint[0]))
        return None

    @staticmethod
    def _coef(bn):
        """host copy of the (scale, shift) the eval epilogue applied (ops.bn_eval_coefficients' cache)"""
        return None if bn is None else host(bn.__dict__["_pcb_bn_coef"]["buf"])

    def attach(self, net):
        self.names = {m: (n or type(net).__name__) for n, m in net.named_modules()}
        for m in net.modules():
            if type(m) in TABLE:
                self.handles.append(m.register_forward_pre_hook(self._pre, with_kwargs=True))
                self.handles.append(m.register_forward_hook(self._post, with_kwargs=True))
        self._wrap()
        return self

    def detach(self):
        for h in self.handles:
            h.remove()
        self.handles = []
        self._unwrap()

    def finish(self, sinks=()):
        """after backward (and the scope's exit): read each handoff and drop every live reference"""
        for u in self.units:
            h = u.live.get("handoff")
            if h is not None:
                u.facts.update(eligible=h.eligible, fused=h.fused, has_bn_sums=h.bn_sums is not None)
            u.live = {}
        self.sinks_used = [s.used for s in sinks]

    def reached(self):
        """the BRANCHES this pass reached"""
        r = set(self.features)
        c = self.calls
        for fn, br in (("pcb_bn_stats_acc", "bn_stats_pass"), ("pcb_bn_stats", "bn_nonvector"), ("pcb_bn_act_backward_small", "bn_bwd_small"),
                       ("pcb_bn_act_backward_reduce_acc", "bn_bwd_reduce_acc"), ("pcb_bn_act_backward_reduce", "bn_bwd_reduce"),
                       ("pcb_bn_act_backward_apply_renorm", "bn_bwd_apply_renorm"), ("pcb_pconv_renorm_backward", "conv_renorm_backward"),
                       ("pcb_upsample2x_backward", "upsampled_full_then_backward")):
            if c.get(fn):
                r.add(br)
        plain_grads = sum(1 for u in self.units if isinstance(u.module, (MB.B200Conv2d, PC.PartialConv1x1))
                          and u.out is not None and (u.out[0] if isinstance(u.out, list) else u.out).tag in self.grads)
        if self.plain_renorm < plain_grads:       # some plain convolution's backward ran no renormalisation pass
            r.add("conv_plain_passthrough")
        if self.with_sinks and c.get("pcb_pconv_backward_weight"):      # a sink was already used: autograd accumulation
            r.add("weight_used_twice")
        for u in self.units:
            f = u.facts
            if f.get("epi_offered"):
                r.add("eval_epilogue_fused" if f.get("epi_fused") else "eval_epilogue_refused")
            if f.get("passthrough"):
                r.add("bn_passthrough")
            if f.get("fused"):
                r.add("handoff_fused")
            if "eligible" in f and not f.get("fused") and isinstance(u.module, PC.PartialConv):
                r.add("handoff_not_fused")
            if f.get("pre_sums"):
                r.add("bn_sums_from_conv_epilogue")
            if "residual" in u.kw:
                r.add("residual_folded_into_bn")
                if any(self._res_tag(u) == t for t in self.grads):
                    r.add("residual_grad")
            if u.inp and isinstance(u.inp[0], list) and u.inp[0] and isinstance(u.inp[0][0], LazyRec) and isinstance(u.module, CONV_LEAVES):
                r.add("lazycat_input")
            if isinstance(u.module, CONV_LEAVES) and u.inp and isinstance(u.inp[0], list) and len(u.inp[0]) > 1 \
                    and isinstance(u.inp[0][1], MaskRec):
                if len(u.inp[0][1].parts) > 1:
                    r.add("holemask_cat")
                if f.get("dense_fallback"):
                    r.add("dense_mask_fallback")
        return r

    @staticmethod
    def _res_tag(u):
        return u.kw["residual"].tag


# ------------------------------------------------------------------------------------------------ fp64 helpers
def _dev(t, dev):
    # NCHW-contiguous: torch's CUDA fp64 avg_pool2d backward on channels_last tensors does not compute the pooling gradient
    # (torch 2.11; its CPU and NCHW CUDA paths agree with each other and with pcb_avgpool_backward), so no reference here
    # runs on the recorded channels_last layout
    return t.to(dev).double().contiguous()


def _dense_mask(mr: MaskRec, dev):
    n, c, h, w = mr.shape
    planes = []
    for p, cc, up in mr.parts:
        q = _dev(p, dev)
        for _ in range(up):
            q = q.repeat_interleave(2, 1).repeat_interleave(2, 2)
        planes.append(q[:, None].expand(n, cc, h, w))
    return torch.cat(planes, 1)


def _up(t, k):
    for _ in range(k):
        t = t.repeat_interleave(2, -2).repeat_interleave(2, -1)
    return t


def _act(z, act):
    code, slope = ops.act_code(act)
    return act_ref(z, code, slope, f32_slope=True)


def _dact(z, act):
    code, slope = ops.act_code(act)
    return _act_grad(z, code, slope)


class Checker:
    """fp64 references of every recorded unit; asserts as it goes, accumulates input- and parameter-gradient contributions"""

    def __init__(self, rec: Recorder, dev, dtype, label):
        self.rec, self.dev, self.dtype, self.label = rec, dev, dtype, label
        self.store = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -24
        self.contrib = {}          # tag -> [sum ref, sum bound, sum |ref|, consumers]
        self.who = {}              # tag -> names of the consumers
        self.current = ""
        self.pref = {}             # id(param) -> [param, sum ref, sum bound]
        self.checked = []

    def _add(self, tag, ref, bd):
        self.who.setdefault(tag, []).append(self.current)
        a = self.contrib.get(tag)
        if a is None:
            self.contrib[tag] = [ref.clone(), bd.clone(), ref.abs(), 1]
        else:
            a[0] += ref; a[1] += bd; a[2] += ref.abs(); a[3] += 1

    def _padd(self, p, ref, bd):
        a = self.pref.get(id(p))
        if a is None:
            self.pref[id(p)] = [p, ref.clone(), bd.clone()]
        else:
            a[1] += ref; a[2] += bd

    def _x(self, r):
        return _dev(r.value, self.dev)

    def _grad(self, r):
        g = self.rec.grads.get(r.tag)
        return None if g is None else _dev(g, self.dev)

    def run(self):
        for u in self.rec.units:
            m = u.module
            name = f"{self.label}: {u.name} ({type(m).__name__})"
            self.current = u.name
            if isinstance(m, CONV_LEAVES):
                self.conv(u, name)
            elif isinstance(m, BN_LEAVES):
                self.bn(u, name)
            elif isinstance(m, PC.DoubleUpSample):
                self.double_upsample(u, name)
            elif isinstance(m, MC.B200AvgPool2d):
                self.pool(u, name)
            elif isinstance(m, MT.B200Upsample):
                self.bilinear_leaf(u, name)
            elif isinstance(m, MC.SpatialChannelSqueezeExcitation):
                self.scse(u, name)
            else:
                self.composite(u, name)
            self.checked.append(u)
        self.params()
        self.inputs()

    # ---------------------------------------------------------------- convolutions
    def conv(self, u, name):
        m, dev = u.module, self.dev
        if isinstance(m, MB.B200Conv2d):
            fc, kind = m, "plain"
            xr, mr = u.inp[0], None
        else:
            fc = m.feature_conv
            kind = "1x1" if isinstance(m, PC.PartialConv1x1) else ("nh" if isinstance(m, PC.PartialConvNoHoles) else "pc")
            xr, mr = u.inp[0][0], u.inp[0][1]
        parts = xr.parts if isinstance(xr, LazyRec) else [xr]
        ups = xr.ups if isinstance(xr, LazyRec) else [0]
        xs = [_up(self._x(p), k) for p, k in zip(parts, ups)]
        x = torch.cat(xs, 1)
        n, cin, h, w = x.shape
        cdt = parts[0].value.dtype
        W = fc.weight.detach().to(cdt).double()
        b = fc.bias.detach().double() if fc.bias is not None else None
        cout, cig, kh, kw = W.shape
        g, st, pd, dl = fc.groups, fc.stride[0], fc.padding, fc.dilation[0]
        geo = dict(stride=st, padding=pd, dilation=dl, groups=g)
        if mr is not None and not isinstance(mr, MaskRec):
            mr = MaskRec([(mr.value[:, 0].to(torch.uint8), cin, 0)], mr.value.shape)        # a dense mask tensor
        M = _dense_mask(mr, dev) if (mr is not None and kind != "1x1") else None
        if M is not None and M.shape[1] == 1 and cin > 1:
            M = M.expand(n, cin, h, w)
        if mr is not None and kind in ("pc", "nh") and len(mr.parts) > _lib.MAX_PARTS:
            u.facts["dense_fallback"] = True
        XM = x * M if (M is not None and kind in ("pc", "nh")) else x
        with torch.backends.cudnn.flags(enabled=False):
            acc = F.conv2d(XM, W, **geo)
            mag = F.conv2d(XM.abs(), W.abs(), **geo)
            if kind == "pc" and m.same_holes:
                s = F.conv2d(M[:, :1], torch.ones(1, 1, kh, kw, dtype=torch.float64, device=dev), stride=st, padding=pd, dilation=dl)
                s = (s * cin).expand_as(acc)
            elif kind in ("pc", "nh"):
                s = F.conv2d(M, torch.ones_like(W), **geo)
            else:
                s = torch.ones_like(acc)
        holes = s == 0
        safe = torch.where(holes, torch.ones_like(s), s)
        routes = u.facts.get("routes", ("generic",) * 3)
        nz = cig * kh * kw
        bb = b[None, :, None, None] if b is not None else 0.0
        v = acc / safe + bb
        e = accumulation_bound(nz, mag, routes[0] == "k2r") / safe + 2.0 ** -22 * (acc.abs() / safe + v.abs())
        if u.facts.get("dense_fallback"):          # the plain convolution's output is stored before the division
            e = e + self.store * (acc.abs() + e) / safe
        guard = kind != "nh"
        v = torch.where(holes, torch.zeros_like(v), v) if guard else v
        e = torch.where(holes, torch.zeros_like(e), e) if guard else e
        yr = u.out[0] if isinstance(u.out, list) else u.out
        y = self._x(yr)
        live = ~holes if not guard else torch.ones_like(holes)
        if not guard:
            assert bool(y[holes].isnan().all()), f"{name}: NaN expected where every tap is a hole (no zero guard)"
        epi = u.facts.get("epi")
        if epi is not None:
            # eval-mode BatchNorm + activation applied in the epilogue: one unit.  The coefficients the kernel applied must be
            # the eval coefficients within the BatchNorm suite's finalize bounds; y = act(v scale + shift) within the
            # conv-route suite's epilogue bound; hole pixels exactly bf16(act(shift))
            bn, act, coef = epi
            if bn is not None:
                sc_k, sh_k = _dev(coef[0], dev), _dev(coef[1], dev)
                inv = 1 / torch.sqrt(bn.running_var.double() + float(torch.tensor(bn.eps, dtype=torch.float32)))
                gam, bet = bn.weight.detach().double(), bn.bias.detach().double()
                sc, sh = gam * inv, bet - bn.running_mean.double() * gam * inv
                assert_within(f"{name}: eval epilogue scale", sc_k, sc, 4 * U * sc.abs())
                assert_within(f"{name}: eval epilogue shift", sh_k, sh, 6 * U * (bn.running_mean.double() * sc).abs() + 2 * U * bet.abs())
            else:
                sc_k, sh_k = torch.ones(cout, dtype=torch.float64, device=dev), torch.zeros(cout, dtype=torch.float64, device=dev)
            P = lambda t: t[None, :, None, None]  # noqa: E731
            z = v * P(sc_k) + P(sh_k)
            va = _act(z, act)
            ev = P(sc_k.abs()) * e + 2.0 ** -23 * (z.abs() + P(sh_k.abs())) + 2.0 ** -23 * va.abs()
            if guard:
                hv = _act(P(sh_k.float()).expand_as(z).contiguous(), act).to(cdt).double()
                assert torch.equal(torch.where(holes, y, hv), hv), f"{name}: hole pixels must be exactly bf16(act(shift))"
                va, ev = torch.where(holes, hv, va), torch.where(holes, torch.zeros_like(ev), ev)
            assert_within(f"{name}: forward act(BN(y)) in the eval epilogue", torch.where(live, y, va), va, ev + self.store * (va.abs() + ev))
        else:
            assert_within(f"{name}: forward y", torch.where(live, y, v), v, e + self.store * (v.abs() + e))
        if yr.pad is not None:
            assert bool((yr.pad == 0).all()), f"{name}: channel padding of y must hold zeros"
        # the new mask, bit-exact
        if kind != "plain":
            om = _dense_mask(u.out[1], dev)
            if kind == "1x1":
                ref = M0 = _dense_mask(mr, dev)[:, :1].expand_as(om)
            elif kind == "nh":
                ref = torch.ones_like(om)
            else:
                ref = (~holes).double()
            assert torch.equal(om, ref), f"{name}: new mask differs from the fp64 box sums in {int((om != ref).sum())} elements"
        G = self._grad(yr)
        if G is None:
            return
        fused = bool(u.facts.get("fused"))
        plain = kind in ("plain", "1x1")
        if fused or plain:
            dc, dc_round = G, 0.0
        else:
            dc = torch.where(holes, torch.zeros_like(G), G / safe)
            dc_round = self.store if cdt == torch.bfloat16 else 2.0 ** -23
        if not guard:
            dc = torch.where(holes, torch.zeros_like(dc), dc)
        if fc.weight.requires_grad:
            with torch.backends.cudnn.flags(enabled=False):
                dw = conv2d_weight(XM, W.shape, dc, **geo)
                wmag = conv2d_weight(XM.abs(), W.shape, dc.abs(), **geo)
            ew = accumulation_bound(n * s.shape[2] * s.shape[3], wmag, routes[2] == "k2r") + dc_round * wmag
            self._padd(fc.weight, dw, ew)
        if fc.bias is not None and fc.bias.requires_grad:
            gl = torch.where(holes, torch.zeros_like(G), G) if guard else G
            cnt = n * gl.shape[2] * gl.shape[3]
            self._padd(fc.bias, gl.sum((0, 2, 3)), cnt * 2.0 ** -23 * gl.abs().sum((0, 2, 3)) + U * gl.sum((0, 2, 3)).abs())
        if not any(self.rec.rg[p.tag] for p in parts):
            return
        with torch.backends.cudnn.flags(enabled=False):
            dx = conv2d_input(x.shape, W, dc, **geo)
            gmag = conv2d_input(x.shape, W.abs(), dc.abs(), **geo)
        if M is not None and kind in ("pc", "nh"):
            dx, gmag = dx * M, gmag * M
        rounds_d = routes[1] == "k2r" or (routes[1] != "none" and u.facts.get("at_src"))
        ed = accumulation_bound(cout // g * kh * kw, gmag, rounds_d) + dc_round * gmag
        off = 0
        for p, k in zip(parts, ups):
            c = p.value.shape[1]
            gp, ep = dx[:, off:off + c], ed[:, off:off + c]
            if k:
                gp, ep = F.avg_pool2d(gp, 2) * 4, F.avg_pool2d(ep + self.store * gp.abs(), 2) * 4
            off += c
            if self.rec.rg[p.tag]:
                self._add(p.tag, gp, ep)

    # ---------------------------------------------------------------- BatchNorm + activation
    def bn(self, u, name):
        m, dev = u.module, self.dev
        bn, act = _bn_of(m)
        xr = u.inp[0][0] if isinstance(u.inp[0], list) else u.inp[0]
        yr = u.out[0] if isinstance(u.out, list) else u.out
        x, y = self._x(xr), self._x(yr)
        if u.facts.get("passthrough"):
            assert torch.equal(x, y), f"{name}: a BatchNorm applied in the convolution epilogue must pass its input through"
            return
        rr = u.kw.get("residual")
        res = self._x(rr) if rr is not None else None
        n, c, h, w = x.shape
        count = n * h * w
        training = bn is not None and bn.training
        if bn is not None:
            gam, bet = bn.weight.detach().double(), bn.bias.detach().double()
        if training:
            L = 2 * count if u.facts.get("pre_sums") else (_chain(count, c, 16) if (c % 8 == 0 and c <= 2048) else math.ceil(count / 256) + 13)
            ax = x.abs()
            S, Q = x.sum((0, 2, 3)), (x * x).sum((0, 2, 3))
            R = _coef_ref(S, Q, (L + 1) * U * ax.sum((0, 2, 3)), (L + 2) * U * (ax * ax).sum((0, 2, 3)), count, gam, bet)
            sc, sh, d_sc, d_sh = R["sc"], R["sh"], R["d_sc"], R["d_sh"]
            mu, inv, dm, d_inv = R["m"], R["inv"], R["dm"], R["d_inv"]
            rm0, rv0, nb0 = u.facts["bn0"]
            rm1, rv1, nb1 = u.facts["bn1"]
            _check_running(name, R, _dev(rm0, dev).float(), _dev(rv0, dev).float(), _dev(rm1, dev), _dev(rv1, dev), count)
            assert nb1 == nb0 + 1, f"{name}: num_batches_tracked must grow by exactly 1, got {nb1 - nb0}"
        elif bn is not None:
            rm, rv = bn.running_mean.double(), bn.running_var.double()
            inv = 1 / torch.sqrt(rv + float(torch.tensor(bn.eps, dtype=torch.float32)))
            sc, sh = gam * inv, bet - rm * gam * inv
            d_sc, d_sh = 4 * U * sc.abs(), 6 * U * (rm * sc).abs() + 2 * U * bet.abs()
            if "bn0" in u.facts:
                assert torch.equal(u.facts["bn0"][0], u.facts["bn1"][0]) and u.facts["bn0"][2] == u.facts["bn1"][2], \
                    f"{name}: eval mode must not touch the running statistics"
        if bn is not None:
            P = lambda t: t[None, :, None, None]  # noqa: E731
            z = x * P(sc) + P(sh)
            dz = x.abs() * P(d_sc) + P(d_sh) + 2 * U * ((x * P(sc)).abs() + P(sh).abs())
        else:
            z, dz = x, torch.zeros_like(x)
        a = _act(z, act)
        v = a + (res if res is not None else 0)
        ev = dz + U * a.abs() + U * v.abs()
        assert_within(f"{name}: forward y", y, v, ev + self.store * (v.abs() + ev))
        G = self._grad(yr)
        if G is None:
            return
        if rr is not None:
            self._add(rr.tag, G, torch.zeros_like(G))
        gz = G * _dact(z, act)
        kink = (_dact(z - dz, act) - _dact(z + dz, act)).abs()
        if training:
            P = lambda t: t[None, :, None, None]  # noqa: E731
            xm = x - P(mu)
            SG, SGX = gz.sum((0, 2, 3)), (gz * xm * P(inv)).sum((0, 2, 3))
            Lb = count + 40
            dSG = (Lb + 1) * U * gz.abs().sum((0, 2, 3)) + (G.abs() * kink).sum((0, 2, 3))
            dSGX = (Lb + 4) * U * (gz * xm * P(inv)).abs().sum((0, 2, 3)) + (G.abs() * kink * xm.abs() * P(inv)).sum((0, 2, 3)) \
                + (gz.abs() * (xm.abs() * P(d_inv) + P(inv * dm))).sum((0, 2, 3))
            B, C = -sc * inv * SGX / count, -sc * SG / count
            dx = P(sc) * gz + P(B) * xm + P(C)
            bd = (P(d_sc) * gz.abs() + P(sc.abs()) * G.abs() * kink
                  + xm.abs() * (P((sc * inv / count).abs()) * P(dSGX) + P((SGX / count).abs()) * (P(d_sc * inv) + P(sc.abs() * d_inv)))
                  + P(B.abs() * dm) + P(sc.abs() / count * dSG + (SG / count).abs() * d_sc)
                  + 6 * U * ((P(sc) * gz).abs() + (P(B) * xm).abs() + P(C.abs())))
            if bn.weight.requires_grad:
                self._padd(bn.weight, SGX, dSGX + U * SGX.abs())
                self._padd(bn.bias, SG, dSG + U * SG.abs())
        elif bn is not None:
            P = lambda t: t[None, :, None, None]  # noqa: E731
            dx = P(sc) * gz
            bd = P(d_sc) * gz.abs() + P(sc.abs()) * G.abs() * kink + U * dx.abs()
        else:
            dx, bd = gz, G.abs() * kink
        conv = self._producer(xr)
        if conv is not None and conv.facts.get("fused"):
            # the renormalisation handoff: the gradient carried into the convolution output is dL/dy / msum, 0 at holes
            s = _dev(conv.facts["msum"], dev)[0][:, None]
            rs = torch.where(s == 0, torch.zeros_like(s), 1 / torch.where(s == 0, torch.ones_like(s), s))
            dx, bd = dx * rs, (bd + 2 * U * dx.abs()) * rs
        self._add(xr.tag, dx, bd)

    def _producer(self, r):
        for u in self.rec.units:
            if isinstance(u.module, CONV_LEAVES) and u.out is not None:
                o = u.out[0] if isinstance(u.out, list) else u.out
                if isinstance(o, Rec) and o.tag == r.tag:
                    return u
        return None

    # ---------------------------------------------------------------- glue
    def double_upsample(self, u, name):
        xr, mr = u.inp[0]
        o = u.out[0]
        assert isinstance(o, LazyRec) and o.parts[0].tag == xr.tag and o.ups == [1], f"{name}: features must become a lazy 2x view"

    def _linear_op(self, u, name, f, terms):
        """a leaf computing a linear map f with nonnegative weights (average pooling, bilinear resampling): y within terms
        2^-22 f(|x|), and the input gradient f^T(G) within terms 2^-22 f^T(|G|) (fp32 sums of at most `terms` products)"""
        xr, yr = u.inp[0], u.out
        x = self._x(xr).requires_grad_(True)
        v = f(x)
        y = self._x(yr)
        with torch.no_grad():
            e = terms * 2.0 ** -22 * f(x.detach().abs())
        assert_within(f"{name}: forward y", y, v.detach(), e + self.store * (v.detach().abs() + e))
        G = self._grad(yr)
        if G is not None and self.rec.rg[xr.tag]:
            (dx,) = torch.autograd.grad(v, x, G)
            xa = x.detach().requires_grad_(True)
            (mag,) = torch.autograd.grad(f(xa), xa, G.abs())
            self._add(xr.tag, dx, terms * 2.0 ** -22 * mag)

    def pool(self, u, name):
        m = u.module
        k, st, p = (v if isinstance(v, int) else v[0] for v in (m.kernel_size, m.stride, m.padding))
        self._linear_op(u, name, lambda t: F.avg_pool2d(t, k, st, p, count_include_pad=True), k * k + 1)

    def bilinear_leaf(self, u, name):
        sf = int(u.module.scale_factor)
        self._linear_op(u, name, lambda t: F.interpolate(t, scale_factor=sf, mode="bilinear", align_corners=False), 4 * sf * sf)

    def scse(self, u, name):
        """y = x (cse[n, c] + s[n, p]), cse = sigmoid(L2(act(L1(mean_p x)))), s = sigmoid(sum_c x ws): every quantity in fp64
        with its error bound carried alongside (fp32 sums of L terms: L 2^-22 times the sum of their magnitudes; sigmoid is
        1/4-Lipschitz, the activation 1-Lipschitz)"""
        m, dev = u.module, self.dev
        xr, yr = u.inp[0], u.out
        x, y = self._x(xr), self._x(yr)
        n, c, h, w = x.shape
        hw = h * w
        l1, act, l2 = m.channel_excite[0], m.channel_excite[1], m.channel_excite[2]
        W1, b1, W2, b2 = (t.detach().double() for t in (l1.weight, l1.bias, l2.weight, l2.bias))
        ws = m.spatial_excite[0].weight.detach().double().reshape(-1)
        mid = W1.shape[0]
        E = 2.0 ** -22
        sq = x.mean((2, 3))
        d_sq = (hw + 1) * E * x.abs().mean((2, 3))
        h1 = sq @ W1.T + b1
        d_h1 = (c + 1) * E * (sq.abs() @ W1.abs().T + b1.abs()) + d_sq @ W1.abs().T
        a1 = _act(h1, act)
        d_a1 = d_h1 + U * a1.abs()
        h2 = a1 @ W2.T + b2
        d_h2 = (mid + 1) * E * (a1.abs() @ W2.abs().T + b2.abs()) + d_a1 @ W2.abs().T
        cse = torch.sigmoid(h2)
        d_cse = d_h2 / 4 + 4 * U
        t = (x * ws[None, :, None, None]).sum(1)
        s_ = torch.sigmoid(t)
        d_s = c * E * (x * ws[None, :, None, None]).abs().sum(1) / 4 + 4 * U
        C4, S4 = cse[:, :, None, None], s_[:, None]
        v = x * (C4 + S4)
        ev = x.abs() * (d_cse[:, :, None, None] + d_s[:, None]) + 2 * U * v.abs()
        assert_within(f"{name}: forward y", y, v, ev + self.store * (v.abs() + ev))
        G = self._grad(yr)
        if G is None:
            return
        gx = G * x
        gcse, d_gcse = gx.sum((2, 3)), hw * E * gx.abs().sum((2, 3))
        gs, d_gs = gx.sum(1), c * E * gx.abs().sum(1)
        gt = gs * s_ * (1 - s_)
        d_gt = d_gs / 4 + gs.abs() * d_s + U * gt.abs()
        dws = (gt[:, None] * x).sum((0, 2, 3))
        d_dws = n * hw * E * (gt[:, None] * x).abs().sum((0, 2, 3)) + (d_gt[:, None] * x.abs()).sum((0, 2, 3))
        gh2 = gcse * cse * (1 - cse)
        d_gh2 = d_gcse / 4 + gcse.abs() * d_cse + U * gh2.abs()
        dW2, d_dW2 = gh2.T @ a1, (n + 1) * E * (gh2.abs().T @ a1.abs()) + d_gh2.T @ a1.abs() + gh2.abs().T @ d_a1
        db2, d_db2 = gh2.sum(0), (n + 1) * E * gh2.abs().sum(0) + d_gh2.sum(0)
        ga1, d_ga1 = gh2 @ W2, (c + 1) * E * (gh2.abs() @ W2.abs()) + d_gh2 @ W2.abs()
        kink = (_dact(h1 - d_h1, act) - _dact(h1 + d_h1, act)).abs()
        gh1 = ga1 * _dact(h1, act)
        d_gh1 = d_ga1 + ga1.abs() * kink + U * gh1.abs()
        dW1, d_dW1 = gh1.T @ sq, (n + 1) * E * (gh1.abs().T @ sq.abs()) + d_gh1.T @ sq.abs() + gh1.abs().T @ d_sq
        db1, d_db1 = gh1.sum(0), (n + 1) * E * gh1.abs().sum(0) + d_gh1.sum(0)
        gsq, d_gsq = gh1 @ W1, (mid + 1) * E * (gh1.abs() @ W1.abs()) + d_gh1 @ W1.abs()
        dx = G * (C4 + S4) + gt[:, None] * ws[None, :, None, None] + (gsq / hw)[:, :, None, None]
        bd = (G.abs() * (d_cse[:, :, None, None] + d_s[:, None]) + d_gt[:, None] * ws.abs()[None, :, None, None]
              + (d_gsq / hw)[:, :, None, None] + 4 * U * (G.abs() * (C4 + S4) + (gt[:, None] * ws[None, :, None, None]).abs()
                                                         + (gsq / hw).abs()[:, :, None, None]))
        # x reaches two Functions inside the module (the gate kernel and the global-average-pool backward): autograd stores
        # each gradient in the compute type before it adds them, one more storage rounding of each part
        gate, sq_part = G * (C4 + S4) + gt[:, None] * ws[None, :, None, None], (gsq / hw)[:, :, None, None]
        bd = bd + self.store * (gate.abs() + sq_part.abs())
        if self.rec.rg[xr.tag]:
            self._add(xr.tag, dx, bd)
        for p, ref, b in ((l1.weight, dW1, d_dW1), (l1.bias, db1, d_db1), (l2.weight, dW2, d_dW2), (l2.bias, db2, d_db2),
                          (m.spatial_excite[0].weight, dws.reshape(1, c, 1, 1), d_dws.reshape(1, c, 1, 1))):
            if p.requires_grad:
                self._padd(p, ref, b)

    # composite glue: y = f(recorded inputs), checked forward; its vector-Jacobian product with the recorded output gradient
    # is each input's share of the gradient
    def relation(self, name, out, ins, f, act_kink=None):
        xs = [self._x(r).requires_grad_(True) for r in ins]
        v = f(*xs)
        with torch.no_grad():
            mag = f(*[x.detach().abs() for x in xs])
        e = 2.0 ** -21 * mag + self.store * mag
        y = self._x(out)
        assert_within(f"{name}: forward glue", y, v.detach(), e + self.store * (v.detach().abs() + e))
        G = self._grad(out)
        if G is None:
            return
        grads = torch.autograd.grad(v, xs, G)
        xa = [x.detach().abs().requires_grad_(True) for x in xs]
        mags = torch.autograd.grad(f(*xa), xa, G.abs())
        kink = 0.0
        if act_kink is not None:        # act(a + b): the sum is rounded before the activation reads its sign
            z = sum(x.detach() for x in xs)
            zm = sum(x.detach().abs() for x in xs)
            kink = G.abs() * ((_dact(z - 2 * self.store * zm, act_kink) - _dact(z + 2 * self.store * zm, act_kink)).abs())
        for r, g, mg in zip(ins, grads, mags):
            if self.rec.rg[r.tag]:
                self._add(r.tag, g, 2.0 ** -21 * mg + kink + U * g.abs())

    @staticmethod
    def _within(u, mod):
        mods = set(mod.modules())
        return [c for c in u.children if c.module in mods]

    def _out(self, u, mod):
        us = self._within(u, mod)
        assert us, f"{u.name}: {type(mod).__name__} not recorded"
        o = us[-1].out
        return o[0] if isinstance(o, list) else o

    def _in(self, u, mod):
        return self._within(u, mod)[0].inp[0]

    def composite(self, u, name):
        m = u.module
        if isinstance(m, (MI.DoublePartialResidual, MM.PartialInvertedResidual)):
            folded = [c for c in u.children if "residual" in c.kw]
            if isinstance(m, MI.DoublePartialResidual):
                # conv2's BatchNorm adds conv1's output
                c1 = u.children[0]
                assert len(folded) == 1, f"{name}: the residual must be folded into conv2's BatchNorm"
                x1 = c1.out[0]
                assert folded[0].kw["residual"].tag == x1.tag, f"{name}: conv2's BatchNorm must add conv1's output"
            elif m.res_connect:
                assert len(folded) == 1 and folded[0].kw["residual"].tag == u.inp[0][0].tag, \
                    f"{name}: the last BatchNorm must add the block input"
        if isinstance(m, (MI.ImageFillOrigin, MI.ImageFillOriginV2, MI.ImageFill)):
            self.unet_head(u, name)
        cat = lambda *t: torch.cat(t, 1)  # noqa: E731
        bil = lambda t, k: F.interpolate(t, scale_factor=k, mode="bilinear", align_corners=False)  # noqa: E731
        add = lambda a, b: a + b  # noqa: E731
        if isinstance(m, MM.InvertedResidual) and m.res_connect:
            folded = [c for c in u.children if "residual" in c.kw]
            if isinstance(m.conv[-1], MB.B200BNAct):
                assert len(folded) == 1 and folded[0].kw["residual"].tag == u.inp[0].tag, f"{name}: the last BatchNorm must add the block input"
            else:
                self.relation(name, u.out, [u.inp[0], self._out(u, m.conv)], add)
        elif isinstance(m, MX.ResidualBlock):
            short = u.inp[0] if m.residual_conv is None else self._out(u, m.residual_conv)
            self.relation(name, u.out, [self._out(u, m.conv), short], add)
        elif isinstance(m, MC.RFB):
            self.relation(name + " concat", self._in(u, m.rfb_linear_conv), [self._out(u, b) for b in m.rfb], cat)
            self.relation(name + " act(sum)", u.out, [self._out(u, m.rfb_linear_conv), self._out(u, m.input_down_channel)],
                          lambda a, b: _act(a + b, m.act_fn), act_kink=m.act_fn)
        elif isinstance(m, MC.ASP):
            self.relation(name + " concat", self._in(u, m.out_conv), [self._out(u, b) for b in m.asp], cat)
            assert self._out(u, m.out_conv).tag == u.out.tag
        elif isinstance(m, MT.TextSegament):
            f = m.encoder.features
            st = [self._out(u, f[i]) for i in range(len(f))]
            pools = [c for c in u.children if c.module is m.feature_avg_pool]
            assert [p.inp[0].tag for p in pools] == [st[0].tag, st[1].tag], f"{name}: the 1/2 maps must be pooled"
            self.relation(name + " shallow concat", self._in(u, m.feature_4x_conv), [pools[0].out, pools[1].out, st[2]], cat)
            self.relation(name + " deep concat", self._in(u, m.feature_pooling), st[3:], cat)
            self.relation(name + " 4x concat", self._in(u, m.smooth_feature_4x_conv),
                          [self._out(u, m.feature_4x_conv), self._out(u, m.feature_pooling)], lambda a, b: cat(a, bil(b, 2)))
            assert self._out(u, m.out_conv).tag == u.out.tag
        elif isinstance(m, MT.XceptionTextSegment):
            x4 = self._out(u, m.encoder.entry_flow_1)
            assert self._in(u, m.feature_4x_conv).tag == x4.tag and self._in(u, m.encoder.entry_flow_2).tag == x4.tag
            self.relation(name + " concat", self._in(u, m.out_conv), [self._out(u, m.feature_pooling), self._out(u, m.feature_4x_conv)],
                          lambda a, b: cat(bil(a, 2), b))
            self.relation(name + " output", u.out, [self._out(u, m.out_conv)], lambda a: bil(a, 4))

    def unet_head(self, u, name):
        """each decoder layer reads LazyCat([x, skip], ups=(1, 0)) and cat([mask.upsampled(), skip mask])"""
        m = u.module

        def layer(l):
            mods = set(l.modules())
            us = [c for c in u.children if c.module in mods]
            assert us, f"{name}: a layer of the network was not recorded"
            return us
        enc = [layer(l) for l in m.encoder]
        dec = [layer(l) for l in m.decoder]
        skips = [(u.inp[0][0], u.inp[0][1])] + [(us[-1].out[0], us[-1].out[1]) for us in enc]
        skips.pop()
        x = enc[-1][-1].out
        if hasattr(m, "dilated_layers"):
            x = layer(m.dilated_layers)[-1].out
        for dus in dec:
            d = dus[0]
            sx, sm = skips.pop()
            xr, mr = d.inp[0]
            assert isinstance(xr, LazyRec) and xr.ups == [1, 0] and [p.tag for p in xr.parts] == [x[0].tag, sx.tag], \
                f"{name}: {d.name} must read LazyCat([x, skip]) of the right tensors"
            want = [(p, c, up + 1) for p, c, up in x[1].parts] + list(sm.parts)
            assert len(want) == len(mr.parts) and all(torch.equal(a[0], b[0]) and a[1:] == b[1:] for a, b in zip(want, mr.parts)), \
                f"{name}: {d.name} must read cat([mask.upsampled(), skip mask])"
            x = dus[-1].out

    # ---------------------------------------------------------------- gradients
    def params(self):
        for p, ref, bd in self.pref.values():
            assert p.grad is not None, f"{self.label}: a parameter with a reference gradient got none"
            assert_within(f"{self.label}: parameter gradient {tuple(p.shape)}", p.grad.detach().double(), ref, bd + 2 * U * ref.abs())

    def inputs(self):
        roots = []
        for tag, g in self.rec.grads.items():
            a = self.contrib.get(tag)
            if a is None:
                roots.append(tag)
                continue
            ref, bd, mag, k = a
            got = _dev(g, self.dev)
            assert_within(f"{self.label}: input gradient of tensor {tag} (consumers {self.who[tag]})", got, ref,
                          bd + k * self.store * (mag + bd))
        self.roots = roots

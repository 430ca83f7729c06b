"""Partial-convolution layer family -- drop-in for the reference's models/partial_convolution.py.

Same constructors, ``forward((x, mask)) -> (y, new_mask)`` and state_dict keys (``feature_conv.weight/bias``,
frozen all-ones ``mask_conv.weight``, ``bn_act.0.*``); the arithmetic runs in libpconv_b200.so:
  * x*mask, the feature conv, the all-ones mask conv, the renormalisation and the mask update
    (reference :49-80) are ONE implicit-GEMM launch (+ a tiny integer box-sum over uint8 planes);
  * the returned mask is a :class:`HoleMask` (uint8 plane(s) + channel counts), never a dense fp32 tensor.
"""
import torch
from torch import nn

from .. import ops
from ..masks import HoleMask, as_hole_mask
from .BaseModels import BaseModule

inplace_batch_norm = False     # the reference's optional InPlaceABN extension is absent there too (:12-17)

CL = torch.channels_last


def _channels_last_(conv: nn.Conv2d):
    # master weights live physically as [cout][kh][kw][cin/g] (KRSC): the layout the kernels (and the
    # weight gradient) use.  Logical shape / state_dict stay OIHW.
    conv.weight.data = conv.weight.data.contiguous(memory_format=CL)


class PartialConv(BaseModule):
    """Hard-gated partial convolution (reference :20-80).  mask: 1 = valid, 0 = hole."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 same_holes=False):
        super().__init__()
        self.feature_conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        nn.init.kaiming_normal_(self.feature_conv.weight)
        _channels_last_(self.feature_conv)
        self.same_holes = same_holes
        # frozen all-ones kernel kept only for checkpoint compatibility (the box sum never reads it)
        m_in, m_out, m_groups = (1, 1, 1) if same_holes else (in_channels, out_channels, groups)
        self.mask_conv = nn.Conv2d(m_in, m_out, kernel_size, stride, padding, dilation, m_groups, bias=False)
        nn.init.constant_(self.mask_conv.weight, 1.0)
        for p in self.mask_conv.parameters():
            p.requires_grad = False
        self._wcache = ops.OperandCache()

    def _conv(self, x, mask, no_guard=False, handoff=None, epilogue=None):
        fc = self.feature_conv
        return ops.partial_conv(x, mask, fc.weight, fc.bias, fc.stride, fc.padding, fc.dilation, fc.groups,
                                same_holes=self.same_holes, no_guard=no_guard, cache=self._wcache, handoff=handoff, epilogue=epilogue)

    def forward(self, args, handoff=None, epilogue=None):
        x, mask = args
        return self._conv(x, mask, handoff=handoff, epilogue=epilogue)


class PartialConv1x1(BaseModule):
    """1x1 conv on the *unmasked* x; the mask's first channel is re-expanded (reference :83-105)."""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=0, dilation=1, groups=1, bias=True):
        super().__init__()
        assert kernel_size == 1 and stride == 1 and padding == 0
        self.feature_conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        nn.init.kaiming_normal_(self.feature_conv.weight)
        _channels_last_(self.feature_conv)
        self._wcache = ops.OperandCache()

    def forward(self, args):
        x, mask = args
        fc = self.feature_conv
        # an ordinary convolution: same kernels, mask ignored, renormaliser forced to 1 (`plain`)
        y, _ = ops.partial_conv(x, None, fc.weight, fc.bias, 1, 0, fc.dilation, fc.groups, cache=self._wcache, plain=True)
        return y, as_hole_mask(mask).expand_channels(y.shape[1])


class PartialConvNoHoles(PartialConv):
    """Decoder-side variant without hole bookkeeping and WITHOUT a zero guard (reference :108-137)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)
        assert self.feature_conv.groups == 1

    def forward(self, args, epilogue=None):
        x, mask = args
        return self._conv(x, mask, no_guard=True, epilogue=epilogue)


def partial_convolution_block(in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=False,
                              BN=True, activation=True, use_1_conv=False, no_holes_1_conv=False, same_holes=False):
    """Factory of reference :163-180: [conv] (+ PartialActivatedBN | PartialActivation) in an nn.Sequential."""
    if use_1_conv:
        m = [PartialConv1x1(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)]
    elif no_holes_1_conv:
        m = [PartialConvNoHoles(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)]
    else:
        m = [PartialConv(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias, same_holes)]
    if BN:
        m.append(PartialActivatedBN(out_channels, activation))
    if not BN and activation:
        m.append(PartialActivation(activation))
    return PartialBlock(*m)


class PartialBlock(nn.Sequential):
    """The nn.Sequential of the reference's factory (same children, same state_dict keys).  When it is exactly
    [PartialConv, PartialActivatedBN] the convolution output has a single consumer by construction, so the BatchNorm
    backward may absorb the convolution's renormalisation backward (ops.RenormHandoff).  For the same reason, inside an
    inference ops.StepScope, an eval-mode [PartialConv | PartialConvNoHoles, PartialActivatedBN | PartialActivation] block
    applies its BatchNorm + activation in the convolution epilogue.  Residual sites never come through
    here: DoublePartialResidual and PartialInvertedResidual call their last convolution and BatchNorm separately."""

    def forward(self, args):
        epi = self._eval_epilogue()
        if epi is not None:
            y, m = self[0](args, epilogue=epi)
            return (y, m) if epi.fused else self[1]((y, m))        # refused by the kernel: the two-pass path
        if len(self) == 2 and type(self[0]) is PartialConv and isinstance(self[1], PartialActivatedBN):
            bn = self[1].bn_act[0]
            h = ops.RenormHandoff(want_stats=bn.training and bn.weight is not None)
            return self[1](self[0](args, handoff=h), handoff=h)
        return super().forward(args)


    def _eval_epilogue(self):
        if len(self) != 2 or type(self[0]) not in (PartialConv, PartialConvNoHoles):
            return None
        tail = self[1]
        if isinstance(tail, PartialActivatedBN):
            return ops.eval_epilogue(tail.bn_act[0], tail.bn_act[1] if len(tail.bn_act) > 1 else None)
        if isinstance(tail, PartialActivation):
            return ops.eval_epilogue(None, tail.act_fn)
        return None


class PartialActivatedBN(BaseModule):
    """BatchNorm2d (+ activation) on x, mask passed through (reference :183-201)."""

    def __init__(self, channel, act_fn):
        super().__init__()
        self.bn_act = nn.Sequential(nn.BatchNorm2d(channel), act_fn) if act_fn else nn.Sequential(nn.BatchNorm2d(channel))

    def forward(self, args, residual=None, handoff=None):
        x, mask = args
        act = self.bn_act[1] if len(self.bn_act) > 1 else None
        return ops.bn_act(x, self.bn_act[0], act, residual=residual, handoff=handoff), mask


class PartialActivation(BaseModule):
    def __init__(self, activation):
        super().__init__()
        self.act_fn = activation

    def forward(self, args):
        x, mask = args
        return ops.activation_only(x, self.act_fn), mask


class DoubleUpSample(nn.Module):
    """Nearest upsampling of features AND mask (reference :224-231).  The mask side is free (index math)."""

    def __init__(self, scale_factor, mode="nearest"):
        super().__init__()
        if scale_factor != 2 or mode != "nearest":
            raise NotImplementedError("only nearest x2 has a GPU kernel (the only use in the reference networks)")
        self.upsample = nn.Upsample(scale_factor=scale_factor, mode=mode)   # kept for attribute compatibility

    def forward(self, args):
        x, mask = args
        # both sides are lazy: the features become a LazyCat (a Tensor subclass the next partial convolution reads in place,
        # also after the reference's own `torch.cat([x_up, skip], dim=1)`), the mask a HoleMask with `up` bumped
        return ops.upsample2x_lazy(x), as_hole_mask(mask).upsampled()

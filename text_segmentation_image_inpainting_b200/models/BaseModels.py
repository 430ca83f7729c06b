"""Module base class and conventions shared by the mirrored layer library.

Boundary contract reproduced from the reference's models/BaseModels.py:12-71 (SURVEY 8b):
lenient ``load_state_dict`` that copies by name and reports instead of raising (:41-52), the two weight
initialisers keyed on ``isinstance(m, nn.Conv2d / nn.BatchNorm2d)`` (:17-39), ``total_parameters`` (:64-68).
"""
import math
from contextlib import contextmanager

import torch
from torch import nn


def _weights_changed():
    """`.data` mutations do not bump tensor version counters: invalidate the cached compute-dtype weight operands."""
    from .. import ops
    ops.bump_weight_epoch()


class BaseModule(nn.Module):
    def __init__(self):
        self.act_fn = None
        super().__init__()

    # -- initialisers -----------------------------------------------------------------------------
    def _trainable(self, kinds):
        return (m for m in self.modules() if isinstance(m, kinds) and m.weight is not None and m.weight.requires_grad)

    def selu_init_params(self):
        for m in self._trainable((nn.Conv2d, nn.Linear)):
            m.weight.data.normal_(0.0, 1.0 / math.sqrt(m.weight.numel()))
            if m.bias is not None:
                m.bias.data.zero_()
        for m in self._trainable(nn.BatchNorm2d):
            m.weight.data.fill_(1)
            m.bias.data.zero_()
        _weights_changed()

    def initialize_weights(self):
        for m in self._trainable(nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="leaky_relu")
            if m.bias is not None:
                m.bias.data.zero_()
        for m in self._trainable(nn.BatchNorm2d):
            m.weight.data.fill_(1)
            m.bias.data.zero_()
        _weights_changed()

    # -- checkpoints ------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, self_state=False):
        """Copy-by-name; never raises (the reference prints and continues)."""
        own = self_state if self_state else self.state_dict()
        for name, value in state_dict.items():
            if name not in own:
                print("Parameter {} is not in the model. ".format(name))
                continue
            try:
                own[name].copy_(value.data if hasattr(value, "data") else value)
            except Exception as exc:  # noqa: BLE001 -- mirror of the reference's lenient behaviour
                print("Parameter {} fails to load.".format(name))
                print("-----------------------------------------")
                print(exc)
        _weights_changed()

    @contextmanager
    def set_activation_inplace(self):
        act = getattr(self, "act_fn", None)
        if act is not None and hasattr(act, "inplace"):
            act.inplace = True
            try:
                yield
            finally:
                act.inplace = False
        else:
            yield

    def total_parameters(self):
        total = sum(p.numel() for p in self.parameters())
        trainable = sum(p.numel() for p in self.parameters() if p.requires_grad)
        print("Total parameters : {}. Trainable parameters : {}".format(total, trainable))
        return total

    def forward(self, *x):
        raise NotImplementedError


# +++++++++++++++++++++++++++++++++++++
#   Convolution wrappers (reference models/BaseModels.py:91-127)
# -------------------------------------
class B200Conv2d(nn.Conv2d):
    """An ``nn.Conv2d`` (isinstance / out_channels / state_dict identical -- SURVEY 8b "attribute conventions")
    whose forward runs on libpconv_b200: dense and 1x1 convolutions on the wgmma implicit-GEMM kernel,
    depthwise ones on the vectorised HBM-bound kernel, anything else on the shape-general kernel."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if self.padding_mode != "zeros" or isinstance(self.padding, str):
            raise NotImplementedError("only explicit zero padding")
        self.weight.data = self.weight.data.contiguous(memory_format=torch.channels_last)
        self._wcache = {}

    def forward(self, x):
        from .. import ops
        # Conv_block linked the BatchNorm(+act) it placed behind this convolution: when that BatchNorm is in training mode the
        # convolution accumulates the per-channel sum / sum of squares of its output in its own epilogue and parks them on the
        # BatchNorm, which then skips its statistics pass over y (keyed by y's address and shape: any other input is ignored).
        hint = self.__dict__.get("_bn_hint")
        handoff = None
        if hint is not None and hint[0].training and hint[0].weight is not None and x.is_cuda:
            handoff = ops.RenormHandoff(want_stats=True)
        y = ops.conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups, cache=self._wcache,
                       handoff=handoff)
        if handoff is not None and handoff.bn_sums is not None:
            hint.__dict__["_pending_stats"] = (y.data_ptr(), tuple(y.shape), handoff.bn_sums)
        return y


class B200BNAct(nn.Sequential):
    """``nn.Sequential(nn.BatchNorm2d(c)[, act])`` (same keys: ``0.weight`` ...) as one statistics pass + one
    apply pass of libpconv_b200."""

    def forward(self, x, residual=None):
        from .. import ops
        act = self[1] if len(self) > 1 else None
        pend = self.__dict__.pop("_pending_stats", None)
        pre = pend[2] if (pend is not None and self[0].training and pend[0] == x.data_ptr() and pend[1] == tuple(x.shape)) else None
        return ops.bn_act(x, self[0], act, residual=residual, pre_sums=pre)


def Conv_block(in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True, BN=False,
               activation=None):
    """Returns the LIST ``[conv, (BN[, act]) | act]`` exactly like the reference factory (BaseModels.py:91-102)."""
    m = [B200Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation, groups, bias)]
    if BN:
        m.append(B200BNAct(nn.BatchNorm2d(out_channels), activation) if activation else B200BNAct(nn.BatchNorm2d(out_channels)))
        m[0].__dict__["_bn_hint"] = m[1]            # plain attribute (not a registered submodule: state_dict keys unchanged)
    if BN is False and activation is not None:
        m.append(activation)
    return m


class DSConvBlock(BaseModule):
    """Depthwise-separable unit: dw kxk (+BN+act) -> pw 1x1 (+BN+act)  (BaseModels.py:105-127)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, bias=True, BN=False,
                 activation_dep=None, activation_point=None):
        super().__init__()
        self.depth_wise_conv = nn.Sequential(*Conv_block(in_channels, in_channels, kernel_size, stride, padding, dilation,
                                                         in_channels, bias, BN=BN, activation=activation_dep))
        self.point_wise_conv = nn.Sequential(*Conv_block(in_channels, out_channels, kernel_size=1, stride=1, padding=0, dilation=1,
                                                         bias=bias, BN=BN, activation=activation_point))

    def forward(self, x):
        return self.point_wise_conv(self.depth_wise_conv(x))

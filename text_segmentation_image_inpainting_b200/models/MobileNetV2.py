"""MobileNetV2 backbones and inverted-residual blocks -- mirror of the hot-path part of the reference's
models/MobileNetV2.py: MobileNetV2 :20-111, InvertedResidual :114-149, PartialInvertedResidual :152-190,
DilatedMobileNetV2 :193-216.  (`MobileNetV2Classifier` -- LSTM/attention pre-training head -- is out of scope, and
`add_partial=True` is broken upstream: SURVEY 2 rows 3-4.)
"""
import torch
from torch import nn

from .. import ops
from .BaseModels import B200BNAct, BaseModule, Conv_block
from .common import SpatialChannelSqueezeExcitation
from .partial_convolution import PartialActivatedBN, partial_convolution_block


class InvertedResidual(BaseModule):
    """1x1 expand (x t) -> BN/act -> depthwise 3x3 (stride, dilation d, pad d) -> BN/act -> 1x1 linear -> BN [-> scSE];
    identity shortcut when stride == 1 and in == out (reference :126-149)."""

    def __init__(self, in_channel, out_channel, stride, expand_ratio, dilation, activation=nn.ReLU6(), bias=False, add_sece=False):
        super().__init__()
        self.stride, self.act_fn, self.bias = stride, activation, bias
        self.in_channels, self.out_channels = in_channel, out_channel
        self.res_connect = self.stride == 1 and in_channel == out_channel
        mid = in_channel * expand_ratio
        m = Conv_block(in_channel, mid, 1, 1, 0, bias=bias, BN=True, activation=activation)
        m += Conv_block(mid, mid, 3, stride, padding=1 + (dilation - 1), dilation=dilation, groups=mid, bias=bias, BN=True,
                        activation=activation)
        m += Conv_block(mid, out_channel, 1, 1, 0, bias=bias, BN=True, activation=None)
        if add_sece:
            m += [SpatialChannelSqueezeExcitation(out_channel, reduction=16, activation=activation)]
        self.conv = nn.Sequential(*m)
        if self.res_connect and isinstance(self.conv[-1], B200BNAct):
            # forward() folds the shortcut into this BatchNorm pass: its convolution must not apply it in the epilogue
            self.conv[-1].__dict__["_pcb_residual_site"] = True

    def forward(self, x):
        if not self.res_connect:
            return self.conv(x)
        last = self.conv[-1]
        if isinstance(last, B200BNAct):                    # no scSE: fold the shortcut into the last BN pass
            return last(self.conv[:-1](x), residual=ops.as_feature(x))
        return x + self.conv(x)


class MobileNetV2(BaseModule):
    """Backbone table walk of reference :20-107 (first conv + 7 inverted-residual stages)."""

    SETTING = [[1, 16, 1, 1, 1], [6, 24, 2, 2, 1], [6, 32, 3, 2, 1], [6, 64, 4, 2, 1], [6, 96, 3, 1, 1], [6, 160, 3, 2, 1],
               [6, 320, 1, 1, 1]]          # t, c, n, s, dilation
    OUT_STRIDE = 32

    def __init__(self, width_mult=1, activation=nn.ReLU6(), bias=False, add_sece=False, add_partial=False, image_channel=3):
        super().__init__()
        if add_partial:
            raise NotImplementedError("add_partial=True is broken in the reference itself (SURVEY 2 row 3)")
        self.add_partial = add_partial
        self.res_block = InvertedResidual
        self.act_fn, self.bias, self.width_mult = activation, bias, width_mult
        self.out_stride = self.OUT_STRIDE
        self.image_channel = image_channel
        self.inverted_residual_setting = [list(r) for r in self.SETTING]
        self.last_channel = 0
        self.features = self.make_inverted_resblocks(self.inverted_residual_setting, add_sece)

    def make_inverted_resblocks(self, settings, add_sece):
        in_channel = self._make_divisible(32 * self.width_mult, divisor=8)
        features = [nn.Sequential(*Conv_block(self.image_channel, in_channel, kernel_size=3, stride=2, padding=1, bias=self.bias,
                                              BN=True, activation=self.act_fn))]
        for t, c, n, s, d in settings:
            out_channel = self._make_divisible(c * self.width_mult, divisor=8)
            block = []
            for i in range(n):
                block.append(self.res_block(in_channel, out_channel, s if i == 0 else 1, t, d, activation=self.act_fn,
                                            bias=self.bias, add_sece=add_sece))
                in_channel = out_channel
            features.append(nn.Sequential(*block))
        self.last_channel = out_channel
        return nn.Sequential(*features)

    def load_pre_train_checkpoint(self, pre_train_checkpoint, free_last_blocks):
        if pre_train_checkpoint:
            if isinstance(pre_train_checkpoint, str):
                self.load_state_dict(torch.load(pre_train_checkpoint, map_location="cpu"))
            else:
                self.load_state_dict(pre_train_checkpoint)
            print("Encoder check point is loaded")
        else:
            print("No check point for the encoder is loaded. ")
        if free_last_blocks >= 0:
            self.freeze_params(free_last_blocks)
        else:
            print("All layers in the encoders are re-trained. ")

    def freeze_params(self, free_last_blocks=2):
        for i in range(len(self.features) - free_last_blocks):
            for p in self.features[i].parameters():
                p.requires_grad = False
        print("{}/{} layers in the encoder are freezed.".format(len(self.features) - free_last_blocks, len(self.features)))

    @staticmethod
    def _make_divisible(v, divisor=8, min_value=None):
        if min_value is None:
            min_value = divisor
        new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
        if new_v < 0.9 * v:
            new_v += divisor
        return new_v

    def forward(self, x):
        return self.features(x)


class DilatedMobileNetV2(MobileNetV2):
    """Output stride 8: the last four stages trade their strides for dilations 2/4/8/16 (reference :193-216)."""

    SETTING = [[1, 16, 1, 1, 1], [6, 24, 2, 2, 1], [6, 32, 3, 2, 1], [6, 64, 4, 1, 2], [6, 96, 3, 1, 4], [6, 160, 3, 1, 8],
               [6, 320, 1, 1, 16]]
    OUT_STRIDE = 8

    def __init__(self, width_mult=2, activation=nn.ReLU6(), bias=False, add_sece=False, add_partial=False, image_channel=3):
        super().__init__(width_mult=width_mult, activation=activation, bias=bias, add_sece=add_sece, add_partial=add_partial,
                         image_channel=image_channel)


class PartialInvertedResidual(BaseModule):
    """1x1 expand -> depthwise kxk (groups = mid, same_holes) -> 1x1 project, each a partial-conv block;
    identity shortcut when stride == 1 and in == out (reference :158,183-190)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, expansion=1, BN=True,
                 activation=True, bias=False, use_1_conv=False, no_holes_1_conv=False, same_holes=False, *args, **kwargs):
        super().__init__()
        self.res_connect = stride == 1 and in_channels == out_channels
        mid = int(in_channels * expansion)
        pw = dict(BN=BN, bias=bias, use_1_conv=use_1_conv, no_holes_1_conv=no_holes_1_conv)
        self.conv = nn.Sequential(
            partial_convolution_block(in_channels, mid, 1, 1, 0, 1, activation=activation, **pw),
            partial_convolution_block(mid, mid, kernel_size, stride, padding, dilation, groups=mid, BN=BN,
                                      activation=activation, bias=bias, same_holes=same_holes),
            partial_convolution_block(mid, out_channels, 1, 1, 0, 1, activation=None, **pw),
        )

    def forward(self, args):
        x, mask = args
        if not self.res_connect:
            return self.conv(args)
        # shortcut fused into the last block's BN(+identity act) pass when that block ends in a BN
        head, last = self.conv[:-1], self.conv[-1]
        y, m = head((x, mask))
        if len(last) == 2 and isinstance(last[1], PartialActivatedBN):
            y, m = last[0]((y, m))
            return last[1]((y, m), residual=ops.as_feature(x))
        y, m = last((y, m))
        return x + y, m

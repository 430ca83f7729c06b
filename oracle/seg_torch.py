"""Functional torch-CPU restatement of the reference's dense segmentation path (Conv_block / DSConvBlock /
InvertedResidual / scSE / RFB / ASP / DilatedMobileNetV2 / Xception / TextSegament / XceptionTextSegment).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pure functions over a reference-format ``state_dict``;
pinned bit-for-bit against the reference's own modules by tests/golden/seg_*.npz.  Citations relative to
the reference checkout.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .pconv_torch import activation, batchnorm


def conv(sd, key, x, stride=1, padding=0, dilation=1, groups=1):
    return F.conv2d(x, sd[key + "weight"], sd.get(key + "bias"), stride, padding, dilation, groups)


def conv_block(sd, prefix, i, x, stride=1, padding=0, dilation=1, groups=1, bn=True, act=None, training=True):
    """Conv_block products inside an nn.Sequential: conv at `<prefix><i>.`, (BN[,act]) at `<prefix><i+1>.0.`
    (models/BaseModels.py:91-102).  Returns (y, next index)."""
    x = conv(sd, f"{prefix}{i}.", x, stride, padding, dilation, groups)
    if bn:
        x = activation(act, batchnorm(x, sd, f"{prefix}{i + 1}.0.", training))
        return x, i + 2
    if act is not None:
        return activation(act, x), i + 2
    return x, i + 1


def ds_conv_block(sd, prefix, x, k, stride, padding, dilation, act_dep, act_point, training=True):
    """DSConvBlock.forward, models/BaseModels.py:105-127 (bias=False, BN=True as used by Xception)."""
    c = x.shape[1]
    x, _ = conv_block(sd, prefix + "depth_wise_conv.", 0, x, stride, padding, dilation, c, True, act_dep, training)
    x, _ = conv_block(sd, prefix + "point_wise_conv.", 0, x, 1, 0, 1, 1, True, act_point, training)
    return x


def scse(sd, prefix, x, act):
    """SpatialChannelSqueezeExcitation.forward, models/common.py:32-43."""
    b, c = x.shape[:2]
    ch = F.adaptive_avg_pool2d(x, 1).view(b, c)
    ch = F.linear(ch, sd[prefix + "channel_excite.0.weight"], sd[prefix + "channel_excite.0.bias"])
    ch = activation(act, ch)
    ch = torch.sigmoid(F.linear(ch, sd[prefix + "channel_excite.2.weight"], sd[prefix + "channel_excite.2.bias"])).view(b, c, 1, 1)
    x_cse = torch.mul(x, ch)                                     # :38  (statement order kept: it fixes autograd's summation order)
    sp = torch.sigmoid(F.conv2d(x, sd[prefix + "spatial_excite.0.weight"]))      # :41
    x_sse = torch.mul(x, sp)                                     # :42
    return torch.add(x_cse, x_sse)                               # :43


def inverted_residual(sd, prefix, x, cin, cout, stride, t, dilation, act, add_sece, training=True):
    """InvertedResidual.forward, models/MobileNetV2.py:114-149."""
    mid = cin * t
    y, _ = conv_block(sd, prefix + "conv.", 0, x, 1, 0, 1, 1, True, act, training)
    y, _ = conv_block(sd, prefix + "conv.", 2, y, stride, 1 + (dilation - 1), dilation, mid, True, act, training)
    y, _ = conv_block(sd, prefix + "conv.", 4, y, 1, 0, 1, 1, True, None, training)
    if add_sece:
        y = scse(sd, prefix + "conv.6.", y, act)
    return x + y if (stride == 1 and cin == cout) else y


def rfb(sd, prefix, x, out_c, act, add_sece, training=True):
    """RFB.forward, models/common.py:148-156 (branches :113-146)."""
    outs = []
    p = prefix + "rfb.0."
    y, _ = conv_block(sd, p, 0, x, 1, 0, 1, 1, True, act, training)
    y, _ = conv_block(sd, p, 2, y, 1, 1, 1, out_c, True, act, training)
    outs.append(y)
    for j, (k, r) in enumerate(zip((3, 5, 7), (5, 17, 29))):
        p = f"{prefix}rfb.{j + 1}."
        pad = (k - 1) // 2
        y, _ = conv_block(sd, p, 0, x, 1, 0, 1, 1, True, act, training)
        y, _ = conv_block(sd, p, 2, y, 1, (0, pad), 1, 1, True, None, training)
        y, _ = conv_block(sd, p, 4, y, 1, (pad, 0), 1, 1, True, None, training)
        y, _ = conv_block(sd, p, 6, y, 1, r, r, out_c, True, act, training)
        outs.append(y)
    y = conv(sd, prefix + "rfb_linear_conv.0.", torch.cat(outs, 1))
    if add_sece:
        y = scse(sd, prefix + "rfb_linear_conv.1.", y, act)
    resi, _ = conv_block(sd, prefix + "input_down_channel.", 0, x, 1, 0, 1, 1, True, act, training)
    return activation(act, y + resi)


def asp(sd, prefix, x, act, rates, training=True):
    """ASP.forward, models/common.py:86-93 (branches :59-71)."""
    y0, _ = conv_block(sd, prefix + "asp.0.", 0, x, 1, 1, 1, 1, True, act, training)
    outs = [y0]
    for j, r in enumerate(rates):
        p = F.avg_pool2d(x, kernel_size=r, stride=1, padding=(r - 1) // 2)
        y, _ = conv_block(sd, f"{prefix}asp.{j + 1}.", 1, p, 1, r, r, 1, True, act, training)
        outs.append(y)
    y, _ = conv_block(sd, prefix + "out_conv.", 0, torch.cat(outs, 1), 1, 0, 1, 1, True, act, training)
    return y


def make_divisible(v, divisor=8):
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


DILATED_SETTING = [[1, 16, 1, 1, 1], [6, 24, 2, 2, 1], [6, 32, 3, 2, 1], [6, 64, 4, 1, 2], [6, 96, 3, 1, 4], [6, 160, 3, 1, 8],
                   [6, 320, 1, 1, 16]]        # models/MobileNetV2.py:206-215


def mobilenet_stage_specs(width_mult):
    cin = make_divisible(32 * width_mult)
    stages = []
    for t, c, n, s, d in DILATED_SETTING:
        cout = make_divisible(c * width_mult)
        blocks = []
        for i in range(n):
            blocks.append((cin, cout, s if i == 0 else 1, t, d))
            cin = cout
        stages.append(blocks)
    return make_divisible(32 * width_mult), stages


def text_segment(sd, x, width_mult=2, training=True):
    """TextSegament.forward, models/text_segmentation.py:60-84."""
    act = ("leaky", 0.3)
    stem_c, stages = mobilenet_stage_specs(width_mult)

    def run_stage(si, x):
        if si == 0:
            y, _ = conv_block(sd, "encoder.features.0.", 0, x, 2, 1, 1, 1, True, act, training)
            return y
        for bi, (ci, co, s, t, d) in enumerate(stages[si - 1]):
            x = inverted_residual(sd, f"encoder.features.{si}.{bi}.", x, ci, co, s, t, d, act, True, training)
        return x
    shallow = []
    for si in range(3):
        x = run_stage(si, x)
        shallow.append(x)
    shallow[0] = F.avg_pool2d(shallow[0], 3, 2, 1)
    shallow[1] = F.avg_pool2d(shallow[1], 3, 2, 1)
    shallow = torch.cat(shallow, 1)
    deep = []
    for si in range(3, 8):
        x = run_stage(si, x)
        deep.append(x)
    x = rfb(sd, "feature_pooling.", torch.cat(deep, 1), 256, act, True, training)
    x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)
    sh_c = shallow.shape[1]
    shallow = inverted_residual(sd, "feature_4x_conv.", shallow, sh_c, 128, 1, 1, 1, act, True, training)
    x = torch.cat([shallow, x], 1)
    x = inverted_residual(sd, "smooth_feature_4x_conv.0.", x, 256 + 128, 128, 1, 1, 2, act, True, training)
    x = inverted_residual(sd, "smooth_feature_4x_conv.1.", x, 128, 128, 1, 1, 1, act, True, training)
    x = conv(sd, "out_conv.0.", x, 1, 1)
    return F.interpolate(x, scale_factor=4, mode="bilinear", align_corners=False)


def xception_residual_block(sd, prefix, x, cin, cout, stride, rate, act, training=True):
    """ResidualBlock.forward, models/Xception.py:13-44 (expand_channel_first=True)."""
    y = ds_conv_block(sd, prefix + "conv.0.", x, 3, 1, rate, rate, act, act, training)
    y = ds_conv_block(sd, prefix + "conv.1.", y, 3, 1, rate, rate, act, act, training)
    y = ds_conv_block(sd, prefix + "conv.2.", y, 3, stride, rate, rate, act, None, training)
    if stride > 1 or cin != cout:
        x, _ = conv_block(sd, prefix + "residual_conv.", 0, x, stride, 0, 1, 1, True, None, training)
    return y + x


def xception(sd, prefix, x, training=True):
    """Xception.forward, models/Xception.py:108-114."""
    act = ("leaky", 0.3)
    y, i = conv_block(sd, prefix + "entry_flow_1.", 0, x, 2, 1, 1, 1, True, act, training)
    y, i = conv_block(sd, prefix + "entry_flow_1.", i, y, 1, 1, 1, 1, True, act, training)
    x4 = xception_residual_block(sd, prefix + f"entry_flow_1.{i}.", y, 64, 128, 2, 1, act, training)
    y = xception_residual_block(sd, prefix + "entry_flow_2.0.", x4, 128, 256, 2, 1, act, training)
    y = xception_residual_block(sd, prefix + "entry_flow_2.1.", y, 256, 512, 1, 2, act, training)
    for j in range(8):
        y = xception_residual_block(sd, prefix + f"middle_flow.{j}.", y, 512, 512, 1, 2 if j < 4 else 4, act, training)
    for j, r in enumerate((2, 2, 1, 1)):
        y = xception_residual_block(sd, prefix + f"exit_flow.{j}.", y, 512, 512, 1, r, act, training)
    return y, x4


def xception_text_segment(sd, x, training=True):
    """XceptionTextSegment.forward, models/text_segmentation.py:104-114."""
    act = ("leaky", 0.3)
    y, x4 = xception(sd, "encoder.", x, training)
    x4, _ = conv_block(sd, "feature_4x_conv.", 0, x4, 1, 0, 1, 1, True, act, training)
    y = asp(sd, "feature_pooling.", y, act, (3, 5, 9), training)
    y = F.interpolate(y, scale_factor=2, mode="bilinear", align_corners=False)
    y = torch.cat([y, x4], 1)
    y, i = conv_block(sd, "out_conv.", 0, y, 1, 1, 1, 1, True, act, training)
    y = conv(sd, f"out_conv.{i}.", y, 1, 1)
    return F.interpolate(y, scale_factor=4, mode="bilinear", align_corners=False)


NETWORKS = {"TextSegament": text_segment, "XceptionTextSegment": xception_text_segment}

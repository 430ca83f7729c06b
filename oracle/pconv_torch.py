"""Functional torch-CPU restatement of the reference's partial-convolution path.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Pinned bit-for-bit against
the reference's own modules by tests/golden/ fixtures.

Everything is a pure function over tensors plus a reference-format
``state_dict`` (same key names as the reference's nn.Modules), so the oracle
can consume a checkpoint of the reference directly.  Citations are relative to
the reference checkout.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------
# storage-precision emulation (bf16 mode of the CUDA path)
# ----------------------------------------------------------------------------
# The CUDA path's tensor-core mode keeps activations and activation gradients in bf16 between kernels (fp32 accumulation
# inside them).  With `storage(torch.bfloat16)` active the oracle rounds at exactly those hand-over points -- and nowhere
# else -- so that a bf16 GPU result can be compared with "the reference algorithm under the same storage precision" at a tight
# tolerance instead of with the fp32 reference at a loose one:
#   forward : conv operands w, x*mask ; conv output y (after renormalisation) ; BN+activation output z ; network output
#   backward: gradient of every conv INPUT use (the data-gradient kernel's output, before the 2x2 sum of an upsampled source),
#             gradient of every block output (sum of its consumers' gradients = a bf16 add / the 2x2 reduction),
#             gradient of the conv's raw accumulator dc = dy / mask_sum (BatchNorm-backward / renorm-backward output)
_STORAGE = None


class storage:
    """Context manager: `with storage(torch.bfloat16): ...` (None = exact fp32, the default)."""

    def __init__(self, dtype):
        self.dtype = dtype

    def __enter__(self):
        global _STORAGE
        self.prev, _STORAGE = _STORAGE, self.dtype

    def __exit__(self, *exc):
        global _STORAGE
        _STORAGE = self.prev
        return False


class _RoundFwd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dtype):
        return x.to(dtype).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g, None


class _RoundBwd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dtype):
        ctx.dtype = dtype
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.to(ctx.dtype).to(g.dtype), None


def _rf(x):
    return x if _STORAGE is None else _RoundFwd.apply(x, _STORAGE)


def _rb(x):
    return x if (_STORAGE is None or not x.requires_grad) else _RoundBwd.apply(x, _STORAGE)


# ----------------------------------------------------------------------------
# L1: the three partial convolutions               models/partial_convolution.py
# ----------------------------------------------------------------------------


def _ones_like_weight(w: torch.Tensor, same_holes: bool) -> torch.Tensor:
    # frozen all-ones mask kernel, partial_convolution.py:38-47
    if same_holes:
        return torch.ones((1, 1) + tuple(w.shape[2:]), dtype=w.dtype)
    return torch.ones_like(w)


def partial_conv(x, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                 same_holes=False):
    """PartialConv.forward, partial_convolution.py:49-80.

    Returns (output, new_mask).  `new_mask` is a stride-0 expand when
    same_holes (partial_convolution.py:76-77).
    """
    x, weight = _rb(x), _rf(weight)                                                     # (storage emulation: no-ops in fp32 mode)
    out = F.conv2d(x * mask, weight, None if _STORAGE is not None else bias, stride, padding, dilation, groups)   # :51
    if _STORAGE is not None:
        out = _rb(out)                                                                  # dc = dy / mask_sum is stored rounded
        if bias is not None:
            out = out + bias.view(1, -1, 1, 1)
    if bias is not None:
        out_bias = bias.view(1, -1, 1, 1).expand_as(out)                                # :52-53
    else:
        out_bias = torch.zeros_like(out)                                                # :55
    with torch.no_grad():                                                               # :57
        ones_w = _ones_like_weight(weight, same_holes)
        if same_holes:
            msum = F.conv2d(mask[:, :1], ones_w, None, stride, padding, dilation, 1)    # :59
            holes = msum == 0                                                           # :60
            msum = msum * weight.shape[1] * groups                                      # :61  (in_channels)
        else:
            msum = F.conv2d(mask, ones_w, None, stride, padding, dilation, groups)      # :63
            holes = msum == 0                                                           # :64
    msum = msum.masked_fill(holes, 1.0)                                                 # :66
    out = _rf(((out - out_bias) / msum + out_bias).masked_fill(holes, 0.0))             # :71-72
    new_mask = torch.ones_like(msum).masked_fill(holes, 0.0)                            # :74-75
    if same_holes:
        new_mask = new_mask.expand_as(out)                                              # :77
    return out, new_mask


def partial_conv_1x1(x, mask, weight, bias=None, groups=1):
    """PartialConv1x1.forward, partial_convolution.py:101-105 (x is NOT masked)."""
    out = _rf(_rb(F.conv2d(_rb(x), _rf(weight), bias, 1, 0, 1, groups)))
    return out, mask[:, :1, :, :].expand_as(out)


def partial_conv_no_holes(x, mask, weight, bias=None, stride=1, padding=0, dilation=1):
    """PartialConvNoHoles.forward, partial_convolution.py:121-137 (no zero guard: NaN on an
    all-hole window, by design of the reference)."""
    x, weight = _rb(x), _rf(weight)
    out = F.conv2d(x * mask, weight, None if _STORAGE is not None else bias, stride, padding, dilation, 1)
    if _STORAGE is not None:
        out = _rb(out)
        if bias is not None:
            out = out + bias.view(1, -1, 1, 1)
    if bias is not None:
        out_bias = bias.view(1, -1, 1, 1).expand_as(out)
    else:
        out_bias = torch.zeros_like(out)
    with torch.no_grad():
        msum = F.conv2d(mask, torch.ones_like(weight), None, stride, padding, dilation, 1)
    out = _rf((out - out_bias) / msum + out_bias)
    return out, torch.ones_like(out)


# ----------------------------------------------------------------------------
# L1: BN / activation / upsample wrappers   partial_convolution.py:183-231
# ----------------------------------------------------------------------------

def activation(kind, x):
    """kind: None | 'relu' | 'relu6' | ('leaky', slope)."""
    if kind is None or kind is False:
        return x
    if kind == "relu":
        return F.relu(x)
    if kind == "relu6":
        return F.relu6(x)
    if isinstance(kind, tuple) and kind[0] == "leaky":
        return F.leaky_relu(x, kind[1])
    raise ValueError(kind)


def batchnorm(x, sd, prefix, training=True, momentum=0.1, eps=1e-5):
    """nn.BatchNorm2d semantics (PartialActivatedBN, partial_convolution.py:193-201;
    Conv_block, BaseModels.py:95-99).  In training mode updates the running buffers inside
    `sd` in place exactly as torch does (unbiased var, momentum 0.1, counter += 1)."""
    w, b = sd[prefix + "weight"], sd[prefix + "bias"]
    rm, rv = sd[prefix + "running_mean"], sd[prefix + "running_var"]
    if training:
        sd[prefix + "num_batches_tracked"] += 1
    return F.batch_norm(x, rm, rv, w, b, training, momentum, eps)


def double_upsample(x, mask, scale=2):
    """DoubleUpSample.forward (nearest on both), partial_convolution.py:229-231."""
    return (F.interpolate(x, scale_factor=scale, mode="nearest"),
            F.interpolate(mask, scale_factor=scale, mode="nearest"))


def pconv_block(sd, prefix, x, mask, *, k, s=1, p=0, d=1, groups=1, bn=True, act=None,
                use_1_conv=False, no_holes_1_conv=False, same_holes=False, training=True, residual=None):
    """partial_convolution_block (+ its BN/act tail), partial_convolution.py:163-180.

    `prefix` addresses the nn.Sequential the factory returns: `<prefix>0.` is the conv,
    `<prefix>1.bn_act.0.` the BatchNorm."""
    w = sd[prefix + "0.feature_conv.weight"]
    b = sd.get(prefix + "0.feature_conv.bias")
    if use_1_conv:
        assert k == 1 and s == 1 and p == 0                                             # :96
        x, mask = partial_conv_1x1(x, mask, w, b, groups)
    elif no_holes_1_conv:
        assert groups == 1                                                              # :119
        x, mask = partial_conv_no_holes(x, mask, w, b, s, p, d)
    else:
        x, mask = partial_conv(x, mask, w, b, s, p, d, groups, same_holes)
    # `residual`: the identity shortcut some callers add to the block output (image_inpainting.py:216, MobileNetV2.py:187).
    # Mathematically the caller's `out + residual`; taken here so that storage emulation rounds the SUM once, like the
    # CUDA path's fused BN + activation + residual pass does.
    if bn:
        x = activation(act, batchnorm(x, sd, prefix + "1.bn_act.0.", training))         # :195-201
    elif act:
        x = activation(act, x)                                                          # :177-178
    if residual is not None:
        x = x + residual
    if bn or act or residual is not None:
        x = _rf(x)
    return _rb(x), mask


# ----------------------------------------------------------------------------
# L2 workloads: the inpainting U-Nets               models/image_inpainting.py
# ----------------------------------------------------------------------------

# (in_c, out_c, k, s, p) -- image_inpainting.py:116-126 / :135-145
ORIGIN_ENCODER = [(64, 128, 5, 2, 2), (128, 256, 5, 2, 2), (256, 512, 3, 2, 1), (512, 512, 3, 2, 1),
                  (512, 512, 3, 2, 1), (512, 512, 3, 2, 1), (512, 512, 3, 2, 1)]
ORIGIN_DECODER = [(1024, 512, 3, 1, 1)] * 4 + [(768, 256, 3, 1, 1), (384, 128, 3, 1, 1), (192, 64, 3, 1, 1)]


def _unet_decode(layers, x, mask, feats, fmasks):
    # shared decoder skeleton, image_inpainting.py:180-191 / :282-290 / :77-86
    feats, fmasks = feats[:-1], fmasks[:-1]
    for layer in layers:
        xu, mu = double_upsample(x, mask)
        x, mask = layer(torch.cat([xu, feats.pop(-1)], 1), torch.cat([mu, fmasks.pop(-1)], 1))
    return x


def image_fill_origin(sd, x, mask, training=True):
    """ImageFillOrigin.forward, image_inpainting.py:164-191 (layer tables :116-153)."""
    feats, fmasks = [x], [mask]
    # encoder.0: 3->64 k7 s2 p3, bias, no BN, ReLU, same_holes          (:132)
    x, mask = pconv_block(sd, "encoder.0.", x, mask, k=7, s=2, p=3, bn=False, act="relu",
                          same_holes=True, training=training)
    feats.append(x); fmasks.append(mask)
    for i, (ci, co, k, s, p) in enumerate(ORIGIN_ENCODER):                             # :133,155-162
        x, mask = pconv_block(sd, f"encoder.{i + 1}.0.", x, mask, k=k, s=s, p=p, bn=True, act="relu",
                              same_holes=True, training=training)
        feats.append(x); fmasks.append(mask)

    def mk(j, k, s, p):
        return lambda xx, mm: pconv_block(sd, f"decoder.{j}.0.", xx, mm, k=k, s=s, p=p, bn=True,
                                          act=("leaky", 0.2), same_holes=False, training=training)
    layers = [mk(j, k, s, p) for j, (ci, co, k, s, p) in enumerate(ORIGIN_DECODER)]     # :152
    # decoder.7: 67->3 k3 p1, bias, no BN, no act                         (:153)
    layers.append(lambda xx, mm: pconv_block(sd, "decoder.7.", xx, mm, k=3, s=1, p=1, bn=False, act=None,
                                             same_holes=False, training=training))
    return _unet_decode(layers, x, mask, feats, fmasks)


# (in_c, out_c) ; all k3 s2 p1                  image_inpainting.py:225-235 / :245-255
V2_ENCODER = [(64, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512)]
V2_DECODER = [(1024, 512), (1024, 512), (768, 256), (512, 256), (512, 256), (384, 128), (192, 64)]


def _double_partial_residual(sd, prefix, x, mask, k, stride, rates, act, same_holes, training):
    """DoublePartialResidual.forward, image_inpainting.py:194-216: padding == dilation == rates[i]
    (the ctor's own `padding`/`dilation` args are ignored, :201-202,206-207)."""
    x1, m1 = pconv_block(sd, prefix + "conv1.", x, mask, k=k, s=stride, p=rates[0], d=rates[0], bn=True,
                         act=act, same_holes=same_holes, training=training)
    y, m2 = pconv_block(sd, prefix + "conv2.", x1, m1, k=k, s=1, p=rates[1], d=rates[1], bn=True,
                        act=act, same_holes=same_holes, training=training, residual=x1)   # x2 + x1, :216
    return y, m2


def image_fill_origin_v2(sd, x, mask, training=True):
    """ImageFillOriginV2.forward, image_inpainting.py:272-290 (tables :225-260)."""
    lk = ("leaky", 0.2)
    feats, fmasks = [x], [mask]
    x, mask = pconv_block(sd, "encoder.0.", x, mask, k=5, s=2, p=2, bn=True, act=lk, same_holes=True,
                          training=training)                                           # :241-242
    feats.append(x); fmasks.append(mask)
    for i in range(len(V2_ENCODER)):
        x, mask = _double_partial_residual(sd, f"encoder.{i + 1}.0.", x, mask, 3, 2, (1, 2), lk, True,
                                           training)                                   # :243
        feats.append(x); fmasks.append(mask)

    def mk(j):
        return lambda xx, mm: _double_partial_residual(sd, f"decoder.{j}.0.", xx, mm, 3, 1, (2, 1), lk, False,
                                                       training)                       # :258
    layers = [mk(j) for j in range(len(V2_DECODER))]
    layers.append(lambda xx, mm: pconv_block(sd, "decoder.7.", xx, mm, k=3, s=1, p=1, bn=False, act="relu",
                                             same_holes=False, training=training))     # :259-260
    return _unet_decode(layers, x, mask, feats, fmasks)


def _partial_inverted_residual(sd, prefix, x, mask, cin, cout, k, s, p, d, t, act, use_1, no_holes, same_holes,
                               training):
    """PartialInvertedResidual.forward, MobileNetV2.py:152-190 (body :164-181)."""
    mid = int(cin * t)
    y, m = pconv_block(sd, prefix + "conv.0.", x, mask, k=1, bn=True, act=act, use_1_conv=use_1,
                       no_holes_1_conv=no_holes, training=training)                    # :170-172
    y, m = pconv_block(sd, prefix + "conv.1.", y, m, k=k, s=s, p=p, d=d, groups=mid, bn=True, act=act,
                       same_holes=same_holes, training=training)                       # :174-176
    y, m = pconv_block(sd, prefix + "conv.2.", y, m, k=1, bn=True, act=None, use_1_conv=use_1,
                       no_holes_1_conv=no_holes, training=training,
                       residual=x if (s == 1 and cin == cout) else None)               # :178-180, shortcut :158,186-187
    return y, m


# in_c, out_c, k, s, p, d, t, n                              image_inpainting.py:15-41
FILL_ENCODER = [(64, 128, 3, 2, 1, 1, 4, 2), (128, 256, 3, 2, 1, 1, 4, 2), (256, 256, 3, 2, 1, 1, 4, 2)]
FILL_DILATED = [(256, 256, 3, 1, 2, 2, 4, 2), (256, 256, 3, 1, 4, 4, 4, 2), (256, 256, 3, 1, 8, 8, 4, 2)]
FILL_DECODER = [(512, 256, 3, 1, 1, 1, 2, 1), (384, 128, 3, 1, 1, 1, 2, 1), (192, 32, 3, 1, 1, 1, 2, 1)]


def _fill_stage(sd, prefix, x, mask, row, act, use_1, no_holes, training):
    # ImageFill.make_layers, image_inpainting.py:46-65: n blocks, first carries the stride
    ci, co, k, s, p, d, t, n = row
    for i in range(n):
        x, mask = _partial_inverted_residual(sd, f"{prefix}{i}.", x, mask, ci, co, k, s if i == 0 else 1, p, d, t,
                                             act, use_1, no_holes, True, training)
        ci = co
    return x, mask


def image_fill(sd, x, mask, training=True):
    """ImageFill.forward, image_inpainting.py:67-86."""
    act = ("leaky", 0.3)                                                                # :12
    feats, fmasks = [x], [mask]
    x, mask = pconv_block(sd, "encoder.0.", x, mask, k=7, s=2, p=3, bn=False, act=act, training=training)  # :23
    feats.append(x); fmasks.append(mask)
    for i, row in enumerate(FILL_ENCODER):                                              # :24
        x, mask = _fill_stage(sd, f"encoder.{i + 1}.", x, mask, row, act, True, False, training)
        feats.append(x); fmasks.append(mask)
    feats, fmasks = feats[:-1], fmasks[:-1]                                             # :77-78
    for i, row in enumerate(FILL_DILATED):                                              # :33,79
        x, mask = _fill_stage(sd, f"dilated_layers.{i}.", x, mask, row, act, False, True, training)
    for j, row in enumerate(FILL_DECODER):                                              # :43,81-85
        xu, mu = double_upsample(x, mask)
        x, mask = _fill_stage(sd, f"decoder.{j}.", torch.cat([xu, feats.pop(-1)], 1),
                              torch.cat([mu, fmasks.pop(-1)], 1), row, act, False, True, training)
    xu, mu = double_upsample(x, mask)
    x, mask = pconv_block(sd, "decoder.3.", torch.cat([xu, feats.pop(-1)], 1),
                          torch.cat([mu, fmasks.pop(-1)], 1), k=3, s=1, p=1, bn=False, act=None,
                          training=training)                                           # :44
    return x


NETWORKS = {"ImageFillOrigin": image_fill_origin, "ImageFillOriginV2": image_fill_origin_v2,
            "ImageFill": image_fill}


def clone_state_dict(sd, requires_grad=False):
    """Detach-clone a state_dict; optionally mark the trainable float tensors as leaves that
    require grad (everything except frozen mask kernels and BN buffers)."""
    out = {}
    for k, v in sd.items():
        t = v.detach().clone()
        if requires_grad and t.is_floating_point() and not (
                k.endswith("mask_conv.weight") or k.endswith("running_mean") or k.endswith("running_var")):
            t.requires_grad_(True)
        out[k] = t
    return out

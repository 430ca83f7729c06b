"""The reference's losses on the GPU under the reference's names and signatures: the inpainting loss (loss.py:185-307:
`InpaintingLoss`, `FeatureExtractor`, `VggExtractor`, `gram_matrix`, `total_variation_loss`) and the segmentation losses
(loss.py:58-121: `BinaryFocalLoss`, `SoftBootstrapCrossEntropy`, csrc/seg_loss.cu).  `MultiClassFocalLoss` (multi-class logits;
both segmentation networks have one output channel) and `BCERegionLoss` (the LSTM classifier head) have no GPU path.

    loss = 1 valid + 6 hole + 0.1 tv + 0.05 perceptual + 120 style          (loss.py:223-224)

The three images the reference runs through VGG16 (composite, output, origin) form ONE batch of 3n images, so every VGG layer
is one launch: the 3x3 convolutions run on this library's convolution kernels in `plain` mode with the ReLU applied in the
forward epilogue where the kernel can; max-pool, pixel terms, perceptual and Gram L1 sums are kernels of `inpaint_loss.cu`;
the Gram products F F^T are the 1x1 weight-gradient problem per image.  Backward goes through the composite and output images
only (2n images, the leading part of every saved activation): frozen VGG weights get no weight gradient, origin is a constant.
Everything is stream-ordered and capturable; the loss and its five terms stay on the device.
"""
from __future__ import annotations

import ctypes
from typing import List

import torch
import torch.nn as nn

from . import _lib, ops
from ._lib import ACT_RELU
from .masks import HoleMask

CL = torch.channels_last
# vgg16.features[:17] split as VggExtractor does (loss.py:248-250): (in, out) channels of each stage's 3x3 convolutions
_VGG_STAGES = (((3, 64), (64, 64)), ((64, 128), (128, 128)), ((128, 256), (256, 256), (256, 256)))
WEIGHTS = (1.0, 6.0, 0.1, 0.05, 120.0)
TERMS = ("valid", "hole", "tv", "perceptual", "style")


def _stream():
    return torch.cuda.current_stream().cuda_stream


_PARTS = None     # optional list: (part, start event, end event) per timed section of the loss (tools/bench_inpaint_loss.py)


def set_part_timing(sink):
    """Pass a list to record CUDA-event-bracketed parts of the loss ("vgg_forward", "vgg_dgrad", "gram", "fused") in eager
    calls, or None to stop."""
    global _PARTS
    _PARTS = sink


class _part:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if _PARTS is not None:
            self.s, self.e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.s.record()

    def __exit__(self, *exc):
        if _PARTS is not None:
            self.e.record()
            _PARTS.append((self.name, self.s, self.e))
        return False


def _strides(t):
    return (ctypes.c_longlong * 4)(*t.stride())


class VggExtractor(nn.Module):
    """VGG16 `features[:17]` as three stages (conv3x3 + ReLU blocks, each ending in a 2x2/2 max-pool), frozen, with the
    reference's `state_dict` keys (`features.0.0.weight`, ...), so torchvision VGG16 weights load.  `pretrained=True` asks
    torchvision for its ImageNet weights (whatever torchvision does on this machine, download included)."""

    def __init__(self, pretrained=True):
        super().__init__()
        stages = []
        for convs in _VGG_STAGES:
            mods = []
            for cin, cout in convs:
                mods += [nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU(inplace=True)]
            mods.append(nn.MaxPool2d(kernel_size=2, stride=2))
            stages.append(nn.Sequential(*mods))
        self.features = nn.Sequential(*stages)
        if pretrained:
            import torchvision
            vgg = torchvision.models.vgg16(pretrained=True)
            sd = {}
            for i, (a, b) in enumerate(((0, 5), (5, 10), (10, 17))):
                for k, v in nn.Sequential(*vgg.features[a:b]).state_dict().items():
                    sd[f"features.{i}.{k}"] = v
            self.load_state_dict(sd)
        for p in self.features.parameters():
            p.requires_grad = False
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                m._wcache = ops.OperandCache(frozen=True)                             # _Vgg.conv_relu, _Vgg.dgrad
                m._k2r_cache = ops.OperandCache(frozen=True, derive=_k2r_image_weight)   # _Vgg.dgrad_image

    def stage_convs(self, s) -> List[nn.Conv2d]:
        return [m for m in self.features[s] if isinstance(m, nn.Conv2d)]

    def forward(self, img):
        """The three stage outputs of `img` (no gradient: the features are frozen and this path has no backward)."""
        return _Vgg(self, len(self.features)).forward(_as_vgg_input(img))[1]


class FeatureExtractor(nn.Module):
    """loss.py:228-241: the first `feature_range` stages of `encoder.features`, frozen."""

    def __init__(self, encoder, feature_range=3):
        super().__init__()
        if not isinstance(encoder, VggExtractor):
            raise NotImplementedError("only VggExtractor has a GPU path (the reference's other extractors raise in forward)")
        if not 1 <= feature_range <= len(encoder.features):
            raise ValueError(f"feature_range must be in 1..{len(encoder.features)}")
        self.__dict__["encoder"] = encoder           # not a submodule: the state_dict keys stay the reference's `layers.*`
        self.feature_range = feature_range
        self.layers = nn.Sequential(*[encoder.features[i] for i in range(feature_range)])
        for p in self.layers.parameters():
            p.requires_grad = False

    def forward(self, x):
        return _Vgg(self.encoder, self.feature_range).forward(_as_vgg_input(x))[1]


def _k2r_image_weight(weight):
    """The fp32 master of conv1_1's kernel-to-row data gradient: W'[tap·3 + ci][co], 27 of 32 rows (pcb_k2r_image_weight)."""
    cout = weight.shape[0]
    wz = torch.empty((32, cout), dtype=torch.float32, device=weight.device)
    _lib.check(_lib.load().pcb_k2r_image_weight(weight.detach().float().contiguous().data_ptr(), cout, wz.data_ptr(), _stream()))
    return wz


def _as_vgg_input(img):
    """[n, 3, h, w] image -> [n, 3, h, w] view of an 8-channel-padded NHWC buffer in its dtype."""
    img = ops.as_feature_padded(img)
    if ops.nhwc_layout(img) == 8:
        return img
    buf = ops.padded_empty(*img.shape, img.dtype, img.device)
    buf.copy_(img)
    return buf


class _Vgg:
    """The VGG stages of one extractor over NHWC batches: forward keeps what the data gradient needs."""

    def __init__(self, enc: VggExtractor, nstages):
        self.enc, self.nstages = enc, nstages
        self.lib = _lib.load()

    def _geom(self, x, conv):
        return ops.ConvGeom([x], [0], conv.out_channels, 3, 1, 1, 1, 1, False, False, [(None, conv.in_channels, 0)], plain=True)

    def operands(self, conv, geom):
        """The operands of a frozen VGG weight (its frozen OperandCache: laid out again only when the weight changes)."""
        return conv._wcache.get(conv.weight, geom)

    def conv_relu(self, conv, x):
        """relu(conv(x) + b), the ReLU in the forward epilogue when the kernel applies one, else in a second pass."""
        lib, dev = self.lib, x.device
        geom = self._geom(x, conv)
        wprep = self.operands(conv, geom)
        c = geom.struct([x])
        y = torch.empty((geom.n, geom.cout, geom.ho, geom.wo), dtype=x.dtype, device=dev, memory_format=CL)
        dummy = torch.empty((16,), dtype=torch.uint8, device=dev)            # plain convolutions write no mask sums
        ws = ops._workspace(lib, c, dev)
        b32 = conv.bias.detach().float().contiguous()
        if lib.pcb_conv_fuses_affine_act(ctypes.byref(c)):
            _lib.check(lib.pcb_pconv_forward_affine_act(ctypes.byref(c), wprep.w_fwd.data_ptr(), b32.data_ptr(), y.data_ptr(), geom.cout,
                                                        dummy.data_ptr(), dummy.data_ptr(), ws.data_ptr(), 0, None, None, ACT_RELU, 0.0,
                                                        _stream()))
        else:
            _lib.check(lib.pcb_pconv_forward(ctypes.byref(c), wprep.w_fwd.data_ptr(), b32.data_ptr(), y.data_ptr(), geom.cout,
                                             dummy.data_ptr(), dummy.data_ptr(), ws.data_ptr(), _stream()))
            _lib.check(lib.pcb_bn_act_forward(y.data_ptr(), geom.dtype, geom.n * geom.ho * geom.wo, geom.cout, None, None, ACT_RELU, 0.0,
                                              None, y.data_ptr(), _stream()))
        return y, wprep

    def forward(self, x):
        """x: [m, 3, h, w] (8-channel-padded NHWC).  Returns (per-stage list of (conv, input, relu output, operands), stage
        outputs)."""
        saved, feats = [], []
        with _part("vgg_forward"):
            for s in range(self.nstages):
                layers = []
                for conv in self.enc.stage_convs(s):
                    y, wprep = self.conv_relu(conv, x)
                    layers.append((conv, x, y, wprep))
                    x = y
                m, c, h, w = x.shape
                p = torch.empty((m, c, h // 2, w // 2), dtype=x.dtype, device=x.device, memory_format=CL)
                _lib.check(self.lib.pcb_maxpool2x2_forward(x.data_ptr(), p.data_ptr(), ops._dtype_code(x), m, h, w, c, _stream()))
                saved.append(layers)
                feats.append(p)
                x = p
        return saved, feats

    def dgrad(self, conv, x, wprep, dc, relu_in=False):
        """Data gradient of one convolution for the first dc.shape[0] images of its input x (no weight gradient: frozen).
        relu_in: x is the output of an in-place ReLU whose backward is applied too -- in the data-gradient epilogue where the
        kernel fuses it, else by a second pass."""
        lib = self.lib
        m = dc.shape[0]
        xs = x[:m]
        if conv.in_channels == 3:
            return self.dgrad_image(conv, xs, dc)
        geom = self._geom(xs, conv)
        c = geom.struct([xs])
        w_fwd, w_dg = wprep
        dx = ops.padded_empty(m, geom.cin, geom.h, geom.w, x.dtype, x.device)
        if relu_in and lib.pcb_conv_dgrad_fuses_relu(ctypes.byref(c)):
            _lib.check(lib.pcb_pconv_backward_data_relu(ctypes.byref(c), dc.data_ptr(), geom.cout, w_dg.data_ptr(), dx.data_ptr(),
                                                        ops.nhwc_layout(dx), xs.data_ptr(), ops.nhwc_layout(xs), _stream()))
            return dx
        ptrs = (ctypes.c_void_p * 1)(dx.data_ptr())
        strides = (ctypes.c_int32 * 1)(ops.nhwc_layout(dx))
        _lib.check(lib.pcb_pconv_backward_data(ctypes.byref(c), dc.data_ptr(), geom.cout, w_fwd.data_ptr(), ops._ptr(w_dg), ptrs, strides,
                                               _stream()))
        return self.relu_backward(dx, xs) if relu_in else dx

    def dgrad_image(self, conv, xs, dc):
        """conv1_1's data gradient (3 input channels) in kernel-to-row form: the 1x1 problem dc (cout) -> Z (27 of 32 columns)
        on the convolution forward kernels, then the streaming tap sum (pcb_k2r_image_dgrad)."""
        lib, dev, dt = self.lib, xs.device, xs.dtype
        m, _, h, w = xs.shape
        cout = conv.out_channels
        geom = ops.ConvGeom([dc], [0], 32, 1, 1, 0, 1, 1, False, False, [(None, cout, 0)], plain=True)
        w_fwd = conv._k2r_cache.get(conv.weight, geom).w_fwd
        c = geom.struct([dc])
        z = torch.empty((m, 32, h, w), dtype=dt, device=dev, memory_format=CL)
        dummy = torch.empty((16,), dtype=torch.uint8, device=dev)
        ws = ops._workspace(lib, c, dev)
        _lib.check(lib.pcb_pconv_forward(ctypes.byref(c), w_fwd.data_ptr(), None, z.data_ptr(), 32, dummy.data_ptr(), dummy.data_ptr(),
                                         ws.data_ptr(), _stream()))
        dx = ops.padded_empty(m, 3, h, w, dt, dev)
        _lib.check(lib.pcb_k2r_image_dgrad(z.data_ptr(), ops._dtype_code(z), m, h, w, dx.data_ptr(), _stream()))
        return dx

    def relu_backward(self, g, y):
        """g * (y > 0) for the ReLU output y (leading g.shape[0] images)."""
        m, c, h, w = g.shape
        out = torch.empty_like(g, memory_format=CL)
        _lib.check(self.lib.pcb_bn_act_backward_apply(g.data_ptr(), y.data_ptr(), ops._dtype_code(g), m * h * w, c, None, None, None, None,
                                                      ACT_RELU, 0.0, None, None, 0, out.data_ptr(), None, None, _stream()))
        return out


class _Gram:
    """Per-image Gram products F F^T (fp32 [m][c][c], unnormalised) as the 1x1 weight-gradient problem with x = dc = F_i, and
    the Gram backward F (S + S^T) as a 1x1 forward with a per-image weight."""

    def __init__(self, f):
        self.lib = _lib.load()
        self.c = f.shape[1]
        self.geom = ops.ConvGeom([f[:1]], [0], self.c, 1, 1, 0, 1, 1, False, False, [(None, self.c, 0)], plain=True)

    def products(self, f):
        lib, c = self.lib, self.c
        g = torch.empty((f.shape[0], c, c), dtype=torch.float32, device=f.device)
        ws = ops._workspace(lib, self.geom.struct([f[:1]]), f.device)
        for i in range(f.shape[0]):
            s = self.geom.struct([f[i:i + 1]])
            _lib.check(lib.pcb_pconv_backward_weight(ctypes.byref(s), f[i:i + 1].data_ptr(), c, g[i].data_ptr(), ws.data_ptr(), _stream()))
        return g

    def backward(self, f, t):
        """out[i] = F_i t[i]^T for the leading t.shape[0] images (t: fp32 [m][c][c], symmetric)."""
        lib, c, m = self.lib, self.c, t.shape[0]
        s0 = self.geom.struct([f[:1]])
        fe, de = ops.Operands.sizes(s0)
        w = torch.empty((m, fe), dtype=f.dtype, device=f.device)
        wd = torch.empty((de,), dtype=f.dtype, device=f.device) if de else None
        out = torch.empty((m, c, f.shape[2], f.shape[3]), dtype=f.dtype, device=f.device, memory_format=CL)
        dummy = torch.empty((16,), dtype=torch.uint8, device=f.device)
        ws = ops._workspace(lib, s0, f.device)
        for i in range(m):
            s = self.geom.struct([f[i:i + 1]])
            ops.Operands.lay_out(s, t[i], w[i], wd)
            _lib.check(lib.pcb_pconv_forward(ctypes.byref(s), w[i].data_ptr(), None, out[i:i + 1].data_ptr(), c, dummy.data_ptr(),
                                             dummy.data_ptr(), ws.data_ptr(), _stream()))
        return out


class _InpaintingLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, crit, raw, origin, plane, output):
        lib = _lib.load()
        n, _, h, w = output.shape
        dt, dev = output.dtype, output.device
        code = ops._dtype_code(output)
        X = ops.padded_empty(3 * n, 3, h, w, dt, dev)                     # comp | output | origin, 8-channel-padded NHWC
        sums = torch.zeros((16,), dtype=torch.float64, device=dev)
        with _part("fused"):
            _lib.check(lib.pcb_inpaint_loss_pixel_forward(raw.data_ptr(), origin.data_ptr(), output.data_ptr(), code, _strides(output),
                                                          plane.data_ptr(), n, h, w, X.data_ptr(), code, sums.data_ptr(), _stream()))
        vgg = _Vgg(crit.feature_encoder.encoder, crit.feature_encoder.feature_range)
        saved, feats = vgg.forward(X)
        inv = [0.0] * 16
        numel = n * 3 * h * w
        inv[0] = inv[1] = 1.0 / numel
        inv[2], inv[3] = 1.0 / (n * 3 * h * (w - 1)), 1.0 / (n * 3 * (h - 1) * w)
        grams = []
        for s, f in enumerate(feats):
            _, c, hs, ws = f.shape
            gm = _Gram(f)
            with _part("gram"):
                g = gm.products(f)
            with _part("fused"):
                _lib.check(lib.pcb_feature_l1_forward(f.data_ptr(), code, n, hs * ws, c, sums[4 + 2 * s:].data_ptr(), _stream()))
                _lib.check(lib.pcb_gram_l1_forward(g.data_ptr(), n, c, float(c * hs * ws), sums[10 + 2 * s:].data_ptr(), _stream()))
            grams.append((gm, g))
            inv[4 + 2 * s] = 1.0 / (n * c * hs * ws)
            inv[10 + 2 * s] = 1.0 / (n * c * c)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        terms = crit._terms_buffer(dev)
        with _part("fused"):
            _lib.check(lib.pcb_inpaint_loss_finalize(sums.data_ptr(), (ctypes.c_double * 16)(*inv), loss.data_ptr(), terms.data_ptr(),
                                                     _stream()))
        ctx.crit, ctx.vgg, ctx.saved_vgg, ctx.feats, ctx.grams, ctx.X = crit, vgg, saved, feats, grams, X
        ctx.raw, ctx.origin, ctx.plane, ctx.output = raw, origin, plane, output
        return loss

    @staticmethod
    def backward(ctx, gloss):
        lib = _lib.load()
        output, vgg = ctx.output, ctx.vgg
        n, _, h, w = output.shape
        code = ops._dtype_code(output)
        gs = gloss.detach().float().contiguous()
        g_next = None
        for s in range(len(ctx.feats) - 1, -1, -1):
            f = ctx.feats[s]
            _, c, hs, ws = f.shape
            gm, g = ctx.grams[s]
            norm = float(c * hs * ws)
            t = torch.empty((2 * n, c, c), dtype=torch.float32, device=f.device)
            with _part("fused"):
                _lib.check(lib.pcb_gram_sign_sym(g.data_ptr(), n, c, norm, t.data_ptr(), _stream()))
            with _part("gram"):
                gg = gm.backward(f, t)
            df = torch.empty((2 * n, c, hs, ws), dtype=f.dtype, device=f.device, memory_format=CL)
            with _part("fused"):
                _lib.check(lib.pcb_feature_loss_backward(f.data_ptr(), code, n, hs * ws, c, ops._ptr(g_next), gg.data_ptr(),
                                                         WEIGHTS[3] / (n * c * hs * ws), WEIGHTS[4] / (n * c * c) / norm, gs.data_ptr(),
                                                         df.data_ptr(), _stream()))
            layers = ctx.saved_vgg[s]
            y_last = layers[-1][2]
            gy = torch.empty((2 * n, c, 2 * hs, 2 * ws), dtype=f.dtype, device=f.device, memory_format=CL)
            with _part("vgg_dgrad"):
                _lib.check(lib.pcb_maxpool2x2_backward(df.data_ptr(), y_last.data_ptr(), gy.data_ptr(), code, 2 * n, 2 * hs, 2 * ws, c, 1,
                                                       _stream()))
                for j in range(len(layers) - 1, -1, -1):
                    conv, x, _, wprep = layers[j]
                    # the input of every convolution but a stage's first is the ReLU output of the one before
                    gy = vgg.dgrad(conv, x, wprep, gy, relu_in=j > 0)
                g_next = gy
        # the gradient in the output's own layout family: NHWC (channel-padded) for NHWC outputs, dense NCHW otherwise
        if ops.nhwc_layout(output) is not None and not output.is_contiguous():
            grad = ops.padded_empty(*output.shape, output.dtype, output.device)
        else:
            grad = torch.empty_like(output)
        coef = (ctypes.c_float * 4)(WEIGHTS[0] / (n * 3 * h * w), WEIGHTS[1] / (n * 3 * h * w), WEIGHTS[2] / (n * 3 * h * (w - 1)),
                                    WEIGHTS[2] / (n * 3 * (h - 1) * w))
        with _part("fused"):
            _lib.check(lib.pcb_inpaint_loss_pixel_backward(ctx.raw.data_ptr(), ctx.origin.data_ptr(), output.data_ptr(), code,
                                                           _strides(output), ctx.plane.data_ptr(), n, h, w, g_next.data_ptr(), code, coef,
                                                           gs.data_ptr(), grad.data_ptr(), _strides(grad), _stream()))
        return None, None, None, None, grad


class InpaintingLoss(nn.Module):
    """loss.py:185-225 on the GPU.  `forward(raw_input, mask, output, origin)`:

    * raw_input, origin: fp32 NCHW [n, 3, h, w] (raw_input = origin * mask in the reference's data path);
    * mask: the reference's {0, 1} [n, 3, h, w] mask (one plane repeated over RGB, 1 = valid) or a `HoleMask`;
    * output: the network output, fp32 NCHW or a bf16 NHWC (channel-padded) view; its dtype is the compute dtype of the VGG pass.

    Returns the scalar loss (device), differentiable w.r.t. `output` only.  `last_terms` holds the five unweighted terms of the
    last call (valid, hole, tv, perceptual, style) as a device fp32 [5] tensor that the next call overwrites."""

    def __init__(self, feature_encoder, feature_range=3):
        super().__init__()
        self.feature_encoder = FeatureExtractor(feature_encoder, feature_range)
        self.last_terms = None

    def _terms_buffer(self, dev):
        if self.last_terms is None or self.last_terms.device != dev:
            self.last_terms = torch.zeros((5,), dtype=torch.float32, device=dev)
        return self.last_terms

    def forward(self, raw_input, mask, output, origin):
        n, c, h, w = output.shape
        if c != 3 or h % 8 or w % 8:
            raise _lib.PcbError(f"InpaintingLoss expects a [n, 3, h, w] output with h, w multiples of 8, got {tuple(output.shape)}")
        if output.dtype not in (torch.float32, torch.bfloat16) or not output.is_cuda:
            raise _lib.PcbError("InpaintingLoss: output must be a CUDA float32 or bfloat16 tensor")
        if not isinstance(mask, HoleMask) and not torch.cuda.is_current_stream_capturing():
            # the kernels take one {0,1} plane per image; outside a graph capture that promise is checked (one device sync)
            m = mask.detach()
            if tuple(m.shape) != (n, 3, h, w) or not bool(((m == 0) | (m == 1)).all()) or not bool((m == m[:, :1]).all()):
                raise ValueError("InpaintingLoss expects a binary [n, 3, h, w] mask with the same plane in every channel")
        hm = mask if isinstance(mask, HoleMask) else HoleMask.from_dense(mask, channel_uniform=True)
        if len(hm.parts) != 1 or hm.parts[0][2] != 0 or tuple(hm.shape[2:]) != (h, w) or hm.shape[0] != n:
            raise _lib.PcbError("InpaintingLoss: the mask must be one hole plane at the output's resolution")
        plane = hm.parts[0][0].contiguous()
        raw = raw_input.detach().float().contiguous()
        origin = origin.detach().float().contiguous()
        if tuple(raw.shape) != (n, 3, h, w) or tuple(origin.shape) != (n, 3, h, w):
            raise _lib.PcbError("InpaintingLoss: raw_input and origin must be [n, 3, h, w] like output")
        return _InpaintingLossFn.apply(self, raw, origin, plane, output)


def gram_matrix(feat):
    """loss.py:294-300 on the GPU (no gradient): F F^T / (c h w) per image, fp32 [b, c, c]."""
    f = ops.as_feature(feat.detach())
    b, c, h, w = f.shape
    return _Gram(f).products(f) / float(c * h * w)


def total_variation_loss(image):
    """loss.py:303-307 on the GPU (no gradient): mean |horizontal differences| + mean |vertical differences| of a 3-channel
    image (the pixel kernel with every pixel valid, so the composite is the image itself)."""
    lib = _lib.load()
    n, c, h, w = image.shape
    if c != 3:
        raise _lib.PcbError("total_variation_loss: 3-channel images only")
    img = image.detach().float().contiguous()
    plane = torch.ones((n, h, w), dtype=torch.uint8, device=img.device)
    X = ops.padded_empty(3 * n, 3, h, w, torch.float32, img.device)
    sums = torch.zeros((16,), dtype=torch.float64, device=img.device)
    _lib.check(lib.pcb_inpaint_loss_pixel_forward(img.data_ptr(), img.data_ptr(), img.data_ptr(), ops._dtype_code(img), _strides(img),
                                                  plane.data_ptr(), n, h, w, X.data_ptr(), ops._dtype_code(img), sums.data_ptr(), _stream()))
    return (sums[2] / (n * 3 * h * (w - 1)) + sums[3] / (n * 3 * (h - 1) * w)).float()


# ------------------------------------------------------------------------------------------------------------------------------
# segmentation losses (loss.py:58-121)
# ------------------------------------------------------------------------------------------------------------------------------
class _SegLossFn(torch.autograd.Function):
    """One forward and one backward launch of csrc/seg_loss.cu over [n, 1, h, w] logits read in place through their strides."""

    @staticmethod
    def forward(ctx, crit, x, target):
        lib = _lib.load()
        n, _, h, w = x.shape
        count = n * h * w
        ws = crit._workspace(x.device, count)
        out = torch.empty((count, 1) if crit._reduction == _lib.SEG_NONE else (), dtype=torch.float32, device=x.device)
        _lib.check(lib.pcb_seg_loss_forward(x.data_ptr(), ops._dtype_code(x), _strides(x), target.data_ptr(), n, h, w, crit._kind,
                                            crit._reduction, *crit._coefs(), ws[0].data_ptr(), ws[1].data_ptr(), out.data_ptr(), _stream()))
        ctx.crit = crit
        ctx.save_for_backward(x, target)
        return out

    @staticmethod
    def backward(ctx, gout):
        lib = _lib.load()
        x, target = ctx.saved_tensors
        crit = ctx.crit
        n, _, h, w = x.shape
        g = gout.detach().float().contiguous()
        # the gradient in the input's own layout family: NHWC (channel-padded) for NHWC views, dense otherwise
        if ops.nhwc_layout(x) is not None and not x.is_contiguous():
            dx = ops.padded_empty(*x.shape, x.dtype, x.device)
        else:
            dx = torch.empty_like(x)
        _lib.check(lib.pcb_seg_loss_backward(x.data_ptr(), ops._dtype_code(x), _strides(x), target.data_ptr(), n, h, w, crit._kind,
                                             crit._reduction, *crit._coefs(), g.data_ptr(), dx.data_ptr(), _strides(dx), _stream()))
        return None, dx, None


class _SegLoss(nn.Module):
    """Shared plumbing: input checks and the device workspace of the deterministic reduction."""

    _kind = _lib.SEG_FOCAL
    _reduction = _lib.SEG_MEAN

    def _coefs(self):
        raise NotImplementedError

    def _workspace(self, dev, count):
        """(fp64 partials, uint32 counter): the counter is zeroed once here and left zero by every forward launch."""
        key = (str(dev), _lib.load().pcb_seg_loss_partials(count))
        ws = self.__dict__.get("_pcb_ws")
        if ws is None or ws[0] != key:
            if torch.cuda.is_current_stream_capturing():
                raise _lib.PcbError(f"{type(self).__name__}: run the loss once before capturing it for this input size")
            ws = (key, (torch.empty((key[1],), dtype=torch.float64, device=dev), torch.zeros((1,), dtype=torch.int32, device=dev)))
            self.__dict__["_pcb_ws"] = ws
        return ws[1]

    def forward(self, input, target):
        assert input.dim() == 4 and input.size(1) == 1          # the reference's flatten_images assertion
        assert target.dim() == 4 and target.size(1) == 1
        if not input.is_cuda or input.dtype not in (torch.float32, torch.bfloat16):
            raise _lib.PcbError(f"{type(self).__name__}: input must be a CUDA float32 or bfloat16 tensor")
        if tuple(target.shape) != tuple(input.shape):
            raise _lib.PcbError(f"{type(self).__name__}: target {tuple(target.shape)} does not match input {tuple(input.shape)}")
        t = target.detach()
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.float().contiguous()
        return _SegLossFn.apply(self, input, t)


class BinaryFocalLoss(_SegLoss):
    """loss.py:58-83 on the GPU: mean(exp(gamma * logsigmoid(-x (2t - 1))) * w * bce(x, t)), w = words_weights where t > 0,
    background_weights elsewhere.  `input`: [n, 1, h, w] logits, fp32 or bf16, dense or the channel-padded NHWC view the
    segmentation networks return (read in place); `target`: [n, 1, h, w] in [0, 1].  Returns the fp32 scalar loss (device);
    the gradient goes to `input` only, through pt as well when gamma != 0."""

    def __init__(self, gamma=0, background_weights=1, words_weights=2):
        super().__init__()
        self.gamma = gamma
        self.background_weights = background_weights
        self.words_weights = words_weights

    def _coefs(self):
        return float(self.gamma), 0.0, float(self.background_weights), float(self.words_weights)


class SoftBootstrapCrossEntropy(_SegLoss):
    """loss.py:86-121 on the GPU: w * bce(x, beta t + (1 - beta) [sigmoid(x) > 0.5]) reduced by mean (default), sum
    (`size_average=False`) or not at all (`reduce=False`: fp32 [n*h*w, 1]).  The indicator carries no gradient; it equals
    torch's CPU float32 `sigmoid(x) > 0.5` for every input value.  Inputs as for BinaryFocalLoss."""

    _kind = _lib.SEG_BOOTSTRAP

    def __init__(self, beta=0.95, background_weight=1, words_weight=2, size_average=True, reduce=True):
        super().__init__()
        self.beta = beta
        self.background_weight = background_weight
        self.words_weight = words_weight
        self.size_average = size_average
        self.reduce = reduce

    @property
    def _reduction(self):
        if self.reduce is not None and not self.reduce:
            return _lib.SEG_NONE
        return _lib.SEG_SUM if self.size_average is not None and not self.size_average else _lib.SEG_MEAN

    def _coefs(self):
        return float(self.beta), float(1 - self.beta), float(self.background_weight), float(self.words_weight)

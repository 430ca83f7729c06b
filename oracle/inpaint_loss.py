"""Functional torch-CPU restatement of the reference's inpainting loss -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

`InpaintingLoss(VggExtractor(), feature_range=3).forward(raw_input, mask, output, origin)` (loss.py:185-225, 244-260,
294-307) as pure functions over tensors and a VGG `state_dict` with the reference's keys (`features.<stage>.<idx>.weight`),
the same ATen ops in the same order.  Pinned bit for bit to tests/golden/inpaint_loss_*.npz, which the reference's own
module produced.

`oracle.pconv_torch.storage(torch.bfloat16)` also applies here: it rounds where the CUDA path hands tensors from kernel to
kernel -- the three VGG input images, every stored feature map (ReLU outputs; the max-pool of bf16 values is exact), the
gradient of every convolution input (data-gradient output) and the gradient arriving at each stage output (perceptual +
style + next stage, summed once).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.pconv_torch import _rb, _rf

# (stage, index inside the stage, in channels, out channels) of the 3x3 convolutions of vgg16.features[:17]
VGG_CONVS = ((0, 0, 3, 64), (0, 2, 64, 64), (1, 0, 64, 128), (1, 2, 128, 128), (2, 0, 128, 256), (2, 2, 256, 256), (2, 4, 256, 256))
STAGE_CONVS = ((0, 2), (0, 2), (0, 2, 4))
WEIGHTS = {"valid": 1.0, "hole": 6.0, "tv": 0.1, "perceptual": 0.05, "style": 120.0}
TERMS = ("valid", "hole", "tv", "perceptual", "style")


def vgg_state_dict(seed=0):
    """Seeded VGG16 feature weights with the reference's `VggExtractor` keys: He-scaled normal weights and non-zero biases
    (torchvision's zero biases would leave the bias path untested).  Shared by the golden generator and the tests."""
    rng = np.random.default_rng(seed)
    sd = {}
    for st, i, cin, cout in VGG_CONVS:
        w = rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (cin * 9))
        b = rng.uniform(-0.05, 0.05, cout)
        sd[f"features.{st}.{i}.weight"] = torch.from_numpy(w.astype(np.float32))
        sd[f"features.{st}.{i}.bias"] = torch.from_numpy(b.astype(np.float32))
    return sd


def vgg_features(x, sd):
    """VggExtractor.forward (loss.py:255-260): the three stage outputs, conv3x3 + bias -> ReLU blocks, each stage ending in a
    2x2/2 max-pool.  No input normalisation (loss.py:192-193 is commented out)."""
    out = []
    x = _rf(x)
    for st, idxs in enumerate(STAGE_CONVS):
        for i in idxs:
            x = _rb(x)
            x = _rf(F.relu(F.conv2d(x, sd[f"features.{st}.{i}.weight"], sd[f"features.{st}.{i}.bias"], 1, 1, 1, 1)))
        x = _rb(F.max_pool2d(x, 2, 2, 0, 1, False, False))
        out.append(x)
    return out


def gram_matrix(feat):
    """loss.py:294-300."""
    b, ch, h, w = feat.size()
    feat = feat.view(b, ch, h * w)
    return torch.bmm(feat, feat.transpose(1, 2)) / (ch * h * w)


def total_variation_loss(image):
    """loss.py:303-307."""
    return torch.mean(torch.abs(image[:, :, :, :-1] - image[:, :, :, 1:])) + \
        torch.mean(torch.abs(image[:, :, :-1, :] - image[:, :, 1:, :]))


def inpainting_loss_terms(raw_input, mask, output, origin, sd):
    """The five unweighted terms of InpaintingLoss.forward (loss.py:195-225) in the reference's order, as a dict."""
    comp = mask * raw_input + (1 - mask) * output
    valid = F.l1_loss(mask * output, mask * origin)
    hole = F.l1_loss((1 - mask) * output, (1 - mask) * origin)
    tv = total_variation_loss(comp)
    f_comp = vgg_features(comp, sd)
    f_out = vgg_features(output, sd)
    f_orig = vgg_features(origin, sd)
    p1 = sum(map(lambda x, y: F.l1_loss(x, y), f_comp, f_orig))
    p2 = sum(map(lambda x, y: F.l1_loss(x, y), f_out, f_orig))
    s1 = sum(map(lambda x, y: F.l1_loss(gram_matrix(x), gram_matrix(y)), f_out, f_orig))
    s2 = sum(map(lambda x, y: F.l1_loss(gram_matrix(x), gram_matrix(y)), f_comp, f_orig))
    return {"valid": valid, "hole": hole, "tv": tv, "perceptual": p1 + p2, "style": s1 + s2}


def combine(terms):
    """loss.py:223-224: 1 valid + 6 hole + 0.1 tv + 0.05 perceptual + 120 style, in that order."""
    return 1.0 * terms["valid"] + 6.0 * terms["hole"] + 0.1 * terms["tv"] + 0.05 * terms["perceptual"] + 120 * terms["style"]


def inpainting_loss(raw_input, mask, output, origin, sd):
    return combine(inpainting_loss_terms(raw_input, mask, output, origin, sd))

"""Generate the committed golden fixtures by running the UNMODIFIED reference on CPU.

Needs a checkout of the reference ($PCB_REFERENCE, default /root/reference); the tests only read the fixtures it writes:

    python tests/golden/make_golden.py

Writes tests/golden/*.npz.  Every fixture stores the inputs, the (deterministic) parameters
or the recipe to regenerate them (oracle/detfill.py), and the reference's outputs.
The reference has no tests / golden vectors of its own (SURVEY 4), so these are the pins.
"""
import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("PCB_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from oracle.detfill import det_fill_state_dict, det_tensor  # noqa: E402
from oracle.masks import random_hole_masks  # noqa: E402

import models.partial_convolution as rpc  # noqa: E402  (the reference)
import models.image_inpainting as rii  # noqa: E402

torch.set_num_threads(8)


def blob_mask(n, c, h, w, seed, per_channel=False):
    """{0,1} masks with rectangular + diagonal-band holes big enough to survive a 3x3 layer."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = np.ones((n, c, h, w), np.float32)
    for i in range(n):
        for ch in range(c if per_channel else 1):
            for _ in range(2):
                y0, x0 = rng.integers(0, h - 3), rng.integers(0, w - 3)
                hh, ww = rng.integers(3, max(4, h // 2)), rng.integers(3, max(4, w // 2))
                if per_channel:
                    m[i, ch, y0:y0 + hh, x0:x0 + ww] = 0
                else:
                    m[i, :, y0:y0 + hh, x0:x0 + ww] = 0
    return m


def save(name, **arrs):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
                                 for k, v in arrs.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


L1_CASES = [
    # name, cls, cin, cout, k, s, p, d, groups, bias, same_holes, (n,h,w), per_channel_mask
    ("pc_k3_blob",        "pc", 4, 6, 3, 1, 1, 1, 1, True,  False, (2, 20, 24), False),
    ("pc_k3_same_holes",  "pc", 4, 6, 3, 1, 1, 1, 1, True,  True,  (2, 20, 24), False),
    ("pc_k3_perchannel",  "pc", 4, 6, 3, 1, 1, 1, 1, False, False, (2, 20, 24), True),
    ("pc_k5_s2",          "pc", 8, 8, 5, 2, 2, 1, 1, False, True,  (2, 21, 26), False),
    ("pc_k7_s2_stem",     "pc", 3, 8, 7, 2, 3, 1, 1, True,  True,  (2, 32, 32), False),
    ("pc_k3_d2",          "pc", 4, 4, 3, 1, 2, 2, 1, False, False, (1, 24, 24), False),
    ("pc_k3_d4",          "pc", 4, 4, 3, 1, 4, 4, 1, True,  True,  (1, 24, 24), False),
    ("pc_k3_d8_s1",       "pc", 2, 4, 3, 1, 8, 8, 1, False, False, (1, 28, 28), True),
    ("pc_dw_same_holes",  "pc", 8, 8, 3, 1, 1, 1, 8, False, True,  (2, 16, 16), False),
    ("pc_dw_s2_d1",       "pc", 8, 8, 3, 2, 1, 1, 8, False, True,  (2, 17, 19), False),
    ("pc_groups2",        "pc", 4, 6, 3, 1, 1, 1, 2, True,  False, (1, 12, 12), True),
    ("pc_nopad",          "pc", 3, 5, 3, 1, 0, 1, 1, True,  False, (1, 10, 12), False),
    ("pc_1x1",            "1x1", 4, 8, 1, 1, 0, 1, 1, True, False, (2, 12, 12), False),
    ("pc_noholes_1x1",    "nh", 6, 4, 1, 1, 0, 1, 1, False, False, (2, 12, 12), True),
    ("pc_noholes_k3_nan", "nh", 4, 4, 3, 1, 1, 1, 1, True,  False, (1, 16, 16), False),
]


def gen_l1():
    for (name, cls, cin, cout, k, s, p, d, g, bias, sh, (n, h, w), pcm) in L1_CASES:
        if cls == "pc":
            m = rpc.PartialConv(cin, cout, k, s, p, d, g, bias, sh)
        elif cls == "1x1":
            m = rpc.PartialConv1x1(cin, cout, k, s, p, d, g, bias)
        else:
            m = rpc.PartialConvNoHoles(cin, cout, k, s, p, d, g, bias)
        m.load_state_dict(det_fill_state_dict(m.state_dict()))
        x = det_tensor(name + ".x", (n, cin, h, w))
        mask = torch.from_numpy(blob_mask(n, cin, h, w, seed=len(name) * 131 + k, per_channel=pcm))
        if name == "pc_noholes_1x1":        # the decoder case: every pixel valid in >=1 channel
            mask[:, 0] = 1.0
        x.requires_grad_(True)
        y, nm = m((x, mask))
        gy = det_tensor(name + ".gy", tuple(y.shape))
        finite = torch.isfinite(y)
        (torch.where(finite, y, torch.zeros_like(y)) * gy).sum().backward()
        out = dict(x=x.detach(), mask=mask, y=y, new_mask=nm.contiguous(), gy=gy, gx=x.grad,
                   gw=m.feature_conv.weight.grad,
                   cfg=np.array([cin, cout, k, s, p, d, g, int(bias), int(sh)], np.int64))
        if bias:
            out["gb"] = m.feature_conv.bias.grad
        for kk, vv in m.state_dict().items():
            out["sd." + kk] = vv
        save(name, **out)


def gen_block_bn():
    """partial_convolution_block with BN + LeakyReLU, two training steps then one eval step
    (running-stat update, SURVEY 8c item 7)."""
    blk = rpc.partial_convolution_block(4, 8, 3, 2, 1, 1, bias=False, BN=True,
                                        activation=nn.LeakyReLU(0.2), same_holes=True)
    blk.load_state_dict(det_fill_state_dict(blk.state_dict()))
    sd0 = {k: v.clone() for k, v in blk.state_dict().items()}
    x = det_tensor("blk.x", (3, 4, 18, 18)); mask = torch.from_numpy(blob_mask(3, 4, 18, 18, 5))
    blk.train()
    x.requires_grad_(True)
    y1, m1 = blk((x, mask))
    gy = det_tensor("blk.gy", tuple(y1.shape))
    (y1 * gy).sum().backward()
    grads = {"g." + k: p.grad for k, p in blk.named_parameters() if p.grad is not None}
    gx = x.grad.clone()
    y2, _ = blk((x.detach() * 0.5 + 0.25, mask))
    sd2 = {k: v.clone() for k, v in blk.state_dict().items()}
    blk.eval()
    y3, _ = blk((x.detach(), mask))
    save("block_bn_leaky", x=x.detach(), mask=mask, y1=y1, m1=m1.contiguous(), gy=gy, gx=gx, y2=y2, y3=y3,
         **{"sd0." + k: v for k, v in sd0.items()}, **{"sd2." + k: v for k, v in sd2.items()}, **grads)


def gen_upsample():
    up = rpc.DoubleUpSample(scale_factor=2, mode="nearest")
    x = det_tensor("up.x", (2, 3, 5, 7)); mask = torch.from_numpy(blob_mask(2, 3, 5, 7, 9))
    xu, mu = up((x, mask))
    save("double_upsample", x=x, mask=mask, xu=xu, mu=mu)


def sub(t, step=8):
    return t[..., ::step, ::step].contiguous()


def gen_network(cls_name, n, hw, grad_keys, step=8, tag=""):
    """End-to-end U-Net: det-filled weights (regenerable from names), seeded blob/line masks,
    train-mode fwd + bwd of loss = out.abs().mean() (SURVEY 8d)."""
    net = getattr(rii, cls_name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net.train()
    x = det_tensor(cls_name + ".x", (n, 3, hw, hw))
    mask = torch.from_numpy(random_hole_masks(n, hw, hw, seed=11))
    out = net((x * mask, mask))                               # Dataloader.py:131 feeds (x*mask, mask)
    loss = out.abs().mean()
    loss.backward()
    params = dict(net.named_parameters())
    sd = net.state_dict()
    bn_keys = [k for k in sd if k.endswith("running_mean") or k.endswith("running_var")]
    save("net_" + cls_name + tag,
         mask_bits=np.packbits(mask[:, 0].numpy().astype(np.uint8)), n=n, hw=hw, step=step,
         out_sub=sub(out, step), out_sum=out.double().sum(), out_abs_sum=out.double().abs().sum(),
         loss=loss, out_row=out[0, :, hw // 2, :],
         **{"g." + k: params[k].grad for k in grad_keys},
         **{"gsum." + k: p.grad.double().abs().sum() for k, p in params.items() if p.grad is not None},
         **{"bn." + k: sd[k] for k in bn_keys[:6] + bn_keys[-4:]})


if __name__ == "__main__":
    torch.set_num_threads(8)          # the count the oracle tests replay with (test_oracle_golden.GOLDEN_THREADS)
    gen_l1()
    gen_block_bn()
    gen_upsample()
    gen_network("ImageFillOrigin", 2, 256,
                ["encoder.0.0.feature_conv.weight", "encoder.0.0.feature_conv.bias",
                 "decoder.7.0.feature_conv.weight", "decoder.6.0.1.bn_act.0.weight",
                 "decoder.6.0.1.bn_act.0.bias", "encoder.7.0.1.bn_act.0.weight"])
    gen_network("ImageFillOriginV2", 2, 256, ["decoder.7.0.feature_conv.weight"])
    gen_network("ImageFill", 2, 128, ["decoder.3.0.feature_conv.weight"])
    # the BENCHMARKED resolution (BASELINE.json configs[2]: 512x512): selects the widest N tiles, row-halo tiles on every
    # full-resolution decoder layer and the concurrent parity-class data gradients that 256x256 never reaches
    gen_network("ImageFillOrigin", 2, 512,
                ["encoder.0.0.feature_conv.weight", "decoder.7.0.feature_conv.weight", "decoder.6.0.0.feature_conv.weight",
                 "decoder.6.0.1.bn_act.0.weight", "decoder.4.0.1.bn_act.0.bias", "encoder.2.0.1.bn_act.0.weight"], step=16, tag="_512")


def gen_state_dict_keys():
    import json
    out = {n: [[k, list(v.shape)] for k, v in getattr(rii, n)().state_dict().items()]
           for n in ("ImageFillOrigin", "ImageFillOriginV2", "ImageFill")}
    json.dump(out, open(os.path.join(HERE, "state_dict_keys.json"), "w"))


if __name__ == "__main__":
    gen_state_dict_keys()

"""Golden fixtures for the dense segmentation path, produced by the UNMODIFIED reference on CPU
(build container only):  python tests/golden/make_golden_seg.py"""
import json
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

import models.BaseModels as rbm  # noqa: E402  (the reference)
import models.MobileNetV2 as rmb  # noqa: E402
import models.common as rcm  # noqa: E402
import models.text_segmentation as rts  # noqa: E402

torch.set_num_threads(8)


def save(name, **arrs):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in arrs.items()})
    print(f"{name}: {os.path.getsize(path) / 1024:.1f} KiB")


def run_block(name, mod, x, grads_of=()):
    mod.load_state_dict(det_fill_state_dict(mod.state_dict()))
    mod.train()
    x = x.clone().requires_grad_(True)
    y = mod(x)
    gy = det_tensor(name + ".gy", tuple(y.shape))
    (y * gy).sum().backward()
    sd_after = {k: v.clone() for k, v in mod.state_dict().items() if "running_" in k}
    params = dict(mod.named_parameters())
    save("seg_" + name, x=x.detach(), y=y, gy=gy, gx=x.grad, **{"g." + k: params[k].grad for k in grads_of},
         **{"bn." + k: v for k, v in list(sd_after.items())[:4]})


def gen_blocks():
    act = nn.LeakyReLU(0.3)
    run_block("dsconv_s2", rbm.DSConvBlock(16, 24, 3, 2, 1, 1, False, True, act, act), det_tensor("dsconv.x", (2, 16, 17, 19)),
              ["depth_wise_conv.0.weight", "point_wise_conv.0.weight", "depth_wise_conv.1.0.weight"])
    run_block("dsconv_d4", rbm.DSConvBlock(16, 16, 3, 1, 4, 4, False, True, act, None), det_tensor("dsconv4.x", (1, 16, 20, 20)),
              ["depth_wise_conv.0.weight", "point_wise_conv.0.weight"])
    run_block("invres_scse", rmb.InvertedResidual(16, 16, 1, 6, 2, activation=act, bias=False, add_sece=True), det_tensor("ir.x", (2, 16, 14, 14)),
              ["conv.0.weight", "conv.2.weight", "conv.4.weight", "conv.6.channel_excite.0.weight", "conv.6.spatial_excite.0.weight", "conv.5.0.weight"])
    run_block("invres_s2", rmb.InvertedResidual(16, 24, 2, 6, 1, activation=act, bias=False, add_sece=False), det_tensor("ir2.x", (2, 16, 15, 15)),
              ["conv.0.weight", "conv.2.weight", "conv.4.weight"])
    run_block("scse", rcm.SpatialChannelSqueezeExcitation(32, reduction=16, activation=act), det_tensor("scse.x", (3, 32, 9, 7)),
              ["channel_excite.0.weight", "channel_excite.2.bias", "spatial_excite.0.weight"])
    run_block("rfb", rcm.RFB(40, 16, activation=act, add_sece=True), det_tensor("rfb.x", (2, 40, 12, 12)),
              ["rfb.0.0.weight", "rfb.0.2.weight", "rfb.3.2.weight", "rfb.3.4.weight", "rfb.3.6.weight", "rfb_linear_conv.0.weight",
               "rfb_linear_conv.0.bias", "input_down_channel.0.weight"])
    run_block("asp", rcm.ASP(24, 16, act, asp_rate=(3, 5, 9)), det_tensor("asp.x", (2, 24, 14, 14)),
              ["asp.0.0.weight", "asp.2.1.weight", "out_conv.0.weight"])
    pool = nn.AvgPool2d(kernel_size=3, stride=2, padding=1)
    xp = det_tensor("pool.x", (2, 8, 9, 11)).requires_grad_(True)
    yp = pool(xp); gyp = det_tensor("pool.gy", tuple(yp.shape)); (yp * gyp).sum().backward()
    xb = det_tensor("bil.x", (2, 8, 5, 7)).requires_grad_(True)
    outs = {}
    for s in (2, 4):
        xb.grad = None
        yb = torch.nn.functional.interpolate(xb, scale_factor=s, mode="bilinear", align_corners=False)
        gyb = det_tensor(f"bil{s}.gy", tuple(yb.shape)); (yb * gyb).sum().backward()
        outs[f"y{s}"] = yb.detach(); outs[f"gy{s}"] = gyb; outs[f"gx{s}"] = xb.grad.clone()
    save("seg_pool_bilinear", xp=xp.detach(), yp=yp, gyp=gyp, gxp=xp.grad, xb=xb.detach(), **outs)


def gen_network(cls_name, n, hw, grad_keys, step=4, tag=""):
    net = getattr(rts, cls_name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net.train()
    x = det_tensor(cls_name + ".x", (n, 3, hw, hw))
    out = net(x)
    loss = out.abs().mean()
    loss.backward()
    params = dict(net.named_parameters())
    sd = net.state_dict()
    bn_keys = [k for k in sd if k.endswith("running_mean") or k.endswith("running_var")]
    save("segnet_" + cls_name + tag, n=n, hw=hw, step=step, out_sub=out[..., ::step, ::step].contiguous(), loss=loss,
         out_row=out[0, :, hw // 2, :], **{"g." + k: params[k].grad for k in grad_keys},
         **{"bn." + k: sd[k] for k in bn_keys[:4] + bn_keys[-2:]})
    keys = [[k, list(v.shape)] for k, v in sd.items()]
    return keys


if __name__ == "__main__":
    torch.set_num_threads(8)          # the count the oracle tests replay with (test_oracle_golden_seg.GOLDEN_THREADS)
    gen_blocks()
    keys = {}
    keys["TextSegament"] = gen_network("TextSegament", 2, 64, ["out_conv.0.weight", "feature_pooling.rfb_linear_conv.0.weight",
                                                               "encoder.features.0.0.weight", "smooth_feature_4x_conv.1.conv.2.weight"])
    keys["XceptionTextSegment"] = gen_network("XceptionTextSegment", 2, 64, ["out_conv.2.weight", "feature_pooling.out_conv.0.weight",
                                                                             "encoder.entry_flow_1.0.weight", "encoder.exit_flow.3.conv.2.depth_wise_conv.0.weight"])
    # 256x256: the 1/8-resolution maps are 32x32, so RFB's dilation-17/29 branches and the d = 8/16 stages see real taps
    # (at 64x64 input they only ever see padding)
    gen_network("TextSegament", 2, 256, ["out_conv.0.weight", "feature_pooling.rfb_linear_conv.0.weight",
                                         "encoder.features.0.0.weight", "smooth_feature_4x_conv.1.conv.2.weight"], step=8, tag="_256")
    gen_network("XceptionTextSegment", 2, 256, ["out_conv.2.weight", "feature_pooling.out_conv.0.weight",
                                                "encoder.entry_flow_1.0.weight", "encoder.exit_flow.3.conv.2.depth_wise_conv.0.weight"],
                step=8, tag="_256")
    path = os.path.join(HERE, "state_dict_keys.json")
    allk = json.load(open(path))
    allk.update(keys)
    json.dump(allk, open(path, "w"))

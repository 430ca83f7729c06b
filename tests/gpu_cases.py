"""Shared GPU parity helpers (used by tests/test_gpu_parity.py and tools/gpu_diag.py).

Every case runs a module of the product package on cuda:0 through the C ABI and compares with the torch-CPU
oracle evaluated on the SAME dtype-rounded operands (so the bf16 tolerance below measures the kernel, not
the input quantisation):
  * fp32 mode  : 1e-4 relative to max|ref|   (north_star bar: 1e-3 relative fp32)
  * bf16 mode  : 2e-2 relative to max|ref|   (outputs/grads are stored in bf16: 2^-8 relative rounding on
                 top of fp32 accumulation; weight gradients are fp32 and typically 1e-3)
  * new masks  : bit-exact always.
"""
import os

import numpy as np
import torch

from oracle import pconv_torch as O
from oracle.detfill import det_fill_state_dict, det_tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = {torch.float32: 1e-4, torch.bfloat16: 2e-2}


def blob(n, c, h, w, seed, per_channel=False):
    rng = np.random.Generator(np.random.PCG64(seed))
    m = np.ones((n, c, h, w), np.float32)
    for i in range(n):
        for ch in range(c if per_channel else 1):
            for _ in range(2):
                y0, x0 = rng.integers(0, max(1, h - 3)), rng.integers(0, max(1, w - 3))
                hh, ww = rng.integers(2, max(3, h // 2)), rng.integers(2, max(3, w // 2))
                if per_channel:
                    m[i, ch, y0:y0 + hh, x0:x0 + ww] = 0
                else:
                    m[i, :, y0:y0 + hh, x0:x0 + ww] = 0
    return torch.from_numpy(m)


def relerr(a, b):
    a = a.detach().float().cpu(); b = b.detach().float().cpu()
    fin = torch.isfinite(b)
    if not torch.equal(torch.isfinite(a), fin):
        return float("inf")
    if not fin.any():
        return 0.0
    return (a[fin] - b[fin]).abs().max().item() / max(b[fin].abs().max().item(), 1e-20)


def rel_l2(a, b, floor=1e-20):
    """||a - b||_2 / ||b||_2 -- the robust metric for bf16 tensors downstream of ReLU/LeakyReLU derivatives: a
    pre-activation within one bf16 ulp of zero flips the derivative of that ELEMENT (an O(1) error at isolated
    elements that max-abs metrics report as failure although the tensor agrees to a few percent in norm)."""
    a = a.detach().float().cpu(); b = b.detach().float().cpu()
    return float((a - b).norm() / b.norm().clamp_min(floor))


# name: (cin, cout, k, s, p, d, groups, bias, same_holes, n, h, w, dtype, mask_kind, cls)
#   mask_kind: "uniform" (one plane over all channels), "perchannel" (<= 8 channels), "two" (two planes split cin/2)
F32, BF = torch.float32, torch.bfloat16
CONV_CASES = {
    # ---- shape-general kernels, exact fp32 mode (mirrors of the committed reference goldens)
    "g_k3": (4, 6, 3, 1, 1, 1, 1, True, False, 2, 20, 24, F32, "uniform", "pc"),
    "g_k3_sh": (4, 6, 3, 1, 1, 1, 1, True, True, 2, 20, 24, F32, "uniform", "pc"),
    "g_k3_perchannel": (4, 6, 3, 1, 1, 1, 1, False, False, 2, 20, 24, F32, "perchannel", "pc"),
    "g_k5_s2": (8, 8, 5, 2, 2, 1, 1, False, True, 2, 21, 26, F32, "uniform", "pc"),
    "g_k7_s2_stem": (3, 8, 7, 2, 3, 1, 1, True, True, 2, 32, 32, F32, "uniform", "pc"),
    "g_d2": (4, 4, 3, 1, 2, 2, 1, False, False, 1, 24, 24, F32, "uniform", "pc"),
    "g_d4_sh": (4, 4, 3, 1, 4, 4, 1, True, True, 1, 24, 24, F32, "uniform", "pc"),
    "g_d8": (2, 4, 3, 1, 8, 8, 1, False, False, 1, 28, 28, F32, "perchannel", "pc"),
    "g_dw_sh": (8, 8, 3, 1, 1, 1, 8, False, True, 2, 16, 16, F32, "uniform", "pc"),
    "g_dw_s2": (8, 8, 3, 2, 1, 1, 8, False, True, 2, 17, 19, F32, "uniform", "pc"),
    "g_groups2": (4, 6, 3, 1, 1, 1, 2, True, False, 1, 12, 12, F32, "perchannel", "pc"),
    "g_nopad": (3, 5, 3, 1, 0, 1, 1, True, False, 1, 10, 12, F32, "uniform", "pc"),
    "g_1x1": (4, 8, 1, 1, 0, 1, 1, True, False, 2, 12, 12, F32, "uniform", "1x1"),
    "g_nh_1x1": (6, 4, 1, 1, 0, 1, 1, False, False, 2, 12, 12, F32, "nh", "nh"),
    "g_nh_k3_nan": (4, 4, 3, 1, 1, 1, 1, True, False, 1, 16, 16, F32, "uniform", "nh"),
    "g_tail_67_3": (67, 3, 3, 1, 1, 1, 1, True, False, 1, 16, 16, F32, "uniform", "pc"),
    "g_bf16_k3": (8, 8, 3, 1, 1, 1, 1, True, False, 2, 12, 12, BF, "uniform", "pc"),
    "g_bf16_dw": (16, 16, 3, 1, 2, 2, 16, False, True, 2, 12, 12, BF, "uniform", "pc"),
    # ---- tensor-core path (bf16, channels % 64 == 0)
    "tc_1x1_k64_n64": (64, 64, 1, 1, 0, 1, 1, False, False, 1, 16, 16, BF, "uniform", "1x1"),
    "tc_1x1_k128_n128": (128, 128, 1, 1, 0, 1, 1, True, False, 1, 16, 16, BF, "uniform", "1x1"),
    "tc_1x1_k256_n64_ragged_m": (256, 64, 1, 1, 0, 1, 1, True, False, 2, 12, 13, BF, "uniform", "1x1"),
    "tc_k3_64_64": (64, 64, 3, 1, 1, 1, 1, True, False, 1, 16, 16, BF, "uniform", "pc"),
    "tc_k3_64_128_sh": (64, 128, 3, 1, 1, 1, 1, False, True, 2, 20, 24, BF, "uniform", "pc"),
    "tc_k3_128_64_two": (128, 64, 3, 1, 1, 1, 1, True, False, 2, 20, 24, BF, "two", "pc"),
    "tc_k5_s2_64_128": (64, 128, 5, 2, 2, 1, 1, False, True, 2, 21, 26, BF, "uniform", "pc"),
    "tc_k3_s2_128_256": (128, 256, 3, 2, 1, 1, 1, False, True, 2, 18, 18, BF, "uniform", "pc"),
    "tc_k3_d2_64_64": (64, 64, 3, 1, 2, 2, 1, False, False, 1, 24, 24, BF, "uniform", "pc"),
    "tc_nh_1x1_128_64_two": (128, 64, 1, 1, 0, 1, 1, False, False, 2, 12, 12, BF, "nh2", "nh"),
    "tc_k3_192_64_two": (192, 64, 3, 1, 1, 1, 1, False, False, 1, 32, 32, BF, "two", "pc"),
    "tc_k3_512_512_tiny": (512, 512, 3, 2, 1, 1, 1, False, True, 2, 4, 4, BF, "uniform", "pc"),
    "tc_k3_320_64_two_odd_split": (320, 64, 3, 1, 1, 1, 1, False, False, 1, 16, 16, BF, "two64", "pc"),
    # ---- channel padding / small-Cin row-packed mode (x lives in an 8-channel-padded NHWC buffer)
    "tc_stem_rowpack_k7_s2": (3, 64, 7, 2, 3, 1, 1, True, True, 2, 40, 44, BF, "uniform3", "pc"),
    # the same stem on a power-of-two grid: its space-to-depth 4x4 problem (conv_stem.cu) runs on the TMA-fed row-halo kernels
    "tc_stem_s2d_k7_s2_tma": (3, 64, 7, 2, 3, 1, 1, True, True, 2, 64, 512, BF, "uniform3", "pc"),
    "tc_rowpack_k3_cin8": (8, 32, 3, 1, 1, 1, 1, False, False, 1, 20, 20, BF, "uniform", "pc"),
    "tc_rowpack_k5_d2_cin4": (4, 128, 5, 1, 4, 2, 1, True, False, 1, 24, 24, BF, "uniform", "pc"),
    "tc_cin72_padded_kblock": (72, 64, 3, 1, 1, 1, 1, True, False, 1, 16, 16, BF, "uniform", "pc"),
    "tc_cout24_padded_n": (64, 24, 3, 1, 1, 1, 1, True, False, 1, 16, 16, BF, "uniform", "pc"),
    "tc_cout3_tail_like": (64, 3, 3, 1, 1, 1, 1, True, False, 2, 16, 16, BF, "uniform", "pc"),
    # ---- TMA-fed path (power-of-two pixel grids): row-halo tiles (w >= 128, stride 1), traversal stride 2, boxes spanning
    #      image rows / several images, N tiles of 32 and 256
    "tma_halo_k3_64_64": (64, 64, 3, 1, 1, 1, 1, True, False, 1, 8, 128, BF, "uniform", "pc"),
    "tma_halo_k3_d2_64_128_w256": (64, 128, 3, 1, 2, 2, 1, False, False, 1, 6, 256, BF, "uniform", "pc"),
    "tma_halo_k5_72_3_n32": (72, 3, 5, 1, 2, 1, 1, True, False, 1, 6, 128, BF, "uniform", "pc"),
    "tma_halo_k3_192_64_two": (192, 64, 3, 1, 1, 1, 1, False, False, 2, 4, 128, BF, "two", "pc"),
    "tma_k5_s2_64_128_box32x4": (64, 128, 5, 2, 2, 1, 1, False, True, 2, 32, 64, BF, "uniform", "pc"),
    "tma_k3_s2_128_256_box_n": (128, 256, 3, 2, 1, 1, 1, False, True, 4, 8, 8, BF, "uniform", "pc"),
    "tma_k3_64_256_n256": (64, 256, 3, 1, 1, 1, 1, False, False, 2, 128, 128, BF, "uniform", "pc"),
    "tma_plain_1x1_128_64": (128, 64, 1, 1, 0, 1, 1, True, False, 2, 16, 16, BF, "uniform", "1x1"),
    # stride-2 data gradient = four stride-1 parity classes on the half-resolution grid (row-halo tiles when w/2 >= 128)
    "tma_k5_s2_halo_dgrad_w256": (64, 64, 5, 2, 2, 1, 1, False, True, 1, 8, 256, BF, "uniform", "pc"),
    "tma_k3_s2_halo_dgrad_w256": (64, 128, 3, 2, 1, 1, 1, True, True, 1, 4, 256, BF, "uniform", "pc"),
    "tma_k7_s2_64_64": (64, 64, 7, 2, 3, 1, 1, False, True, 2, 16, 32, BF, "uniform", "pc"),
    # few output tiles: the K blocks of a tile are split across CTAs (fp32 partial sums + finish kernel)
    "tma_splitk_k3_256_128_8x8": (256, 128, 3, 1, 1, 1, 1, True, False, 2, 8, 8, BF, "uniform", "pc"),
    "tma_splitk_k3_320_64_two_8x16": (320, 64, 3, 1, 1, 1, 1, False, False, 1, 8, 16, BF, "two64", "pc"),
}
PADDED_X = {"tc_stem_rowpack_k7_s2", "tc_stem_s2d_k7_s2_tma", "tc_rowpack_k5_d2_cin4"}


def make_mask(kind, n, cin, h, w, seed):
    """Returns (dense fp32 mask for the oracle, builder(dev) -> mask object for the device module)."""
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    if kind == "uniform3":                 # dense 3-channel repeated plane, declared channel-uniform by the caller
        m = blob(n, cin, h, w, seed)
        return m, lambda dev: HoleMask.from_dense(m.to(dev), channel_uniform=True)
    if kind in ("uniform",):
        m = blob(n, cin, h, w, seed)
        if cin <= 8:
            return m, lambda dev: m.to(dev)
        return m, lambda dev: HoleMask.from_plane(m[:, 0].to(dev).to(torch.uint8).contiguous(), cin)
    if kind == "perchannel":
        m = blob(n, cin, h, w, seed, per_channel=True)
        return m, lambda dev: m.to(dev)
    if kind == "nh":                       # decoder case: every pixel valid in at least one channel
        m = blob(n, cin, h, w, seed, per_channel=True)
        m[:, 0] = 1.0
        return m, lambda dev: m.to(dev)
    # two planes: channels [0, c0) and [c0, cin)
    c0 = {"two": cin // 2, "two64": 64, "nh2": cin // 2}[kind]
    a = blob(n, 1, h, w, seed)[:, 0]
    b = blob(n, 1, h, w, seed + 977)[:, 0]
    if kind == "nh2":
        a = torch.ones_like(a)
    m = torch.cat([a[:, None].expand(n, c0, h, w), b[:, None].expand(n, cin - c0, h, w)], 1).contiguous()
    def build(dev):
        pa = HoleMask.from_plane(a.to(dev).to(torch.uint8).contiguous(), c0)
        pb = HoleMask.from_plane(b.to(dev).to(torch.uint8).contiguous(), cin - c0)
        return torch.cat([pa, pb], dim=1)
    return m, build


def conv_case(tag, dev, dump_dir=None):
    if "splitk" in tag:
        os.environ["PCB_SPLITK"] = "1"
    try:
        return _conv_case(tag, dev, dump_dir)
    finally:
        os.environ.pop("PCB_SPLITK", None)


def _conv_case(tag, dev, dump_dir=None):
    """fwd + bwd of one PartialConv* module on the GPU vs the oracle.  Returns dict of errors + flags."""
    from text_segmentation_image_inpainting_b200 import _lib, ops
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    cin, cout, k, s, p, d, g, bias, same_holes, n, h, w, dtype, mkind, cls = CONV_CASES[tag]
    if cls == "pc":
        mod = PC.PartialConv(cin, cout, k, s, p, d, g, bias, same_holes)
    elif cls == "1x1":
        mod = PC.PartialConv1x1(cin, cout, k, s, p, d, g, bias)
    else:
        mod = PC.PartialConvNoHoles(cin, cout, k, s, p, d, g, bias)
    sd = det_fill_state_dict(mod.state_dict())
    mod.load_state_dict(sd)
    x = det_tensor(tag + ".x", (n, cin, h, w))
    mask, build_mask = make_mask(mkind, n, cin, h, w, seed=len(tag) * 7 + k)
    wq = sd["feature_conv.weight"].to(dtype).float()
    xq = x.to(dtype).float()
    bq = sd["feature_conv.bias"] if bias else None
    xo = xq.clone().requires_grad_(True); wo = wq.clone().requires_grad_(True)
    bo = bq.clone().requires_grad_(True) if bias else None
    if cls == "pc":
        yo, mo = O.partial_conv(xo, mask, wo, bo, s, p, d, g, same_holes)
    elif cls == "1x1":
        yo, mo = O.partial_conv_1x1(xo, mask, wo, bo, g)
    else:
        yo, mo = O.partial_conv_no_holes(xo, mask, wo, bo, s, p, d)
    gy = det_tensor(tag + ".gy", tuple(yo.shape)).to(dtype).float()
    (torch.where(torch.isfinite(yo), yo, torch.zeros_like(yo)) * gy).sum().backward()
    with torch.no_grad():
        mod.feature_conv.weight.copy_(wq)
    mod = mod.to(dev)
    if tag in PADDED_X:
        buf = torch.zeros((n, 8, h, w), dtype=dtype, device=dev).contiguous(memory_format=torch.channels_last)
        buf[:, :cin].copy_(xq.to(dev).to(dtype))
        xd = buf[:, :cin].detach().requires_grad_(True)
    else:
        xd = xq.to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    yd, md = mod((xd, build_mask(dev)))
    gyd = gy.to(dev).to(dtype)
    if not torch.isfinite(yo).all():          # NoHoles NaN case: backprop only through the finite outputs
        gyd = torch.where(torch.isfinite(yd), gyd, torch.zeros_like(gyd))
        (torch.where(torch.isfinite(yd), yd, torch.zeros_like(yd)) * gyd).sum().backward()
    else:
        yd.backward(gyd)
    torch.cuda.synchronize()
    res = {"y": relerr(yd, yo), "gx": relerr(xd.grad, xo.grad), "gw": relerr(mod.feature_conv.weight.grad, wo.grad),
           "gb": relerr(mod.feature_conv.bias.grad, bo.grad) if bias else 0.0,
           "mask_equal": torch.equal(md.dense().cpu(), mo.contiguous())}
    c = ops.ConvGeom([xd.detach()], [0], cout, k, s, p, d, g, same_holes, cls == "nh", [(None, cin, 0)]).struct([xd.detach()])
    res["tc"] = int(_lib.load().pcb_conv_uses_tensor_cores(_lib.ctypes.byref(c)))
    res["tol"] = TOL[dtype]
    res["ok"] = all(res[k2] <= res["tol"] for k2 in ("y", "gx", "gw", "gb")) and res["mask_equal"]
    if dump_dir and not res["ok"]:
        for nm, a in (("y_dev", yd), ("y_ref", yo), ("gw_dev", mod.feature_conv.weight.grad), ("gw_ref", wo.grad),
                      ("gx_dev", xd.grad), ("gx_ref", xo.grad)):
            np.save(os.path.join(dump_dir, f"dump_{tag}_{nm}.npy"), a.detach().float().cpu().numpy())
    return res


# (ca at half resolution -> 2x nearest upsampled, cb at full resolution, cout, bias): the decoder / tail input pattern
LAZYCAT_CASES = {"lc_128up_64_to_64": (128, 64, 64, False), "lc_256up_64_to_128": (256, 64, 128, False),
                 "lc_tail_64up_3_to_3": (64, 3, 3, True), "lc_64up_8_to_16": (64, 8, 16, True),
                 # TMA-fed path: the upsampled source is materialised in the workspace; second one uses row-halo tiles
                 "lc_tma_128up_64_to_64": (128, 64, 64, False, (2, 32, 32)), "lc_tma_halo_tail_64up_3_to_3": (64, 3, 3, True, (1, 8, 128)),
                 "lc_tma_splitk_256up_64_to_128": (256, 64, 128, False, (2, 8, 8)),
                 # kernel-to-row tails (conv_k2r.cu) with the 1x1 problem on the TMA-fed kernels; 4-channel second part, 2 outputs
                 "lc_k2r_tail_64up_3_to_3": (64, 3, 3, True, (2, 32, 64)), "lc_k2r_64up_4_to_2": (64, 4, 2, False, (2, 32, 32))}


def lazycat_case(tag, dev, dtype=BF):
    if "splitk" in tag:
        os.environ["PCB_SPLITK"] = "1"
    try:
        return _lazycat_case(tag, dev, dtype)
    finally:
        os.environ.pop("PCB_SPLITK", None)


def _lazycat_case(tag, dev, dtype=BF):
    """PartialConv over LazyCat([up2x(a), b]) with HoleMask cat([mask_a.upsampled(), mask_b]) vs the oracle on the
    materialised cat (image_inpainting.py:183-186)."""
    import torch.nn.functional as F
    from text_segmentation_image_inpainting_b200 import _lib, ops
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    ca, cb, cout, bias = LAZYCAT_CASES[tag][:4]
    n, h, w = LAZYCAT_CASES[tag][4] if len(LAZYCAT_CASES[tag]) > 4 else (2, 24, 20)
    mod = PC.PartialConv(ca + cb, cout, 3, 1, 1, 1, 1, bias, False)
    sd = det_fill_state_dict(mod.state_dict()); mod.load_state_dict(sd)
    wq = sd["feature_conv.weight"].to(dtype).float()
    a = det_tensor(tag + ".a", (n, ca, h // 2, w // 2)).to(dtype).float()
    b = det_tensor(tag + ".b", (n, cb, h, w)).to(dtype).float()
    pa = blob(n, 1, h // 2, w // 2, 11)[:, 0]; pb = blob(n, 1, h, w, 23)[:, 0]
    mask = torch.cat([F.interpolate(pa[:, None], scale_factor=2, mode="nearest").expand(n, ca, h, w), pb[:, None].expand(n, cb, h, w)], 1)
    ao, bo, wo = a.clone().requires_grad_(True), b.clone().requires_grad_(True), wq.clone().requires_grad_(True)
    bio = sd["feature_conv.bias"].clone().requires_grad_(True) if bias else None
    yo, mo = O.partial_conv(torch.cat([F.interpolate(ao, scale_factor=2, mode="nearest"), bo], 1), mask.contiguous(), wo, bio, 1, 1, 1, 1, False)
    gy = det_tensor(tag + ".gy", tuple(yo.shape)).to(dtype).float()
    (yo * gy).sum().backward()
    with torch.no_grad():
        mod.feature_conv.weight.copy_(wq)
    mod = mod.to(dev)
    ad = a.to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    if cb % 8:
        buf = torch.zeros((n, 8, h, w), dtype=dtype, device=dev).contiguous(memory_format=torch.channels_last)
        buf[:, :cb].copy_(b.to(dev).to(dtype)); bd = buf[:, :cb].detach().requires_grad_(True)
    else:
        bd = b.to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    hm = torch.cat([HoleMask.from_plane(pa.to(dev).to(torch.uint8).contiguous(), ca).upsampled(),
                    HoleMask.from_plane(pb.to(dev).to(torch.uint8).contiguous(), cb)], dim=1)
    x = ops.LazyCat([ad, bd], ups=(1, 0))
    yd, md = mod((x, hm))
    yd.backward(gy.to(dev).to(dtype))
    torch.cuda.synchronize()
    res = {"y": relerr(yd, yo), "ga": relerr(ad.grad, ao.grad), "gb_in": relerr(bd.grad, bo.grad),
           "gw": relerr(mod.feature_conv.weight.grad, wo.grad), "gbias": relerr(mod.feature_conv.bias.grad, bio.grad) if bias else 0.0,
           "mask_equal": torch.equal(md.dense().cpu(), mo.contiguous())}
    # the materialised path must agree too
    ym, _ = mod((x.materialize(), hm))
    res["vs_materialized"] = relerr(ym, yd)
    c = ops.ConvGeom(x.xs, x.ups, cout, 3, 1, 1, 1, 1, False, False, hm.parts).struct(x.xs)
    res["tc"] = int(_lib.load().pcb_conv_uses_tensor_cores(_lib.ctypes.byref(c)))
    res["tol"] = TOL[dtype]
    res["ok"] = all(res[k2] <= res["tol"] for k2 in ("y", "ga", "gb_in", "gw", "gbias", "vs_materialized")) and res["mask_equal"]
    return res


# well-conditioned quantities only in bf16: the count-2/8 BatchNorm layers at the bottom of ImageFillOrigin make the
# deep-layer gradients numerically ill-posed (x_hat = +-1), so bf16 compares outputs, loss and decoder-side grads.
def run_net(cls_name, dev, dtype, tag=""):
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.models import image_inpainting as PII
    g = np.load(os.path.join(ROOT, "tests", "golden", f"net_{cls_name}{tag}.npz"))
    n, hw, step = int(g["n"]), int(g["hw"]), int(g["step"])
    net = getattr(PII, cls_name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(dev).train()
    plane = np.unpackbits(g["mask_bits"])[: n * hw * hw].reshape(n, 1, hw, hw).astype(np.float32)
    mask = torch.from_numpy(np.repeat(plane, 3, 1))
    x = det_tensor(cls_name + ".x", (n, 3, hw, hw))
    xin = (x * mask).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    out = net((xin, mask.to(dev)))
    loss = ops.l1_mean(out)
    loss.backward()
    torch.cuda.synchronize()
    errs = {"out": relerr(out[..., ::step, ::step], torch.from_numpy(g["out_sub"])),
            "out_row": relerr(out[0, :, hw // 2, :], torch.from_numpy(g["out_row"])),
            "loss": abs(float(loss.detach()) - float(g["loss"])) / abs(float(g["loss"]))}
    params = dict(net.named_parameters())
    sdn = net.state_dict()
    if dtype == F32:
        for k in g.files:
            if k.startswith("g."):
                errs[k] = relerr(params[k[2:]].grad, torch.from_numpy(g[k]))
            if k.startswith("bn."):
                errs[k] = relerr(sdn[k[3:]], torch.from_numpy(g[k]))
        return errs
    for k in g.files:
        if k.startswith("bn.") and (".encoder.1." in k or ".encoder.0." in k):
            errs[k] = relerr(sdn[k[3:]], torch.from_numpy(g[k]))
    # bf16 mode: gradients against the oracle evaluated under the same storage precision (every parameter, not a sample)
    ref_loss, ref_grads = oracle_bf16_step(cls_name, x, mask)
    errs["loss_vs_bf16_oracle"] = abs(float(loss.detach()) - ref_loss) / abs(ref_loss)
    # Error of a gradient tensor relative to max|ref| of that tensor -- but never relative to less than 1 % of the typical
    # (median) gradient magnitude of tensors of the same kind: some gradients are mathematically ZERO (a conv weight under a
    # BatchNorm that sees 2 values per channel; a BatchNorm shift followed by a mask-free 1x1 conv + BatchNorm, whose input
    # gradient sums to zero) and what either side holds there is rounding noise.
    kinds = {}
    for k, gr in ref_grads.items():
        kinds.setdefault((gr.dim(), k.rsplit(".", 1)[-1]), []).append(float(gr.abs().max()))
    floors = {kk: 1e-2 * float(np.median(v)) for kk, v in kinds.items()}
    num, den = {}, {}
    for k, gr in ref_grads.items():
        kind = (gr.dim(), k.rsplit(".", 1)[-1])
        got = params[k].grad.detach().float().cpu()
        denom = max(float(gr.abs().max()), floors[kind], 1e-30)
        errs["g." + k] = float((got - gr).abs().max()) / denom
        num[kind] = num.get(kind, 0.0) + float((got - gr).double().pow(2).sum())
        den[kind] = den.get(kind, 0.0) + float(gr.double().pow(2).sum())
    # and per KIND of parameter (conv weights / BatchNorm scales / BatchNorm shifts / conv biases): relative L2 over the
    # concatenation of all tensors of the kind -- insensitive to which individual tensors are mathematically zero
    for kind in num:
        errs[f"gl2.{kind[0]}d.{kind[1]}"] = (num[kind] / max(den[kind], 1e-60)) ** 0.5
    return errs


def oracle_bf16_step(cls_name, x, mask, sd0=None):
    """fwd + bwd of the reference algorithm on the host with bf16 STORAGE emulation (oracle.pconv_torch.storage): the loss and
    every parameter gradient the CUDA path's tensor-core mode should reproduce."""
    from text_segmentation_image_inpainting_b200.models import image_inpainting as PII
    if sd0 is None:
        sd0 = det_fill_state_dict(getattr(PII, cls_name)().state_dict())
    sd = O.clone_state_dict(sd0, requires_grad=True)
    with O.storage(torch.bfloat16):
        xin = (x * mask).to(torch.bfloat16).float()
        out = O.NETWORKS[cls_name](sd, xin, mask, training=True)
        out = O._rb(O._rf(out))                       # network output stored in bf16; d loss / d out stored in bf16
        loss = out.abs().mean()
        loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in sd.items() if v.grad is not None}


# ---------------------------------------------------------------------------------------------------------------
# dense segmentation path: modules of the product package on the GPU vs goldens produced by the reference itself
# ---------------------------------------------------------------------------------------------------------------
def seg_block_builders():
    from torch import nn
    from text_segmentation_image_inpainting_b200.models import BaseModels as MB, MobileNetV2 as MM, common as MC
    act = lambda: nn.LeakyReLU(0.3)  # noqa: E731
    return {
        "dsconv_s2": lambda: MB.DSConvBlock(16, 24, 3, 2, 1, 1, False, True, act(), act()),
        "dsconv_d4": lambda: MB.DSConvBlock(16, 16, 3, 1, 4, 4, False, True, act(), None),
        "invres_scse": lambda: MM.InvertedResidual(16, 16, 1, 6, 2, activation=act(), bias=False, add_sece=True),
        "invres_s2": lambda: MM.InvertedResidual(16, 24, 2, 6, 1, activation=act(), bias=False, add_sece=False),
        "scse": lambda: MC.SpatialChannelSqueezeExcitation(32, reduction=16, activation=act()),
        "rfb": lambda: MC.RFB(40, 16, activation=act(), add_sece=True),
        "asp": lambda: MC.ASP(24, 16, act(), asp_rate=(3, 5, 9)),
    }


def seg_block_case(name, dev, dtype):
    g = np.load(os.path.join(ROOT, "tests", "golden", f"seg_{name}.npz"))
    mod = seg_block_builders()[name]()
    mod.load_state_dict(det_fill_state_dict(mod.state_dict()))
    mod = mod.to(dev).train()
    x = torch.from_numpy(g["x"]).to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = mod(x)
    y.backward(torch.from_numpy(g["gy"]).to(dev).to(dtype))
    torch.cuda.synchronize()
    # bf16 gradients: relative L2 (see rel_l2).  Gradients that are mathematically ~0 in the reference (a conv weight
    # directly under a BatchNorm is scale-invariant; RFB's dilation-29 depthwise conv sees only its centre tap on a
    # 12x12 map) are pure rounding noise there: floor the denominator at 1 % of the largest gradient norm.
    floor = 0.01 * max([float(np.linalg.norm(g[k])) for k in g.files if k.startswith("g.")] + [1e-20])
    m = relerr if dtype == F32 else (lambda a, b: rel_l2(a, b, floor))
    errs = {"y": relerr(y, torch.from_numpy(g["y"])), "gx": (relerr if dtype == F32 else rel_l2)(x.grad, torch.from_numpy(g["gx"]))}
    params = dict(mod.named_parameters())
    sdn = mod.state_dict()
    for k in g.files:
        if k.startswith("g."):
            errs[k] = m(params[k[2:]].grad, torch.from_numpy(g[k]))
        if k.startswith("bn."):
            errs[k] = relerr(sdn[k[3:]], torch.from_numpy(g[k]))
    return errs


def pool_bilinear_case(dev, dtype):
    from text_segmentation_image_inpainting_b200 import ops
    g = np.load(os.path.join(ROOT, "tests", "golden", "seg_pool_bilinear.npz"))
    errs = {}
    xp = torch.from_numpy(g["xp"]).to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    yp = ops.avg_pool2d(xp, 3, 2, 1)
    yp.backward(torch.from_numpy(g["gyp"]).to(dev).to(dtype))
    errs["pool_y"], errs["pool_gx"] = relerr(yp, torch.from_numpy(g["yp"])), relerr(xp.grad, torch.from_numpy(g["gxp"]))
    for s in (2, 4):
        xb = torch.from_numpy(g["xb"]).to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        yb = ops.bilinear_upsample(xb, s)
        yb.backward(torch.from_numpy(g[f"gy{s}"]).to(dev).to(dtype))
        errs[f"bil{s}_y"], errs[f"bil{s}_gx"] = relerr(yb, torch.from_numpy(g[f"y{s}"])), relerr(xb.grad, torch.from_numpy(g[f"gx{s}"]))
    return errs


def run_segnet(cls_name, dev, dtype, tag=""):
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.models import text_segmentation as MT
    g = np.load(os.path.join(ROOT, "tests", "golden", f"segnet_{cls_name}{tag}.npz"))
    n, hw, step = int(g["n"]), int(g["hw"]), int(g["step"])
    net = getattr(MT, cls_name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(dev).train()
    x = det_tensor(cls_name + ".x", (n, 3, hw, hw)).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    out = net(x)
    loss = ops.l1_mean(out)
    loss.backward()
    torch.cuda.synchronize()
    m = relerr if dtype == F32 else rel_l2
    errs = {"out": m(out[..., ::step, ::step], torch.from_numpy(g["out_sub"])),
            "out_row": m(out[0, :, hw // 2, :], torch.from_numpy(g["out_row"])),
            "loss": abs(float(loss.detach()) - float(g["loss"])) / abs(float(g["loss"]))}
    params = dict(net.named_parameters())
    sdn = net.state_dict()
    for k in g.files:
        if k.startswith("g."):
            errs[k] = m(params[k[2:]].grad, torch.from_numpy(g[k]))
        if k.startswith("bn."):
            errs[k] = relerr(sdn[k[3:]], torch.from_numpy(g[k]))
    return errs

"""GPU tests of inference: the eval-mode BatchNorm + activation fused into the convolution epilogues
(pcb_pconv_forward_affine_act), the graph-captured engines (engine.InferStep / SegInferStep) and the text-mask
post-processing kernel (ops.text_mask_postprocess).

Per layer, the fused epilogue is compared with today's two-pass eval path of the SAME module (eager, no_grad, switch off):
new masks, hole pixels (= bf16(act(shift))), padded channels, NaN positions and activation-only ReLU are bit-identical; every
other element is within 2^-7 |unfused| + 2^-8 |scale| |conv_out| + 1e-6.  The fused path rounds to bf16 once instead of twice:
the unfused path reads the convolution output rounded to bf16 (up to 2^-8 |conv_out| off, times |scale|), and the two final
roundings may land on neighbouring bf16 values -- one bf16 ulp, up to 2^-7 of the value.  Where the convolution output is not
finite (PartialConvNoHoles' 0/0) the two paths must agree exactly.

Networks: running statistics are calibrated deterministically by one training-mode forward of the GPU net on the test batch
with momentum 1 (running statistics = that batch's statistics), so eval activations are O(1).  U-Nets: the engine output is
within 2e-2 relative L2 of the fp32 oracle in eval mode (the bf16 forward bar) and within 1e-2 of the eager eval path.
Segmentation networks: with these statistics the eager bf16 eval path itself is 5-6 % (relative L2) from the oracle after
~100 BatchNorm layers (measured on an H100: TextSegament 256² 6.4 %, XceptionTextSegment 600² 5.1 %), and TextSegament's is
not run-to-run deterministic (float atomics in its reductions); there the engine must be no further from the oracle than the
eager path, and replays must be bitwise equal wherever two eager runs are."""
import os

import numpy as np
import pytest
import torch
from torch import nn

from gpu_cases import ROOT
from oracle.detfill import det_fill_state_dict, det_tensor

pytestmark = pytest.mark.gpu

CL = torch.channels_last
DEV = torch.device("cuda:0")


def _lib():
    from text_segmentation_image_inpainting_b200 import _lib as L
    return L


def _ops():
    from text_segmentation_image_inpainting_b200 import ops
    return ops


def _pipeline_ok():
    import ctypes
    code = ctypes.c_int(0)
    torch.cuda.synchronize()
    _lib().check(_lib().load().pcb_debug_pipeline_status(ctypes.byref(code)))
    assert code.value == 0


def _randomise_bn(mod, seed):
    g = torch.Generator().manual_seed(seed)
    for m in mod.modules():
        if isinstance(m, nn.BatchNorm2d):
            c = m.num_features
            with torch.no_grad():
                m.weight.copy_(torch.randn(c, generator=g) * 0.5 + 1.0)
                m.bias.copy_(torch.randn(c, generator=g) * 0.2)
                m.running_mean.copy_(torch.randn(c, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(c, generator=g) + 0.5)


def _act(kind):
    return {"relu": nn.ReLU(), "leaky": nn.LeakyReLU(0.2), "relu6": nn.ReLU6(), "none": None}[kind]


def _torch_act(kind, z):
    if kind == "relu":
        return torch.relu(z)
    if kind == "leaky":
        return torch.where(z > 0, z, z * 0.2)
    if kind == "relu6":
        return z.clamp(0, 6)
    return z


def _feature(n, c, h, w, seed):
    from text_segmentation_image_inpainting_b200.ops import padded_empty
    x = padded_empty(n, c, h, w, torch.bfloat16, DEV)
    x.copy_(det_tensor(f"infer.x{seed}", (n, c, h, w)).to(DEV))
    return x


def _padded_channels(y):
    """the channels [cout, cstride) of y's NHWC buffer, or None when y is not channel-padded"""
    from text_segmentation_image_inpainting_b200.ops import nhwc_layout
    n, c, h, w = y.shape
    cs = nhwc_layout(y)
    if cs == c:
        return None
    return y.as_strided((n, cs, h, w), (h * w * cs, 1, w * cs, cs))[:, c:]


def _check_layer(fused, unfused, conv_out, scale, shift, act, hole=None, exact=False):
    """hole: bool [n, 1, ho, wo] of output holes (new mask 0) or None"""
    f, u, co = fused.float().cpu(), unfused.float().cpu(), conv_out.float().cpu()
    pad = _padded_channels(fused)
    if pad is not None:
        assert not bool(pad.any()), "padded channels must be zero"
    assert torch.equal(torch.isnan(f), torch.isnan(u)), "NaN positions differ"
    if exact:
        assert torch.equal(f.nan_to_num(), u.nan_to_num())
        return
    c = f.shape[1]
    sc = scale.float().cpu().view(1, c, 1, 1) if scale is not None else torch.ones(1, c, 1, 1)
    if hole is not None and bool(hole.any()):
        hv = _torch_act(act, shift.float().cpu() if shift is not None else torch.zeros(c)).to(torch.bfloat16).float()
        hm = hole.cpu().expand_as(f)
        assert torch.equal(f[hm], hv.view(1, c, 1, 1).expand_as(f)[hm]), "hole pixels must hold bf16(act(shift))"
        assert torch.equal(f[hm], u[hm])
    fin = torch.isfinite(u) & torch.isfinite(co)
    assert torch.equal(f[~fin].nan_to_num(), u[~fin].nan_to_num())
    bound = 2.0 ** -7 * u.abs() + 2.0 ** -8 * sc.abs() * co.abs() + 1e-6
    err = (f - u).abs()
    assert bool((err[fin] <= bound[fin]).all()), f"max excess {float((err - bound)[fin].max())}"


def _run_block(block, args):
    """(fused output, unfused output, conv output, new mask) of a partial-convolution block in eval mode"""
    ops = _ops()
    block = block.to(DEV).eval()
    with torch.no_grad():
        yu, mu = block(args)
        conv_out, _ = block[0](args)
        with ops.StepScope(DEV, training=False) as scope:
            yf, mf = block(args)
    torch.cuda.synchronize()
    return yf, yu, conv_out, mf, mu, {"fused": scope.fused_sites, "unfused": scope.unfused_sites}


def _bn_coef(block):
    tail = block[1]
    if not hasattr(tail, "bn_act"):
        return None, None
    return _ops().bn_eval_coefficients(tail.bn_act[0])


PCONV_CASES = {
    # name: (cin, cout, k, s, p, d, n, h, w, same_holes, no_holes)
    "tma_k3_64x64_8x128": (64, 64, 3, 1, 1, 1, 2, 8, 128, False, False),
    "tma_k5_s2": (64, 128, 5, 2, 2, 1, 2, 32, 64, False, False),
    "gather_75x75": (64, 64, 3, 1, 1, 1, 1, 75, 75, False, False),
    "no_holes_k3": (64, 64, 3, 1, 1, 1, 1, 16, 32, False, True),
}


@pytest.mark.parametrize("act", ["relu", "leaky", "relu6", "none"])
@pytest.mark.parametrize("bn", [True, False], ids=["bn", "nobn"])
@pytest.mark.parametrize("case", list(PCONV_CASES))
def test_partial_block_fused_epilogue(case, bn, act):
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models.partial_convolution import partial_convolution_block
    from gpu_cases import blob
    if not bn and act == "none":
        pytest.skip("a bare convolution has no epilogue to fuse")
    cin, cout, k, s, p, d, n, h, w, same, noh = PCONV_CASES[case]
    torch.manual_seed(7)
    block = partial_convolution_block(cin, cout, k, s, p, d, BN=bn, activation=_act(act) if act != "none" else None,
                                      no_holes_1_conv=noh, same_holes=same)
    _randomise_bn(block, 3)
    x = _feature(n, cin, h, w, 1)
    m = blob(n, 1, h, w, 5)
    if noh:
        m[:, :, :, : w // 2] = 0                          # box sums of 0: NoHoles divides by zero (NaN like the reference)
    hm = HoleMask.from_dense(m.expand(n, cin, h, w).contiguous().to(DEV), channel_uniform=True)
    yf, yu, co, mf, mu, sites = _run_block(block, (x, hm))
    assert sites["fused"] == 1 and sites["unfused"] == 0
    assert torch.equal(mf.dense(), mu.dense())
    scale, shift = _bn_coef(block)
    hole = None if noh else (mu.dense()[:, :1] == 0)
    _check_layer(yf, yu, co, scale, shift, act, hole, exact=(not bn and act == "relu"))


def test_partial_block_lazy_upsampled_concat():
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models.partial_convolution import partial_convolution_block
    from gpu_cases import blob
    torch.manual_seed(8)
    block = partial_convolution_block(128 + 64, 64, 3, 1, 1, 1, BN=True, activation=nn.LeakyReLU(0.2))
    _randomise_bn(block, 4)
    a, sx = _feature(2, 128, 16, 32, 2), _feature(2, 64, 32, 64, 3)
    ma, ms = blob(2, 1, 16, 32, 6), blob(2, 1, 32, 64, 7)
    ha = HoleMask.from_dense(ma.expand(2, 128, 16, 32).contiguous().to(DEV), channel_uniform=True)
    hs = HoleMask.from_dense(ms.expand(2, 64, 32, 64).contiguous().to(DEV), channel_uniform=True)
    xh = ops.LazyCat([a, sx], ups=(1, 0))
    mh = torch.cat([ha.upsampled(), hs], dim=1)
    yf, yu, co, mf, mu, sites = _run_block(block, (xh, mh))
    assert sites["fused"] == 1
    assert torch.equal(mf.dense(), mu.dense())
    scale, shift = _bn_coef(block)
    _check_layer(yf, yu, co, scale, shift, "leaky", mu.dense()[:, :1] == 0)


@pytest.mark.parametrize("hw", [64, 75])
def test_stem_7x7_s2_activation_only_relu(hw):
    """the ImageFillOrigin stem, [PartialConv(3 -> 64, k7 s2, same_holes), PartialActivation(ReLU)]: bit-identical"""
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models.partial_convolution import partial_convolution_block
    from gpu_cases import blob
    torch.manual_seed(9)
    block = partial_convolution_block(3, 64, 7, 2, 3, 1, BN=False, activation=nn.ReLU(), same_holes=True)
    x = _feature(2, 3, hw, hw, 4)
    m = blob(2, 1, hw, hw, 8)
    hm = HoleMask.from_dense(m.expand(2, 3, hw, hw).contiguous().to(DEV), channel_uniform=True)
    yf, yu, co, mf, mu, sites = _run_block(block, (x, hm))
    assert sites["fused"] == 1
    assert torch.equal(mf.dense(), mu.dense())
    _check_layer(yf, yu, co, None, None, "relu", exact=True)


CONV_CASES = {
    # name: (cin, cout, k, s, p, d, groups, n, h, w)
    "dw3_d1": (64, 64, 3, 1, 1, 1, 64, 2, 32, 40),
    "dw3_d2": (64, 64, 3, 1, 2, 2, 64, 2, 32, 40),
    "dw3_s2": (64, 64, 3, 2, 1, 1, 64, 2, 33, 40),
    "pw_1x1": (64, 96, 1, 1, 0, 1, 1, 2, 24, 40),
    "dense_k3": (64, 64, 3, 1, 1, 1, 1, 1, 30, 30),
}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("act", ["leaky", "relu6", "none"])
@pytest.mark.parametrize("case", list(CONV_CASES))
def test_conv_block_fused_epilogue(case, act, dtype):
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.models.BaseModels import Conv_block
    cin, cout, k, s, p, d, groups, n, h, w = CONV_CASES[case]
    if dtype == torch.float32 and groups == 1:
        pytest.skip("the dense kernels fuse in bf16 (tensor cores); the fp32 exact mode stays two-pass")
    torch.manual_seed(10)
    seq = nn.Sequential(*Conv_block(cin, cout, k, s, p, d, groups, bias=False, BN=True, activation=_act(act) if act != "none" else None))
    _randomise_bn(seq, 5)
    seq = seq.to(DEV).eval()
    x = det_tensor(f"infer.conv.{case}", (n, cin, h, w)).to(DEV).to(dtype).contiguous(memory_format=CL)
    with torch.no_grad():
        yu = seq(x)
        co = seq[0](x)
        with ops.StepScope(DEV, training=False) as scope:
            yf = seq(x)
    assert (scope.fused_sites, scope.unfused_sites) == (1, 0)
    assert "_pcb_fused_out" not in seq[1].__dict__
    scale, shift = ops.bn_eval_coefficients(seq[1][0])
    if dtype == torch.float32:
        f, u = yf.cpu(), yu.cpu()
        assert float((f - u).abs().max()) <= 1e-5 * (1 + float(u.abs().max()))
    else:
        _check_layer(yf, yu, co, scale, shift, act)


def test_residual_batchnorm_is_not_fused():
    """InvertedResidual folds its shortcut into the last BatchNorm pass: that convolution must stay two-pass"""
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.models.MobileNetV2 import InvertedResidual
    torch.manual_seed(11)
    blk = InvertedResidual(32, 32, 1, 2, 1, activation=nn.ReLU6())
    _randomise_bn(blk, 6)
    blk = blk.to(DEV).eval()
    x = det_tensor("infer.ir", (2, 32, 16, 24)).to(DEV).to(torch.bfloat16).contiguous(memory_format=CL)
    with torch.no_grad():
        yu = blk(x)
        with ops.StepScope(DEV, training=False) as scope:
            yf = blk(x)
    assert (scope.fused_sites, scope.unfused_sites) == (2, 1)
    assert float((yf.float() - yu.float()).abs().max()) <= 3e-2 * float(yu.float().abs().max())


def test_affine_act_rejects_refused_problem():
    """a problem pcb_conv_fuses_affine_act refuses (the fp32 generic kernels) is rejected with a message"""
    import ctypes
    from text_segmentation_image_inpainting_b200 import ops
    x = torch.randn(1, 16, 8, 8, device=DEV).contiguous(memory_format=CL)
    wt = torch.randn(16, 16, 3, 3, device=DEV).contiguous(memory_format=CL)
    geom = ops.ConvGeom([x], [0], 16, (3, 3), 1, 1, 1, 1, False, False, [(None, 16, 0)], plain=True)
    lib = _lib().load()
    c = geom.struct([x])
    assert lib.pcb_conv_fuses_affine_act(ctypes.byref(c)) == 0
    y = torch.empty_like(x)
    msum = torch.empty(1, 8, 8, device=DEV)
    nm = torch.empty(1, 8, 8, dtype=torch.uint8, device=DEV)
    rc = lib.pcb_pconv_forward_affine_act(ctypes.byref(c), wt.data_ptr(), None, y.data_ptr(), 16, msum.data_ptr(), nm.data_ptr(), None, 0,
                                          None, None, 1, 0.0, None)
    assert rc != 0 and b"fuses_affine_act" in lib.pcb_last_error()


# ------------------------------------------------------------------------------------------------ networks
def _calibrate(net, run_train):
    """running statistics = the statistics of one training-mode forward on the test batch (momentum 1)"""
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    for m in bns:
        m.momentum = 1.0
    net.train()
    with torch.no_grad():
        run_train()
    torch.cuda.synchronize()
    for m in bns:
        m.momentum = 0.1
    net.eval()


def _rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


UNETS = {
    "ImageFillOrigin_512_b1": ("ImageFillOrigin", 512, 1),
    "ImageFillOrigin_256_b2": ("ImageFillOrigin", 256, 2),
    "ImageFillOriginV2_256_b2": ("ImageFillOriginV2", 256, 2),     # batch 2: the 1x1 bottleneck needs two values per
    "ImageFill_256_b2": ("ImageFill", 256, 2),                     # channel for the training-mode calibration
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(UNETS))
def test_infer_step_unet(case):
    from oracle import pconv_torch as O
    from text_segmentation_image_inpainting_b200 import _lib as L
    from text_segmentation_image_inpainting_b200.engine import InferStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    name, hw, batch = UNETS[case]
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    torch.manual_seed(12)
    net = getattr(II, name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(DEV)
    x = det_tensor("infer.net.x", (batch, 3, hw, hw))
    mask = torch.from_numpy(random_hole_masks(batch, hw, hw, seed=31))
    xd, md = x.to(DEV), mask.to(DEV)
    step = InferStep(net)
    _calibrate(net, lambda: net(step._prepare(xd, md)))
    with torch.no_grad():                                    # today's eager eval path
        before = L.launch_count()
        eager = net(step._prepare(xd, md)).float()
        eager_launches = L.launch_count() - before
    out = step.run(xd, md).clone()
    out2 = step.run(xd, md).clone()
    _pipeline_ok()
    assert torch.equal(out, out2)
    assert step.fused_sites > 0
    assert eager_launches - step.launches_per_run >= step.fused_sites
    assert _rel_l2(out, eager) <= 1e-2
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref = {"ImageFillOrigin": O.image_fill_origin, "ImageFillOriginV2": O.image_fill_origin_v2, "ImageFill": O.image_fill}[name]
    with torch.no_grad():
        oracle = ref(O.clone_state_dict(sd), x * mask, mask, training=False)
    assert _rel_l2(out, oracle) <= 2e-2


SEGS = {
    "TextSegament_256_b2": ("TextSegament", 256, 2),
    "XceptionTextSegment_600_b1": ("XceptionTextSegment", 600, 1),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(SEGS))
def test_seg_infer_step(case):
    from oracle import seg_torch as S
    from text_segmentation_image_inpainting_b200 import _lib as L
    from text_segmentation_image_inpainting_b200.engine import SegInferStep
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    name, hw, batch = SEGS[case]
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    torch.manual_seed(13)
    net = getattr(TS, name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(DEV)
    x = det_tensor("infer.seg.x", (batch, 3, hw, hw))
    xd = x.to(DEV)
    step = SegInferStep(net)
    _calibrate(net, lambda: step._forward(xd))
    with torch.no_grad():
        before = L.launch_count()
        eager = step._forward(xd).float()
        eager_launches = L.launch_count() - before
        eager2 = step._forward(xd).float()
    out = step.run(xd).clone()
    out2 = step.run(xd).clone()
    _pipeline_ok()
    if torch.equal(eager, eager2):
        assert torch.equal(out, out2)
    assert step.fused_sites > 0
    assert eager_launches - step.launches_per_run >= step.fused_sites
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        oracle = S.text_segment(sd, x, training=False) if name == "TextSegament" else S.xception_text_segment(sd, x, training=False)
    assert _rel_l2(out, oracle) <= _rel_l2(eager, oracle) + 5e-3
    assert _rel_l2(out, oracle) <= 0.1


def test_infer_step_refresh_after_load_state_dict():
    from text_segmentation_image_inpainting_b200.engine import InferStep
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    torch.manual_seed(14)
    net = ImageFillOrigin()
    sd0 = det_fill_state_dict(net.state_dict())
    net.load_state_dict(sd0)
    _randomise_bn(net, 8)
    net = net.to(DEV).eval()
    x = det_tensor("infer.refresh.x", (1, 3, 256, 256)).to(DEV)
    mask = torch.from_numpy(random_hole_masks(1, 256, 256, seed=32)).to(DEV)
    step = InferStep(net)
    first = step.run(x, mask).clone()
    sd1 = {k: (v * 0.9 + 0.01 if v.is_floating_point() and "running_var" not in k else v) for k, v in net.state_dict().items()}
    net.load_state_dict(sd1)
    after = step.run(x, mask).clone()
    fresh_net = ImageFillOrigin()
    fresh_net.load_state_dict({k: v.cpu() for k, v in sd1.items()})
    fresh = InferStep(fresh_net.to(DEV)).run(x, mask).clone()
    _pipeline_ok()
    assert not torch.equal(first, after)
    assert torch.equal(after, fresh)


# ------------------------------------------------------------------------------------------------ post-processing
@pytest.mark.parametrize("layout", ["f32_nchw", "bf16_nhwc_padded"])
def test_text_mask_postprocess_matches_golden(layout):
    from text_segmentation_image_inpainting_b200 import ops
    g = np.load(os.path.join(ROOT, "tests", "golden", "seg_postprocess.npz"))
    names = sorted({k.split(".")[0] for k in g.files})
    for name in names:
        logits = torch.from_numpy(g[name + ".logits"]).to(DEV)
        if layout == "bf16_nhwc_padded":
            n, _, h, w = logits.shape
            buf = torch.randn(n, 8, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=CL)
            buf[:, :1].copy_(logits)
            logits = buf[:, :1]
        before = _lib().launch_count()
        out = ops.text_mask_postprocess(logits, tuple(g[name + ".pad"]), tuple(g[name + ".out_hw"]))
        assert _lib().launch_count() - before == 1
        assert out.dtype == torch.uint8 and torch.equal(out.cpu(), torch.from_numpy(g[name + ".mask"])), name

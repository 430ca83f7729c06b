"""GPU parity tests (run with -m gpu on an H100): the CUDA path, called through the module surface ->
autograd Functions -> ctypes -> C ABI (include/pconv_b200.h), against the oracle."""
import pytest
import torch

from gpu_cases import BF, CONV_CASES, F32, LAZYCAT_CASES, conv_case, lazycat_case, relerr, run_net
from oracle import pconv_torch as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from text_segmentation_image_inpainting_b200 import _lib
    _lib.load()
    return torch.device("cuda:0")


def _pipeline_clean():
    from text_segmentation_image_inpainting_b200 import _lib
    code = _lib.ctypes.c_int(0)
    torch.cuda.synchronize()
    _lib.check(_lib.load().pcb_debug_pipeline_status(_lib.ctypes.byref(code)))
    return code.value == 0


@pytest.mark.parametrize("tag", sorted(CONV_CASES))
def test_partial_conv_module_fwd_bwd(tag, dev):
    res = conv_case(tag, dev)
    assert _pipeline_clean(), "a tensor-core pipeline wait timed out"
    assert res["mask_equal"], "binary mask update must be bit-exact"
    if tag.startswith("tc_"):
        assert res["tc"] == 1, "this case must run on the tensor-core path"
    for k in ("y", "gx", "gw", "gb"):
        assert res[k] <= res["tol"], (k, res)


@pytest.mark.parametrize("tag", sorted(LAZYCAT_CASES))
def test_partial_conv_over_lazy_upsample_concat(tag, dev):
    """The decoder pattern: conv(cat([up2x(a), b])) without materialising the upsample or the concat."""
    res = lazycat_case(tag, dev)
    assert _pipeline_clean() and res["mask_equal"] and res["tc"] == 1, res
    for k in ("y", "ga", "gb_in", "gw", "gbias", "vs_materialized"):
        assert res[k] <= res["tol"], (k, res)


NET_GOLDENS = [("ImageFillOrigin", ""), ("ImageFillOriginV2", ""), ("ImageFill", ""), ("ImageFillOrigin", "_512")]     # "_512": the benchmarked resolution (BASELINE.json configs[2])
SEG_GOLDENS = [("TextSegament", ""), ("XceptionTextSegment", ""), ("TextSegament", "_256"), ("XceptionTextSegment", "_256")]


@pytest.mark.parametrize("cls_name,tag", NET_GOLDENS)
def test_network_fp32_matches_reference_golden(cls_name, tag, dev):
    """exact mode end to end: forward within 1e-3 relative of the reference's CPU forward (north_star bar);
    gradients within 2e-3 (fp32 re-association noise amplified by the tiny-batch BatchNorms at the bottom)."""
    errs = run_net(cls_name, dev, F32, tag)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    assert errs["out"] <= 1e-3 and errs["out_row"] <= 1e-3 and errs["loss"] <= 1e-5, worst
    assert max(errs.values()) <= (5e-3 if tag == "_512" else 2e-3), worst


@pytest.mark.parametrize("cls_name,tag", NET_GOLDENS)
def test_network_bf16_tensor_core_mode(cls_name, tag, dev):
    """bf16 storage + tensor cores: 16+ layers of bf16 rounding -> a few 1e-3 on the output and loss.  Gradients of the
    BatchNorm scales see LeakyReLU sign flips of pre-activations within one bf16 ulp of zero (a systematic, not a
    random, perturbation): a few percent of max|grad|; convolution weight grads stay at the 1e-3 level."""
    errs = run_net(cls_name, dev, BF, tag)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    assert _pipeline_clean()
    # forward / loss / running statistics against the fp32 REFERENCE golden
    assert errs["out"] <= 2e-2 and errs["loss"] <= 2e-3, worst
    assert all(v <= 2e-2 for k, v in errs.items() if k.startswith("bn.")), worst
    # every gradient against the oracle run under the SAME storage precision (oracle.pconv_torch.storage(bfloat16): activations
    # and activation gradients rounded to bf16 exactly where the CUDA path hands them from kernel to kernel).  Against the fp32
    # reference these gradients differ by tens of percent on ill-conditioned channels (a BatchNorm channel whose spread is
    # below one bf16 ulp of its mean) -- tests/test_oracle_golden.py::test_bf16_storage_emulation documents that gap on CPU.
    assert all(v <= 5e-2 for k, v in errs.items() if k.startswith("gl2.")), worst
    if cls_name == "ImageFillOrigin":      # the benchmarked network: every single tensor as well
        # 5e-2: the sub-pixel data gradient multiplies by SUMS of taps rounded to bf16 once (w1 + w2 -> bf16), the oracle by
        # individually rounded taps -- a different, equally legitimate bf16 rounding of the same fp32 weights, amplified like any
        # other perturbation by the ill-conditioned BatchNorm channels upstream
        assert all(v <= 5e-2 for k, v in errs.items() if k.startswith("g.")), worst


@pytest.mark.parametrize("c", [24, 256])       # 256 channels x 297 rows: the one-launch small-tensor backward (pcb_bn_act_backward_small)
def test_bn_act_and_running_stats(c, dev):
    from oracle.detfill import det_fill_state_dict, det_tensor
    from text_segmentation_image_inpainting_b200 import ops
    for dtype, tol in ((F32, 2e-5), (BF, 2e-2)):
        for act in (torch.nn.ReLU(), torch.nn.LeakyReLU(0.2), None, torch.nn.ReLU6()):
            bn = torch.nn.BatchNorm2d(c); sd = det_fill_state_dict(bn.state_dict()); bn.load_state_dict(sd)
            ref = torch.nn.BatchNorm2d(c); ref.load_state_dict(sd)
            xq = (det_tensor("bn.x", (3, c, 9, 11)) * 2 + 0.3).to(dtype).float()
            xr = xq.clone().requires_grad_(True)
            yr = ref(xr); yr = act(yr) if act else yr
            gy = det_tensor("bn.gy", tuple(yr.shape)).to(dtype).float()
            (yr * gy).sum().backward()
            bn = bn.to(dev)
            xd = xq.to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            yd = ops.bn_act(xd, bn, act)
            yd.backward(gy.to(dev).to(dtype))
            for a, b in ((yd, yr), (xd.grad, xr.grad), (bn.weight.grad, ref.weight.grad), (bn.bias.grad, ref.bias.grad),
                         (bn.running_mean, ref.running_mean), (bn.running_var, ref.running_var)):
                assert relerr(a, b) <= tol
            assert int(bn.num_batches_tracked) == 1
            bn.eval(); ref.eval()
            assert relerr(ops.bn_act(xd.detach(), bn, act), act(ref(xq)) if act else ref(xq)) <= tol
            bn.train()
            if c >= 256:                  # the two-launch path must agree with the one-launch path
                ops.set_bn_small_kernel(False)
                try:
                    bn.zero_grad(set_to_none=True)
                    x2 = xd.detach().clone().requires_grad_(True)
                    ops.bn_act(x2, bn, act).backward(gy.to(dev).to(dtype))
                    assert relerr(x2.grad, xd.grad) <= (1e-5 if dtype == F32 else 1e-2) and relerr(bn.weight.grad, ref.weight.grad) <= tol
                finally:
                    ops.set_bn_small_kernel(True)


@pytest.mark.parametrize("shape", [(64, 128, 3, 1, 1, (2, 24, 20)), (64, 64, 3, 1, 1, (2, 8, 128)), (128, 256, 3, 2, 1, (2, 32, 32)),
                                   (192, 320, 1, 1, 0, (1, 16, 16))])
def test_bn_statistics_fused_into_conv_epilogue(shape, dev):
    """PartialConv -> BatchNorm(train) -> LeakyReLU block: the per-channel sums accumulated in the tensor-core epilogue
    (pcb_pconv_forward_bn) against the separate statistics pass (ops.set_fused_bn_stats(False)) and against the oracle."""
    from gpu_cases import blob
    from oracle.detfill import det_fill_state_dict, det_tensor
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    cin, cout, k, s, p, (n, h, w) = shape
    blk = PC.partial_convolution_block(cin, cout, k, s, p, 1, bias=False, BN=True, activation=torch.nn.LeakyReLU(0.2), same_holes=True)
    sd = det_fill_state_dict(blk.state_dict())
    x = det_tensor("fbn.x", (n, cin, h, w)).to(BF)
    mask = blob(n, cin, h, w, 3)
    gy = None
    res = {}
    for fused in (True, False):
        ops.set_fused_bn_stats(fused)
        try:
            blk.load_state_dict(sd)
            m = blk.to(dev).train()
            m.zero_grad(set_to_none=True)
            xd = x.to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            y, _ = m((xd, mask.to(dev)))
            if gy is None:
                gy = det_tensor("fbn.gy", tuple(y.shape)).to(BF)
            y.backward(gy.to(dev))
            torch.cuda.synchronize()
            res[fused] = (y.detach().float().cpu(), xd.grad.float().cpu(), m[1].bn_act[0].running_mean.cpu().clone(),
                          m[1].bn_act[0].running_var.cpu().clone(), m[1].bn_act[0].weight.grad.cpu().clone(), m[0].feature_conv.weight.grad.cpu().clone())
        finally:
            ops.set_fused_bn_stats(True)
    assert _pipeline_clean()
    for a, b in zip(res[True], res[False]):
        assert relerr(a, b) <= 2e-2, relerr(a, b)
    # the statistics themselves are sums of the same bf16-rounded values: only the summation order differs
    assert relerr(res[True][2], res[False][2]) <= 1e-5 and relerr(res[True][3], res[False][3]) <= 1e-4
    # the oracle under the same storage precision (conv output and BN+activation output rounded to bf16, like the two kernels
    # store them): reference semantics of the whole block, partial_convolution.py:49-80 + :193-201
    sdo = O.clone_state_dict(sd, requires_grad=True)
    xo = x.float().clone().requires_grad_(True)
    with O.storage(BF):
        zo, _ = O.pconv_block(sdo, "", xo, mask, k=k, s=s, p=p, bn=True, act=("leaky", 0.2), same_holes=True, training=True)
        (zo * gy.float()).sum().backward()
    assert relerr(res[True][0], zo) <= 2e-2, relerr(res[True][0], zo)
    assert relerr(res[True][2], sdo["1.bn_act.0.running_mean"]) <= 1e-2 and relerr(res[True][3], sdo["1.bn_act.0.running_var"]) <= 1e-2
    assert relerr(res[True][5], sdo["0.feature_conv.weight"].grad) <= 3e-2 and relerr(res[True][1], xo.grad) <= 3e-2


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_general_per_channel_masks_beyond_part_table(dtype, dev):
    """partial_convolution.py:62-64 accepts ANY [N,C,H,W] mask.  12 genuinely different mask planes (more than PCB_MAX_PARTS = 8)
    into a dense PartialConv, then a 16-group non-same_holes conv whose 16-plane output mask feeds a third layer: the general
    dense-mask route must reproduce the oracle (masks bit-exact)."""
    from gpu_cases import blob
    from oracle.detfill import det_fill_state_dict, det_tensor
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    n, h, w = 2, 20, 24
    mods = [PC.PartialConv(12, 32, 3, 1, 1, 1, 1, True, False), PC.PartialConv(32, 32, 3, 1, 1, 1, 16, False, False),
            PC.PartialConv(32, 8, 3, 2, 1, 1, 1, True, False)]
    sds = [det_fill_state_dict(m.state_dict()) for m in mods]
    x = det_tensor("pcm.x", (n, 12, h, w)).to(dtype).float()
    mask = blob(n, 12, h, w, 17, per_channel=True)
    assert len({mask[0, c].numpy().tobytes() for c in range(12)}) > 8
    xo = x.clone().requires_grad_(True)
    ws = [sd["feature_conv.weight"].to(dtype).float().requires_grad_(True) for sd in sds]
    yo, mo = xo, mask
    for sd, wq, (s_, g_) in zip(sds, ws, ((1, 1), (1, 16), (2, 1))):
        yo, mo = O.partial_conv(yo, mo.contiguous(), wq, sd.get("feature_conv.bias"), s_, 1, 1, g_, False)
    gy = det_tensor("pcm.gy", tuple(yo.shape)).to(dtype).float()
    (yo * gy).sum().backward()
    yd = x.to(dev).to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    xd, md = yd, mask.to(dev)
    for m, sd, wq in zip(mods, sds, ws):
        m.load_state_dict(sd)
        with torch.no_grad():
            m.feature_conv.weight.copy_(wq.detach())
        m.to(dev)
        yd, md = m((yd, md))
    yd.backward(gy.to(dev).to(dtype))
    torch.cuda.synchronize()
    tol = 1e-4 if dtype == F32 else 3e-2
    assert torch.equal(md.dense().cpu(), mo.contiguous())
    assert relerr(yd, yo) <= tol and relerr(xd.grad, xo.grad) <= tol
    for m, wq in zip(mods, ws):
        assert relerr(m.feature_conv.weight.grad, wq.grad) <= tol


def test_concat_upsample_and_masks(dev):
    import torch.nn.functional as F
    from oracle.detfill import det_tensor
    from gpu_cases import blob
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    for dtype, tol in ((F32, 1e-6), (BF, 2e-2)):
        for ca, cb in ((16, 8), (64, 3)):
            a = det_tensor("cat.a", (2, ca, 5, 6)).to(dtype); b = det_tensor("cat.b", (2, cb, 10, 12)).to(dtype)
            ar = a.float().clone().requires_grad_(True); br = b.float().clone().requires_grad_(True)
            yr = torch.cat([F.interpolate(ar, scale_factor=2, mode="nearest"), br], 1)
            gy = det_tensor("cat.gy", tuple(yr.shape)).to(dtype).float()
            (yr * gy).sum().backward()
            ad = a.detach().to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            bd = b.detach().to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            yd = ops.concat_features([ad, bd], ups=(1, 0))
            yd.backward(gy.to(dev).to(dtype))
            assert relerr(yd, yr) <= tol and relerr(ad.grad, ar.grad) <= tol and relerr(bd.grad, br.grad) <= tol
    m = blob(2, 3, 8, 10, 3, per_channel=True)
    hm = HoleMask.from_dense(m.to(dev))
    up = F.interpolate(m, scale_factor=2, mode="nearest")
    assert torch.equal(hm.dense().cpu(), m) and torch.equal(hm.upsampled().dense().cpu(), up)
    cat = torch.cat([hm.upsampled(), HoleMask.from_dense(up.to(dev))], 1)
    assert torch.equal(cat.dense().cpu(), torch.cat([up, up], 1))
    assert torch.equal((cat * 1.0).cpu(), torch.cat([up, up], 1))          # unknown op -> dense fallback, same values


def test_full_size_properties_cfg1_and_hole_semantics(dev):
    """BASELINE cfg 1 (PartialConv 3->64 k3 @256^2 b1) and size-independent properties at full size:
    hole interior -> y == 0 and m' == 0; a 32x32 hole under k3 p1 shrinks to 30x30; same_holes == full-mask path
    for channel-uniform masks; linearity in x."""
    from oracle.detfill import det_fill_state_dict, det_tensor
    from oracle import pconv_torch as O
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    mod = PC.PartialConv(3, 64, 3, 1, 1)
    sd = det_fill_state_dict(mod.state_dict()); mod.load_state_dict(sd); mod = mod.to(dev)
    x = det_tensor("cfg1.x", (1, 3, 256, 256)); mask = torch.ones_like(x); mask[:, :, 100:132, 60:92] = 0
    y, nm = mod((x.to(dev).contiguous(memory_format=torch.channels_last), mask.to(dev)))
    yo, mo = O.partial_conv(x, mask, sd["feature_conv.weight"], sd["feature_conv.bias"], 1, 1, 1, 1, False)
    assert relerr(y, yo) <= 1e-4                                  # north_star: <= 1e-3 relative fp32
    nmd = nm.dense().cpu()
    assert torch.equal(nmd, mo) and int((nmd[0, 0] == 0).sum()) == 30 * 30
    assert bool((y.cpu()[nmd == 0] == 0).all())
    mod2 = PC.PartialConv(3, 64, 3, 1, 1, same_holes=True).to(dev)
    with torch.no_grad():
        mod2.feature_conv.weight.copy_(sd["feature_conv.weight"]); mod2.feature_conv.bias.copy_(sd["feature_conv.bias"])
    y2, nm2 = mod2((x.to(dev).contiguous(memory_format=torch.channels_last), mask.to(dev)))
    assert relerr(y2, y) <= 1e-6 and torch.equal(nm2.dense(), nm.dense())
    # linearity of the masked convolution part: f(2x) - b == 2 (f(x) - b)
    y3, _ = mod(((2 * x.to(dev)).contiguous(memory_format=torch.channels_last), mask.to(dev)))
    b = sd["feature_conv.bias"].to(dev).view(1, -1, 1, 1) * nm.dense()
    assert relerr(y3 - b, 2 * (y - b)) <= 1e-5


def test_train_step_engine_graph_matches_eager(dev):
    """CUDA-graph replay of the whole step == eager steps (same data): losses agree step by step."""
    from text_segmentation_image_inpainting_b200.engine import TrainStep
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(3)).to(dev)
    mask = torch.from_numpy(random_hole_masks(2, 256, 256, seed=5)).to(dev)
    losses = []
    for use_graph in (False, True):
        torch.manual_seed(0)
        ts = TrainStep(ImageFillOrigin().to(dev), use_graph=use_graph, lr=1e-3)
        # the graph path runs one extra (side-stream) step before capture: give eager one more warm-up step
        ts.warmup_and_capture(x, mask, eager_warmup=2 if use_graph else 3)
        if use_graph:
            assert ts.graph is not None
        losses.append([float(ts.step(x, mask)) for _ in range(3)])
    assert losses[0][0] > 0 and all(abs(a - b) <= 2e-2 * abs(a) for a, b in zip(*losses)), losses


def test_gradient_sink_matches_autograd_accumulation(dev):
    """engine.FlatParams registers in-place gradient sinks on the conv weights (ops.GradSink, written from a side stream and
    joined by ops.join_side_streams): the arena must hold the gradients autograd would have accumulated (fp32 split-K adds
    are unordered: compare to 1e-4 of max)."""
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import FlatParams
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    x = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(7)).to(dev)      # 8 stride-2 levels: >= 256
    mask = torch.from_numpy(random_hole_masks(2, 256, 256, seed=9)).to(dev)

    def run(with_sinks):
        torch.manual_seed(0)
        net = ImageFillOrigin().to(dev).train()
        flat = FlatParams(net) if with_sinks else None
        buf = torch.zeros((2, 8, 256, 256), dtype=torch.bfloat16, device=dev).contiguous(memory_format=torch.channels_last)
        xin = buf[:, :3]
        xin.copy_(x * mask)
        ops.bump_weight_epoch()
        out = net((xin, HoleMask.from_dense(mask, channel_uniform=True)))
        ops.l1_mean(out).backward()
        ops.join_side_streams()
        torch.cuda.synchronize()
        if with_sinks:
            unused = [i for i, sk in enumerate(flat.sinks) if not sk.used]
            assert flat.sinks and not unused, unused
        return {n: p.grad.detach().float().clone() for n, p in net.named_parameters() if p.grad is not None}

    ref, got = run(False), run(True)
    bad = {n: relerr(got[n], ref[n]) for n in ref if relerr(got[n], ref[n]) > 1e-4}
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------
# dense segmentation path (Conv_block / DSConvBlock / InvertedResidual / scSE / RFB / ASP / pooling / bilinear)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["dsconv_s2", "dsconv_d4", "invres_scse", "invres_s2", "scse", "rfb", "asp"])
@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_segmentation_blocks_vs_reference_golden(name, dtype, dev):
    from gpu_cases import seg_block_case
    errs = seg_block_case(name, dev, dtype)
    assert _pipeline_clean()
    if dtype == F32:
        assert max(errs.values()) <= 2e-4, errs
    else:   # bf16: forward max-abs; gradients in relative L2 (activation-derivative flips, see gpu_cases.rel_l2)
        assert errs["y"] <= 2e-2 and max(errs.values()) <= 0.15, errs


@pytest.mark.parametrize("dtype", [F32, BF], ids=["f32", "bf16"])
def test_avgpool_and_bilinear_vs_reference_golden(dtype, dev):
    from gpu_cases import pool_bilinear_case
    errs = pool_bilinear_case(dev, dtype)
    assert max(errs.values()) <= (1e-5 if dtype == F32 else 2e-2), errs


@pytest.mark.parametrize("cls_name,tag", SEG_GOLDENS)
def test_segmentation_network_fp32_matches_reference_golden(cls_name, tag, dev):
    from gpu_cases import run_segnet
    errs = run_segnet(cls_name, dev, F32, tag)
    assert errs["out"] <= 1e-3 and errs["out_row"] <= 1e-3 and errs["loss"] <= 1e-4, errs      # north_star bar on the forward
    # gradients: fp32 re-association noise is amplified through ~70 BatchNorm'd layers of a randomly initialised net
    # (the late layers agree to 1e-6, the first conv to ~5e-3)
    assert max(errs.values()) <= 2e-2, errs


@pytest.mark.parametrize("cls_name,tag", SEG_GOLDENS)
def test_segmentation_network_bf16(cls_name, tag, dev):
    from gpu_cases import run_segnet
    errs = run_segnet(cls_name, dev, BF, tag)
    assert _pipeline_clean()
    assert errs["out"] <= 0.15 and errs["loss"] <= 2e-2, errs          # relative L2 of the logit map after ~70 bf16 layers

"""Every module of the five networks against fp64 on the operands the network handed it (tests/module_sites.py), through the
autograd glue of ops.py and models/: the renormalisation handoff, BatchNorm statistics from the convolution epilogue, gradient
sinks, residuals folded into the BatchNorm pass, LazyCat decoder inputs and HoleMask concatenation, the segmentation
networks' concatenations, bilinear resampling and residual sums, and the fused eval epilogue.

Runs per network: (a) bf16 training forward + ops.l1_mean backward with autograd gradients; (b) the same with engine.FlatParams
gradient sinks, parameter gradients read from the arena after the training ops.StepScope exits; (c) an eval forward in an
inference ops.StepScope with randomised BatchNorm running statistics, where a convolution and the BatchNorm + activation
fused into its epilogue are one unit.  Plus fp32 training runs of ImageFillOrigin and TextSegament (generic kernels,
handoffs that are never eligible).  Hand-built module cases reach the glue branches the networks do not reach at these shapes.
Every case records the branches it reached (module_sites.Recorder.reached); test_branch_coverage runs whatever case has not
run yet in the session and asserts that the union covers module_sites.BRANCHES."""
import time

import pytest
import torch
from torch import nn

from gpu_cases import blob
from module_sites import BRANCHES, NOT_CALLED, TABLE, Checker, Recorder
from oracle.detfill import det_fill_state_dict, det_tensor
from test_gpu_inference import _randomise_bn
from text_segmentation_image_inpainting_b200 import ops
from text_segmentation_image_inpainting_b200.engine import FlatParams
from text_segmentation_image_inpainting_b200.masks import HoleMask
from text_segmentation_image_inpainting_b200.models import MobileNetV2 as MM
from text_segmentation_image_inpainting_b200.models import image_inpainting as MI
from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
from text_segmentation_image_inpainting_b200.models import text_segmentation as MT
from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
NETS = {"ImageFillOrigin": 512, "ImageFillOriginV2": 256, "ImageFill": 256, "TextSegament": 256, "XceptionTextSegment": 256}
INPAINT = {"ImageFillOrigin", "ImageFillOriginV2", "ImageFill"}
REACHED = {}                  # case -> the BRANCHES it reached (cases that passed)


def _expected_units(net, rec):
    """(names of the table modules the forward must call, names of those a parent bypasses).  Bypassed, each by name: the
    last block of a DoublePartialResidual / residual PartialInvertedResidual (the parent calls its convolution and BatchNorm
    itself to fold the residual), and in eval the BatchNorm + activation tail of a PartialBlock whose convolution applied it
    in its epilogue"""
    root = type(net).__name__
    names = {(n or root) for n, m in net.named_modules() if type(m) in TABLE and n.split(".")[-1] not in NOT_CALLED}
    bypassed = set()
    for n, m in net.named_modules():
        if isinstance(m, MI.DoublePartialResidual):
            bypassed.add(f"{n}.conv2")
        if isinstance(m, MM.PartialInvertedResidual) and m.res_connect:
            bypassed.add(f"{n}.conv.2")
    for u in rec.units:
        if isinstance(u.module, PC.PartialConv) and u.facts.get("epi_fused"):
            bypassed.add(u.name.rsplit(".", 1)[0] + ".1")
    assert bypassed <= names, sorted(bypassed - names)[:4]
    return names - bypassed, bypassed


def _check_units(rec, net, label):
    called = {u.name for u in rec.units}
    want, bypassed = _expected_units(net, rec)
    missing = sorted(want - called)
    assert not missing, f"{label}: table modules never called (so never checked): {missing[:8]}"
    assert not (called & bypassed), f"{label}: modules listed as bypassed were called: {sorted(called & bypassed)[:4]}"
    assert len(called) == len(want), (len(called), len(want))
    print(f"{label}: {len(called)} table modules checked ({len(rec.units)} calls), {len(bypassed)} bypassed by their parent")


def _run(net, call, dev, dtype, label, sinks=None, train=True):
    rec = Recorder().attach(net)
    rec.with_sinks = sinks is not None
    try:
        with ops.StepScope(dev, training=train):
            if train:
                ops.l1_mean(call()).backward()
            else:
                with torch.no_grad():
                    call()
        torch.cuda.synchronize()
    finally:
        rec.detach()
    rec.finish(sinks.sinks if sinks is not None else ())
    if sinks is not None:
        # sinks on parameters no kernel writes (nn.Linear biases, the scSE spatial weight) stay unused: autograd accumulates
        # into the arena view instead, and Checker.params compares every gradient either way
        assert any(rec.sinks_used), f"{label}: no gradient sink was written"
        if any(getattr(p, "_pcb_grad_sink", None) is not None and p._pcb_grad_sink.used for n, p in net.named_parameters()
               if p.dim() == 1 and (n.endswith("feature_conv.bias") or (n.endswith(".bias") and "bn" not in n and ".1." not in n))):
            rec.features.add("bias_grad_sink")
    t0 = time.time()
    Checker(rec, dev, dtype, label).run()
    print(f"{label}: checked in {time.time() - t0:.1f} s")
    return rec


def _net(name, dev):
    torch.manual_seed(0)
    mod = MI if name in INPAINT else MT
    net = getattr(mod, name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    return net.to(dev).train()


def _call(net, name, hw, dtype, dev, seed):
    x = det_tensor(f"module_sites.{seed}", (2, 3, hw, hw))
    if name not in INPAINT:
        xin = x.to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
        return lambda: net(xin)
    mask = torch.from_numpy(random_hole_masks(2, hw, hw, seed=seed)).to(dev)
    if dtype == BF:
        buf = torch.zeros((2, 8, hw, hw), dtype=dtype, device=dev).contiguous(memory_format=torch.channels_last)
        xin = buf[:, :3]
        xin.copy_(x.to(dev) * mask)
    else:
        xin = (x.to(dev) * mask).contiguous(memory_format=torch.channels_last)
    hm = HoleMask.from_dense(mask, channel_uniform=True)
    return lambda: net((xin, hm))


def _network_case(name, mode, dtype=BF):
    dev = torch.device("cuda:0")
    hw = NETS[name] if dtype == BF else 256
    net = _net(name, dev)
    label = f"{name} {'bf16' if dtype == BF else 'fp32'} {mode}"
    flat = FlatParams(net) if mode == "sinks" else None
    if mode == "eval":
        _randomise_bn(net, seed=len(name))
        net.eval()
    ops.bump_weight_epoch()
    rec = _run(net, _call(net, name, hw, dtype, dev, seed=len(name)), dev, dtype, label, flat, train=mode != "eval")
    _check_units(rec, net, label)
    return rec.reached()


# ------------------------------------------------------------------------------------------------ hand-built module cases
class _Twice(nn.Module):
    """the same block applied twice in one pass"""

    def __init__(self, block):
        super().__init__()
        self.block = block

    def forward(self, args):
        return self.block(self.block(args))


def _hand(name, dev):
    """(module, input x, input mask, dtype, with sinks) of one hand case"""
    lk = nn.LeakyReLU(0.2)
    if name == "bn_c12_nonvector":                 # c % 8 != 0: no handoff eligibility, the non-vector BatchNorm path
        mod, cin, hw, dt = PC.partial_convolution_block(8, 12, 3, 1, 1, activation=lk), 8, 20, BF
    elif name == "bn_eval_backward":                # eval-mode BatchNorm with a gradient
        mod, cin, hw, dt = PC.partial_convolution_block(16, 16, 3, 1, 1, activation=lk), 16, 16, BF
    elif name == "weight_used_twice":
        mod, cin, hw, dt = _Twice(PC.partial_convolution_block(64, 64, 3, 1, 1, activation=lk)), 64, 16, BF
    elif name == "rowpacked_input_grad":
        mod, cin, hw, dt = PC.partial_convolution_block(8, 32, 3, 1, 1, activation=nn.ReLU()), 8, 20, BF
    elif name == "dense_mask_fallback":             # 12 distinct planes: past PCB_MAX_PARTS
        mod, cin, hw, dt = PC.partial_convolution_block(12, 16, 3, 1, 1, BN=False, activation=False, bias=True), 12, 16, BF
    else:
        raise KeyError(name)
    mod.load_state_dict(det_fill_state_dict(mod.state_dict()))
    mod = mod.to(dev).train()
    if name == "bn_eval_backward":
        mod[1].eval()
    x = det_tensor(f"module_sites.{name}", (2, cin, hw, hw)).to(dev).to(dt).contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    if name == "dense_mask_fallback":
        m = blob(2, cin, hw, hw, 5, per_channel=True).to(dev)
        hm = HoleMask.from_dense(m, channel_uniform=False)
        assert len(hm.parts) > 8
    else:
        hm = HoleMask.from_plane(blob(2, 1, hw, hw, 7)[:, 0].to(dev).to(torch.uint8).contiguous(), cin)
    return mod, x, hm, dt, name == "weight_used_twice"


HAND = ["bn_c12_nonvector", "bn_eval_backward", "weight_used_twice", "rowpacked_input_grad", "dense_mask_fallback"]


class _Head(nn.Module):
    def __init__(self, mod):
        super().__init__()
        self.mod = mod

    def forward(self, args):
        out = self.mod(args)
        return out[0] if isinstance(out, tuple) else out


def _hand_case(name):
    dev = torch.device("cuda:0")
    mod, x, hm, dt, sinks = _hand(name, dev)
    net = _Head(mod)
    flat = FlatParams(net) if sinks else None
    ops.bump_weight_epoch()
    rec = _run(net, lambda: net((x, hm)), dev, dt, name, flat)
    if name == "weight_used_twice":
        w = mod.block[0].feature_conv.weight
        assert sum(u.module is mod.block[0] for u in rec.units) == 2 and w._pcb_grad_sink.used
    assert x.grad is not None
    return rec.reached()


CASES = {**{f"{n}-{m}": (lambda n=n, m=m: _network_case(n, m)) for n in NETS for m in ("autograd", "sinks", "eval")},
         "ImageFillOrigin-fp32": lambda: _network_case("ImageFillOrigin", "autograd", F32),
         "TextSegament-fp32": lambda: _network_case("TextSegament", "autograd", F32),
         **{f"hand-{h}": (lambda h=h: _hand_case(h)) for h in HAND}}


def _case(name):
    if name not in REACHED:
        REACHED[name] = CASES[name]()
    return REACHED[name]


@pytest.mark.parametrize("mode", ["autograd", "sinks", "eval"])
@pytest.mark.parametrize("name", sorted(NETS))
def test_network_modules_vs_fp64(name, mode):
    _case(f"{name}-{mode}")


def test_image_fill_origin_fp32_modules_vs_fp64():
    _case("ImageFillOrigin-fp32")


def test_text_segament_fp32_modules_vs_fp64():
    _case("TextSegament-fp32")


@pytest.mark.parametrize("name", HAND)
def test_hand_module_cases_vs_fp64(name):
    _case(f"hand-{name}")


@pytest.mark.timeout(900)
def test_branch_coverage():
    """the union of every case (each run here if it has not run yet) reaches every glue branch of module_sites.BRANCHES"""
    reached = set().union(*(_case(c) for c in CASES))
    missing = sorted(set(BRANCHES) - reached)
    assert not missing, f"glue branches no case reached: {missing}"

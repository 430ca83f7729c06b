"""The cyclical learning rate on the device and the training-state checkpoint (engine.CyclicLR, TrainStep.state_dict /
load_state_dict) on the GPU:

  * pcb_lr_cyclic against the reference's own CyclicLR (the staged, unmodified models/utils/cls.py) over >= 3 cycles:
    triangular and triangular2 bit-identical in fp32 and fp64 (the kernel rounds every operation once, in numpy's order);
    exp_range, whose gamma ** iteration is CUDA's pow (within 2 ulp), equal to fp32(ref) or one ulp away and within 4 ulp in
    fp64;
  * pcb_sgd_step_dev bitwise equal to pcb_sgd_step_scaled at the same rate (one templated kernel), and each step of a changing
    rate within the fp64 bound of test_gpu_glue_ops.py's SGD cases;
  * the captured scheduled step against the reference recipe (oracle network, torch.optim.SGD, the reference's CyclicLR),
    warm-up updates counted on both sides;
  * resume in graph mode (TrainStep, and SegLossTrainStep with its batcher): the loaded state is bitwise the saved one, and
    the replays that follow track the uninterrupted run within the rounding of the unordered split-K weight gradients;
  * torch.optim.SGD interop and the refusals on the device step; a two-rank resume (skipped below 2 devices)."""
import importlib.util
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_cases import ROOT
from kernel_harness import assert_within, traced
from oracle import pconv_torch as O
from oracle.detfill import det_fill_state_dict, det_tensor
from text_segmentation_image_inpainting_b200 import _lib, ops
from text_segmentation_image_inpainting_b200.engine import CyclicLR, SegLossTrainStep, TrainStep, _flat_view

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _ref_cyclic():
    from oracle.stage_reference import reference_dir
    ref = reference_dir()
    path = os.path.join(ref, "models", "utils", "cls.py") if ref else None
    if path is None or not os.path.exists(path):
        pytest.skip("reference not staged in oracle/_ref")
    spec = importlib.util.spec_from_file_location("reference_cls", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.CyclicLR


class _StubOptimizer:
    def __init__(self):
        self.param_groups = [{}]


def _reference_rates(mode, base, top, step, gamma, k, count):
    """rates of iterations k+1 .. k+count as the reference sets them: batch_step() before every batch"""
    s = _ref_cyclic()(_StubOptimizer(), base, top, step_size=step, mode=mode, gamma=gamma, last_batch_iteration=k)
    out = []
    with np.errstate(over="ignore"):            # triangular2: numpy's 2.0 ** (cycle - 1) overflows to inf past cycle 1024
        for _ in range(count):
            s.batch_step()
            out.append(float(s.optimizer.param_groups[0]["lr"]))
    return out


SCHEDULES = {
    "tri_s1": ("triangular", 1e-3, 6e-3, 1, 1.0, -1),
    "tri_recipe_s7": ("triangular", 1e-4, 4e-4, 7, 1.0, -1),
    "tri_recipe_resume": ("triangular", 1e-4, 4e-4, 7, 1.0, 100),
    "tri2_recipe_s7": ("triangular2", 1e-4, 4e-4, 7, 1.0, -1),
    "tri2_s1_resume": ("triangular2", 1e-3, 6e-3, 1, 1.0, 12),
    # base 0: the rate is height * 2^-(cycle-1) itself, so iteration 2047's subnormal 4e-4 * 2^-1023 and iteration 2049's 0 (numpy's
    # 2.0 ** 1024 overflows to inf) both show
    "tri2_s1_past_cycle_1024": ("triangular2", 0.0, 4e-4, 1, 1.0, 2040),
    "exp_recipe_s7": ("exp_range", 1e-4, 4e-4, 7, 0.99994, -1),
    "exp_s1_resume": ("exp_range", 1e-3, 6e-3, 1, 0.9, 20),
}


@pytest.mark.parametrize("name", sorted(SCHEDULES))
def test_lr_cyclic_kernel_matches_reference(name):
    mode, base, top, step, gamma, k = SCHEDULES[name]
    count = 3 * 2 * step + 3
    want = _reference_rates(mode, base, top, step, gamma, k, count)
    sched = CyclicLR(base, top, step, mode, gamma, last_batch_iteration=k)
    code = CyclicLR.MODES[mode]
    it = torch.tensor([k + 1], dtype=torch.int64, device="cuda")
    lr32 = torch.full((1,), float("nan"), device="cuda")
    lr64 = torch.full((), float("nan"), dtype=torch.float64, device="cuda")

    def check(records):
        assert set(records) == {("lr_cyclic_kernel", ())} and records[("lr_cyclic_kernel", ())] == 1, sorted(records)
    traced(name, lambda: ops.lr_cyclic(it, lr32, lr64, base, top, step, code, gamma), check, [(it, k + 1), (lr32, float("nan"))])
    assert int(it) == k + 2
    it.fill_(k + 1)
    got32, got64 = [], []
    for _ in range(count):
        ops.lr_cyclic(it, lr32, lr64, base, top, step, code, gamma)
        got32.append(lr32.clone())
        got64.append(lr64.clone())
    got32, got64 = torch.cat(got32).cpu(), torch.stack(got64).cpu()
    assert int(it) == k + 1 + count
    ref = torch.tensor(want, dtype=torch.float64)
    ref32 = ref.float()
    if mode == "exp_range":
        up, down = torch.nextafter(ref32, torch.full_like(ref32, math.inf)), torch.nextafter(ref32, torch.full_like(ref32, -math.inf))
        assert bool(((got32 == ref32) | (got32 == up) | (got32 == down)).all()), (got32, ref32)
        ulp = torch.tensor([math.ulp(v) for v in want], dtype=torch.float64)
        assert bool(((got64 - ref).abs() <= 4 * ulp).all()), ((got64 - ref) / ulp)
    else:
        assert torch.equal(got64, ref), [(i, a, b) for i, (a, b) in enumerate(zip(got64.tolist(), want)) if a != b][:4]
        assert torch.equal(got32, ref32)
    # the host formula (the rate a step reports before its first update) is the reference's, operation for operation
    assert [sched.rate(k + 1 + i) for i in range(count)] == want
    assert len(set(want)) > 1
    if name == "tri2_s1_past_cycle_1024":
        assert want[2047 - (k + 1)] == 4e-4 * 2.0 ** -1023 > 0.0 and want[2049 - (k + 1)] == 0.0


def _sgd_buffers(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(n, generator=g, device="cuda") for _ in range(3)]


@pytest.mark.parametrize("mom,nest", [(0.0, 0), (0.9, 0), (0.9, 1)])
def test_sgd_dev_is_bitwise_the_constant_rate_kernel(mom, nest):
    lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream
    n, lr, wd, gs = 100003, 2.5e-4, 1e-3, 0.5
    p, g, b = _sgd_buffers(n, 3)
    p1, b1, p2, b2 = p.clone(), b.clone(), p.clone(), b.clone()
    _lib.check(lib.pcb_sgd_step_scaled(p1.data_ptr(), g.data_ptr(), b1.data_ptr(), n, lr, mom, wd, nest, 0, gs, st))
    lr_dev = torch.tensor([lr], dtype=torch.float32, device="cuda")

    def check(records):
        assert set(records) == {("sgd_kernel", ("true",))}, sorted(records)
    traced("sgd_dev", lambda: ops.sgd_step_dev(p2, g, b2, lr_dev, mom, wd, bool(nest), grad_scale=gs), check, [(p2, p), (b2, b)])
    assert torch.equal(p1, p2) and torch.equal(b1, b2)
    assert not torch.equal(p1, p)


def _assert_nesterov_step(name, p, buf, p0, b0, g, lr, mom, wd, gs=1.0):
    """p, buf: the kernel's fp32 result of one Nesterov step from the stored p0, b0 and gradient g at rate lr; against
    torch.optim.SGD in fp64 on the same values, with test_gpu_glue_ops.py's bound (each product and sum rounds once)"""
    p64 = torch.nn.Parameter(p0.double())
    p64.grad = g.double() * gs
    opt = torch.optim.SGD([p64], lr=lr, momentum=mom, weight_decay=wd, nesterov=True)
    opt.state[p64]["momentum_buffer"] = b0.double().clone()
    opt.step()
    P, G = p0.double(), g.double() * gs
    d = G + wd * P
    e_d = 3 * U * (G.abs() + wd * P.abs())
    b = mom * b0.double() + d
    e_b = e_d + 2 * U * (mom * b0.double().abs() + d.abs())
    assert_within(f"{name}: momentum buffer", buf, opt.state[p64]["momentum_buffer"], e_b)
    dn = d + mom * b
    e_dn = e_d + mom * e_b + 2 * U * (d.abs() + mom * b.abs())
    assert_within(f"{name}: parameters", p, p64.detach(), lr * e_dn + 2 * U * (P.abs() + lr * dn.abs()))


def test_sgd_dev_steps_with_a_changing_rate_track_torch_fp64():
    """four steps at the rates of a triangular2 schedule; each one against torch.optim.SGD in fp64 on the kernel's own stored
    state, with test_gpu_glue_ops.py's bound (starting from the zero buffer: the first step needs no flag)"""
    n, gs = 77777, 0.5
    mom, wd = (float(torch.tensor(v, dtype=torch.float32)) for v in (0.9, 1e-3))      # the values the kernel multiplies by
    p, _, _ = _sgd_buffers(n, 5)
    buf = torch.zeros(n, device="cuda")
    it = torch.zeros(1, dtype=torch.int64, device="cuda")
    lr32, lr64 = torch.zeros(1, device="cuda"), torch.zeros((), dtype=torch.float64, device="cuda")
    rates = set()
    for t in range(4):
        g = _sgd_buffers(n, 10 + t)[1]
        p0, b0 = p.clone(), buf.clone()
        ops.lr_cyclic(it, lr32, lr64, 1e-3, 4e-3, 3, _lib.CLR_TRIANGULAR2)
        ops.sgd_step_dev(p, g, buf, lr32, mom, wd, True, grad_scale=gs)
        lr = float(lr32)
        rates.add(lr)
        _assert_nesterov_step(f"step {t}", p, buf, p0, b0, g, lr, mom, wd, gs)
    assert len(rates) == 4


# ------------------------------------------------------------------------------------------------ the captured step
def _inpaint_setup(seed=5):
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    net = ImageFillOrigin()
    sd0 = det_fill_state_dict(net.state_dict())
    net.load_state_dict(sd0)
    x = det_tensor("engine.x", (2, 3, 256, 256))
    mask = torch.from_numpy(random_hole_masks(2, 256, 256, seed=seed))
    return net, sd0, x, mask


RECIPE = dict(momentum=0.9, weight_decay=1e-3, nesterov=True)
# segmentation resume in fp32, measured on an H100: over five resumes the three replays after the load stayed within 3.6e-5 of
# the uninterrupted run's losses and its parameters within 6.6e-3 of how far they moved; two runs never interrupted (eight steps
# apart from the same start) within 2.4e-4 and 3.9e-2.  A momentum or rate that was not restored moves both by far more.
SEG_LOSS_TOL, SEG_PARAM_TOL = 1e-3, 5e-2


def test_captured_scheduled_step_follows_the_reference_recipe():
    """graph replays with CyclicLR(1e-4, 4e-4, step_size=2, triangular2) against the oracle stepped by torch.optim.SGD and the
    reference's CyclicLR; the three warm-up updates of warmup_and_capture are iterations 0-2 on both sides.  The losses agree
    to the bf16 step's tolerance; that the captured SGD node consumes the scheduled rate is checked tightly on every replay: the
    parameter and momentum arenas against one fp64 Nesterov step at fp32(the reference's rate) from the arenas before the
    replay and the gradient it left behind (a rate off by more than a few ulp fails)."""
    ref_clr = _ref_cyclic()
    net, sd0, x, mask = _inpaint_setup()
    warm, replays = 3, 4
    sd = O.clone_state_dict(sd0, requires_grad=True)
    opt = torch.optim.SGD([v for v in sd.values() if v.requires_grad], lr=1.0, **RECIPE)
    sched = ref_clr(opt, 1e-4, 4e-4, step_size=2, mode="triangular2")
    ref, rates = [], []
    for _ in range(warm + replays):
        sched.batch_step()
        opt.zero_grad(set_to_none=True)
        loss = O.image_fill_origin(sd, x * mask, mask, training=True).abs().mean()
        loss.backward()
        opt.step()
        ref.append(float(loss))
        rates.append(float(opt.param_groups[0]["lr"]))
    ts = TrainStep(net.cuda(), lr_schedule=CyclicLR(1e-4, 4e-4, step_size=2, mode="triangular2"), use_graph=True, **RECIPE)
    xd, md = x.cuda(), mask.cuda()
    ts.warmup_and_capture(xd, md, eager_warmup=2)
    assert ts.graph is not None and ts.iteration == warm
    assert float(ts.last_lr) == rates[warm - 1]
    mom, wd = (float(torch.tensor(RECIPE[k], dtype=torch.float32)) for k in ("momentum", "weight_decay"))
    fl = ts.flat
    got, got_rates = [], []
    for j in range(replays):
        p0, b0 = fl.flat_p.clone(), fl.flat_m.clone()
        got.append(float(ts.step(xd, md)))
        got_rates.append(float(ts.last_lr))
        lr = float(torch.tensor(rates[warm + j], dtype=torch.float32))
        _assert_nesterov_step(f"replay {j}", fl.flat_p, fl.flat_m, p0, b0, fl.flat_g, lr, mom, wd)
    assert ts.iteration == warm + replays
    assert got_rates == rates[warm:], (got_rates, rates[warm:])
    assert all(abs(a - b) <= 1e-2 * abs(b) for a, b in zip(got, ref[warm:])), (got, ref[warm:])
    assert ref[-1] != ref[0] and len(set(rates)) > 2


# ------------------------------------------------------------------------------------------------ resume
def _momentum_views(ts):
    return [_flat_view(ts.flat.flat_m, o, p.data) for p, o in zip(ts.flat.params, ts.flat.offsets)]


def _assert_state_is(ts, sd):
    """ts's live state equals the saved one bitwise"""
    for k, v in ts.net.state_dict().items():
        assert torch.equal(v.cpu(), sd["model"][k]), k
    for i, m in enumerate(_momentum_views(ts)):
        assert torch.equal(m.cpu(), sd["optimizer"]["state"][i]["momentum_buffer"]), i
    assert ts.iteration == sd["last_batch_iteration"] + 1
    if "batcher_rng" in sd:
        assert torch.equal(ts.batcher.rng.cpu(), sd["batcher_rng"])


def _assert_tracks(losses_a, losses_b, params_a, params_b, saved, loss_tol, param_tol):
    """The first loss after the resume is the forward of the restored state on the same batch (1e-4: the BatchNorm statistics
    are unordered sums too); the updates that follow
    carry the unordered split-K weight-gradient sums, so later losses and the parameters agree within the network's own
    run-to-run spread: loss_tol relative, parameters within param_tol of how far they moved since the save."""
    assert abs(losses_a[0] - losses_b[0]) <= 1e-4 * abs(losses_a[0]), (losses_a, losses_b)
    assert all(abs(a - b) <= loss_tol * abs(a) for a, b in zip(losses_a, losses_b)), (losses_a, losses_b)
    moved = max(float((params_a[k] - saved[k]).abs().max()) for k in params_a)
    diff = max(float((params_a[k] - params_b[k]).abs().max()) for k in params_a)
    print(f"resume: loss A {losses_a} B {losses_b}; parameters differ by {diff:.3e}, moved {moved:.3e}")
    assert moved > 0 and diff <= param_tol * moved, (diff, moved)


def _params(ts):
    return {k: v.detach().float().cpu().clone() for k, v in ts.net.named_parameters() if v.requires_grad}


def test_train_step_resume_in_graph_mode(tmp_path):
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    net, _, x, mask = _inpaint_setup(seed=9)
    xd, md = x.cuda(), mask.cuda()
    sched = dict(base_lr=1e-3, max_lr=4e-3, step_size=2, mode="triangular")
    k, m = 3, 3
    a = TrainStep(net.cuda(), lr_schedule=CyclicLR(**sched), use_graph=True, **RECIPE)
    a.warmup_and_capture(xd, md)
    for _ in range(k):
        a.step(xd, md)
    path = tmp_path / "ckpt.pt"
    torch.save(a.state_dict(), path)
    saved = {k_: v.float() for k_, v in torch.load(path)["model"].items()}
    la = [float(a.step(xd, md)) for _ in range(m)]
    pa = _params(a)
    a.close()

    torch.manual_seed(123)
    b = TrainStep(ImageFillOrigin().cuda(), lr_schedule=CyclicLR(**sched), use_graph=True, **RECIPE)
    b.warmup_and_capture(xd, md)
    sd = torch.load(path)
    b.load_state_dict(sd)
    _assert_state_is(b, sd)
    lb = [float(b.step(xd, md)) for _ in range(m)]
    _assert_tracks(la, lb, pa, _params(b), saved, 2e-3, 5e-2)
    assert b.iteration == 3 + k + m


def test_seg_loss_train_step_resume_with_batcher_in_graph_mode(tmp_path):
    """fp32 compute, so that the replays after the resume differ from the uninterrupted run only by fp32 rounding of the
    unordered sums (in bf16 a one-ulp difference can flip a weight's bf16 rounding and grow over a few steps)"""
    import seg_ref as S
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    src = [S.sources(40 + i, h, w) for i, (h, w) in enumerate([(300, 420), (512, 380)])]
    sched = dict(base_lr=1e-4, max_lr=4e-4, step_size=2, mode="exp_range", gamma=0.9)

    def make(seed, batcher_seed):
        torch.manual_seed(seed)
        net = TS.TextSegament()
        if seed == 0:
            net.load_state_dict(det_fill_state_dict(net.state_dict()))
        bat = SegBatcher(2, (512, 512), image_size=128, seed=batcher_seed, compute_dtype=torch.float32)
        bat.stage(src)
        ts = SegLossTrainStep(net.cuda(), bat, BinaryFocalLoss(), lr_schedule=CyclicLR(**sched), use_graph=True, **RECIPE)
        ts.warmup_and_capture(eager_warmup=2)
        return ts

    def run(ts, count):
        losses, draws = [], []
        for _ in range(count):
            ts.batcher.stage(src)
            losses.append(float(ts.step()))
            draws.append(ts.batcher.params.clone())
        return losses, draws

    k, m = 2, 3
    a = make(0, 11)
    run(a, k)
    path = tmp_path / "seg.pt"
    torch.save(a.state_dict(), path)
    saved = {k_: v.float() for k_, v in torch.load(path)["model"].items()}
    la, da = run(a, m)
    pa = _params(a)
    a.close()

    b = make(7, 99)                             # other weights, other generator seed: the load replaces both
    sd = torch.load(path)
    assert "batcher_rng" in sd
    b.load_state_dict(sd)
    _assert_state_is(b, sd)
    lb, db = run(b, m)
    assert all(torch.equal(x, y) for x, y in zip(da, db))        # the same crops and jitter draws
    _assert_tracks(la, lb, pa, _params(b), saved, SEG_LOSS_TOL, SEG_PARAM_TOL)


# ------------------------------------------------------------------------------------------------ interop
def test_torch_sgd_checkpoints_load_and_continue():
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    # 1. a torch.optim.SGD state dict over ALL of net.parameters() of the reference-shaped module (frozen mask convolutions
    #    included, without state)
    cpu_net = ImageFillOrigin()
    cpu_net.load_state_dict(det_fill_state_dict(cpu_net.state_dict()))
    every = list(cpu_net.parameters())
    assert any(not p.requires_grad for p in every)
    opt = torch.optim.SGD(every, lr=2e-4, **RECIPE)
    gen = torch.Generator().manual_seed(0)
    for p in every:
        if p.requires_grad:
            p.grad = torch.randn(p.shape, generator=gen)
    opt.step()
    torch.manual_seed(1)
    ts = TrainStep(ImageFillOrigin().cuda(), lr_schedule=CyclicLR(1e-4, 4e-4, step_size=5), use_graph=False, **RECIPE)
    ts.load_state_dict({"model": cpu_net.state_dict(), "optimizer": opt.state_dict(), "last_batch_iteration": 6})
    trainable = [p for p in every if p.requires_grad]
    for p, v in zip(trainable, _momentum_views(ts)):
        assert torch.equal(v.cpu(), opt.state[p]["momentum_buffer"])
    for k, v in ts.net.state_dict().items():
        assert torch.equal(v.cpu(), cpu_net.state_dict()[k]), k

    # 2. ts.state_dict()["optimizer"] back into torch.optim.SGD: the same next update
    sd = ts.state_dict()
    params = [sd["model"][k].clone().requires_grad_(True) for k, p in ts.net.named_parameters() if p.requires_grad]
    opt2 = torch.optim.SGD(params, lr=1.0, **RECIPE)
    opt2.load_state_dict(sd["optimizer"])
    rate = float(torch.tensor(CyclicLR(1e-4, 4e-4, step_size=5).rate(7), dtype=torch.float32))
    opt2.param_groups[0]["lr"] = rate
    grads = [torch.randn(p.shape, generator=gen) for p in params]
    for p, g in zip(params, grads):
        p.grad = g
    opt2.step()
    with torch.no_grad():
        for p, g in zip(ts.flat.params, grads):
            p.grad.copy_(g)
    ts._update(False)
    assert float(ts.last_lr) == CyclicLR(1e-4, 4e-4, step_size=5).rate(7) and ts.iteration == 8
    for p, q in zip(ts.flat.params, params):
        assert torch.allclose(p.detach().cpu(), q.detach(), rtol=1e-5, atol=1e-7)
    for v, q in zip(_momentum_views(ts), params):
        assert torch.allclose(v.cpu(), opt2.state[q]["momentum_buffer"], rtol=1e-5, atol=1e-5)     # O(1) terms that cancel

    # 3. the refusals, before anything is written
    sd = ts.state_dict()
    g = sd["optimizer"]["param_groups"][0]
    before = ts.flat.flat_p.clone()
    for bad in (dict(g, momentum=0.5), dict(g, nesterov=False), dict(g, dampening=0.1), dict(g, maximize=True),
                dict(g, params=g["params"][:-1])):
        with pytest.raises(ValueError):
            ts.load_state_dict(dict(sd, optimizer=dict(sd["optimizer"], param_groups=[bad])))
    first = next(iter(sd["model"]))
    with pytest.raises(ValueError):
        ts.load_state_dict(dict(sd, model=dict(sd["model"], **{first: torch.zeros(1)})))
    assert torch.equal(ts.flat.flat_p, before)


# ------------------------------------------------------------------------------------------------ two ranks
_RANK_SCRIPT = r"""
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, {root!r})
from oracle.detfill import det_fill_state_dict
from text_segmentation_image_inpainting_b200.engine import CyclicLR, TrainStep
from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
from oracle.detfill import det_tensor
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
net = ImageFillOrigin()
net.load_state_dict(det_fill_state_dict(net.state_dict()))
ts = TrainStep(net.to(dev), lr_schedule=CyclicLR(1e-4, 4e-4, step_size=5), process_group=dist.group.WORLD, use_graph=True,
               momentum=0.9, weight_decay=1e-3, nesterov=True)
B, HW = 2, 256
x = det_tensor("ddp.x", (world * B, 3, HW, HW))[rank * B:(rank + 1) * B].to(dev)
mask = torch.from_numpy(random_hole_masks(world * B, HW, HW, seed=31))[rank * B:(rank + 1) * B].to(dev)
ts.warmup_and_capture(x, mask, eager_warmup=2)  # the supported order: capture (collectives included), then load
g = torch.Generator(device=dev).manual_seed(3)
ts.flat.flat_m.copy_(torch.randn(ts.flat.numel, generator=g, device=dev))
sd = ts.state_dict()
sd["last_batch_iteration"] = 17
if rank == 1:                                   # a checkpoint perturbed on purpose: rank 1 must end with rank 0's state
    for b in sd["optimizer"]["state"].values():
        b["momentum_buffer"].add_(0.25)
    for v in sd["model"].values():
        if v.is_floating_point():
            v.add_(0.5)
    sd["last_batch_iteration"] = 3
ts.load_state_dict(sd)


def same(expect_iter):
    ms = [torch.empty_like(ts.flat.flat_m) for _ in range(world)]
    ps = [torch.empty_like(ts.flat.flat_p) for _ in range(world)]
    its = [torch.empty_like(ts._lr_iter) for _ in range(world)]
    dist.all_gather(ms, ts.flat.flat_m)
    dist.all_gather(ps, ts.flat.flat_p)
    dist.all_gather(its, ts._lr_iter)
    return (all(torch.equal(ms[0], t) for t in ms) and all(torch.equal(ps[0], t) for t in ps)
            and [int(t) for t in its] == [expect_iter] * world)


ok_load = same(18)
loss = float(ts.step(x, mask))                  # the captured graph (overlapped all-reduce included) replays from the loaded state
torch.cuda.synchronize()
ok_step = same(19) and loss == loss
if rank == 0:
    with open({out!r}, "w") as f:
        f.write("ok" if ok_load and ok_step else f"differ: after load {{ok_load}}, after a replay {{ok_step}}")
ts.close()                                      # graphs with captured collectives must die before the communicator
dist.barrier()
dist.destroy_process_group()
"""


def test_two_rank_resume_adopts_rank0_state(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "result.txt")
    script = tmp_path / "rank.py"
    script.write_text(_RANK_SCRIPT.format(root=ROOT, out=out))
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=420)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert open(out).read() == "ok"

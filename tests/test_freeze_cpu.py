"""Frozen parameters and training in stages on one TrainStep (FlatParams(retrainable=...), TrainStep.update_trainable), on CPU:
the arena layout and checkpoint format without `retrainable` are the ones a step always had; with it, frozen parameters get
slots, the SGD ranges and all-reduce buckets cover the trainable slots only and follow update_trainable(), checkpoints load
across stages and from torch.optim.SGD(net.parameters()), and data-parallel replicas adopt rank 0's frozen parameters
(world size 2 over gloo)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from text_segmentation_image_inpainting_b200.engine import FlatParams, TrainStep, _flat_view

RECIPE = dict(lr=1e-3, momentum=0.9, weight_decay=1e-4, nesterov=True)


class Staged(torch.nn.Module):
    """An encoder of three convolution + BatchNorm stages, a head, and a mask-like convolution that is always frozen."""

    def __init__(self):
        super().__init__()
        self.encoder = torch.nn.Sequential(*[torch.nn.Sequential(torch.nn.Conv2d(8, 8, 3, bias=False), torch.nn.BatchNorm2d(8))
                                             for _ in range(3)])
        self.head = torch.nn.Conv2d(8, 3, 1, bias=True)
        self.mask_conv = torch.nn.Conv2d(1, 1, 3, bias=False)
        self.mask_conv.weight.requires_grad = False
        for m in self.modules():
            if isinstance(m, torch.nn.Conv2d):
                m.weight.data = m.weight.data.contiguous(memory_format=torch.channels_last)

    def freeze_encoder(self, free_last_blocks):
        """MobileNetV2.freeze_params: 0 freezes all stages, k the first len - k."""
        for i, stage in enumerate(self.encoder):
            stage.requires_grad_(i >= len(self.encoder) - free_last_blocks)


def _net(seed=0):
    torch.manual_seed(seed)
    return Staged()


def _old_offsets(net):
    """the arena layout of a step without `retrainable`: trainable parameters only, each padded to 4 elements"""
    offs, off = [], 0
    for p in net.parameters():
        if p.requires_grad:
            offs.append(off)
            off += (p.numel() + 3) // 4 * 4
    return offs, off


def test_without_retrainable_the_layout_and_checkpoint_are_unchanged():
    net = _net()
    net.freeze_encoder(1)
    offs, numel = _old_offsets(net)
    trainable = [p for p in net.parameters() if p.requires_grad]
    ts = TrainStep(net, use_graph=False, **RECIPE)
    assert ts.flat.params == trainable and ts.flat.offsets == offs and ts.flat.numel == numel
    assert ts.flat.ranges == [[0, numel]]
    assert ts.buckets == [[0, numel, list(range(len(trainable)))]]
    opt = ts.state_dict()["optimizer"]
    assert opt["param_groups"][0]["params"] == list(range(len(trainable))) and sorted(opt["state"]) == list(range(len(trainable)))
    # frozen parameters keep their own storage and carry no gradient sink
    assert all(not hasattr(p, "_pcb_grad_sink") for p in net.encoder[0].parameters())


def test_retrainable_slots_ranges_and_buckets_follow_update_trainable():
    net = _net()
    net.freeze_encoder(1)                               # stages 0 and 1 frozen
    ptrs = {n: p.data_ptr() for n, p in net.named_parameters()}
    ts = TrainStep(net, use_graph=False, retrainable=net.encoder, bucket_mb=1, **RECIPE)
    fp = ts.flat
    every = list(net.parameters())
    assert fp.params == [p for p in every if p is not net.mask_conv.weight]
    # every slot, frozen or not, lives in the arena; the always-frozen convolution keeps its storage
    base, end = fp.flat_p.data_ptr(), fp.flat_p.data_ptr() + 4 * fp.numel
    assert all(base <= p.data_ptr() < end for p in fp.params)
    assert net.mask_conv.weight.data_ptr() == ptrs["mask_conv.weight"]
    first_trainable = next(i for i, p in enumerate(fp.params) if p.requires_grad)
    assert fp.ranges == [[fp.offsets[first_trainable], fp.numel]]
    assert [b[:2] for b in ts.buckets] == [[fp.offsets[first_trainable], fp.numel]]
    assert sorted(i for b in ts.buckets for i in b[2]) == list(range(first_trainable, len(fp.params)))
    assert set(fp.sink_of) <= set(range(first_trainable, len(fp.params)))
    assert all(not hasattr(p, "_pcb_grad_sink") for p in fp.params[:first_trainable])

    # stage 2: everything trainable, nothing moves
    moved = {n: p.data_ptr() for n, p in net.named_parameters()}
    net.encoder.requires_grad_(True)
    ts.update_trainable()
    assert {n: p.data_ptr() for n, p in net.named_parameters()} == moved
    assert fp.ranges == [[0, fp.numel]] and [b[:2] for b in ts.buckets] == [[0, fp.numel]]
    assert sorted(i for b in ts.buckets for i in b[2]) == list(range(len(fp.params)))
    assert all(hasattr(p, "_pcb_grad_sink") for p in net.encoder.parameters())

    # a frozen stage in the middle: two ranges, and no bucket crosses the gap
    net.encoder[1].requires_grad_(False)
    ts.bucket_elems = 100
    ts.update_trainable()
    slot = {id(p): i for i, p in enumerate(fp.params)}
    lo, hi = slot[id(net.encoder[1][0].weight)], slot[id(net.encoder[2][0].weight)]
    assert fp.ranges == [[0, fp.offsets[lo]], [fp.offsets[hi], fp.numel]]
    for s, e, mem in ts.buckets:
        assert any(rs <= s and e <= re_ for rs, re_ in fp.ranges), (s, e)
        assert all(fp.params[i].requires_grad for i in mem)
    assert sorted(i for b in ts.buckets for i in b[2]) == [i for i, p in enumerate(fp.params) if p.requires_grad]

    # a parameter without a slot cannot be unfrozen: that would move its storage
    net.mask_conv.weight.requires_grad_(True)
    before = [list(r) for r in fp.ranges]
    with pytest.raises(ValueError, match="mask_conv.weight"):
        ts.update_trainable()
    assert fp.ranges == before


def test_retrainable_refuses_foreign_parameters():
    net = _net()
    with pytest.raises(ValueError):
        FlatParams(net, retrainable=torch.nn.Conv2d(1, 1, 1))


def test_overlap_reports_ignore_frozen_slots():
    net = _net()
    net.freeze_encoder(0)
    ts = TrainStep(net, use_graph=False, retrainable=net.encoder, **RECIPE)
    launched = []
    ts._comm_stream = None
    ts._launch_bucket = lambda b: launched.append(b)
    ts._hooks_installed = True
    ts._arm_overlap(True)
    for i in range(len(ts.flat.params)):
        ts._param_ready(i)
    assert launched == [0] and len(ts.buckets) == 1


def _momentum_by_param(ts):
    return {id(p): _flat_view(ts.flat.flat_m, o, p.data) for p, o in zip(ts.flat.params, ts.flat.offsets)}


def test_checkpoints_load_across_stages():
    # stage 1: encoder frozen; every slot carries a (distinct) momentum buffer
    a_net = _net(0)
    a_net.freeze_encoder(0)
    a = TrainStep(a_net, use_graph=False, retrainable=a_net.encoder, **RECIPE)
    a.flat.flat_m.copy_(torch.arange(a.flat.numel, dtype=torch.float32))
    sd1 = a.state_dict()
    every = list(a_net.parameters())
    g = sd1["optimizer"]["param_groups"][0]
    assert g["params"] == list(range(len(every)))
    assert sorted(sd1["optimizer"]["state"]) == [j for j, p in enumerate(every) if p is not a_net.mask_conv.weight]

    # ... into a stage-2 step (everything trainable) built from another seed: weights and every buffer, frozen slots' included
    b_net = _net(1)
    b = TrainStep(b_net, use_graph=False, retrainable=b_net.encoder, **RECIPE)
    b.load_state_dict(sd1)
    for k, v in b_net.state_dict().items():
        assert torch.equal(v, sd1["model"][k]), k
    mb = _momentum_by_param(b)
    for j, p in enumerate(b_net.parameters()):
        if j in sd1["optimizer"]["state"]:
            assert torch.equal(mb[id(p)], sd1["optimizer"]["state"][j]["momentum_buffer"]), j

    # ... and back: a stage-2 checkpoint into a stage-1 step
    b.flat.flat_m.normal_()
    sd2 = b.state_dict()
    a.load_state_dict(sd2)
    ma = _momentum_by_param(a)
    for j, p in enumerate(a_net.parameters()):
        if j in sd2["optimizer"]["state"]:
            assert torch.equal(ma[id(p)], sd2["optimizer"]["state"][j]["momentum_buffer"]), j

    # a checkpoint of a step without `retrainable` at stage 1 (trainable parameters only) loads into the staged step
    c_net = _net(2)
    c_net.freeze_encoder(0)
    c = TrainStep(c_net, use_graph=False, **RECIPE)
    c.flat.flat_m.normal_()
    sd_plain = c.state_dict()
    a.flat.flat_m.fill_(7.0)
    a.load_state_dict(sd_plain)
    ma = _momentum_by_param(a)
    for i, p in enumerate(q for q in a_net.parameters() if q.requires_grad):
        assert torch.equal(ma[id(p)], sd_plain["optimizer"]["state"][i]["momentum_buffer"])
    assert all(float(ma[id(p)].abs().sum()) == 0 for p in a_net.encoder.parameters())     # no state: zeros

    # without `retrainable` a frozen parameter has no slot, and a buffer for it is still refused
    with pytest.raises(ValueError):
        c.load_state_dict(sd1)


def test_torch_sgd_over_all_parameters_loads():
    """the reference's way: torch.optim.SGD(net.parameters()) after a stage-2 step, so every parameter with a gradient has a
    buffer; the frozen mask convolution never had a gradient and has none"""
    ref = _net(3)
    opt = torch.optim.SGD(ref.parameters(), **RECIPE)
    gen = torch.Generator().manual_seed(0)
    for p in ref.parameters():
        if p.requires_grad:
            p.grad = torch.randn(p.shape, generator=gen)
    opt.step()
    net = _net(4)
    net.freeze_encoder(0)
    ts = TrainStep(net, use_graph=False, retrainable=net.encoder, **RECIPE)
    ts.load_state_dict({"model": ref.state_dict(), "optimizer": opt.state_dict()})
    m = _momentum_by_param(ts)
    for p, q in zip(net.parameters(), ref.parameters()):
        if q.requires_grad:
            assert torch.equal(m[id(p)], opt.state[q]["momentum_buffer"])
    # and the step's own checkpoint loads into torch.optim.SGD over all parameters
    opt2 = torch.optim.SGD(_net(5).parameters(), **RECIPE)
    opt2.load_state_dict(ts.state_dict()["optimizer"])


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok = True
    for retrainable in (False, True):
        net = _net(10 + rank)                                  # replicas built from DIFFERENT seeds
        net.freeze_encoder(1)
        net.mask_conv.weight.data.fill_(float(rank + 1))
        TrainStep(net, use_graph=False, process_group=dist.group.WORLD, retrainable=net.encoder if retrainable else None,
                  **RECIPE)
        for name, p in net.named_parameters():
            got = [torch.empty_like(p.data) for _ in range(world)]
            dist.all_gather(got, p.data.contiguous())
            ok = ok and all(torch.equal(got[0], t) for t in got)
        ok = ok and float(net.mask_conv.weight.flatten()[0]) == 1.0
    out[rank] = ok
    dist.destroy_process_group()


def test_replicas_adopt_rank0_frozen_parameters_gloo_world2():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert dict(out) == {0: True, 1: True}

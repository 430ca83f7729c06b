"""Host side of the training schedule and checkpoints (engine.CyclicLR, TrainStep.state_dict / load_state_dict) on CPU: argument
validation, the host rate formula at exactly representable points, the checkpoint's keys, index order and logical shapes (a
channels-last convolution weight), the in-place round trip, torch.optim.SGD interop, the refusals, and the data-parallel
broadcast of momentum and counter after a resume (world size 2 over gloo)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_engine_cpu import Tiny
from text_segmentation_image_inpainting_b200.engine import CyclicLR, TrainStep, _flat_view

SCHED = dict(base_lr=1e-4, max_lr=4e-4, step_size=3, mode="triangular2")


def _step(seed=0, **kw):
    torch.manual_seed(seed)
    net = Tiny()
    kw.setdefault("lr_schedule", CyclicLR(**SCHED))
    return TrainStep(net, use_graph=False, weight_decay=1e-3, **kw)


def _momentum_views(ts):
    return [_flat_view(ts.flat.flat_m, o, p.data) for p, o in zip(ts.flat.params, ts.flat.offsets)]


@pytest.mark.parametrize("kw", [dict(scale_fn=lambda x: 1.0), dict(mode="cosine"), dict(step_size=0), dict(step_size=-2),
                                dict(base_lr=[1e-4]), dict(max_lr=float("nan")), dict(gamma=float("inf")),
                                dict(last_batch_iteration=-2), dict(last_batch_iteration=1.5)])
def test_cyclic_lr_refuses_what_the_device_cannot_run(kw):
    with pytest.raises(ValueError):
        CyclicLR(**kw)


def test_cyclic_lr_defaults_and_rates():
    s = CyclicLR()
    assert (s.base_lr, s.max_lr, s.step_size, s.mode, s.gamma, s.last_batch_iteration) == (1e-3, 6e-3, 2000, "triangular", 1.0, -1)
    # base 1, max 3, half cycle 2: every rate below is exact in fp64
    assert [CyclicLR(1.0, 3.0, 2).rate(i) for i in range(9)] == [1, 2, 3, 2, 1, 2, 3, 2, 1]
    assert [CyclicLR(1.0, 3.0, 2, "triangular2").rate(i) for i in range(9)] == [1, 2, 3, 2, 1, 1.5, 2, 1.5, 1]
    assert [CyclicLR(1.0, 3.0, 2, "exp_range", gamma=0.5).rate(i) for i in range(4)] == [1, 1.5, 1.5, 1.125]
    assert CyclicLR(1.0, 3.0, 1, "triangular2").rate(2 * 1100 + 1) == 1.0      # 2 ** (cycle - 1) overflows: scale 0


def test_scheduled_step_counter_rate_and_lr_assignment():
    ts = _step(lr_schedule=CyclicLR(**dict(SCHED, last_batch_iteration=4)))
    assert ts.iteration == 5 and ts.last_lr.dtype == torch.float64
    assert float(ts.last_lr) == CyclicLR(**SCHED).rate(5)            # before the first update: the rate it will use
    with pytest.raises(AttributeError):
        ts.lr = 1e-3
    plain = _step(lr_schedule=None)
    plain.lr = 1e-3
    assert plain.lr == 1e-3 and plain.iteration is None and plain.last_lr is None


def test_state_dict_keys_order_and_channels_last_shapes():
    ts = _step(lr_schedule=CyclicLR(**dict(SCHED, last_batch_iteration=9)))
    ts.flat.flat_m.copy_(torch.arange(ts.flat.numel, dtype=torch.float32))
    sd = ts.state_dict()
    assert set(sd) == {"model", "optimizer", "last_batch_iteration"} and sd["last_batch_iteration"] == 9
    assert list(sd["model"]) == list(ts.net.state_dict())
    assert all(v.device.type == "cpu" for v in sd["model"].values())
    g = sd["optimizer"]["param_groups"]
    assert len(g) == 1 and g[0]["params"] == [0, 1, 2, 3]
    assert {k: g[0][k] for k in ("momentum", "dampening", "weight_decay", "nesterov", "maximize")} == \
        dict(momentum=0.9, dampening=0, weight_decay=1e-3, nesterov=True, maximize=False)
    assert g[0]["lr"] == CyclicLR(**SCHED).rate(10)
    params = [p for p in ts.net.parameters() if p.requires_grad]
    state = sd["optimizer"]["state"]
    assert sorted(state) == [0, 1, 2, 3]
    for i, p in enumerate(params):
        assert state[i]["momentum_buffer"].shape == p.shape
    # the conv weight is channels-last: its arena slice is [co][kh][kw][ci]; the buffer comes back in logical [co][ci][kh][kw]
    w = state[0]["momentum_buffer"]
    assert torch.equal(w.permute(0, 2, 3, 1).reshape(-1), torch.arange(w.numel(), dtype=torch.float32))
    assert "batcher_rng" not in sd
    # the saved tensors are copies: later updates do not reach them
    ts.flat.flat_m.zero_()
    assert float(state[1]["momentum_buffer"].abs().sum()) > 0


def test_round_trip_restores_in_place():
    a = _step(seed=0, lr_schedule=CyclicLR(**dict(SCHED, last_batch_iteration=6)))
    a.flat.flat_m.normal_()
    a.net.bn.running_mean.normal_()
    a.net.bn.num_batches_tracked.fill_(17)
    sd = a.state_dict()
    b = _step(seed=1)
    ptrs = (b.flat.flat_p.data_ptr(), b.flat.flat_m.data_ptr(), b.net.bn.running_mean.data_ptr(), b._lr_iter.data_ptr())
    b.first = True
    b.load_state_dict(sd)
    assert ptrs == (b.flat.flat_p.data_ptr(), b.flat.flat_m.data_ptr(), b.net.bn.running_mean.data_ptr(), b._lr_iter.data_ptr())
    for k, v in b.net.state_dict().items():
        assert torch.equal(v, sd["model"][k]), k
    for i, m in enumerate(_momentum_views(b)):
        assert torch.equal(m, sd["optimizer"]["state"][i]["momentum_buffer"])
    assert b.iteration == 7 and float(b.last_lr) == CyclicLR(**SCHED).rate(7) and not b.first
    # without "last_batch_iteration" (a checkpoint of the reference modules) the schedule's own start is used
    del sd["last_batch_iteration"]
    b.load_state_dict(sd)
    assert b.iteration == 0


def test_torch_sgd_state_dicts_load_both_ways():
    ts = _step()
    net = ts.net
    every = list(net.parameters())
    opt = torch.optim.SGD(every, lr=0.1, momentum=0.9, weight_decay=1e-3, nesterov=True)
    for p in every:
        if p.requires_grad:
            p.grad = torch.randn_like(p)
    opt.step()                                  # momentum for the trainable parameters; the frozen conv has none
    ts.load_state_dict({"model": net.state_dict(), "optimizer": opt.state_dict()})
    trainable = [p for p in every if p.requires_grad]
    for p, m in zip(trainable, _momentum_views(ts)):
        assert torch.equal(m, opt.state[p]["momentum_buffer"])
    # and back: the step's optimizer entry loads into torch.optim.SGD over the trainable parameters
    opt2 = torch.optim.SGD(trainable, lr=0.1, momentum=0.9, weight_decay=1e-3, nesterov=True)
    opt2.load_state_dict(ts.state_dict()["optimizer"])
    for p in trainable:
        assert torch.equal(opt2.state[p]["momentum_buffer"], opt.state[p]["momentum_buffer"])


def _bad(sd):
    opt = sd["optimizer"]
    g = opt["param_groups"][0]
    bufs = opt["state"]
    yield "momentum", dict(sd, optimizer=dict(opt, param_groups=[dict(g, momentum=0.5)]))
    yield "nesterov", dict(sd, optimizer=dict(opt, param_groups=[dict(g, nesterov=False)]))
    yield "dampening", dict(sd, optimizer=dict(opt, param_groups=[dict(g, dampening=0.1)]))
    yield "maximize", dict(sd, optimizer=dict(opt, param_groups=[dict(g, maximize=True)]))
    yield "two groups", dict(sd, optimizer=dict(opt, param_groups=[g, g]))
    yield "count", dict(sd, optimizer=dict(opt, param_groups=[dict(g, params=[0, 1, 2])]))
    yield "buffer shape", dict(sd, optimizer=dict(opt, state={**bufs, 0: {"momentum_buffer": torch.zeros(5, 3, 3)}}))
    frozen_state = {**bufs, 4: {"momentum_buffer": torch.zeros(1, 1, 3, 3)}}
    yield "frozen with state", dict(sd, optimizer=dict(opt, state=frozen_state, param_groups=[dict(g, params=[0, 1, 2, 3, 4])]))
    yield "model shape", dict(sd, model=dict(sd["model"], **{"conv.bias": torch.zeros(6)}))
    yield "model keys", dict(sd, model={k: v for k, v in sd["model"].items() if k != "bn.running_var"})
    yield "no optimizer", {"model": sd["model"]}


def test_load_refuses_mismatched_state_before_writing():
    ts = _step()
    ts.flat.flat_m.normal_()
    sd = ts.state_dict()
    before = (ts.flat.flat_p.clone(), ts.flat.flat_m.clone())
    for what, bad in _bad(sd):
        with pytest.raises(ValueError):
            ts.load_state_dict(bad)
        assert torch.equal(ts.flat.flat_p, before[0]) and torch.equal(ts.flat.flat_m, before[1]), what


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ts = _step(seed=0, process_group=dist.group.WORLD)
    torch.manual_seed(100)
    ts.flat.flat_m.normal_()
    sd = ts.state_dict()
    sd["last_batch_iteration"] = 41
    if rank == 1:                               # a rank that loads a different checkpoint must adopt rank 0's
        for b in sd["optimizer"]["state"].values():
            b["momentum_buffer"].add_(1.0)
        sd["last_batch_iteration"] = 7
    ts.load_state_dict(sd)
    m = [torch.empty_like(ts.flat.flat_m) for _ in range(world)]
    it = [torch.empty_like(ts._lr_iter) for _ in range(world)]
    dist.all_gather(m, ts.flat.flat_m)
    dist.all_gather(it, ts._lr_iter)
    out[rank] = all(torch.equal(m[0], x) for x in m) and all(int(x) == 42 for x in it)
    dist.destroy_process_group()


def test_load_broadcasts_momentum_and_counter_from_rank0_gloo_world2():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert dict(out) == {0: True, 1: True}

"""Training the segmentation networks with a frozen encoder, and unfreezing it in place (TrainStep(retrainable=...),
update_trainable), on the GPU:

  * the frozen stage, captured, in fp32, for TextSegament with freeze_params(k), k in {0, 2}, and XceptionTextSegment with its
    encoder frozen: frozen parameters bitwise unchanged over the replays, every trainable update one fp64 Nesterov step from
    the arenas before it and the gradient it left behind (test_gpu_train_state.py's bound);
  * the frozen BatchNorm layers keep training mode: their running statistics after eager steps match the oracle network
    (oracle/seg_torch.py) run with the same freezing;
  * no backward and no operand refresh for any convolution or BatchNorm of the frozen prefix, and fewer launches per step than
    the all-trainable step;
  * the stage switch: no parameter moves, an evaluation graph captured before the switch still returns the logits of a freshly
    built SegEvalStep bitwise, stage-1 momentum carries over, new slots start from zeros, the schedule counter continues."""
import pytest
import torch

import seg_ref as S
from test_gpu_train_state import _assert_nesterov_step
from text_segmentation_image_inpainting_b200 import _lib, ops

pytestmark = pytest.mark.gpu

LR = 2.0 ** -10                                   # exact in fp32: the kernel's rate is the one the fp64 check uses
RECIPE = dict(momentum=0.9, weight_decay=1e-4, nesterov=True)
MOM, WD = (float(torch.tensor(RECIPE[k], dtype=torch.float32)) for k in ("momentum", "weight_decay"))
CASES = {"TextSegament_k0": ("TextSegament", 0, 128), "TextSegament_k2": ("TextSegament", 2, 128),
         "XceptionTextSegment_frozen": ("XceptionTextSegment", None, 256)}


def _net(name, k):
    """the network with deterministic weights, frozen the reference's way (k: MobileNetV2.freeze_params; None: the whole
    encoder; -1: nothing)"""
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    net = getattr(TS, name)()
    sd0 = det_fill_state_dict(net.state_dict())
    net.load_state_dict(sd0)
    if k is None:
        net.encoder.requires_grad_(False)
    elif k == "mid":                              # a frozen block between trainable ones: two SGD ranges with `retrainable`
        net.encoder.features[2:4].requires_grad_(False)
    elif k >= 0:
        net.encoder.freeze_params(k)
    return net, sd0


def _batcher(size, seed, dtype=torch.float32):
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    return SegBatcher(2, (512, 512), image_size=size, seed=seed, compute_dtype=dtype)


def _src(seed):
    return [S.sources(seed + i, h, w) for i, (h, w) in enumerate([(300, 420), (512, 380)])]


def _step(net, b, **kw):
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    kw.setdefault("lr", LR)
    return SegLossTrainStep(net, b, BinaryFocalLoss(gamma=2), **RECIPE, **kw)


def _check_updates(name, ts, p0, b0):
    fl = ts.flat
    assert fl.ranges
    for s, e in fl.ranges:
        _assert_nesterov_step(f"{name} [{s}, {e})", fl.flat_p[s:e], fl.flat_m[s:e], p0[s:e], b0[s:e], fl.flat_g[s:e], LR, MOM, WD)


CAPTURED = dict(CASES, TextSegament_mid=("TextSegament", "mid", 128))


@pytest.mark.parametrize("retrainable", [False, True], ids=["no_slots", "retrainable"])
@pytest.mark.parametrize("case", list(CAPTURED))
def test_frozen_stage_captured_updates_only_the_trainable_part(case, retrainable):
    """Without `retrainable` frozen parameters have no arena slot; with it they have one inside the arena, and the SGD runs over
    the trainable ranges only (one that does not start at 0, or two around a frozen block)"""
    name, k, size = CAPTURED[case]
    net, _ = _net(name, k)
    frozen = {n: p.detach().clone() for n, p in net.cuda().named_parameters() if not p.requires_grad}
    assert frozen and any(p.requires_grad for p in net.parameters())
    b = _batcher(size, 7)
    src = _src(80)
    b.stage(src)
    ts = _step(net, b, use_graph=True, retrainable=net.encoder if retrainable else None)
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None
    fl = ts.flat
    trainable = torch.zeros(fl.numel, dtype=torch.bool, device="cuda")
    for s, e in fl.ranges:
        trainable[s:e] = True
    if retrainable:
        assert any(not p.requires_grad for p in fl.params)
        # the encoder comes first: a frozen prefix leaves one range after it, a frozen block in the middle two
        assert (len(fl.ranges), fl.ranges[0][0] > 0) == ((2, False) if k == "mid" else (1, True))
    else:
        assert fl.ranges == [[0, fl.numel]]
    moved = torch.zeros(fl.numel, dtype=torch.bool, device="cuda")
    for j in range(3):
        p0, b0 = fl.flat_p.clone(), fl.flat_m.clone()
        b.stage(src)
        ts.step()
        torch.cuda.synchronize()
        _check_updates(f"{case} replay {j}", ts, p0, b0)
        # frozen slots: parameters and momentum bitwise as before the replay
        assert torch.equal(fl.flat_p[~trainable], p0[~trainable]) and torch.equal(fl.flat_m[~trainable], b0[~trainable])
        moved |= fl.flat_p != p0
    for n, p in net.named_parameters():
        if n in frozen:
            assert torch.equal(p.detach(), frozen[n]), n
    assert bool(moved.any())
    assert not bool(fl.flat_m[~trainable].any())             # a frozen slot's momentum was never written


def test_capture_without_eager_warmup_captures_no_frozen_refresh(monkeypatch):
    """eager_warmup=0: the operand caches are created by the step just before the capture; their modes are set before it, so
    no frozen weight is laid out inside the captured graph"""
    net, _ = _net("TextSegament", 2)
    net.cuda()
    b = _batcher(128, 7)
    b.stage(_src(80))
    ts = _step(net, b, use_graph=True)
    captured = []
    refresh = ops.Operands.refresh

    def operands_refresh(self_):
        if torch.cuda.is_current_stream_capturing():
            captured.append(id(self_.weight))
        return refresh(self_)
    monkeypatch.setattr(ops.Operands, "refresh", operands_refresh)
    ts.warmup_and_capture(eager_warmup=0)
    monkeypatch.undo()
    frozen = {id(p) for p in net.parameters() if not p.requires_grad}
    assert ts.graph is not None and captured                  # the trainable ones are refreshed by every replay
    assert not (set(captured) & frozen)
    assert all(c.frozen == (not c.current.weight.requires_grad) for _, _, c in ops.operand_caches(net) if c.current is not None)


def _bn_prefixes(net):
    """state_dict prefixes of the BatchNorm layers whose parameters are frozen"""
    return [n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d) and not m.weight.requires_grad]


@pytest.mark.parametrize("case", list(CASES))
def test_frozen_batchnorm_running_statistics_follow_the_oracle(case):
    """two eager fp32 steps on one drawn batch against two training-mode forwards of the oracle network: the frozen prefix sees
    the same input on both sides whatever the trainable part does, so its statistics must agree"""
    from oracle import pconv_torch as O
    from oracle import seg_torch as OS
    name, k, size = CASES[case]
    b = _batcher(size, 7)
    b.stage(_src(80))
    x, _ = b.prepare()
    params = b.params.cpu().numpy()
    x = x.float().cpu().contiguous()
    net, sd0 = _net(name, k)
    bns = _bn_prefixes(net)
    assert bns
    sd = O.clone_state_dict(sd0)
    fwd = OS.text_segment if name == "TextSegament" else OS.xception_text_segment
    with torch.no_grad():
        for _ in range(2):
            fwd(sd, x, training=True)
    ts = _step(net.cuda(), b, use_graph=False)
    for _ in range(2):
        ts.step(params=params)
    torch.cuda.synchronize()
    got = net.state_dict()
    for prefix in bns:
        for buf in ("running_mean", "running_var"):
            key = f"{prefix}.{buf}"
            want, have = sd[key].detach(), got[key].cpu()
            scale = float(want.abs().max())
            assert torch.allclose(have, want, rtol=1e-3, atol=1e-4 * scale), (key, float((have - want).abs().max()), scale)
        assert int(got[f"{prefix}.num_batches_tracked"]) == 2


class _Record:
    """The convolutions and BatchNorm layers whose backward runs, and the weights whose operands are laid out again, keyed by
    the parameter's id"""

    def __init__(self, monkeypatch):
        self.backward, self.refresh = set(), set()
        conv_bwd, bn_bwd, refresh = ops.PartialConvFn.backward, ops.BNActFn.backward, ops.Operands.refresh
        rec = self

        def conv_backward(ctx, *grads):
            rec.backward.add(id(ctx.weight_ref))
            return conv_bwd(ctx, *grads)

        def bn_backward(ctx, gy):
            for p in getattr(ctx, "params", ()) or ():
                if p is not None:
                    rec.backward.add(id(p))
            return bn_bwd(ctx, gy)

        def operands_refresh(self_):
            rec.refresh.add(id(self_.weight))
            return refresh(self_)
        monkeypatch.setattr(ops.PartialConvFn, "backward", staticmethod(conv_backward))
        monkeypatch.setattr(ops.BNActFn, "backward", staticmethod(bn_backward))
        monkeypatch.setattr(ops.Operands, "refresh", operands_refresh)


@pytest.mark.parametrize("case", list(CASES))
def test_no_backward_and_no_operand_refresh_in_the_frozen_prefix(case, monkeypatch):
    name, k, size = CASES[case]
    src = _src(80)
    counts = {}
    for stage in ("frozen", "all"):
        net, _ = _net(name, k if stage == "frozen" else -1)
        b = _batcher(size, 7)
        b.stage(src)
        ts = _step(net.cuda(), b, use_graph=False)
        for _ in range(2):                              # operand caches exist, frozen ones laid out once in their mode
            b.stage(src)
            ts.step()
        torch.cuda.synchronize()
        rec = _Record(monkeypatch)
        before = _lib.launch_count()
        b.stage(src)
        ts.step()
        torch.cuda.synchronize()
        counts[stage] = _lib.launch_count() - before
        monkeypatch.undo()
        frozen = {id(p) for p in net.parameters() if not p.requires_grad}
        trainable = {id(p) for p in net.parameters() if p.requires_grad}
        assert rec.backward & trainable, f"{stage}: no backward recorded at all"          # the recorder intercepts
        assert not (rec.backward & frozen), f"{stage}: backward ran for {len(rec.backward & frozen)} frozen parameters"
        assert not (rec.refresh & frozen), f"{stage}: operands of {len(rec.refresh & frozen)} frozen weights laid out again"
        conv_weights = {id(c.current.weight) for _, _, c in ops.operand_caches(net) if c.current is not None}
        assert conv_weights & trainable <= rec.refresh           # every trainable convolution is refreshed
        if stage == "frozen":
            assert all(c.frozen == (not c.current.weight.requires_grad) for _, _, c in ops.operand_caches(net) if c.current is not None)
    print(f"{case}: {counts['frozen']} launches per step frozen, {counts['all']} all-trainable")
    assert counts["frozen"] < counts["all"]


def test_stage_switch_in_place():
    """XceptionTextSegment (its forward is deterministic, so two evaluation graphs on the same weights agree bitwise): train
    with the encoder frozen, capture an evaluation, unfreeze, switch, recapture, train"""
    from text_segmentation_image_inpainting_b200.engine import CyclicLR, SegEvalStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    net, sd0 = _net("XceptionTextSegment", None)
    net.cuda()
    tb = _batcher(256, 7)
    src, eval_src = _src(80), _src(90)
    tb.stage(src)
    sched = CyclicLR(1e-4, 4e-4, step_size=3)
    ts = _step(net, tb, use_graph=True, lr_schedule=sched, retrainable=net.encoder)
    ptrs = {n: p.data_ptr() for n, p in net.named_parameters()}
    ts.warmup_and_capture(eager_warmup=2)
    for _ in range(2):
        tb.stage(src)
        ts.step()
    eb = _batcher(256, 2)
    eb.stage(eval_src)
    ev = SegEvalStep(net, eb, BinaryFocalLoss(gamma=2))
    ev.warmup_and_capture()
    torch.cuda.synchronize()
    fl = ts.flat
    enc = {id(p) for p in net.encoder.parameters()}
    enc_slots = torch.zeros(fl.numel, dtype=torch.bool, device="cuda")
    for p, o in zip(fl.params, fl.offsets):
        if id(p) in enc:
            enc_slots[o:o + p.numel()] = True
    m1, it1 = fl.flat_m.clone(), ts.iteration
    assert bool((m1[enc_slots] == 0).all()) and bool((m1[~enc_slots] != 0).any())

    net.encoder.requires_grad_(True)
    ts.update_trainable()
    assert ts.graph is None and fl.ranges == [[0, fl.numel]]
    assert torch.equal(fl.flat_m, m1) and ts.iteration == it1
    # the first stage-2 update: the encoder from zero momentum, the rest from the stage-1 buffers
    p0, b0 = fl.flat_p.clone(), fl.flat_m.clone()
    tb.stage(src)
    ts.step()
    torch.cuda.synchronize()
    lr = float(torch.tensor(sched.rate(it1), dtype=torch.float32))
    _assert_nesterov_step("first stage-2 update", fl.flat_p, fl.flat_m, p0, b0, fl.flat_g, lr, MOM, WD)
    assert bool((fl.flat_p[enc_slots] != p0[enc_slots]).any())
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None and ts.iteration == it1 + 1 + 3
    for _ in range(2):
        tb.stage(src)
        ts.step()
    torch.cuda.synchronize()
    assert {n: p.data_ptr() for n, p in net.named_parameters()} == ptrs
    assert ts.iteration == it1 + 1 + 3 + 2

    # the evaluation graph captured in stage 1 sees the stage-2 weights, bitwise as a fresh one
    eb.reseed(2)
    eb.stage(eval_src)
    old = ev.run().clone()
    copy, _ = _net("XceptionTextSegment", -1)
    copy.cuda().load_state_dict(net.state_dict())
    eb2 = _batcher(256, 2)
    eb2.stage(eval_src)
    fresh = SegEvalStep(copy, eb2, BinaryFocalLoss(gamma=2))
    new = fresh.run().clone()
    torch.cuda.synchronize()
    assert torch.equal(old, new)
    ts.close()


def test_load_refreshes_the_frozen_operands_the_captured_step_holds():
    """the frozen weights change outside the step and an eager forward gives their caches new records; load_state_dict()
    still rewrites the records the captured graph reads"""
    net, _ = _net("TextSegament", 2)
    net.cuda()
    b = _batcher(128, 7)
    b.stage(_src(80))
    ts = _step(net, b, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    held = [r for r in ts._captured_operands if not r.weight.requires_grad]
    assert held
    sd = ts.state_dict()
    for n, p in net.named_parameters():
        if not p.requires_grad:
            sd["model"][n] = sd["model"][n] * 1.5
    net.load_state_dict(sd["model"])
    with torch.no_grad():
        net(b.prepare()[0])
    torch.cuda.synchronize()
    assert any(c.current is not r for r in held for _, _, c in ops.operand_caches(net) if c.current is not None
               and c.current.weight is r.weight)
    ts.load_state_dict(sd)
    for r in held:
        fresh = ops.Operands(r.weight, r.geom)
        assert torch.equal(r.w_fwd, fresh.w_fwd)
        assert (r.w_dg is None) == (fresh.w_dg is None) and (r.w_dg is None or torch.equal(r.w_dg, fresh.w_dg))

"""GPU tests of the pixel average precision (metrics.PixelAveragePrecision, csrc/seg_loss.cu pcb_seg_score_*) and of held-out
segmentation evaluation (engine.SegEvalStep).

The histogram and the five counts are integer sums, so they are compared bit for bit with the numpy restatement
(seg_score_ref.py) on every bf16 bit pattern, on fp32 values at and beside the bf16 rounding midpoints, at the sigmoid > 0.5
threshold and the target > 0.5 label boundary, through every layout the logits arrive in.  The AP is held to the recorded
sklearn fixture and to an exact rational evaluation, and must be bit-identical however the pixels are batched.

SegEvalStep: both networks, graph against eager, fp32 against the oracle, interleaved with a captured SegLossTrainStep, and
reseeded passes.  XceptionTextSegment's eval forward is deterministic and is held bit for bit.  TextSegament's is not: the
squeeze of its scSE blocks (pcb_gap_forward) adds per-chunk partial sums with float atomics, so two runs of the same batch may
differ in the last bits and bf16 carries that through ~100 BatchNorm layers (see test_gpu_inference.py).  Its logits are
compared within NONDET_TOL instead; its score is still held exactly to the restatement on the logits the step returned."""
import os

import numpy as np
import pytest
import torch

import seg_ref as S
import seg_score_ref as R
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CL = torch.channels_last


def _score():
    from text_segmentation_image_inpainting_b200.metrics import PixelAveragePrecision
    return PixelAveragePrecision(DEV)


def _bf16_tensor(bits, shape):
    return torch.from_numpy(np.asarray(bits, np.uint16).view(np.int16).copy()).view(torch.bfloat16).reshape(shape)


def _layout(x, kind):
    """x: [n, 1, h, w] on the device -> the same logical values in the given memory layout."""
    n, _, h, w = x.shape
    if kind == "nchw":
        return x.contiguous()
    if kind in ("nhwc8", "nhwc16"):
        c = 8 if kind == "nhwc8" else 16
        buf = torch.full((n, c, h, w), float("nan"), dtype=x.dtype, device=x.device).contiguous(memory_format=CL)
        v = buf[:, :1]
        v.copy_(x)
        return v
    if kind == "transposed":
        t = x.transpose(2, 3).contiguous().transpose(2, 3)
        assert not t.is_contiguous()
        return t
    if kind == "strided":
        big = torch.full((n, 3, h, 2 * w), float("nan"), dtype=x.dtype, device=x.device)
        v = big[:, 1:2, :, ::2]
        v.copy_(x)
        return v
    raise ValueError(kind)


def _check_exact(logits, target):
    """One update on a fresh score; hist and counts must equal the restatement's."""
    sc = _score()
    sc.update(logits, target)
    torch.cuda.synchronize()
    x = logits.detach().cpu().contiguous()
    if x.dtype == torch.bfloat16:
        ref = R.score_counts(x.view(torch.int16).numpy().view(np.uint16), target.cpu().numpy(), bf16=True)
    else:
        ref = R.score_counts(x.numpy(), target.cpu().numpy())
    assert np.array_equal(sc.hist.cpu().numpy(), ref[0])
    assert np.array_equal(sc.counts_tensor.cpu().numpy(), ref[1])
    return sc, ref


def _targets(rng, size):
    """Targets on both sides of the label boundary: 0, 0.5, nextafter(0.5, 1), 1 and uniform values."""
    t = rng.random(size).astype(np.float32)
    pick = rng.integers(0, 5, size)
    t[pick == 0] = 0.5
    t[pick == 1] = np.nextafter(np.float32(0.5), np.float32(1))
    t[pick == 2] = 0.0
    t[pick == 3] = 1.0
    return t


# ------------------------------------------------------------------------------------------------ hist and counts
def test_every_bf16_bit_pattern_in_one_call():
    rng = np.random.default_rng(1)
    bits = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    x = _bf16_tensor(bits, (1, 1, 256, 256)).to(DEV)
    t = torch.from_numpy(_targets(rng, 65536).reshape(1, 1, 256, 256)).to(DEV)
    sc, (hist, counts) = _check_exact(x, t)
    assert counts[4] == 2 * 127                          # every NaN pattern: all-ones exponent, non-zero mantissa, either sign
    assert hist[0].sum() + counts[4] == 65536
    assert hist[0][0x8000] == 2                          # +0 and -0 share a key
    assert np.isnan(sc.average_precision())


def _fp32_cases(rng, size):
    """fp32 logits on and beside bf16 rounding midpoints, and in [2^-25, 2^-23) and their negatives (the threshold)."""
    base = rng.integers(0, 0x7F7F, size // 2).astype(np.uint32) | (rng.integers(0, 2, size // 2).astype(np.uint32) << 15)
    mid = (base << 16) | 0x8000
    near = (mid.astype(np.int64) + rng.integers(-1, 2, mid.size)).astype(np.uint32)
    small = rng.uniform(2.0 ** -25, 2.0 ** -23, size - size // 2).astype(np.float32)
    small[::2] *= -1
    edge = np.array([2 ** -25, 1.5 * 2 ** -24, np.nextafter(np.float32(1.5 * 2 ** -24), np.float32(1)), -2 ** -24], np.float32)
    small[:min(4, small.size)] = edge[:min(4, small.size)]
    x = np.concatenate([near.view(np.float32), small])
    return x[rng.permutation(x.size)]


LAYOUTS = ["nchw", "nhwc8", "nhwc16", "transposed", "strided"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", LAYOUTS)
def test_midpoints_thresholds_and_labels_through_every_layout(kind, dtype):
    rng = np.random.default_rng(2 + LAYOUTS.index(kind))
    n, h, w = 3, 37, 61
    x = torch.from_numpy(_fp32_cases(rng, n * h * w).reshape(n, 1, h, w)).to(dtype).to(DEV)
    t = torch.from_numpy(_targets(rng, n * h * w).reshape(n, 1, h, w)).to(DEV)
    _, (hist, counts) = _check_exact(_layout(x, kind), t)
    assert counts[0] > 0 and counts[1] > 0 and counts[2] > 0 and counts[3] > 0 and counts[4] == 0


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (1, 1, 1, 9), (1, 1, 9, 1), (4, 1, 1, 1), (2, 1, 1, 300), (5, 1, 7, 1)])
@pytest.mark.parametrize("kind", ["nchw", "nhwc8"])
def test_degenerate_shapes(shape, kind):
    rng = np.random.default_rng(sum(shape))
    size = int(np.prod(shape))
    x = torch.from_numpy(_fp32_cases(rng, max(size, 2))[:size].reshape(shape)).to(DEV)
    t = torch.from_numpy(_targets(rng, size).reshape(shape)).to(DEV)
    _check_exact(_layout(x, kind), t)


@pytest.mark.parametrize("batch,pad", [(8, 8), (16, 8), (16, 16)])
def test_training_step_logit_shapes_at_512(batch, pad):
    """The [n, 1, 512, 512] bf16 logits of TextSegament (batch 8) and XceptionTextSegment (batch 16) training at 512^2: clustered
    values, as a network's (many pixels per bin)."""
    g = torch.Generator(device=DEV).manual_seed(batch + pad)
    x = (torch.randn((batch, 1, 512, 512), generator=g, device=DEV) * 3 - 5).to(torch.bfloat16)
    t = (torch.rand((batch, 1, 512, 512), generator=g, device=DEV) < 0.1).float()
    _check_exact(_layout(x, "nhwc8" if pad == 8 else "nhwc16"), t)


# ------------------------------------------------------------------------------------------------ the AP
def test_ap_matches_the_recorded_sklearn_scores():
    g = np.load(os.path.join(GOLDEN, "seg_ap.npz"))
    for k in range(len(g["ap"])):
        bits, labels, ap = g[f"bits_{k}"], g[f"labels_{k}"].astype(np.float32), float(g["ap"][k])
        sc = _score()
        sc.update(_bf16_tensor(bits, (1, 1, 1, bits.size)).to(DEV), torch.from_numpy(labels).reshape(1, 1, 1, -1).to(DEV))
        got = sc.average_precision()
        assert abs(got - ap) <= 1e-12 * max(abs(ap), 1e-300), (k, got, ap)


def test_ap_is_bit_identical_across_calls_replays_and_batch_splits():
    rng = np.random.default_rng(7)
    x = torch.from_numpy(np.concatenate([rng.normal(-4, 3, 8 * 64 * 64 - 64), np.zeros(32), -np.zeros(32)]).astype(np.float32))
    x = x[torch.from_numpy(rng.permutation(x.numel()))].reshape(8, 1, 64, 64).to(torch.bfloat16).to(DEV)
    t = torch.from_numpy(_targets(rng, 8 * 64 * 64).reshape(8, 1, 64, 64)).to(DEV)
    results = []
    for parts in (1, 2, 8):
        sc = _score()
        for xs, ts in zip(x.chunk(parts), t.chunk(parts)):
            sc.update(_layout(xs, "nhwc8"), ts.contiguous())
        results.append((sc.hist.clone(), sc.finalize().clone(), sc.finalize().clone()))
    # a captured update, replayed over a pass of two batches
    sc = _score()
    static_x, static_t = _layout(x[:4].clone(), "nhwc8"), t[:4].clone()
    sc.update(static_x, static_t)
    torch.cuda.synchronize()
    sc.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sc.update(static_x, static_t)
    for _ in range(2):
        sc.reset()
        for half in range(2):
            static_x.copy_(x[4 * half:4 * half + 4])
            static_t.copy_(t[4 * half:4 * half + 4])
            graph.replay()
        results.append((sc.hist.clone(), sc.finalize().clone(), sc.finalize().clone()))
    torch.cuda.synchronize()
    h0, a0, _ = results[0]
    ref = R.average_precision(h0.cpu().numpy())
    assert abs(float(a0) - ref) <= 1e-12 * ref
    for h, a, b in results:
        assert torch.equal(h, h0)
        assert a.view(torch.int64).item() == a0.view(torch.int64).item() == b.view(torch.int64).item()


def test_ap_edge_values():
    sc = _score()
    x = torch.randn((2, 1, 16, 16), device=DEV)
    sc.update(x, torch.zeros_like(x))
    assert sc.average_precision() == 0.0
    sc.reset()
    sc.update(x, torch.ones_like(x))
    assert sc.average_precision() == 1.0
    assert sc.counts == {"tp": int((x > 8.940696716308594e-08).sum()), "fp": 0, "fn": int((x <= 8.940696716308594e-08).sum()),
                         "tn": 0, "nan": 0, "pixels": 512}
    x[1, 0, 3, 4] = float("nan")
    sc.update(x, torch.ones_like(x))
    assert np.isnan(sc.average_precision()) and sc.counts["nan"] == 1 and sc.counts["pixels"] == 1024


def test_finalize_with_counts_beyond_32_bits_matches_exact_rationals():
    rng = np.random.default_rng(9)
    hist = np.zeros((2, R.KEYS), np.int64)
    keys = rng.choice(R.KEYS, 3000, replace=False)
    hist[0][keys] = rng.integers(1, 2 ** 40, keys.size)
    hist[1][keys] = (hist[0][keys] * rng.random(keys.size)).astype(np.int64)
    hist[0][keys[:5]] = 2 ** 45 + 12345
    hist[1][keys[:5]] = 2 ** 44 + 777
    assert hist[0].sum() > 2 ** 32 and hist[1].sum() > 2 ** 32
    sc = _score()
    sc.hist.copy_(torch.from_numpy(hist))
    got = sc.average_precision()
    exact = float(R.average_precision_exact(hist))
    assert abs(got - exact) <= 1e-12 * exact, (got, exact)


def test_refused_updates_launch_and_write_nothing():
    from text_segmentation_image_inpainting_b200 import _lib
    sc = _score()
    sentinel = torch.arange(2 * R.KEYS, dtype=torch.int64, device=DEV).reshape(2, R.KEYS)
    sc.hist.copy_(sentinel)
    sc.counts_tensor.fill_(3)
    torch.cuda.synchronize()
    x = torch.randn((2, 1, 8, 8), device=DEV)
    t = torch.rand((2, 1, 8, 8), device=DEV)
    bad = [
        (x.cpu(), t.cpu()),                                                 # CPU tensors
        (x, t.cpu()),
        (torch.randn((2, 2, 8, 8), device=DEV), torch.rand((2, 2, 8, 8), device=DEV)),   # a second channel
        (x, torch.rand((2, 1, 8, 9), device=DEV)),                          # target of another shape
        (x, t.double()),                                                    # ... or dtype
        (x, t.to(torch.bfloat16)),
        (x, torch.rand((2, 1, 8, 8), device=DEV).transpose(2, 3)),          # non-contiguous target
        (x.half(), t),                                                      # unsupported logits dtype
        (x[:, :, :0], t[:, :, :0]),                                         # empty
    ]
    before = _lib.launch_count()
    for lg, tg in bad:
        with pytest.raises((_lib.PcbError, TypeError)):
            sc.update(lg, tg)
    torch.cuda.synchronize()
    assert _lib.launch_count() == before
    assert torch.equal(sc.hist, sentinel) and bool((sc.counts_tensor == 3).all())


# ------------------------------------------------------------------------------------------------ SegEvalStep
NETS = {"TextSegament": 128, "XceptionTextSegment": 256}
DETERMINISTIC = {"TextSegament": False, "XceptionTextSegment": True}
# logits of two runs of a non-deterministic forward on the same batch (relative L2), and their APs, agree within this
NONDET_TOL = 2e-2


def _net(name):
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    net = getattr(TS, name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    return net


def _batcher(size, seed, dtype=torch.bfloat16):
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    return SegBatcher(2, (512, 512), image_size=size, seed=seed, compute_dtype=dtype)


def _src(seed):
    return [S.sources(seed + i, h, w) for i, (h, w) in enumerate([(300, 420), (512, 380)])]


def _calibrate(net, b):
    """Running statistics = one training-mode forward's batch statistics on a prepared batch (momentum 1), so the eval
    activations are O(1); the batcher's generator is left as it was."""
    bns = [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    rng = b.rng.clone()
    for m in bns:
        m.momentum = 1.0
    net.train()
    with torch.no_grad():
        net(b.prepare()[0])
    torch.cuda.synchronize()
    for m in bns:
        m.momentum = 0.1
    b.rng.copy_(rng)


def _eager_eval(net, b, crit, sc):
    """prepare + eval-mode forward with the fused epilogues + loss + score, eagerly under no_grad."""
    from text_segmentation_image_inpainting_b200 import ops
    training = net.training
    net.eval()
    try:
        with ops.StepScope(b.device, training=False), torch.no_grad():
            x, target = b.prepare()
            out = net(x)
            loss = crit(out, target) if crit is not None else None
            sc.update(out, target)
    finally:
        net.train(training)
    torch.cuda.synchronize()
    return out.float(), loss


def _rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name,loss", [("TextSegament", "BinaryFocalLoss"), ("XceptionTextSegment", "SoftBootstrapCrossEntropy"),
                                       ("TextSegament", None)])
def test_eval_step_matches_eager_evaluation(name, loss):
    from text_segmentation_image_inpainting_b200 import loss as L
    from text_segmentation_image_inpainting_b200.engine import SegEvalStep
    from text_segmentation_image_inpainting_b200.metrics import PixelAveragePrecision
    seed = 21
    b = _batcher(NETS[name], seed)
    b.stage(_src(40))
    net = _net(name).cuda()
    _calibrate(net, b)
    net.train()
    crit = getattr(L, loss)(gamma=2) if loss == "BinaryFocalLoss" else (getattr(L, loss)() if loss else None)
    ev = SegEvalStep(net, b, crit)
    ev.warmup_and_capture()
    assert int(b.rng[1]) == 0 and net.training
    assert int(ev.score.hist.sum()) == 0 and int(ev.score.counts_tensor.sum()) == 0
    out = ev.run().clone()
    target = b.target.clone()
    hist, counts = ev.score.hist.clone(), ev.score.counts_tensor.clone()
    e_loss = None
    torch.cuda.synchronize()
    assert net.training and ev.fused_sites > 0 and out.dtype == torch.float32 and out.is_contiguous()
    # exact: the step's score is the restatement's on the step's own logits
    ref_hist, ref_counts = R.score_counts(out.cpu().numpy().astype(np.float32), target.cpu().numpy())
    assert np.array_equal(hist.cpu().numpy(), ref_hist) and np.array_equal(counts.cpu().numpy(), ref_counts)
    assert int(counts.sum()) == out.numel() and int(counts[0]) + int(counts[2]) > 0
    # against eager evaluation of the same batch
    b.reseed(seed)
    sc = PixelAveragePrecision(DEV)
    e_out, e_loss = _eager_eval(net, b, crit, sc)
    deterministic = DETERMINISTIC[name]
    if deterministic:
        assert torch.equal(out, e_out)
        assert torch.equal(hist, sc.hist) and torch.equal(counts, sc.counts_tensor)
    else:
        assert _rel_l2(out, e_out) <= NONDET_TOL
    assert torch.equal(b.target, target)
    if crit is not None:
        tol = 1e-6 if deterministic else 1e-3
        assert torch.allclose(ev.last_loss, e_loss, rtol=tol, atol=0), (float(ev.last_loss), float(e_loss))
    ap = ev.score.average_precision()
    assert abs(ap - R.average_precision(ref_hist, ref_counts)) <= 1e-12 * ap


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(NETS))
def test_eval_step_fp32_against_the_oracle(name):
    from oracle import seg_torch as OS
    from text_segmentation_image_inpainting_b200.engine import SegEvalStep
    from text_segmentation_image_inpainting_b200.metrics import PixelAveragePrecision
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    b = _batcher(NETS[name], 5, dtype=torch.float32)
    b.stage(_src(60))
    net = _net(name).cuda()
    _calibrate(net, b)
    ev = SegEvalStep(net, b, compute_dtype=torch.float32)
    out = ev.run().clone()                                   # captures first: the score counts this batch once
    x, target = b.x.float().cpu().contiguous(), b.target.cpu()
    ap, counts = ev.score.average_precision(), ev.score.counts
    assert counts["pixels"] == out.numel()
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        oracle = OS.text_segment(sd, x, training=False) if name == "TextSegament" else OS.xception_text_segment(sd, x, training=False)
    b.reseed(5)
    e_out, _ = _eager_eval(net, b, None, PixelAveragePrecision(DEV))
    assert _rel_l2(out, oracle) <= _rel_l2(e_out, oracle) + 5e-3
    assert _rel_l2(out, oracle) <= 0.1
    # the step's AP is the restatement's AP on the logits the step returned
    ref_hist, ref_counts = R.score_counts(out.cpu().numpy(), target.numpy())
    ref_ap = R.average_precision(ref_hist, ref_counts)
    assert abs(ap - ref_ap) <= 1e-12 * ref_ap
    assert dict(zip(R.COUNTS, ref_counts.tolist())) == {k: v for k, v in counts.items() if k != "pixels"}


def _state(ts):
    return [ts.flat.flat_p.clone(), ts.flat.flat_m.clone()] + [t.clone() for t in ts.net.buffers()]


def _operand_bits(ts):
    return [t.view(torch.uint8).clone() for v in ts._captured_operands if v is not None for t in v if t is not None]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", list(NETS))
def test_eval_interleaved_with_training_changes_nothing_and_sees_every_update(name):
    from text_segmentation_image_inpainting_b200.engine import SegEvalStep, SegLossTrainStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    size = NETS[name]
    tb = _batcher(size, 1)
    train_src = _src(80)
    tb.stage(train_src)
    crit = BinaryFocalLoss(gamma=2)
    net = _net(name).cuda()
    _calibrate(net, tb)
    net.train()
    ts = SegLossTrainStep(net, tb, crit, lr=1e-3, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    eb = _batcher(size, 2)
    eval_src = _src(90)
    eb.stage(eval_src)
    ev = SegEvalStep(ts.net, eb, crit)
    ev.warmup_and_capture()
    outs = []
    for _ in range(3):
        tb.stage(train_src)
        ts.step()
        torch.cuda.synchronize()
        before, ops_before = _state(ts), _operand_bits(ts)
        passes = []
        for _ in range(2):                                  # two reseeded passes of two batches: one refresh
            ev.reset()
            eb.reseed(2)
            logits = []
            for _ in range(2):
                eb.stage(eval_src)
                logits.append(ev.run().clone())
            passes.append((logits, ev.score.hist.clone(), ev.score.average_precision(), ev.last_loss.clone()))
        torch.cuda.synchronize()
        assert ts.net.training
        for a, c in zip(before, _state(ts)):
            assert torch.equal(a, c)
        for a, c in zip(ops_before, _operand_bits(ts)):
            assert torch.equal(a, c)
        deterministic = DETERMINISTIC[name]
        if deterministic:
            assert torch.equal(passes[0][1], passes[1][1]) and passes[0][2] == passes[1][2]
        outs.append(passes[-1])
        # a fresh evaluation step on a copy of the state at this point
        copy = _net(name).cuda()
        copy.load_state_dict(ts.net.state_dict())
        eb2 = _batcher(size, 2)
        eb2.stage(eval_src)
        fresh = SegEvalStep(copy, eb2, BinaryFocalLoss(gamma=2))
        fresh.warmup_and_capture()
        f_logits = []
        for _ in range(2):
            eb2.stage(eval_src)
            f_logits.append(fresh.run().clone())
        f_ap = fresh.score.average_precision()
        if deterministic:
            assert all(torch.equal(a, c) for a, c in zip(f_logits, outs[-1][0]))
            assert torch.equal(fresh.score.hist, outs[-1][1]) and f_ap == outs[-1][2]
            assert torch.allclose(fresh.last_loss, outs[-1][3], rtol=1e-6, atol=0)
        else:
            rel = [_rel_l2(a, c) for a, c in zip(f_logits, outs[-1][0])]
            assert max(rel) <= NONDET_TOL and abs(f_ap - outs[-1][2]) <= NONDET_TOL, (rel, f_ap, outs[-1][2])
    assert not torch.equal(outs[0][0][0], outs[-1][0][0])      # the evaluations followed the updates
    assert 0.0 <= outs[-1][2] <= 1.0


@pytest.mark.parametrize("name", list(NETS))
def test_reseeded_validation_passes_repeat(name):
    from text_segmentation_image_inpainting_b200.engine import SegEvalStep
    sizes = [[(300, 420), (512, 380)], [(260, 261), (400, 512)], [(512, 512), (333, 444)]]
    sources = [[S.sources(100 + 10 * i + j, h, w) for j, (h, w) in enumerate(s)] for i, s in enumerate(sizes)]
    b = _batcher(NETS[name], 3)
    b.stage(sources[0])
    net = _net(name).cuda()
    _calibrate(net, b)
    ev = SegEvalStep(net, b)
    ev.warmup_and_capture()
    passes = []
    for _ in range(2):
        ev.reset()
        b.reseed(3)
        outs = []
        for src in sources:
            b.stage(src)
            outs.append((ev.run().clone(), b.target.clone()))
        passes.append((outs, ev.score.hist.clone(), ev.score.counts_tensor.clone(), ev.score.finalize().clone()))
    torch.cuda.synchronize()
    same = DETERMINISTIC[name]
    for (o1, t1), (o2, t2) in zip(passes[0][0], passes[1][0]):
        assert torch.equal(t1, t2)
        assert torch.equal(o1, o2) if same else _rel_l2(o1, o2) <= NONDET_TOL
    if same:
        assert torch.equal(passes[0][1], passes[1][1]) and torch.equal(passes[0][2], passes[1][2])
        assert passes[0][3].view(torch.int64).item() == passes[1][3].view(torch.int64).item()
    # either way the pass's score is the restatement's over the logits the step returned, pixel for pixel
    x = torch.cat([o for o, _ in passes[1][0]]).cpu().numpy()
    t = torch.cat([t for _, t in passes[1][0]]).cpu().numpy()
    ref_hist, ref_counts = R.score_counts(x, t)
    assert np.array_equal(passes[1][1].cpu().numpy(), ref_hist) and np.array_equal(passes[1][2].cpu().numpy(), ref_counts)
    assert int(passes[1][2].sum()) == 3 * passes[1][0][0][0].numel()

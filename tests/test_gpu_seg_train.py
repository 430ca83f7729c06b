"""The segmentation training step on the reference's data and losses (engine.SegLossTrainStep): graph replays against eager
steps on the same staged batch and draws, and three fp32 SGD steps against the oracle network (oracle/seg_torch.py), the
reference's own loss module and torch.optim.SGD."""
import numpy as np
import pytest
import torch

import seg_ref as S

pytestmark = pytest.mark.gpu


def _net(name="TextSegament"):
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    net = getattr(TS, name)()
    sd0 = det_fill_state_dict(net.state_dict())
    net.load_state_dict(sd0)
    return net, sd0


def _sources(sizes, seed):
    return [S.sources(seed + i, h, w) for i, (h, w) in enumerate(sizes)]


@pytest.mark.parametrize("loss_name", ["BinaryFocalLoss", "SoftBootstrapCrossEntropy"])
def test_graph_replays_match_eager_steps(loss_name):
    from text_segmentation_image_inpainting_b200 import loss as L
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep
    sizes = [(300, 420), (512, 380)]
    src = _sources(sizes, 70)
    kw = dict(lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False)
    crit = getattr(L, loss_name)()
    bg = SegBatcher(2, (512, 512), image_size=128, seed=11)
    bg.stage(src)
    ts = SegLossTrainStep(_net()[0].cuda(), bg, crit, use_graph=True, **kw)
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None
    counter = int(bg.rng[1])
    be = SegBatcher(2, (512, 512), image_size=128, seed=11)
    be.reseed(11, counter)
    eager = SegLossTrainStep(_net()[0].cuda(), be, getattr(L, loss_name)(), use_graph=False, **kw)
    for _ in range(3):
        bg.stage(src)
        be.stage(src)
        lg = ts.step()
        le = eager.step()
        torch.cuda.synchronize()
        assert torch.equal(bg.params, be.params)
        assert torch.equal(bg.x, be.x) and torch.equal(bg.target, be.target)
        # the batch is bit-identical; the bf16 network's reductions (BatchNorm statistics, split-K) run in no fixed order
        assert np.isfinite(float(lg)) and abs(float(lg) - float(le)) <= 2e-3 * abs(float(le)), (float(lg), float(le))


def test_three_fp32_sgd_steps_track_the_oracle_and_the_reference_loss():
    from oracle import pconv_torch as O
    from oracle import seg_torch as OS
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    ref_loss = S.reference_loss_module()
    if ref_loss is None:
        pytest.skip("reference not staged in oracle/_ref")
    b = SegBatcher(2, (512, 512), image_size=128, seed=7, compute_dtype=torch.float32)
    b.stage(_sources([(300, 420), (512, 380)], 80))
    x, target = b.prepare()
    params = b.params.cpu().numpy()
    x, target = x.float().cpu().contiguous(), target.cpu()
    net, sd0 = _net()
    kw = dict(lr=1e-3, momentum=0.9, weight_decay=1e-4, nesterov=True)
    sd = O.clone_state_dict(sd0, requires_grad=True)
    opt = torch.optim.SGD([v for v in sd.values() if v.requires_grad], **kw)
    crit_ref = ref_loss.BinaryFocalLoss(gamma=2)
    ref = []
    for _ in range(3):
        opt.zero_grad(set_to_none=True)
        loss = crit_ref(OS.text_segment(sd, x, training=True), target)
        loss.backward()
        opt.step()
        ref.append(float(loss))
    ts = SegLossTrainStep(net.cuda(), b, BinaryFocalLoss(gamma=2), use_graph=False, **kw)
    got = [float(ts.step(params=params)) for _ in range(3)]
    assert all(abs(a - r) <= 1e-2 * abs(r) for a, r in zip(got, ref)), (got, ref)
    assert ref[-1] != ref[0] and got[-1] != got[0]


def test_capture_after_a_partial_convolution_step_in_the_same_process():
    """A partial-convolution training step leaves the mask and prefetch streams behind; capturing a segmentation step (which
    never uses the mask stream) afterwards must not wait on them."""
    from test_gpu_inpaint_data import _small_net
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep, TrainStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    x = torch.rand(2, 3, 256, 256, device="cuda")
    m = torch.ones(2, 3, 256, 256, device="cuda")
    m[:, :, 64:160, 80:176] = 0
    pconv = TrainStep(_small_net().cuda(), lr=1e-3, use_graph=False)
    pconv.step(x, m)
    torch.cuda.synchronize()
    mask_stream = ops._aux_stream("mask", x.device)
    assert mask_stream in pconv._scope.streams
    b = SegBatcher(2, (512, 512), image_size=128, seed=3)
    b.stage(_sources([(300, 420), (512, 380)], 90))
    ts = SegLossTrainStep(_net()[0].cuda(), b, BinaryFocalLoss(), lr=1e-3, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None
    assert mask_stream not in ts._scope.streams          # the scope of the capture
    losses = []
    for _ in range(2):
        b.stage(_sources([(300, 420), (512, 380)], 90))
        losses.append(float(ts.step()))
    torch.cuda.synchronize()
    assert all(np.isfinite(v) for v in losses)

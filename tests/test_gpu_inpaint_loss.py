"""The inpainting loss on the GPU (text_segmentation_image_inpainting_b200/loss.py, csrc/inpaint_loss.cu): fp32 mode against the
reference's goldens, bf16 mode against the emulating oracle, the Gram products against fp64, exact features away from holes,
the ReLU backward in the data-gradient epilogue, and the training step: graph replay against eager, SGD against the oracle,
two ranks.  The kernels of inpaint_loss.cu one by one: test_gpu_inpaint_loss_kernels.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import inpaint_loss as OL
from oracle import pconv_torch as O
from test_inpaint_loss_golden_cpu import CASES, load_case

pytestmark = pytest.mark.gpu
CL = torch.channels_last


def _criterion(seed=0):
    from text_segmentation_image_inpainting_b200 import loss as L
    vgg = L.VggExtractor(pretrained=False)
    vgg.load_state_dict(OL.vgg_state_dict(seed))
    return L.InpaintingLoss(vgg.cuda())


def _rel(a, b):
    return float((a.double().cpu() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _run(crit, clean, mask, output):
    out = output.cuda().requires_grad_(True)
    c = clean.cuda()
    loss = crit(c * mask.cuda(), mask.cuda(), out, c)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach().cpu(), crit.last_terms.cpu(), out.grad


@pytest.mark.parametrize("name", CASES)
def test_fp32_against_reference_goldens(name):
    g, clean, mask, output = load_case(name)
    loss, terms, grad = _run(_criterion(int(g["cfg"][2])), clean, mask, output)
    assert abs(float(loss) - float(g["loss"])) <= 1e-3 * abs(float(g["loss"]))
    for k in range(5):
        ref = float(g["terms"][k])
        assert abs(float(terms[k]) - ref) <= 1e-3 * abs(ref) + 1e-9, (OL.TERMS[k], float(terms[k]), ref)
    assert _rel(grad, torch.from_numpy(g["grad"])) <= 2e-3


@pytest.mark.parametrize("name", CASES[:2])
def test_bf16_against_emulating_oracle(name):
    from text_segmentation_image_inpainting_b200 import ops
    g, clean, mask, output = load_case(name)
    ob = output.to(torch.bfloat16).float()
    sd = OL.vgg_state_dict(0)
    with O.storage(torch.bfloat16):
        o = ob.clone().requires_grad_(True)
        lo = OL.inpainting_loss(clean * mask, mask, o, clean, sd)
        lo.backward()
    crit = _criterion(0)
    n, _, h, w = output.shape
    out = ops.padded_empty(n, 3, h, w, torch.bfloat16, torch.device("cuda"))     # the networks' NHWC channel-padded output
    with torch.no_grad():
        out.copy_(ob.cuda())
    out.requires_grad_(True)
    c = clean.cuda()
    loss = crit(c * mask.cuda(), mask.cuda(), out, c)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(lo)) <= 2e-3 * abs(float(lo))
    assert out.grad.dtype == torch.bfloat16
    assert _rel(out.grad.float(), o.grad) <= 5e-2


def test_features_away_from_holes_are_exact():
    """With holes and output != origin, comp equals origin outside the holes, so every feature whose receptive field holds no
    hole pixel is bit-identical in F(comp) and F(origin), and the perceptual gradient arriving there is exactly 0."""
    from text_segmentation_image_inpainting_b200 import _lib
    from text_segmentation_image_inpainting_b200.loss import _Vgg
    g, clean, _, output = load_case("inpaint_loss_b1_128")
    crit = _criterion(0)
    n, _, h, w = output.shape
    mask = torch.ones((n, 3, h, w))
    mask[:, :, 40:60, 30:75] = 0                      # one hole block: plenty of feature pixels far from it at every stage
    c = clean.cuda()
    out = output.cuda().to(torch.bfloat16)
    hole = (mask[:, :1] == 0).float()
    # receptive field of stage k: 3x3 convs and 2x2 pools -> a feature pixel sees a box of the input; dilate the hole mask by it
    reach = {0: (2, 6), 1: (6, 16), 2: (16, 44)}     # (pool factor, conservative half-width in input pixels) per stage
    feats = []
    for img in (c * mask.cuda() + (1 - mask.cuda()) * out.float(), c):
        feats.append(crit.feature_encoder(img.to(torch.bfloat16)))
    checked = 0
    for k, (fa, fo) in enumerate(zip(*feats)):
        s, r = 2 ** (k + 1), reach[k][1]
        near = F.max_pool2d(F.pad(hole, (r, r, r, r)), 2 * r + 1, 1)                  # any hole within r pixels
        far = F.max_pool2d(near, s, s)[:, 0] == 0                                    # [n, h/s, w/s] feature pixels far from holes
        assert far.any() and not far.all()
        a, b = fa.float().cpu().permute(0, 2, 3, 1)[far], fo.float().cpu().permute(0, 2, 3, 1)[far]
        assert torch.equal(a, b), k
        checked += int(far.sum())
    assert checked > 0
    # the perceptual-only gradient of stage 0 at those pixels: sign(F(comp) - F(origin)) = 0 there, checked through the kernel
    lib = _lib.load()
    f0 = feats[0][0]
    stack = torch.cat([f0, f0, feats[1][0]]).contiguous(memory_format=torch.channels_last)     # comp | output(=comp) | origin
    df = torch.empty_like(stack[:2 * n])
    one = torch.ones((), device="cuda")
    _lib.check(lib.pcb_feature_loss_backward(stack.data_ptr(), 1, n, stack.shape[2] * stack.shape[3], stack.shape[1], None, None, 1.0,
                                             0.0, one.data_ptr(), df.data_ptr(), None))
    torch.cuda.synchronize()
    hole0 = F.max_pool2d(F.max_pool2d(F.pad(hole, (6,) * 4), 13, 1), 2, 2)[:, 0] == 0
    assert torch.equal(df[:n].float().cpu().permute(0, 2, 3, 1)[hole0], torch.zeros_like(df[:n].float().cpu().permute(0, 2, 3, 1)[hole0]))
    assert float(df[:n].float().abs().sum()) > 0


def test_dgrad_relu_epilogue_matches_separate_pass():
    """The ReLU backward applied in the TMA-fed data-gradient epilogue equals the data gradient followed by the separate
    activation-backward pass, bit for bit (a select on the same bf16 values)."""
    import ctypes

    from text_segmentation_image_inpainting_b200 import _lib, ops
    from text_segmentation_image_inpainting_b200.loss import _Vgg
    crit = _criterion(0)
    vgg = _Vgg(crit.feature_encoder.encoder, 1)
    conv = crit.feature_encoder.encoder.stage_convs(0)[1]               # 64 -> 64
    torch.manual_seed(4)
    m, h, w = 2, 64, 128
    x = torch.relu(torch.randn(m, 64, h, w, device="cuda")).to(torch.bfloat16).contiguous(memory_format=CL)
    dc = torch.randn(m, 64, h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    geom = vgg._geom(x, conv)
    c = geom.struct([x])
    lib = _lib.load()
    assert lib.pcb_conv_dgrad_fuses_relu(ctypes.byref(c)) == 1
    wprep = vgg.operands(conv, geom)
    fused = vgg.dgrad(conv, x, wprep, dc, relu_in=True)
    plain = vgg.dgrad(conv, x, wprep, dc, relu_in=False)
    sep = vgg.relu_backward(plain, x)
    torch.cuda.synchronize()
    assert torch.equal(fused, sep)
    assert int((fused == 0).sum()) > int((plain == 0).sum())


def test_gram_matches_fp64():
    from text_segmentation_image_inpainting_b200.loss import gram_matrix
    torch.manual_seed(1)
    f = torch.relu(torch.randn(3, 128, 32, 32)).to(torch.bfloat16)
    g = gram_matrix(f.cuda().contiguous(memory_format=CL)).cpu().double()
    fd = f.double().view(3, 128, -1)
    ref = torch.bmm(fd, fd.transpose(1, 2)) / (128 * 32 * 32)
    assert float((g - ref).abs().max() / ref.abs().max()) <= 1e-5


def test_total_variation_matches_reference_formula():
    from text_segmentation_image_inpainting_b200.loss import total_variation_loss
    img = torch.rand(2, 3, 24, 40)
    ref = OL.total_variation_loss(img.double())
    assert abs(float(total_variation_loss(img.cuda())) - float(ref)) <= 1e-6 * float(ref)


def test_train_step_graph_replay_matches_eager():
    from test_gpu_inpaint_data import _small_net, _sources
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintLossTrainStep
    from text_segmentation_image_inpainting_b200.loss import VggExtractor
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(OL.vgg_state_dict(0))
    vgg = vgg.cuda()
    src = _sources([(300, 420), (512, 380)], 40)
    b = InpaintBatcher(2, (512, 512), image_size=256, add_random_masks=True, seed=5)
    b.stage(src)
    kw = dict(lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False)
    ts = InpaintLossTrainStep(_small_net().cuda(), b, vgg, use_graph=True, **kw)
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None
    # the frozen VGG is not in the gradient arena
    assert ts.flat.true_numel == sum(p.numel() for p in ts.net.parameters() if p.requires_grad)
    assert not any(p.requires_grad for p in vgg.parameters())
    loss = float(ts.step())
    terms = ts.last_terms.clone()
    torch.cuda.synchronize()
    params = b.params.cpu().numpy()                                  # what the replay drew
    eager = InpaintLossTrainStep(_small_net().cuda(), b, vgg, use_graph=False, **kw)
    le = float(eager.step(params=params))
    torch.cuda.synchronize()
    assert np.isfinite(loss) and abs(loss - le) <= 1e-5 * abs(le), (loss, le)
    assert torch.allclose(terms, eager.last_terms, rtol=1e-5, atol=0)
    assert float(terms[3]) > 0 and float(terms[4]) > 0


def test_train_step_sgd_tracks_oracle():
    """Three steps with the optimiser (SGD + Nesterov + weight decay) on one fp32 batch against torch.optim.SGD on the CPU
    oracle of the network and the loss: the loss trajectories agree."""
    from oracle.detfill import det_fill_state_dict
    from test_gpu_inpaint_data import _sources
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintLossTrainStep
    from text_segmentation_image_inpainting_b200.loss import VggExtractor
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    vsd = OL.vgg_state_dict(0)
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(vsd)
    b = InpaintBatcher(2, (512, 512), image_size=256, add_random_masks=True, seed=7, compute_dtype=torch.float32)
    b.stage(_sources([(300, 420), (512, 380)], 50))
    _, hm, clean = b.prepare()
    params = b.params.cpu().numpy()
    x, mask = clean.cpu(), hm.dense().cpu()
    net = ImageFillOrigin()
    sd0 = det_fill_state_dict(net.state_dict())
    net.load_state_dict(sd0)
    kw = dict(lr=1e-3, momentum=0.9, weight_decay=1e-4, nesterov=True)
    sd = O.clone_state_dict(sd0, requires_grad=True)
    opt = torch.optim.SGD([v for v in sd.values() if v.requires_grad], **kw)
    ref = []
    for _ in range(3):
        opt.zero_grad(set_to_none=True)
        out = O.image_fill_origin(sd, x * mask, mask, training=True)
        loss = OL.inpainting_loss(x * mask, mask, out, x, vsd)
        loss.backward()
        opt.step()
        ref.append(float(loss))
    ts = InpaintLossTrainStep(net.cuda(), b, vgg.cuda(), use_graph=False, **kw)
    got = [float(ts.step(params=params)) for _ in range(3)]
    assert all(abs(a - r) <= 1e-2 * abs(r) for a, r in zip(got, ref)), (got, ref)
    assert ref[-1] != ref[0] and got[-1] != got[0]


_RANK_SCRIPT = r"""
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
from oracle.detfill import det_fill_state_dict
from oracle.inpaint_loss import vgg_state_dict
from test_gpu_inpaint_data import _sources
from text_segmentation_image_inpainting_b200.data import InpaintBatcher
from text_segmentation_image_inpainting_b200.engine import InpaintLossTrainStep
from text_segmentation_image_inpainting_b200.loss import VggExtractor
from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
rank = int(os.environ["RANK"])
torch.cuda.set_device(rank)
dev = torch.device("cuda", rank)
dist.init_process_group("nccl", device_id=dev)
net = ImageFillOrigin()
net.load_state_dict(det_fill_state_dict(net.state_dict()))
vgg = VggExtractor(pretrained=False)
vgg.load_state_dict(vgg_state_dict(0))
b = InpaintBatcher(2, (512, 512), image_size=256, add_random_masks=True, seed=11 + rank)
b.stage(_sources([(300, 420), (512, 380)], 60 + 2 * rank))
ts = InpaintLossTrainStep(net.to(dev), b, vgg.to(dev), lr=1e-3, process_group=dist.group.WORLD, use_graph={graph})
ts.warmup_and_capture(eager_warmup=2)
loss = float(ts.step())
torch.cuda.synchronize()
torch.save({{"p": ts.flat.flat_p.cpu(), "loss": loss}}, {out!r}.format(rank))
ts.close()
dist.barrier()
dist.destroy_process_group()
"""


@pytest.mark.parametrize("graph", [False, True])
def test_two_rank_train_step(tmp_path, graph):
    """Two ranks over NCCL on different batches: both finish with finite losses and identical parameters (the gradient exchange
    keeps the replicas together)."""
    import socket
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from conftest import ROOT
    out = str(tmp_path / "rank{}.pt")
    script = tmp_path / "rank.py"
    script.write_text(_RANK_SCRIPT.format(root=ROOT, out=out, graph=graph))
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), str(script)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    r0, r1 = torch.load(out.format(0)), torch.load(out.format(1))
    assert np.isfinite(r0["loss"]) and np.isfinite(r1["loss"]) and r0["loss"] != r1["loss"]
    assert torch.equal(r0["p"], r1["p"])

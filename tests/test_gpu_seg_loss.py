"""The segmentation losses as modules (loss.BinaryFocalLoss, loss.SoftBootstrapCrossEntropy): every constructor's reduction
option, output value and shape, and gradient against direct kernel calls and the fp64 oracle (oracle/seg_loss.py), fp32 and
bf16 logits, dense and the channel-padded view the networks return; the bootstrap indicator against torch's CPU sigmoid for
every bf16 value and a dense fp32 sweep; determinism; graph replay; the Xception output view fed in place.  The kernels
themselves, element by element against the fp64 oracle at every dtype, layout, reduction and call-site geometry, are
tests/test_gpu_seg_loss_kernels.py."""
import numpy as np
import pytest
import torch

from oracle import seg_loss as OL

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24


def _padded(x):
    """x [n, 1, h, w] as the [:, :1] view of an 8-channel NHWC buffer (ops.bilinear_upsample's output layout)."""
    n, _, h, w = x.shape
    buf = torch.empty((n, 8, h, w), dtype=x.dtype, device="cuda", memory_format=torch.channels_last).zero_()
    buf[:, :1].copy_(x)
    return buf[:, :1]


def _inputs(seed, shape=(3, 1, 40, 56), hard=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * 3
    x.view(-1)[::11] = torch.tensor([0.0, 1e-9, -1e-9, 8.9e-8, 9e-8, 1.2e-7, -20.0, 20.0]).repeat(x.numel())[: x.view(-1)[::11].numel()]
    t = (torch.rand(shape, generator=g) < 0.3).float() if hard else torch.rand(shape, generator=g)
    if not hard:
        t.view(-1)[::5] = 0
        t.view(-1)[2::9] = 1
    return x, t


def _grad_scale(kind, x, t, kw, gout):
    """Per element, the size of what the fp32 gradient sums: w f (gamma |s| sig(xs) bce + sig(x) + |t|) |gout| / N."""
    x, t = x.numpy().astype(np.float64).ravel(), t.numpy().astype(np.float64).ravel()
    n = x.size if kw.get("reduction", "mean") == "mean" else 1
    if kind == "focal":
        gamma = kw.get("gamma", 0)
        w = np.where(t > 0, 2.0, 1.0)
        s = 2 * t - 1
        f = np.exp(gamma * OL.log_sigmoid(-x * s))
        return w * f * (gamma * np.abs(s) * OL.sigmoid(x * s) * OL.bce(x, t) + OL.sigmoid(x) + np.abs(t)) * np.abs(gout) / n
    w = np.where(t > 0, 2.0, 1.0)
    return w * (OL.sigmoid(x) + np.abs(t) + 0.05) * np.abs(gout) / n


def _oracle(kind, x32, t, kw, gout):
    if kind == "focal":
        loss, grad = OL.focal(x32.numpy().ravel(), t.numpy().ravel(), **kw)
    else:
        loss, grad = OL.bootstrap(x32.numpy().ravel(), t.numpy().ravel(), x32=x32.numpy().ravel(), **kw)
    return loss, grad * gout


CASES = [("focal", {"gamma": 0}), ("focal", {"gamma": 2}), ("bootstrap", {"reduction": "mean"}), ("bootstrap", {"reduction": "sum"}),
         ("bootstrap", {"reduction": "none"})]


def _module(kind, kw):
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss, SoftBootstrapCrossEntropy
    if kind == "focal":
        return BinaryFocalLoss(gamma=kw["gamma"])
    red = kw["reduction"]
    return SoftBootstrapCrossEntropy(size_average=red != "sum", reduce=red != "none")


def _direct(kind, kw, x, t, gout=None, dx=None):
    """the kernels called directly through the C ABI with the loss, reduction and fp32 coefficients the case names (not the
    module's): the forward output (gout None), else the backward into dx"""
    import ctypes

    from text_segmentation_image_inpainting_b200 import _lib
    lib = _lib.load()
    n, _, h, w = x.shape
    loss = _lib.SEG_FOCAL if kind == "focal" else _lib.SEG_BOOTSTRAP
    red = {"mean": _lib.SEG_MEAN, "sum": _lib.SEG_SUM, "none": _lib.SEG_NONE}[kw.get("reduction", "mean")]
    coefs = (float(kw["gamma"]), 0.0, 1.0, 2.0) if kind == "focal" else (0.95, 1 - 0.95, 1.0, 2.0)
    code = _lib.PCB_BF16 if x.dtype == torch.bfloat16 else _lib.PCB_F32
    xs = (ctypes.c_longlong * 4)(*x.stride())
    st = torch.cuda.current_stream().cuda_stream
    if gout is None:
        out = torch.full((n * h * w, 1) if red == _lib.SEG_NONE else (), float("nan"), device="cuda")
        partials = torch.empty(lib.pcb_seg_loss_partials(n * h * w), dtype=torch.float64, device="cuda")
        counter = torch.zeros(1, dtype=torch.int32, device="cuda")
        _lib.check(lib.pcb_seg_loss_forward(x.data_ptr(), code, xs, t.data_ptr(), n, h, w, loss, red, *coefs, partials.data_ptr(),
                                            counter.data_ptr(), out.data_ptr(), st))
        return out
    _lib.check(lib.pcb_seg_loss_backward(x.data_ptr(), code, xs, t.data_ptr(), n, h, w, loss, red, *coefs, gout.data_ptr(), dx.data_ptr(),
                                         (ctypes.c_longlong * 4)(*dx.stride()), st))
    return dx


@pytest.mark.parametrize("layout", ["dense", "padded"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("hard", [False, True])
def test_loss_and_gradient_against_the_fp64_oracle(case, dtype, layout, hard):
    """The modules with each reduction option (BinaryFocalLoss(gamma=0 / 2); SoftBootstrapCrossEntropy() mean,
    size_average=False sum, reduce=False none), a scalar upstream gradient of 0.75 or a per-element one.  The output has the
    reduction's shape ((n*h*w, 1) for none, () otherwise) and equals, bit for bit, the forward kernel called directly with
    the case's loss and reduction codes, so a module that maps its options to the wrong code fails.  The gradient equals
    fl32(g * gs) of the raw per-element gradient g (an fp32 call with gs = 1: focal mean with gout = count, bootstrap sum with
    gout = 1), gs = fl32(fl64(gout) / count) for mean, gout for sum and gout_e for none, stored in the logits' dtype.  Both
    are also within the stated tolerances of the fp64 oracle."""
    kind, kw = CASES[case]
    x, t = _inputs(case + 10 * hard, hard=hard)
    xd = x.to(dtype)
    x32 = xd.float()                                       # the values the kernel sees
    xin = (_padded(xd.cuda()) if layout == "padded" else xd.cuda()).requires_grad_(True)
    crit = _module(kind, kw)
    raw = []
    xin.register_hook(lambda g: raw.append(g))              # the gradient as the kernel wrote it, before accumulation
    td = t.cuda()
    loss = crit(xin, td)
    n = x.numel()
    none = kw.get("reduction") == "none"
    gout = torch.rand(n, 1) + 0.5 if none else torch.tensor(0.75)
    loss.backward(gout.cuda())
    torch.cuda.synchronize()
    ref_loss, ref_grad = _oracle(kind, x32, t, kw, gout.numpy().ravel() if none else float(gout))
    got = loss.detach().cpu().double().numpy()
    if none:
        assert got.shape == (n, 1)
        scale = 2 * (np.abs(x32.double().numpy().ravel()) + 1)         # w (|x| + log 2) bounds what each element sums
        assert np.all(np.abs(got.ravel() - ref_loss) <= 8 * EPS32 * scale)
    else:
        assert got.shape == ()
        assert abs(float(got) - ref_loss) <= 1e-6 * abs(ref_loss), (float(got), ref_loss)
    direct = _direct(kind, kw, xin.detach(), td)
    torch.cuda.synchronize()
    assert direct.shape == loss.shape and torch.equal(loss.detach(), direct), "the module's output is not the kernel's for its reduction"
    g = raw[0]
    assert g.dtype == dtype and g.shape == xin.shape and g.stride() == xin.stride()
    # exactly one fp32 multiply of the raw per-element gradient
    raw_kw = dict(kw, reduction="mean" if kind == "focal" else "sum")
    g_raw = _direct(kind, raw_kw, x32.cuda(), td, torch.tensor([float(n) if kind == "focal" else 1.0], device="cuda"),
                    torch.full(tuple(x.shape), float("nan"), device="cuda"))
    torch.cuda.synchronize()
    if none:
        gs = gout.cuda().view(x.shape).double()
    else:
        gs = float(np.float32(0.75 / n)) if kw.get("reduction", "mean") == "mean" else 0.75     # fl32(fl64(0.75) / count)
    want = (g_raw.double() * gs).float().to(dtype)
    assert torch.equal(g, want), f"{int((g != want).sum())} gradient elements are not fl32(g * gs)"
    g = g.float().cpu().double().numpy().ravel()
    bound = 64 * EPS32 * _grad_scale(kind, x32, t, kw, gout.numpy().ravel() if none else float(gout))
    if dtype == torch.bfloat16:                            # one rounding of the stored gradient
        bound = bound * (1 + 2.0 ** -8) + 2.0 ** -8 * np.abs(ref_grad)
    assert np.all(np.abs(g - ref_grad) <= bound), float(np.max(np.abs(g - ref_grad) / np.maximum(bound, 1e-300)))


def _indicator_on_gpu(x32):
    """sigmoid(x) > 0.5 as the bootstrap kernel decides it, read from the reduce=False gradient at t = 0 (w = 1):
    dL/dx = sigmoid(x) - 0.05 [indicator]."""
    from text_segmentation_image_inpainting_b200.loss import SoftBootstrapCrossEntropy
    x = x32.reshape(1, 1, 1, -1).cuda().requires_grad_(True)
    loss = SoftBootstrapCrossEntropy(reduce=False)(x, torch.zeros_like(x))
    loss.backward(torch.ones_like(loss))
    g = x.grad.double().cpu().ravel()
    d = OL.sigmoid(x32.double().numpy().ravel()) - g.numpy()
    assert np.all((np.abs(d) < 1e-3) | (np.abs(d - 0.05) < 1e-3))
    return torch.from_numpy(d > 0.025)


def test_bootstrap_indicator_is_torch_cpu_sigmoid_for_every_bf16_value_and_around_zero():
    b = torch.arange(0, 65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    b = b[~torch.isnan(b.float())]
    xb = b.cuda().reshape(1, 1, 1, -1).requires_grad_(True)
    from text_segmentation_image_inpainting_b200.loss import SoftBootstrapCrossEntropy
    loss = SoftBootstrapCrossEntropy(reduce=False)(xb, torch.zeros(xb.shape, device="cuda"))
    loss.backward(torch.ones_like(loss))
    g = xb.grad.float().cpu().double().ravel().numpy()
    sig = OL.sigmoid(b.float().double().numpy())
    ind_ref = (torch.sigmoid(b.float()) > 0.5).numpy()
    # bf16 gradient: sigmoid - 0.05 ind rounded once; the two candidates are far apart in bf16 near 0.5 and share a sign elsewhere
    err_with = np.abs(g - (sig - 0.05 * ind_ref))
    err_without = np.abs(g - (sig - 0.05 * ~ind_ref))
    near = np.abs(sig - 0.5) < 0.2
    assert np.all(err_with[near] < err_without[near])
    assert np.all(err_with <= 2.0 ** -8 * np.abs(sig - 0.05 * ind_ref) + 2.0 ** -125)     # + the subnormal range
    # every float in [2^-25, 2^-23) (the threshold lies inside), and a strided sweep of all magnitudes below 2^-20
    bits = np.concatenate([np.arange(0x33000000, 0x34000000, dtype=np.int64), np.arange(0, 0x35800000, 4099, dtype=np.int64)])
    bits = bits.astype(np.int32)
    x = np.concatenate([bits.view(np.float32), -bits.view(np.float32), [OL.BOOT_THRESHOLD, np.nextafter(OL.BOOT_THRESHOLD, 1)]])
    x32 = torch.from_numpy(x.astype(np.float32))
    assert torch.equal(_indicator_on_gpu(x32), torch.sigmoid(x32) > 0.5)


def test_repeated_calls_are_bit_identical_and_graph_replay_equals_eager():
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    x, t = _inputs(3, shape=(4, 1, 256, 256))
    xd, td = _padded(x.to(torch.bfloat16).cuda()), t.cuda()
    crit = BinaryFocalLoss(gamma=2)
    outs = []
    for _ in range(3):
        xi = xd.detach().requires_grad_(True)
        loss = crit(xi, td)
        loss.backward()
        outs.append((loss.detach().clone(), xi.grad.clone()))
    assert all(torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1]) for o in outs)
    static_x = xd.detach().requires_grad_(True)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        crit(static_x, td).backward()
    torch.cuda.current_stream().wait_stream(s)
    static_x.grad = None
    with torch.cuda.graph(graph):
        static_loss = crit(static_x, td)
        static_loss.backward()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static_loss, outs[0][0]) and torch.equal(static_x.grad, outs[0][1])


def test_xception_output_view_feeds_the_loss_in_place():
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.loss import SoftBootstrapCrossEntropy
    from text_segmentation_image_inpainting_b200.models.text_segmentation import XceptionTextSegment
    net = XceptionTextSegment()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.cuda().train()
    buf = torch.empty((2, 8, 128, 128), dtype=torch.bfloat16, device="cuda", memory_format=torch.channels_last).zero_()
    buf[:, :3].copy_(torch.rand(2, 3, 128, 128))
    out = net(buf[:, :3])
    assert out.shape == (2, 1, 128, 128) and not out.is_contiguous()
    out.retain_grad()
    t = (torch.rand(2, 1, 128, 128) < 0.2).float()
    loss = SoftBootstrapCrossEntropy()(out, t.cuda())
    loss.backward()
    torch.cuda.synchronize()
    x32 = out.detach().float().cpu()
    ref_loss, ref_grad = OL.bootstrap(x32.numpy().ravel(), t.numpy().ravel(), x32=x32.numpy().ravel())
    assert abs(float(loss) - ref_loss) <= 1e-6 * abs(ref_loss)
    bound = 64 * EPS32 * _grad_scale("bootstrap", x32, t, {}, 1.0) * (1 + 2.0 ** -8) + 2.0 ** -8 * np.abs(ref_grad)
    assert np.all(np.abs(out.grad.float().cpu().double().numpy().ravel() - ref_grad) <= bound)
    assert any(p.grad is not None and bool(p.grad.abs().sum() > 0) for p in net.parameters())

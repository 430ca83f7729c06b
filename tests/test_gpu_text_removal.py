"""GPU tests of text removal: the glue kernels of csrc/text_removal.cu (ops.removal_seg_input, removal_holes,
removal_composite) bit-exact against the golden fixture recorded from the reference's own statements
(tests/golden/text_removal.npz) and against torch, and engine.TextRemovalStep end to end:

  * every stage the step leaves behind is checked against the CPU restatement (tests/text_removal_ref.py) applied to the
    step's own previous stage, exactly; the fill equals InferStep on the same U-Net input bitwise; the networks' outputs are
    within the inference tests' bounds of the fp32 oracles;
  * the launch count is the sum of its parts;
  * weight reloads on either network, a second page shape and refused inputs.

Networks: deterministic weights, BatchNorm running statistics calibrated on the test batch (as test_gpu_inference does), and
the segmentation output bias shifted so that about 0.5 % of the logits are positive (more when that leaves fewer than 5 % of
the page as hole), so both branches of the composite are exercised."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import text_removal_ref as R
from gpu_cases import ROOT
from oracle.detfill import det_fill_state_dict

pytestmark = pytest.mark.gpu

CL = torch.channels_last
DEV = torch.device("cuda:0")
DEMO = ((0.4935, 0.4563, 0.4544), (0.3769, 0.3615, 0.3566))


def _lib():
    from text_segmentation_image_inpainting_b200 import _lib as L
    return L


def _ops():
    from text_segmentation_image_inpainting_b200 import ops
    return ops


def _full8(x):
    """the whole 8-channel NHWC buffer behind a [n, 3, h, w] view"""
    n, _, h, w = x.shape
    return x.as_strided((n, 8, h, w), (h * w * 8, 1, w * 8, 8))


def _golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "text_removal.npz"))
    return g, sorted({k.split(".")[0] for k in g.files})


def _count(fn):
    before = _lib().launch_count()
    out = fn()
    return out, _lib().launch_count() - before


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("layout", ["f32_nchw", "bf16_nhwc_padded"])
def test_removal_holes_matches_golden(layout):
    ops = _ops()
    g, names = _golden()
    for name in names:
        logits = torch.from_numpy(g[name + ".logits"]).to(DEV)
        page = torch.from_numpy(g[name + ".page"]).to(DEV)
        n, _, h, w = page.shape
        if layout == "bf16_nhwc_padded":
            buf = torch.randn(n, 8, *logits.shape[2:], device=DEV).to(torch.bfloat16).contiguous(memory_format=CL)
            buf[:, :1].copy_(logits)
            logits = buf[:, :1]
        mask = ops.text_mask_postprocess(logits, tuple(int(v) for v in g[name + ".pad"]), (h, w))
        assert torch.equal(mask.cpu(), torch.from_numpy(g[name + ".mask"])), name
        hole = torch.from_numpy(g[name + ".hole"])
        want = torch.from_numpy(g[name + ".corrupted"])
        for hu, wu in (((h + 15) // 16 * 16, (w + 15) // 16 * 16), (h, w), (h + 37, w + 3)):
            for dt in (torch.float32, torch.bfloat16):
                (corrupted, valid), launches = _count(lambda: ops.removal_holes(mask, page, hu, wu, dt))
                assert launches == 1
                assert corrupted.shape == (n, 3, hu, wu) and corrupted.dtype == dt and valid.shape == (n, hu, wu)
                v, full = valid.cpu(), _full8(corrupted).cpu()
                assert torch.equal(v[:, :h, :w], 1 - hole), (name, hu, wu)
                assert not bool(v[:, h:].any()) and not bool(v[:, :, w:].any()), "the padding is hole"
                assert torch.equal(full[:, :3, :h, :w], want.to(dt)), (name, hu, wu, dt)
                assert not bool(full[:, 3:].any()), "padded channels are zero"
                assert not bool(full[:, :, h:].any()) and not bool(full[:, :, :, w:].any()), "padded pixels are zero"
        # the fixture's own mask gives the same
        corrupted, valid = ops.removal_holes(torch.from_numpy(g[name + ".mask"]).to(DEV), page, h, w, torch.float32)
        assert torch.equal(valid.cpu(), 1 - hole) and torch.equal(corrupted.cpu().contiguous(), want)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("normalize", [True, False], ids=["demo", "none"])
def test_removal_seg_input_matches_torch(normalize, dtype):
    ops = _ops()
    gen = torch.Generator().manual_seed(21)
    for n, h, w in ((1, 37, 53), (2, 64, 48), (3, 5, 9)):
        page = torch.rand((n, 3, h, w), generator=gen)
        page[0, 0, 0, :3] = torch.tensor([0.0, 1.0, 0.4935])                     # a zero, a one and the mean itself
        hs, ws = (h + 7) // 8 * 8, (w + 7) // 8 * 8
        for phs, pws in ((hs, ws), (h, w), (hs + 8, ws + 16)):
            x, launches = _count(lambda: ops.removal_seg_input(page.to(DEV), DEMO if normalize else None, phs, pws, dtype))
            assert launches == 1
            want = page.clone()
            if normalize:                                                         # torchvision's Normalize: sub_ then div_
                mean, std = (torch.as_tensor(v, dtype=torch.float32) for v in DEMO)
                want.sub_(mean[:, None, None]).div_(std[:, None, None])
            want = F.pad(want, (0, pws - w, 0, phs - h), value=0.0).to(dtype)
            full = _full8(x).cpu()
            assert x.shape == (n, 3, phs, pws) and x.dtype == dtype and ops.nhwc_layout(x) == 8
            assert torch.equal(full[:, :3], want)
            assert not bool(full[:, 3:].any())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("layout", ["nhwc_padded8", "nhwc_dense"])
def test_removal_composite_matches_where(layout, dtype):
    ops = _ops()
    gen = torch.Generator().manual_seed(22)
    for n, h, w, hu, wu in ((1, 37, 53, 48, 64), (2, 30, 20, 30, 20), (2, 61, 44, 256, 256)):
        page = torch.rand((n, 3, h, w), generator=gen)
        valid = (torch.rand((n, hu, wu), generator=gen) > 0.5).to(torch.uint8)
        f = torch.randn((n, 3, hu, wu), generator=gen).to(dtype)
        if layout == "nhwc_padded8":
            fill = ops.padded_empty(n, 3, hu, wu, dtype, DEV)
            fill.copy_(f)
            assert ops.nhwc_layout(fill) == 8
        else:
            fill = f.to(DEV).contiguous(memory_format=CL)
        out, launches = _count(lambda: ops.removal_composite(fill, page.to(DEV), valid.to(DEV)))
        assert launches == 1 and out.dtype == torch.float32 and out.shape == (n, 3, h, w) and out.is_contiguous()
        want = torch.where(valid[:, None, :h, :w].bool(), page, f[:, :, :h, :w].float())
        assert torch.equal(out.cpu(), want)
        assert torch.equal(R.composite(f, page, valid), want)


def test_removal_ops_refuse_bad_arguments():
    ops, L = _ops(), _lib()
    page = torch.rand(1, 3, 20, 30, device=DEV)
    mask = torch.zeros(1, 1, 20, 30, dtype=torch.uint8, device=DEV)
    before = L.launch_count()
    bad = [
        lambda: ops.removal_seg_input(page.cpu(), DEMO, 24, 32),
        lambda: ops.removal_seg_input(page.double(), DEMO, 24, 32),
        lambda: ops.removal_seg_input(page[:, :2], DEMO, 24, 32),
        lambda: ops.removal_seg_input(page[0], DEMO, 24, 32),
        lambda: ops.removal_seg_input(page, DEMO, 16, 32),
        lambda: ops.removal_seg_input(page, DEMO, 24, 32, torch.float16),
        lambda: ops.removal_holes(mask.float(), page, 32, 32),
        lambda: ops.removal_holes(mask[:, :, :10], page, 32, 32),
        lambda: ops.removal_holes(mask, page, 32, 16),
        lambda: ops.removal_composite(torch.zeros(1, 3, 32, 32, device=DEV), page, torch.ones(1, 16, 32, dtype=torch.uint8, device=DEV)),
        lambda: ops.removal_composite(torch.zeros(1, 3, 16, 32, device=DEV), page, torch.ones(1, 32, 32, dtype=torch.uint8, device=DEV)),
    ]
    for i, fn in enumerate(bad):
        with pytest.raises((L.PcbError, ValueError)):
            fn()
    assert L.launch_count() == before
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    v = torch.empty(1, 32, 32, dtype=torch.uint8, device=DEV)
    c = torch.empty(1, 32, 32, 8, device=DEV)
    assert lib.pcb_removal_holes(None, page.data_ptr(), 1, 20, 30, 32, 32, v.data_ptr(), c.data_ptr(), 1, st) != 0
    assert lib.pcb_removal_holes(mask.data_ptr(), page.data_ptr(), 1, 20, 30, 32, 32, v.data_ptr(), c.data_ptr(), 7, st) != 0
    assert lib.pcb_removal_holes(mask.data_ptr(), page.data_ptr(), 1, 20, 30, 19, 32, v.data_ptr(), c.data_ptr(), 1, st) != 0
    assert lib.pcb_removal_seg_input(page.data_ptr(), 1, 20, 30, None, 24, 29, c.data_ptr(), 0, st) != 0
    assert lib.pcb_removal_composite(c.data_ptr(), 0, 2, page.data_ptr(), v.data_ptr(), 1, 20, 30, 32, 32, page.data_ptr(), st) != 0
    assert L.launch_count() == before


# ------------------------------------------------------------------------------------------------ end to end
def _calibrate(net, run_train):
    """running statistics = the statistics of one training-mode forward on the test batch (momentum 1)"""
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    for m in bns:
        m.momentum = 1.0
    net.train()
    with torch.no_grad():
        run_train()
    torch.cuda.synchronize()
    for m in bns:
        m.momentum = 0.1
    net.eval()


def _rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / b.norm())


def _out_bias(seg_net):
    return [m for m in seg_net.modules() if getattr(m, "out_channels", None) == 1 and getattr(m, "bias", None) is not None][-1].bias


def _nets(seg_name, fill_name, page, seed):
    """deterministic networks on DEV, calibrated on `page`, with the segmentation bias shifted (see the module docstring)"""
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    ops = _ops()
    torch.manual_seed(seed)
    seg, fill = getattr(TS, seg_name)(), getattr(II, fill_name)()
    seg.load_state_dict(det_fill_state_dict(seg.state_dict()))
    fill.load_state_dict(det_fill_state_dict(fill.state_dict()))
    seg, fill = seg.to(DEV), fill.to(DEV)
    n, _, h, w = page.shape
    hs, ws = (h + 7) // 8 * 8, (w + 7) // 8 * 8
    m = 2 ** len(fill.decoder)
    hu, wu = (h + m - 1) // m * m, (w + m - 1) // m * m
    x = ops.removal_seg_input(page, DEMO, hs, ws, torch.bfloat16)
    _calibrate(seg, lambda: seg(x))
    with torch.no_grad():
        logits = seg(x).float().cpu()
    for q in (0.995, 0.99, 0.98, 0.95, 0.9):
        shift = float(torch.quantile(logits.flatten()[::7], q))
        hole = R.holes(R.text_mask(logits - shift, h, w))
        if 0.05 <= float(hole.float().mean()) <= 0.95:
            break
    with torch.no_grad():
        _out_bias(seg).sub_(shift)
    ops.bump_weight_epoch()
    with torch.no_grad():
        mask = ops.text_mask_postprocess(seg(x), (0, ws - w, 0, hs - h), (h, w))
    corrupted, valid = ops.removal_holes(mask, page, hu, wu, torch.bfloat16)
    _calibrate(fill, lambda: fill((corrupted, HoleMask.from_plane(valid, 3))))
    return seg, fill


def _page(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    # smooth colour fields with some texture, in [0, 1]
    base = F.interpolate(torch.rand((n, 3, h // 16 + 2, w // 16 + 2), generator=g), size=(h, w), mode="bilinear", align_corners=False)
    return (0.8 * base + 0.2 * torch.rand((n, 3, h, w), generator=g)).clamp(0, 1).to(DEV)


PAIRS = {
    "xception_origin": ("XceptionTextSegment", "ImageFillOrigin"),
    "textseg_fill": ("TextSegament", "ImageFill"),
}


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("pair", list(PAIRS))
def test_text_removal_step_end_to_end(pair):
    from oracle import pconv_torch as O
    from oracle import seg_torch as S
    from text_segmentation_image_inpainting_b200.engine import InferStep, SegInferStep, TextRemovalStep
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    ops, L = _ops(), _lib()
    seg_name, fill_name = PAIRS[pair]
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    n, h, w = 2, 300, 420
    page = _page(n, h, w, 23)
    seg, fill = _nets(seg_name, fill_name, page, 24)
    step = TextRemovalStep(seg, fill)
    (hs, ws), (hu, wu) = step.padded_sizes(h, w)
    assert (hs, ws) == (304, 424) and (hu, wu) == ((512, 512) if fill_name == "ImageFillOrigin" else (304, 432))

    out = step.run(page).clone()
    text_mask, valid, logits, fill_out = (t.clone() for t in (step.text_mask, step.valid, step.last_logits, step.last_fill))
    out2 = step.run(page).clone()
    logits2 = step.last_logits.clone()
    torch.cuda.synchronize()
    assert out.shape == (n, 3, h, w) and out.dtype == torch.float32
    assert text_mask.shape == (n, 1, h, w) and text_mask.dtype == torch.uint8 and valid.shape == (n, hu, wu)
    assert logits.shape == (n, 1, hs, ws) and fill_out.shape == (n, 3, hu, wu)

    holes = 1.0 - float(valid[:, :h, :w].float().mean())
    assert 0.05 <= holes <= 0.95, holes                                    # both branches of the composite
    # every stage against the restatement applied to the step's own previous stage
    assert torch.equal(text_mask.cpu(), R.text_mask(logits, h, w))
    v_ref, c_ref = R.unet_input(text_mask, page, hu, wu)
    assert torch.equal(valid.cpu(), v_ref)
    assert torch.equal(out.cpu(), R.composite(fill_out, page, valid))
    # the fill is InferStep's on the same U-Net input
    page_pad = F.pad(page, (0, wu - w, 0, hu - h))
    valid3 = valid[:, None].expand(n, 3, hu, wu).float().contiguous()
    infer = InferStep(fill)
    fill_ref = infer.run(page_pad, valid3).clone()
    assert torch.equal(fill_out.float(), fill_ref)
    # replays repeat wherever two eager forwards do (TextSegament's reductions use float atomics)
    x = ops.removal_seg_input(page, DEMO, hs, ws, torch.bfloat16)
    with torch.no_grad():
        e1, e2 = seg(x).float(), seg(x).float()
    if torch.equal(e1, e2):
        assert torch.equal(logits, logits2) and torch.equal(out, out2)
    # launches: the parts, without InferStep's dense-mask conversion, plus the four glue launches
    seg_step = SegInferStep(seg)
    x32 = F.pad((page - torch.tensor(DEMO[0], device=DEV)[:, None, None]) / torch.tensor(DEMO[1], device=DEV)[:, None, None],
                (0, ws - w, 0, hs - h))
    with torch.no_grad():
        eager_logits = seg_step._forward(x32).float()
    seg_step.run(x32)
    _, dense_to_plane = _count(lambda: HoleMask.from_dense(valid3, channel_uniform=True))
    assert step.launches_per_run == seg_step.launches_per_run + infer.launches_per_run - dense_to_plane + 4
    assert step.fused_sites == seg_step.fused_sites + infer.fused_sites
    assert step.unfused_sites == seg_step.unfused_sites + infer.unfused_sites
    assert step.fused_sites > 0
    # the networks against the fp32 oracles
    sd_seg = {k: v.detach().cpu() for k, v in seg.state_dict().items()}
    with torch.no_grad():
        oracle = (S.text_segment if seg_name == "TextSegament" else S.xception_text_segment)(sd_seg, x32.cpu(), training=False)
    assert _rel_l2(logits, oracle) <= _rel_l2(eager_logits, oracle) + 5e-3
    assert _rel_l2(logits, oracle) <= 0.1
    sd_fill = {k: v.detach().cpu() for k, v in fill.state_dict().items()}
    ref = {"ImageFillOrigin": O.image_fill_origin, "ImageFill": O.image_fill}[fill_name]
    m3 = valid3.cpu()
    with torch.no_grad():
        oracle_fill = ref(O.clone_state_dict(sd_fill), page_pad.cpu() * m3, m3, training=False)
    assert _rel_l2(fill_out, oracle_fill) <= 2e-2


def _fresh(seg_name, fill_name, sd_seg, sd_fill):
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    seg, fill = getattr(TS, seg_name)(), getattr(II, fill_name)()
    seg.load_state_dict({k: v.cpu() for k, v in sd_seg.items()})
    fill.load_state_dict({k: v.cpu() for k, v in sd_fill.items()})
    return TextRemovalStep(seg.to(DEV), fill.to(DEV))


def _products(step):
    return [t.clone() for t in (step.text_mask, step.valid, step.last_logits, step.last_fill)]


def _perturbed(sd):
    """a small change of every floating-point parameter and buffer but the running variances: the page keeps text and
    background, so neither network sees an input that is all hole"""
    return {k: (v * 0.99 + 0.001 if v.is_floating_point() and "running_var" not in k else v) for k, v in sd.items()}


def _same(a, b):
    """bitwise equal, NaN where NaN (a U-Net's no-holes convolution divides 0 by 0 under a window that is all hole)"""
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(), b.nan_to_num())


@pytest.mark.timeout(900)
def test_text_removal_step_reload_and_shapes():
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    page_a, page_b = _page(1, 150, 230, 25), _page(2, 97, 64, 26)
    seg, fill = _nets("XceptionTextSegment", "ImageFill", page_a, 27)
    step = TextRemovalStep(seg, fill)
    first = step.run(page_a).clone()
    first_products = _products(step)
    # a second shape captures its own graph and leaves the first shape's replays unchanged
    out_b = step.run(page_b).clone()
    assert out_b.shape == (2, 3, 97, 64) and step.valid.shape == (2, 112, 64) and len(step._graphs) == 2
    again = step.run(page_a).clone()
    assert torch.equal(again, first) and all(torch.equal(a, b) for a, b in zip(_products(step), first_products))
    # reloading the segmentation network, then the U-Net, is picked up by the next run
    for which in ("seg", "fill"):
        net = seg if which == "seg" else fill
        net.load_state_dict(_perturbed(net.state_dict()))
        out = step.run(page_a).clone()
        got = _products(step)
        fresh = _fresh("XceptionTextSegment", "ImageFill", seg.state_dict(), fill.state_dict())
        want = fresh.run(page_a).clone()
        assert _same(out, want), which
        assert all(_same(a, b) for a, b in zip(got, _products(fresh))), which
        changed = got[2] if which == "seg" else got[3]
        assert not _same(changed, first_products[2] if which == "seg" else first_products[3]), which
    # the second shape's graph follows the reloads too
    assert _same(step.run(page_b).clone(), fresh.run(page_b).clone())


def test_text_removal_step_refuses_bad_inputs():
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    L = _lib()
    seg, fill = TS.XceptionTextSegment(), II.ImageFill()
    with pytest.raises(TypeError):
        TextRemovalStep(fill, seg)
    with pytest.raises(TypeError):
        TextRemovalStep(seg, nn.Conv2d(3, 3, 3))
    with pytest.raises(TypeError):
        TextRemovalStep(nn.Conv2d(3, 1, 3), fill)
    with pytest.raises(ValueError):                                          # networks on different devices
        TextRemovalStep(seg.to(DEV), fill)
    step = TextRemovalStep(seg.to(DEV), fill.to(DEV))
    page = torch.rand(1, 3, 40, 48, device=DEV)
    before = L.launch_count()
    for bad in (page.cpu(), page.double(), page.half(), page[:, :2], torch.rand(1, 4, 40, 48, device=DEV), page[0], page[None]):
        with pytest.raises(L.PcbError):
            step.run(bad)
    with pytest.raises(L.PcbError):
        step.run(page.cpu().numpy())
    assert L.launch_count() == before and not step._graphs and step.text_mask is None

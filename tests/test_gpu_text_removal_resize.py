"""GPU tests of EvaluateSet's page resize in text removal: the kernels behind ops.page_resize_bicubic (csrc/text_removal.cu)
bit-exact against the golden fixture recorded from the reference's own EvaluateSet (tests/golden/evaluate_set.npz) and against
the numpy restatement of Pillow's resampler (tests/evaluate_set_ref.py), and engine.TextRemovalStep(..., seg_resize=600)
end to end: every stage product against the restatement applied to the step's own previous stage, the networks against
SegInferStep and InferStep on the step's own inputs, graph replays against the eager forward, weight reloads, and
seg_resize=None against a step built without it.

Networks and pages as tests/test_gpu_text_removal.py makes them, with the segmentation network calibrated on the resized page
it sees here."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import evaluate_set_ref as E
import text_removal_ref as R
from gpu_cases import ROOT
from test_gpu_text_removal import _calibrate, _full8, _out_bias, _page, _perturbed, _same

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DEMO = ((0.4935, 0.4563, 0.4544), (0.3769, 0.3615, 0.3566))


def _lib():
    from text_segmentation_image_inpainting_b200 import _lib as L
    return L


def _ops():
    from text_segmentation_image_inpainting_b200 import ops
    return ops


def _count(fn):
    before = _lib().launch_count()
    out = fn()
    return out, _lib().launch_count() - before


def _resize_into_sentinel(page, rh, rw):
    """the C ABI into an output prefilled with NaN, so an unwritten pixel shows"""
    L = _lib()
    lib = L.load()
    n, _, h, w = page.shape
    ws = torch.empty((lib.pcb_page_resize_workspace(n, h, w, rh, rw),), dtype=torch.uint8, device=DEV)
    out = torch.full((n, 3, rh, rw), float("nan"), device=DEV)
    L.check(lib.pcb_page_resize_bicubic(page.data_ptr(), n, h, w, rh, rw, ws.data_ptr(), out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    return out


# ------------------------------------------------------------------------------------------------ kernel
def test_page_resize_matches_golden():
    ops = _ops()
    g = np.load(os.path.join(ROOT, "tests", "golden", "evaluate_set.npz"))
    names = sorted({k.split(".")[0] for k in g.files if "." in k})
    for name in names:
        chw = np.ascontiguousarray(g[name + ".page"].transpose(2, 0, 1))
        want = torch.from_numpy(E.to_tensor(np.ascontiguousarray(g[name + ".resized"].transpose(2, 0, 1))))
        rh, rw = want.shape[1:]
        (grh, grw), pad = ops.evaluate_set_geometry(chw.shape[1], chw.shape[2], int(g[name + ".resize"]))
        assert (grh, grw) == (rh, rw) and pad == tuple(int(v) for v in g[name + ".pad"]), name
        page = torch.from_numpy(E.to_tensor(chw))[None].to(DEV)
        got = _resize_into_sentinel(page, rh, rw)
        assert torch.equal(got[0].cpu(), want), name
        # a batch of two: the page and its mirror image
        pages = torch.cat([page, page.flip(3)]).contiguous()
        out, launches = _count(lambda: ops.page_resize_bicubic(pages, rh, rw))
        assert launches == 3 and out.shape == (2, 3, rh, rw) and out.dtype == torch.float32
        assert torch.equal(out[0].cpu(), want), name
        assert torch.equal(out[1].cpu(), torch.from_numpy(E.page_resize(pages[1:].cpu().numpy(), rh, rw))[0]), name
        # then the demo's Normalize and pad through the existing kernel, against the reference's tensor
        x = ops.removal_seg_input(out[:1], DEMO, rh + pad[3], rw + pad[1], torch.float32)
        assert torch.equal(x.cpu(), torch.from_numpy(g[name + ".input"])), name


# (batch, h, w, rh, rw): the reduction limit on each axis, upscaling, an identity axis, single pixels
SWEEP = [(1, 1024, 1000, 64, 63), (2, 640, 1600, 40, 100), (1, 333, 517, 333, 40), (3, 257, 311, 31, 311),
         (2, 120, 90, 600, 500), (1, 1, 1, 7, 5), (1, 16, 16, 1, 1), (2, 1700, 1200, 592, 416)]


@pytest.mark.parametrize("n,h,w,rh,rw", SWEEP, ids=[f"b{c[0]}_{c[1]}x{c[2]}_to_{c[3]}x{c[4]}" for c in SWEEP])
def test_page_resize_matches_restatement(n, h, w, rh, rw):
    gen = torch.Generator().manual_seed(h * 7 + w)
    page = torch.rand((n, 3, h, w), generator=gen)
    if h * w > 64:
        # values to_pil_image clamps: outside [0, 1], infinities and NaN (their bytes are 0 or 255)
        flat = page.view(-1)
        idx = torch.randint(0, flat.numel(), (64,), generator=gen)
        flat[idx] = torch.tensor([-0.5, 1.5, float("inf"), -float("inf"), float("nan"), 1.0, 0.0, 0.999999]).repeat(8)
    got = _resize_into_sentinel(page.to(DEV), rh, rw)
    assert torch.equal(got.cpu(), torch.from_numpy(E.page_resize(page.numpy(), rh, rw)))


def test_page_resize_refuses_bad_arguments():
    ops, L = _ops(), _lib()
    page = torch.rand(1, 3, 64, 80, device=DEV)
    before = L.launch_count()
    for bad in (lambda: ops.page_resize_bicubic(page.cpu(), 8, 8),
                lambda: ops.page_resize_bicubic(page.double(), 8, 8),
                lambda: ops.page_resize_bicubic(page[:, :2], 8, 8),
                lambda: ops.page_resize_bicubic(page[0], 8, 8),
                lambda: ops.page_resize_bicubic(page, 0, 8),
                lambda: ops.page_resize_bicubic(page, 3, 8),                   # 64 / 3 > 16
                lambda: ops.page_resize_bicubic(page, 8, 4)):                  # 80 / 4 > 16
        with pytest.raises(L.PcbError):
            bad()
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.pcb_page_resize_workspace(1, 64, 80, 0, 8) == 0 and lib.pcb_page_resize_workspace(0, 64, 80, 8, 8) == 0
    ws = torch.empty((lib.pcb_page_resize_workspace(1, 64, 80, 8, 8) + 256,), dtype=torch.uint8, device=DEV)
    out = torch.empty(1, 3, 8, 8, device=DEV)
    p, w, o = page.data_ptr(), ws.data_ptr(), out.data_ptr()
    for args in ((None, 1, 64, 80, 8, 8, w, o), (p, 1, 64, 80, 8, 8, None, o), (p, 1, 64, 80, 8, 8, w, None),
                 (p, 0, 64, 80, 8, 8, w, o), (p, 1, 0, 80, 8, 8, w, o), (p, 1, 64, 80, 0, 8, w, o), (p, 1, 64, 80, 8, 0, w, o),
                 (p, 1, 64, 80, 3, 8, w, o), (p, 1, 64, 80, 8, 4, w, o), (p, 1, 64, 80, 8, 8, w + 4, o)):
        assert lib.pcb_page_resize_bicubic(*args, st) != 0, args
        assert L.load().pcb_last_error()
    assert L.launch_count() == before


# ------------------------------------------------------------------------------------------------ end to end
def _nets(page, seed):
    """XceptionTextSegment (run-to-run deterministic, so its logits can be compared bitwise) and ImageFillOrigin, calibrated
    on `page` as the step with seg_resize=600 feeds them"""
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    ops = _ops()
    torch.manual_seed(seed)
    seg, fill = TS.XceptionTextSegment(), II.ImageFillOrigin()
    seg.load_state_dict(det_fill_state_dict(seg.state_dict()))
    fill.load_state_dict(det_fill_state_dict(fill.state_dict()))
    seg, fill = seg.to(DEV), fill.to(DEV)
    n, _, h, w = page.shape
    (rh, rw), pad = ops.evaluate_set_geometry(h, w, 600)
    x = ops.removal_seg_input(ops.page_resize_bicubic(page, rh, rw), DEMO, rh + pad[3], rw + pad[1], torch.bfloat16)
    _calibrate(seg, lambda: seg(x))
    with torch.no_grad():
        logits = seg(x).float()
        _out_bias(seg).sub_(float(torch.quantile(logits.flatten()[::7].cpu(), 0.99)))
    ops.bump_weight_epoch()
    with torch.no_grad():
        mask = ops.text_mask_postprocess(seg(x), pad, (h, w))
    m = 2 ** len(fill.decoder)
    corrupted, valid = ops.removal_holes(mask, page, (h + m - 1) // m * m, (w + m - 1) // m * m, torch.bfloat16)
    _calibrate(fill, lambda: fill((corrupted, HoleMask.from_plane(valid, 3))))
    return seg, fill


def _resize_mask(logits, pad, h, w):
    """the demo's mask by torch on the CPU: sigmoid > 0.5, 3x3 max-pool, unpad, bilinear to h x w (align_corners=False), > 0"""
    b = (torch.sigmoid(logits.float().cpu()[:, :1]) > 0.5).float()
    b = F.max_pool2d(b, 3, stride=1, padding=1)
    b = b[:, :, :b.shape[2] - pad[3], :b.shape[3] - pad[1]]
    return (F.interpolate(b, size=(h, w), mode="bilinear", align_corners=False) > 0).to(torch.uint8)


PAGES = [(1, 1700, 1200), (1, 1200, 1700), (1, 800, 1109), (2, 800, 1109), (2, 1109, 800), (1, 400, 300), (2, 400, 300)]


@pytest.mark.timeout(2400)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
def test_text_removal_step_seg_resize_stages(dtype):
    from text_segmentation_image_inpainting_b200.engine import InferStep, SegInferStep, TextRemovalStep
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    ops = _ops()
    torch.set_num_threads(max(1, min(32, os.cpu_count() or 1)))
    seg, fill = _nets(_page(1, 1700, 1200, 31), 32)
    step = TextRemovalStep(seg, fill, compute_dtype=dtype, seg_resize=600)
    some_text = 0
    for i, (n, h, w) in enumerate(PAGES):
        # fresh engines per page: two pages can share a segmentation grid, and the launch counts come from each capture
        seg_step, fill_step = SegInferStep(seg, compute_dtype=dtype), InferStep(fill, compute_dtype=dtype)
        page = _page(n, h, w, 40 + i)
        (rh, rw), pad = ops.evaluate_set_geometry(h, w, 600)
        (hs, ws), (hu, wu) = step.padded_sizes(h, w)
        assert (hs, ws) == (rh + pad[3], rw + pad[1]) and max(hs, ws) == 600
        out = step.run(page).clone()
        text_mask, valid, resized, logits, fill_out = (t.clone() for t in (step.text_mask, step.valid, step.last_resized,
                                                                           step.last_logits, step.last_fill))
        full = _full8(step.last_seg_input).clone()                              # the whole 8-channel NHWC input
        x = full[:, :3]
        case = (n, h, w)
        assert out.shape == (n, 3, h, w) and text_mask.shape == (n, 1, h, w) and valid.shape == (n, hu, wu), case
        assert resized.shape == (n, 3, rh, rw) and x.shape == (n, 3, hs, ws) and logits.shape == (n, 1, hs, ws), case
        assert fill_out.shape == (n, 3, hu, wu), case
        # each stage against the restatement applied to the step's own previous stage
        assert torch.equal(resized.cpu(), torch.from_numpy(E.page_resize(page.cpu().numpy(), rh, rw))), case
        want_x = torch.from_numpy(E.normalize_pad(resized.cpu().numpy(), *DEMO, hs, ws)).to(dtype)
        assert torch.equal(full[:, :3].cpu(), want_x) and not bool(full[:, 3:].any()), case
        assert torch.equal(logits.float().cpu(), seg_step.run(x.float()).cpu()), case
        assert torch.equal(text_mask, ops.text_mask_postprocess(logits, pad, (h, w))), case
        assert torch.equal(text_mask.cpu(), _resize_mask(logits, pad, h, w)), case
        v_ref, _ = R.unet_input(text_mask, page, hu, wu)
        assert torch.equal(valid.cpu(), v_ref), case
        page_pad = F.pad(page, (0, wu - w, 0, hu - h))
        valid3 = valid[:, None].expand(n, 3, hu, wu).float().contiguous()
        assert _same(fill_out.float(), fill_step.run(page_pad, valid3)), case
        assert _same(out.cpu(), R.composite(fill_out, page, valid)), case
        some_text += int(text_mask.any())
        # the graph's replay against the eager forward of the same page
        again = step.run(page).clone()
        assert _same(again, out), case
        with torch.no_grad():
            eager = step._run_forward(page)
        eager_products = step._cur
        step._cur = None
        assert _same(eager, out), case
        for a, b in zip((text_mask, valid, resized, x, logits, fill_out), eager_products):
            assert _same(a.float(), b.float()), case
        # launches: the resize's three on top of the parts
        _, dense_to_plane = _count(lambda: HoleMask.from_dense(valid3, channel_uniform=True))
        assert step.launches_per_run == 3 + seg_step.launches_per_run + fill_step.launches_per_run - dense_to_plane + 4, case
    assert some_text >= len(PAGES) - 2


@pytest.mark.timeout(1200)
def test_text_removal_step_seg_resize_reload():
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    page = _page(1, 1109, 800, 33)
    seg, fill = _nets(page, 34)
    step = TextRemovalStep(seg, fill, seg_resize=600)
    step.run(page)
    first = [t.clone() for t in (step.last_logits, step.last_fill)]
    for which in ("seg", "fill"):
        net = seg if which == "seg" else fill
        net.load_state_dict(_perturbed(net.state_dict()))
        out = step.run(page).clone()
        got = [t.clone() for t in (step.text_mask, step.valid, step.last_resized, step.last_logits, step.last_fill)]
        s2, f2 = TS.XceptionTextSegment(), II.ImageFillOrigin()
        s2.load_state_dict({k: v.cpu() for k, v in seg.state_dict().items()})
        f2.load_state_dict({k: v.cpu() for k, v in fill.state_dict().items()})
        fresh = TextRemovalStep(s2.to(DEV), f2.to(DEV), seg_resize=600)
        assert _same(out, fresh.run(page).clone()), which
        want = (fresh.text_mask, fresh.valid, fresh.last_resized, fresh.last_logits, fresh.last_fill)
        assert all(_same(a.float(), b.float()) for a, b in zip(got, want)), which
        changed = got[3] if which == "seg" else got[4]
        assert not _same(changed, first[0] if which == "seg" else first[1]), which


def test_text_removal_step_seg_resize_none_is_unchanged():
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    page = _page(2, 150, 230, 35)
    seg, fill = _nets(page, 36)
    outs = []
    for kwargs in ({}, {"seg_resize": None}):
        step = TextRemovalStep(seg, fill, **kwargs)
        assert step.padded_sizes(150, 230) == ((152, 232), (256, 256))
        out = step.run(page).clone()
        assert step.last_resized is None
        outs.append((out, step.text_mask.clone(), step.valid.clone(), step.last_seg_input.clone(), step.last_logits.clone(),
                     step.last_fill.clone(), step.launches_per_run))
    a, b = outs
    assert a[-1] == b[-1]
    assert all(_same(x.float(), y.float()) for x, y in zip(a[:-1], b[:-1]))


def test_text_removal_step_seg_resize_refuses():
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    L = _lib()
    seg, fill = TS.XceptionTextSegment().to(DEV), II.ImageFill().to(DEV)
    for bad in (0, -600, 12, 600.0, True, "600"):
        with pytest.raises(ValueError):
            TextRemovalStep(seg, fill, seg_resize=bad)
    step = TextRemovalStep(seg, fill, seg_resize=64)
    before = L.launch_count()
    for h, w in ((2000, 10), (1100, 1100)):                     # a side that resizes to 0; a reduction beyond 16x
        with pytest.raises(ValueError):
            step.run(torch.rand(1, 3, h, w, device=DEV))
    assert L.launch_count() == before and not step._graphs and step.text_mask is None

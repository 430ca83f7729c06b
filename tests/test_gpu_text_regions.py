"""GPU tests of the segmentation demo's region image (ops.text_region_hulls, csrc/text_regions.cu; DESIGN 4.14): byte for
byte against the fixture drawn by the reference's own draw_bounding_box (tests/golden/text_regions.npz) and against the numpy
restatement (tests/text_regions_ref.py) on page-sized masks, including union-find's worst cases; repeatability, `out=`, graph
capture and refusals; and engine.TextRemovalStep(region_hulls=...)."""
import os

import numpy as np
import pytest
import torch

import text_regions_ref as R
from gpu_cases import ROOT
from test_gpu_text_removal import _same
from test_gpu_text_removal_resize import _nets, _page

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


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


def test_matches_golden():
    g = np.load(os.path.join(ROOT, "tests", "golden", "text_regions.npz"))
    names = sorted({k.split(".")[0] for k in g.files if "." in k})
    assert len(names) >= 12
    for name in names:
        mask, page = torch.from_numpy(g[name + ".mask"]).to(DEV), torch.from_numpy(g[name + ".page"]).to(DEV)
        out, launches = _count(lambda: _ops().text_region_hulls(mask, page, float(g[name + ".threshold"])))
        assert launches == _ops().TEXT_REGION_LAUNCHES, name
        assert np.array_equal(out.cpu().numpy(), g[name + ".out"]), name


# ------------------------------------------------------------------------------------------------ page-sized masks
def _noise_pixels(h, w, rng):
    """isolated single pixels on the even grid: about h * w / 4 components, union-find's most roots"""
    m = np.zeros((h, w), np.uint8)
    m[::2, ::2] = rng.random(((h + 1) // 2, (w + 1) // 2)) < 0.95
    return m


def _noise20(h, w, rng):
    return (rng.random((h, w)) < 0.2).astype(np.uint8)


def _page_wide(h, w, rng):
    """one component across the whole page, with holes and islands in them"""
    m = np.ones((h, w), np.uint8)
    m[5:-5, 5:-5] = rng.random((h - 10, w - 10)) < 0.7
    m[h // 2, :] = 1
    m[:, w // 2] = 1
    return m


def _serpent(h, w, rng):
    """one text component snaking down the page row by row (the longest union chains)"""
    m = np.zeros((h, w), np.uint8)
    for i, y in enumerate(range(0, h - 2, 3)):
        m[y, 1:w - 1] = 1
        c = w - 2 if i % 2 == 0 else 1
        m[y:y + 4, c] = 1
    return m


def _corridor(h, w, rng):
    """a text block with a serpentine background corridor that opens to the outside at one end: all of it is exterior"""
    m = np.ones((h, w), np.uint8)
    for i, y in enumerate(range(2, h - 3, 3)):
        m[y, 2:w - 2] = 0
        c = w - 3 if i % 2 == 0 else 2
        m[y:y + 4, c] = 0
    m[2, w - 3:] = 0                                                     # the mouth on the right border
    return m


def _manga(h, w, rng):
    from text_segmentation_image_inpainting_b200.synthetic import manga_text_mask
    return manga_text_mask(h, w, int(rng.integers(0, 1 << 30)))


PAGE_CASES = [
    ("manga", 1700, 1200, 500), ("manga", 1700, 1200, 0), ("manga", 3508, 2480, 500),
    ("noise_pixels", 1700, 1200, 500), ("noise_pixels", 3508, 2480, 500), ("noise_pixels", 301, 399, -1),
    ("noise20", 1700, 1200, 100), ("noise20", 3508, 2480, 500),
    ("page_wide", 3508, 2480, 500), ("page_wide", 1700, 1200, 0),
    ("serpent", 1700, 1200, 500), ("serpent", 3508, 2480, 100),
    ("corridor", 1700, 1200, 0), ("corridor", 3508, 2480, 500),
]


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("style,h,w,threshold", PAGE_CASES, ids=[f"{s}_{h}x{w}_t{t}" for s, h, w, t in PAGE_CASES])
def test_matches_restatement_at_page_size(style, h, w, threshold):
    rng = np.random.default_rng([sum(map(ord, style)), h, w, threshold + 1])
    mask = globals()["_" + style](h, w, rng)
    page = rng.integers(0, 256, (1, 3, h, w), dtype=np.uint8).astype(np.float32) / 255
    got = _ops().text_region_hulls(torch.from_numpy(mask[None, None]).to(DEV), torch.from_numpy(page).to(DEV), threshold)
    want = R.text_region_hulls(mask, page[0], threshold)
    assert np.array_equal(got[0].cpu().numpy(), want)


def test_batch_repeat_out_and_capture():
    """a 3-page batch: each page equals the restatement, two calls agree, out= is written in place, a captured call replays
    the eager result, and pages that are not multiples of anything are fine"""
    ops = _ops()
    rng = np.random.default_rng(11)
    h, w = 517, 389
    masks = np.stack([_manga(h, w, rng), _noise20(h, w, rng), _serpent(h, w, rng)])[:, None]
    page = torch.from_numpy(rng.random((3, 3, h, w), dtype=np.float32)).to(DEV)
    page[0, 0, 0, :4] = torch.tensor([float("nan"), -1.0, 2.0, 1.0])                   # to_pil_image's clamps and NaN
    mask = torch.from_numpy(masks).to(DEV)
    a = ops.text_region_hulls(mask, page, 20)
    want = R.text_region_hulls_batch(masks, page.cpu().numpy(), 20)
    assert np.array_equal(a.cpu().numpy(), want)
    b = ops.text_region_hulls(mask, page, 20)
    assert torch.equal(a, b)
    out = torch.full((3, h, w, 3), 7, dtype=torch.uint8, device=DEV)
    r = ops.text_region_hulls(mask, page, 20, out=out)
    assert r is out and torch.equal(out, a)
    static = torch.zeros_like(a)
    ops.text_region_hulls(mask, page, 20, out=static)                                    # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.text_region_hulls(mask, page, 20, out=static)
    static.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, a)
    # the replay follows new mask contents
    mask.copy_(torch.from_numpy(masks[::-1].copy()).to(DEV))
    graph.replay()
    want2 = R.text_region_hulls_batch(masks[::-1], page.cpu().numpy(), 20)
    assert np.array_equal(static.cpu().numpy(), want2)


def test_refuses_bad_arguments():
    ops, L = _ops(), _lib()
    page = torch.rand((2, 3, 20, 30), device=DEV)
    mask = torch.zeros((2, 1, 20, 30), dtype=torch.uint8, device=DEV)
    before = L.launch_count()
    bad = [
        (mask.float(), page, 500, None), (mask[:1], page, 500, None), (mask[:, :, :, :29], page, 500, None),
        (mask.cpu(), page, 500, None), (mask.transpose(2, 3).contiguous().transpose(2, 3), page, 500, None),
        (mask, page.double(), 500, None), (mask, page[:, :2], 500, None), (mask, page.cpu(), 500, None),
        (mask, page.to(torch.bfloat16), 500, None),
        (mask, page, float("nan"), None), (mask, page, float("inf"), None), (mask, page, "500", None), (mask, page, True, None),
        (mask, page, 500, torch.empty((2, 20, 30, 3), dtype=torch.float32, device=DEV)),
        (mask, page, 500, torch.empty((2, 20, 30, 4), dtype=torch.uint8, device=DEV)),
        (mask, page, 500, torch.empty((2, 3, 20, 30), dtype=torch.uint8, device=DEV).permute(0, 2, 3, 1)),
        (mask, page, 500, torch.empty((2, 20, 30, 3), dtype=torch.uint8)),
    ]
    for i, (m, p, t, o) in enumerate(bad):
        with pytest.raises((L.PcbError, TypeError)):
            ops.text_region_hulls(m, p, t, out=o)
    lib = L.load()
    assert lib.pcb_text_regions_workspace(0, 20, 30) == 0 and lib.pcb_text_regions_workspace(1, 1 << 16, 1 << 16) == 0
    st = torch.cuda.current_stream().cuda_stream
    ws = torch.empty((lib.pcb_text_regions_workspace(2, 20, 30),), dtype=torch.uint8, device=DEV)
    o = torch.empty((2, 20, 30, 3), dtype=torch.uint8, device=DEV)
    args = (mask.data_ptr(), page.data_ptr(), 2, 20, 30, 500.0, ws.data_ptr(), o.data_ptr(), st)
    assert lib.pcb_text_region_hulls(*args) == 0
    after_ok = L.launch_count()
    for k, v in ((0, None), (5, float("nan")), (6, ws.data_ptr() + 16), (2, 0), (4, 0)):
        a = list(args)
        a[k] = v
        assert lib.pcb_text_region_hulls(*a) != 0, k
        assert lib.pcb_last_error()
    assert L.launch_count() == after_ok == before + ops.TEXT_REGION_LAUNCHES


# ------------------------------------------------------------------------------------------------ engine
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("seg_resize", [None, 600], ids=["page_size", "resize600"])
def test_text_removal_step_region_hulls(seg_resize):
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    ops = _ops()
    page = _page(2, 400, 300, 51)
    seg, fill = _nets(page, 52)
    plain = TextRemovalStep(seg, fill, seg_resize=seg_resize)
    assert plain.region_hulls is None
    want_out = plain.run(page).clone()
    assert plain.text_regions is None
    want = {k: getattr(plain, k) for k in plain._PRODUCTS if k != "text_regions"}
    step = TextRemovalStep(seg, fill, seg_resize=seg_resize, region_hulls=500)
    out = step.run(page).clone()
    assert _same(out, want_out)
    for k, v in want.items():
        got = getattr(step, k)
        assert (got is None and v is None) or _same(got.float(), v.float()), k
    assert step.text_mask.any()
    regions = step.text_regions.clone()
    assert regions.shape == (2, 400, 300, 3) and regions.dtype == torch.uint8
    assert torch.equal(regions, ops.text_region_hulls(step.text_mask, page, 500))
    assert np.array_equal(regions.cpu().numpy(), R.text_region_hulls_batch(step.text_mask.cpu().numpy(), page.cpu().numpy(), 500))
    assert step.launches_per_run == plain.launches_per_run + ops.TEXT_REGION_LAUNCHES
    # every replay rewrites the product
    step.text_regions.zero_()
    step.run(page)
    assert torch.equal(step.text_regions, regions)
    # a lower threshold paints at least as much
    low = TextRemovalStep(seg, fill, seg_resize=seg_resize, region_hulls=0)
    low.run(page)
    color = torch.tensor((50, 128, 30), dtype=torch.uint8, device=DEV)
    painted = lambda t: int((t == color).all(-1).sum())                                      # noqa: E731
    assert painted(low.text_regions) >= painted(regions)
    for bad in (float("nan"), "500", True):
        with pytest.raises(ValueError):
            TextRemovalStep(seg, fill, region_hulls=bad)

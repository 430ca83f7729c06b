"""The GPU segmentation data path (csrc/seg_data.cu, data.SegBatcher) on the device: bit-exact against the reference's
recorded outputs and the numpy restatement, the bf16 and normalized variants, the device draws against the restated stream and
the reference's distributions, seeding, and source-size changes across graph replays."""
import ctypes
import os

import numpy as np
import pytest
import torch

import seg_ref as S
from conftest import GOLDEN
from oracle import inpaint_data as OI
from oracle import seg_data as OS

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN, "seg_data.npz"))


def _batcher(sources, size, dtype=torch.float32, **kw):
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    cap = (max(p.shape[0] for p, _ in sources), max(p.shape[1] for p, _ in sources))
    b = SegBatcher(len(sources), cap, image_size=size, compute_dtype=dtype, **kw)
    b.stage(sources)
    return b


def _expected(sources, params, size):
    out = [OS.process(pg, m, p, size) for (pg, m), p in zip(sources, params)]
    page = torch.from_numpy(np.stack([OS.to_tensor(o[0]) for o in out]))
    mask = torch.from_numpy(np.stack([OS.to_tensor(o[1]) for o in out]))
    return page, mask


@pytest.mark.parametrize("k", range(len(S.CASES)))
def test_golden_cases_are_bit_exact_in_fp32_and_rounded_once_in_bf16(k):
    size = int(G["cases"][k][3])
    src = [S.case_sources(k)]
    p = G[f"params{k}"][None]
    page = torch.from_numpy(G[f"page{k}"]).float()[None, None] / 255
    mask = torch.from_numpy(G[f"mask{k}"]).float()[None, None] / 255
    b32 = _batcher(src, size)
    x32, t32 = (v.clone() for v in b32.prepare(p))
    b16 = _batcher(src, size, torch.bfloat16)
    x16, t16 = b16.prepare(p)
    torch.cuda.synchronize()
    assert torch.equal(x32.cpu(), page.expand(1, 3, size, size))
    assert torch.equal(t32.cpu(), mask) and torch.equal(t16.cpu(), mask)
    assert torch.equal(x16.cpu(), x32.cpu().to(torch.bfloat16))
    for b in (b32, b16):
        assert not bool(b._xbuf[:, 3:].any())
        assert torch.equal(b._xbuf[:, 0], b._xbuf[:, 1]) and torch.equal(b._xbuf[:, 0], b._xbuf[:, 2])


def test_random_parameters_match_the_restatement():
    rng = np.random.default_rng(3)
    sizes = [(300, 220), (64, 500), (700, 640), (45, 60), (512, 512)]
    src = [S.sources(20 + i, h, w) for i, (h, w) in enumerate(sizes)]
    for size, seed in ((128, 1), (96, 2)):
        params = OS.sample(seed, 5, sizes)
        params[rng.integers(0, len(sizes)), 4] ^= 1
        b = _batcher(src, size)
        x, t = b.prepare(params)
        page, mask = _expected(src, params, size)
        torch.cuda.synchronize()
        assert torch.equal(x.cpu(), page.expand(-1, 3, -1, -1))
        assert torch.equal(t.cpu(), mask)


def test_normalize_is_torchvision_normalize_of_the_fp32_output():
    from torchvision.transforms import Normalize
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    src = [S.sources(30 + i, 300 + 40 * i, 280) for i in range(3)]
    params = OS.sample(4, 0, [p.shape for p, _ in src])
    plain = _batcher(src, 128).prepare(params)[0].cpu()
    for dtype in (torch.float32, torch.bfloat16):
        x = _batcher(src, 128, dtype, normalize=(mean, std)).prepare(params)[0]
        ref = Normalize(mean, std)(plain.clone())
        torch.cuda.synchronize()
        assert torch.equal(x.cpu(), ref.to(dtype))


def _device_draws(seed, counter, sizes):
    from text_segmentation_image_inpainting_b200 import _lib
    n = len(sizes)
    table = np.zeros(n, dtype=[("a", "<u8"), ("b", "<u8"), ("h", "<i4"), ("w", "<i4"), ("sa", "<i4"), ("sb", "<i4")])
    table["a"] = table["b"] = 1
    table["h"], table["w"] = [s[0] for s in sizes], [s[1] for s in sizes]
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    rng = torch.tensor([seed, counter], dtype=torch.int64, device="cuda")
    params = torch.empty((n, OS.PARAM_INTS), dtype=torch.int32, device="cuda")
    _lib.check(_lib.load().pcb_seg_sample(tab.data_ptr(), n, rng.data_ptr(), params.data_ptr(),
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert int(rng[1]) == counter + 1
    return params.cpu().numpy()


def test_device_sampler_is_the_restated_stream():
    rng = np.random.default_rng(0)
    sizes = [(int(h), int(w)) for h, w in rng.integers(20, 2000, (300, 2))] + [(100, 900), (900, 100)]
    for seed, counter in ((0, 0), (123456789012, 7), (5, 2 ** 33 + 1)):
        np.testing.assert_array_equal(_device_draws(seed, counter, sizes), OS.sample(seed, counter, sizes))


def test_device_draws_follow_the_reference_distributions():
    from scipy import stats
    from torchvision.transforms import ColorJitter, RandomResizedCrop
    H, W, N = 181, 256, 4096
    dev = np.concatenate([_device_draws(99, c, [(H, W)] * 1024) for c in range(N // 1024)])
    torch.manual_seed(99)
    cj = ColorJitter(brightness=0.2, contrast=0.2, saturation=0.2, hue=0.2)
    img = torch.zeros(1, H, W)
    ref = []
    for _ in range(N):
        box = RandomResizedCrop.get_params(img, scale=(0.1, 2), ratio=(3. / 4., 4. / 3.))
        fn_idx, b, c, _, _ = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        idx = [int(v) for v in fn_idx]
        ref.append(OS.params_row(box, idx.index(0) < idx.index(1), b, c))
    ref = np.stack(ref)
    alpha = 1e-4

    def scale(a):
        return a[:, 2] * a[:, 3] / float(H * W)

    def log_aspect(a):
        return np.log(a[:, 3] / a[:, 2])

    for f in (scale, log_aspect, lambda a: a[:, 0], lambda a: a[:, 1]):
        assert stats.ks_2samp(f(dev), f(ref)).pvalue > alpha
    table = np.array([[(a[:, 4] == v).sum() for v in (0, 1)] for a in (dev, ref)])
    assert stats.chi2_contingency(table)[1] > alpha
    assert stats.chisquare(table[0]).pvalue > alpha                       # brightness first with probability 1/2
    for col in (0, 1):
        fd, fr = (np.array([OS.factors(p)[col] for p in a]) for a in (dev, ref))
        assert stats.ks_2samp(fd, fr).pvalue > alpha
        assert fd.min() >= np.float32(0.8) and fd.max() <= np.float32(1.2)
    assert (dev[:, 2] * dev[:, 3] < 128 * 128).mean() > 0.2             # small boxes, upscaled to the output, are common


def test_reseed_and_graph_replays_with_new_source_sizes():
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    seed, size = 17, 128
    sizes_a, sizes_b = [(300, 420), (512, 380)], [(260, 261), (100, 512)]
    src_a = [S.sources(40 + i, h, w) for i, (h, w) in enumerate(sizes_a)]
    src_b = [S.sources(50 + i, h, w) for i, (h, w) in enumerate(sizes_b)]
    b = SegBatcher(2, (512, 512), image_size=size, seed=seed, compute_dtype=torch.float32)
    b.stage(src_a)
    b.prepare()                                               # eager warm-up (draw 0)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    b.activate()
    with torch.cuda.graph(graph):
        b.prepare()
    torch.cuda.synchronize()
    counter = int(b.rng[1])
    seen = []
    for step, (sizes, src) in enumerate([(sizes_a, src_a), (sizes_b, src_b), (sizes_a, src_a)]):
        b.stage(src)
        b.activate()
        graph.replay()
        b.release()
        torch.cuda.synchronize()
        p = b.params.cpu().numpy()
        np.testing.assert_array_equal(p, OS.sample(seed, counter + step, sizes))
        page, mask = _expected(src, p, size)
        assert torch.equal(b.x.cpu(), page.expand(-1, 3, -1, -1)) and torch.equal(b.target.cpu(), mask)
        seen.append(b.x.clone())
    assert not torch.equal(seen[0], seen[2])                  # same sources, fresh draws
    b.reseed(seed, counter)
    b.stage(src_a)
    b.prepare()
    torch.cuda.synchronize()
    assert torch.equal(b.x, seen[0])                          # the same seed and counter reproduce the batch


def test_validation_rejects_bad_parameters():
    from text_segmentation_image_inpainting_b200._lib import PcbError
    src = [S.sources(60, 100, 120)]
    b = _batcher(src, 64)
    for bad in ((0, 0, 101, 50, 0, 1.0, 1.0), (0, 100, 10, 30, 0, 1.0, 1.0), (0, 0, 100, 120, 2, 1.0, 1.0),
                (0, 0, 100, 120, 0, float("nan"), 1.0)):
        with pytest.raises(PcbError):
            b.prepare(OS.params_row(bad[:4], bad[4], bad[5], bad[6])[None] if bad[4] != 2 else
                      np.array([[0, 0, 100, 120, 2, 0, 0, 0]], np.int32))
    with pytest.raises(ValueError):
        b.stage([(np.zeros((600, 600), np.uint8), np.zeros((600, 600), np.uint8))])
    with pytest.raises(ValueError):
        _batcher([(np.zeros((600, 600), np.uint8), np.zeros((600, 600), np.uint8))], 64)   # > 8x the output

"""The GPU inpainting data path (csrc/inpaint_data.cu, data.InpaintBatcher, engine.InpaintTrainStep) on the device: bit-exact
against the reference's recorded outputs without strokes, bit-exact against the numpy stroke rule with them, the device draws
against the reference's distributions, seeding and graph replays, and the training step against TrainStep."""
import ctypes
import os

import numpy as np
import pytest
import torch

import inpaint_ref as R
from conftest import GOLDEN
from oracle import inpaint_data as OI

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN, "inpaint_data.npz"))
STROKE_FREE = [k for k, c in enumerate(G["cases"]) if not c[4]]
STROKED = [k for k, c in enumerate(G["cases"]) if c[4]]


def _case(k):
    seed, H, W, size, strokes, _ = (int(v) for v in G["cases"][k])
    rgb, mask = R.sources(seed, H, W)
    hole = np.unpackbits(G[f"hole{k}"])[:size * size].reshape(size, size).astype(bool)
    return rgb, mask, size, bool(strokes), G[f"params{k}"], G[f"clean{k}"].transpose(1, 2, 0), hole  # clean HWC


def _prepare_one(rgb, mask, size, strokes, params, dtype):
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    b = InpaintBatcher(1, mask.shape, image_size=size, add_random_masks=strokes, compute_dtype=dtype)
    b.stage([(rgb, mask)])
    x, hm, clean = b.prepare(params[None])
    torch.cuda.synchronize()
    return b, x, hm, clean


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", STROKE_FREE)
def test_stroke_free_cases_are_bit_exact_against_the_reference(k, dtype):
    rgb, mask, size, strokes, p, clean_u8, hole = _case(k)
    b, x, hm, clean = _prepare_one(rgb, mask, size, strokes, p, dtype)
    ref_clean = torch.from_numpy(clean_u8).permute(2, 0, 1).float() / 255
    binary = 1 - torch.from_numpy(hole).float() * 255 / 255
    assert torch.equal(clean[0].cpu(), ref_clean)
    assert torch.equal(b.plane[0].cpu(), torch.from_numpy(~hole).to(torch.uint8))
    assert torch.equal(hm.dense()[0].cpu(), binary.expand(3, -1, -1))
    assert torch.equal(x[0].cpu(), (ref_clean * binary).to(dtype))
    assert not bool(b._xbuf[:, 3:].any())


@pytest.mark.parametrize("k", STROKED)
def test_stroke_cases_match_the_rule_exactly_and_pillow_within_two_percent(k):
    rgb, mask, size, strokes, p, clean_u8, hole = _case(k)
    b, x, hm, clean = _prepare_one(rgb, mask, size, strokes, p, torch.bfloat16)
    rule_clean, rule_hole = OI.process(rgb, mask, p, size, strokes=True)
    got_hole = b.plane[0].cpu().numpy() == 0
    np.testing.assert_array_equal(got_hole, rule_hole)
    assert torch.equal(clean[0].cpu(), torch.from_numpy(rule_clean).permute(2, 0, 1).float() / 255)
    np.testing.assert_array_equal(rule_clean, clean_u8)
    assert (got_hole != hole).sum() <= 0.02 * hole.sum(), ((got_hole != hole).sum(), hole.sum())


def _device_draws(seed, counter, sizes, out, strokes=True):
    """Call the sampler alone on a table that only carries source sizes."""
    from text_segmentation_image_inpainting_b200 import _lib
    n = len(sizes)
    table = np.zeros(n, dtype=[("rgb", "<u8"), ("mask", "<u8"), ("h", "<i4"), ("w", "<i4"), ("rs", "<i4"), ("ms", "<i4")])
    table["rgb"] = table["mask"] = 1
    table["h"], table["w"] = [s[0] for s in sizes], [s[1] for s in sizes]
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    rng = torch.tensor([seed, counter], dtype=torch.int64, device="cuda")
    params = torch.empty((n, OI.PARAM_INTS), dtype=torch.int32, device="cuda")
    _lib.check(_lib.load().pcb_inpaint_sample(tab.data_ptr(), n, out, int(strokes), rng.data_ptr(), params.data_ptr(),
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert int(rng[1]) == counter + 1
    return params.cpu().numpy()


def test_device_sampler_is_the_restated_stream():
    rng = np.random.default_rng(0)
    sizes = [(int(h), int(w)) for h, w in rng.integers(40, 2000, (300, 2))] + [(100, 900), (900, 100)]
    for seed, counter in ((0, 0), (123456789012, 7), (5, 2 ** 33 + 1)):
        np.testing.assert_array_equal(_device_draws(seed, counter, sizes, 512), OI.sample(seed, counter, sizes, 512))
    np.testing.assert_array_equal(_device_draws(3, 1, sizes, 256, strokes=False), OI.sample(3, 1, sizes, 256, strokes=False))


def test_device_draws_follow_the_reference_distributions():
    import random

    from PIL import Image
    from scipy import stats
    from torchvision.transforms import RandomResizedCrop
    if R.dataloader() is None:
        pytest.skip("reference not staged in oracle/_ref")
    H, W, size, N = 181, 256, 512, 4096
    dev = np.concatenate([_device_draws(99, c, [(H, W)] * 1024, size) for c in range(N // 1024)])
    random.seed(99)
    torch.manual_seed(99)
    ref = []
    img = torch.zeros(1, H, W)
    for _ in range(N):
        with R.recording() as rec:
            rec["box"] = RandomResizedCrop.get_params(img, scale=(0.5, 2.0), ratio=(3. / 4., 4. / 3.))
            rec["gray"] = int(torch.rand(1) < 0.4)
            R.dataloader().random_masks(Image.new("L", (1, 1)), size=size, offset=10)
        ref.append(R.params_of(rec))
    ref = np.stack(ref)
    alpha = 1e-4
    for col in (4, 5, 6):                                              # grayscale, line count, ellipse count
        cats = np.union1d(dev[:, col], ref[:, col])
        table = np.array([[(a[:, col] == c).sum() for c in cats] for a in (dev, ref)])
        assert stats.chi2_contingency(table)[1] > alpha, col
    widths = [a[a[:, 5] >= 1][:, OI.LINE0 + 4] for a in (dev, ref)]
    cats = np.arange(15, 21)
    assert stats.chi2_contingency(np.array([[(w == c).sum() for c in cats] for w in widths]))[1] > alpha
    for col in (0, 1, 2, 3, OI.LINE0, OI.LINE0 + 2, OI.ELL0, OI.ELL0 + 1, OI.ELL0 + 2, OI.ELL0 + 3):   # crop box, stroke geometry
        assert stats.ks_2samp(dev[:, col], ref[:, col]).pvalue > alpha, col


def _small_net():
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    net = ImageFillOrigin()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    return net


def _sources(sizes, seed):
    return [R.sources(seed + i, h, w) for i, (h, w) in enumerate(sizes)]


def test_inpaint_train_step_matches_train_step_on_the_same_batch():
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintTrainStep, TrainStep
    dev = torch.device("cuda")
    sizes = [(300, 420), (512, 380)]
    b = InpaintBatcher(2, (512, 512), image_size=256, add_random_masks=True, seed=3)
    b.stage(_sources(sizes, 10))
    _, hm, clean = b.prepare()
    params = b.params.cpu().numpy()
    clean, dense = clean.clone(), hm.dense().clone()
    ref = TrainStep(_small_net().to(dev), lr=1e-3, use_graph=False)
    loss_ref = ref.step(clean, dense)
    ts = InpaintTrainStep(_small_net().to(dev), b, lr=1e-3, use_graph=False)
    loss = ts.step(params=params)
    torch.cuda.synchronize()
    assert torch.equal(loss, loss_ref), (float(loss), float(loss_ref))
    # the weight-gradient kernels' split-K adds are unordered fp32, so the updated weights agree to rounding, not bitwise
    assert float((ts.flat.flat_p - ref.flat.flat_p).abs().max()) <= 1e-6


def test_graph_replays_draw_fresh_batches_and_take_new_source_sizes():
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintTrainStep
    seed, size = 17, 256
    sizes_a, sizes_b = [(300, 420), (512, 380)], [(260, 261), (400, 512)]
    b = InpaintBatcher(2, (512, 512), image_size=size, add_random_masks=True, seed=seed)
    src_a, src_b = _sources(sizes_a, 20), _sources(sizes_b, 30)
    b.stage(src_a)
    ts = InpaintTrainStep(_small_net().cuda(), b, lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    assert ts.graph is not None
    counter = int(b.rng[1])                                   # two eager steps and the side-stream run drew
    assert counter == 3
    seen = []
    for step, (sizes, src) in enumerate([(sizes_a, src_a), (sizes_b, src_b), (sizes_a, src_a)]):
        b.stage(src)
        loss = ts.step()
        torch.cuda.synchronize()
        assert np.isfinite(float(loss))
        p = b.params.cpu().numpy()
        np.testing.assert_array_equal(p, OI.sample(seed, counter + step, sizes, size))
        clean_u8, hole = OI.process(*src[1], p[1], size)
        assert torch.equal(b.clean[1].cpu(), torch.from_numpy(clean_u8).permute(2, 0, 1).float() / 255)
        np.testing.assert_array_equal(b.plane[1].cpu().numpy() == 0, hole)
        seen.append(b.plane.clone())
    assert not torch.equal(seen[0], seen[2])                 # same sources, fresh draws
    b.reseed(seed, counter)
    b.stage(src_a)
    ts.step()
    torch.cuda.synchronize()
    assert torch.equal(b.plane, seen[0])                      # the same seed and counter reproduce the batch

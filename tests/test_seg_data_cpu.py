"""The numpy restatement of the segmentation data path (oracle/seg_data.py) against the reference's own code on the CPU:
Pillow's blends behind ColorJitter's brightness and contrast, the whole process_images with recorded and forced parameters,
and the sampler's mapping from uniforms to RandomResizedCrop.get_params(scale=(0.1, 2)) and ColorJitter.get_params."""
import os
import random
import unittest.mock as um

import numpy as np
import pytest
import torch

import inpaint_ref as R
import seg_ref as S
from conftest import GOLDEN
from oracle import inpaint_data as OI
from oracle import seg_data as OS

needs_ref = pytest.mark.skipif(R.dataloader() is None, reason="reference not staged in oracle/_ref")


def test_blends_match_image_enhance():
    from PIL import Image, ImageEnhance
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (40, 50), dtype=np.uint8)
    img[0, :8] = (0, 1, 127, 128, 212, 213, 254, 255)
    pil = Image.fromarray(img, "L")
    factors = [0.8, 1.2, 1.0, np.nextafter(np.float32(0.8), np.float32(1))] + list(rng.uniform(0.8, 1.2, 300))
    for f in factors:
        f = float(np.float32(f))
        np.testing.assert_array_equal(OS.blend(0, img, f), np.array(ImageEnhance.Brightness(pil).enhance(f)))
        np.testing.assert_array_equal(OS.blend(OS.contrast_mean(img), img, f), np.array(ImageEnhance.Contrast(pil).enhance(f)))


def test_contrast_mean_rounds_half_up_at_the_boundary():
    page, _ = S.half_page(64, 64)
    assert int(page.astype(np.int64).sum()) * 2 == 201 * page.size        # mean 100.5 exactly
    assert OS.contrast_mean(page) == 101


@needs_ref
@pytest.mark.parametrize("k", range(len(S.CASES)))
def test_process_images_is_the_restatement(k):
    seed, _, _, out, force = S.CASES[k]
    page, mask = S.case_sources(k)
    random.seed(seed)
    torch.manual_seed(seed)
    for _ in range(3):
        (pg, m), p = S.run_reference(page, mask, out, **force)
        op, om = OS.process(page, mask, p, out)
        np.testing.assert_array_equal(OS.to_tensor(op), pg)
        np.testing.assert_array_equal(OS.to_tensor(om), m)


@needs_ref
def test_process_images_with_natural_draws_is_the_restatement():
    random.seed(1)
    torch.manual_seed(1)
    orders = set()
    for t in range(120):
        H, W = (int(v) for v in np.random.default_rng(t).integers(20, 400, 2))
        page, mask = S.sources(t, H, W)
        (pg, m), p = S.run_reference(page, mask, 48)
        op, om = OS.process(page, mask, p, 48)
        np.testing.assert_array_equal(OS.to_tensor(op), pg)
        np.testing.assert_array_equal(OS.to_tensor(om), m)
        orders.add(int(p[4]))
    assert orders == {0, 1}


class _Draws:
    """Serves the sampler's uniforms in the order the reference draws."""

    def __init__(self, u):
        self.u = list(u)

    def next(self):
        return float(self.u.pop(0))


def test_crop_mapping_matches_get_params_for_the_segmentation_scale_range():
    from torchvision.transforms import RandomResizedCrop
    rng = np.random.default_rng(5)
    for trial in range(400):
        H, W = (int(v) for v in rng.integers(20, 1600, 2))
        u = OI.uniforms(2000 + trial, trial, 1)[0]
        if trial % 7 == 0:
            W = H * 5                                   # no attempt fits: the fallback branch
            u[0:40:4] = np.float32(0.999)
        elif trial % 5 == 0:
            u[0:40:4] = np.float32(0.001)               # scale near 0.1: boxes smaller than the output, upscaled
        d = _Draws(u[:40])
        calls = [0]

        class FakeEmpty:
            def uniform_(self, lo, hi):
                lo, hi = np.float32(float(lo)), np.float32(float(hi))
                return torch.tensor([lo + (hi - lo) * np.float32(d.next())], dtype=torch.float32)

        def fake_empty(*a, **k):
            calls[0] += 1
            if calls[0] % 2 == 1 and calls[0] > 1:      # an attempt that did not fit skips its top / left slots
                d.next()
                d.next()
            return FakeEmpty()

        def fake_randint(lo, hi, size):
            return torch.tensor([lo + int(np.float64(d.next()) * (hi - lo))])

        with um.patch.object(torch, "empty", fake_empty), um.patch.object(torch, "randint", fake_randint):
            ref = RandomResizedCrop.get_params(torch.zeros(1, H, W), scale=(0.1, 2), ratio=(3. / 4., 4. / 3.))
        got = OS.crop_from_uniforms(H, W, u)
        assert tuple(ref) == got, (H, W, trial)
        if trial % 7 == 0:                              # the centre crop of a 5:1 source at the widest ratio
            w = int(np.rint(H * 4 / 3))
            assert got == (0, (W - w) // 2, H, w)


def test_jitter_mapping_matches_color_jitter_get_params():
    from torchvision.transforms import ColorJitter
    cj = ColorJitter(brightness=0.2, contrast=0.2, saturation=0.2, hue=0.2)
    for trial in range(300):
        u = OI.uniforms(77, trial, 1)[0]
        if trial < 4:
            u[41:43] = np.float32([0.0, 1 - 2.0 ** -24, 0.5, 0.25][trial])
        bfirst, b, c = OS.jitter_from_uniforms(u)
        d = _Draws(u[41:43])

        class FakeEmpty:
            def uniform_(self, lo, hi):
                lo, hi = np.float32(float(lo)), np.float32(float(hi))
                v = np.float32(d.next()) if d.u else np.float32(0.5)      # saturation and hue: not drawn by the sampler
                return torch.tensor([lo + (hi - lo) * v], dtype=torch.float32)

        perm = torch.tensor([0, 1, 2, 3] if u[40] < 0.5 else [1, 0, 2, 3])
        with um.patch.object(torch, "empty", lambda *a, **k: FakeEmpty()), um.patch.object(torch, "randperm", lambda n: perm):
            fn_idx, rb, rc, _, _ = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        idx = [int(v) for v in fn_idx]
        assert (int(idx.index(0) < idx.index(1)), np.float32(rb), np.float32(rc)) == (bfirst, b, c), trial
        assert np.float32(0.8) <= b <= np.float32(1.2) and np.float32(0.8) <= c <= np.float32(1.2)


def test_golden_fixture_is_the_restatement():
    g = np.load(os.path.join(GOLDEN, "seg_data.npz"))
    assert len(g["cases"]) == len(S.CASES)
    for k, (seed, H, W, size) in enumerate(g["cases"]):
        page, mask = S.case_sources(k)
        assert page.shape == (H, W)
        op, om = OS.process(page, mask, g[f"params{k}"], int(size))
        np.testing.assert_array_equal(op, g[f"page{k}"])
        np.testing.assert_array_equal(om, g[f"mask{k}"])

"""The numpy restatement of the inpainting data path (oracle/inpaint_data.py) against the reference's own code on the CPU:
Pillow's bicubic crop + resize, torchvision's grayscale and ToTensor, cv2.dilate, RandomResizedCrop.get_params and random_masks
given the same draws, and the distance of the documented stroke rule from Pillow's rasteriser."""
import random
import unittest.mock as um

import numpy as np
import pytest
import torch

import inpaint_ref as R
from oracle import inpaint_data as OI

needs_ref = pytest.mark.skipif(R.dataloader() is None, reason="reference not staged in oracle/_ref")


@pytest.mark.parametrize("H,W,box,out", [
    (300, 200, (10, 20, 150, 110), 256),      # upscale
    (300, 200, (0, 0, 300, 200), 64),         # downscale, whole source
    (181, 240, (33, 7, 97, 181), 128),        # mixed: up in one axis, down in the other
    (97, 61, (5, 3, 61, 40), 61),             # identity width
    (1448, 1024, (200, 100, 1180, 900), 512),
])
def test_resized_crop_matches_pillow(H, W, box, out):
    from PIL import Image
    from torchvision.transforms.functional import resized_crop
    rgb, mask = R.sources(H + W, H, W)
    i, j, h, w = box
    ref = np.array(resized_crop(Image.fromarray(rgb), i, j, h, w, size=(out, out), interpolation=Image.BICUBIC))
    np.testing.assert_array_equal(OI.resized_crop(rgb, box, out), ref)
    ref_l = np.array(resized_crop(Image.fromarray(mask), i, j, h, w, size=(out, out), interpolation=Image.BICUBIC))
    np.testing.assert_array_equal(OI.resized_crop(mask[..., None], box, out)[..., 0], ref_l)


def test_grayscale_matches_torchvision():
    from PIL import Image
    import torchvision.transforms.functional as F
    rgb = np.random.default_rng(1).integers(0, 256, (64, 80, 3), dtype=np.uint8)
    ref = np.array(F.rgb_to_grayscale(Image.fromarray(rgb), num_output_channels=3))
    np.testing.assert_array_equal(OI.grayscale(rgb), ref)


def test_threshold_and_dilation_match_cv2_at_borders():
    import cv2
    rng = np.random.default_rng(2)
    m = rng.integers(0, 256, (53, 47)).astype(np.uint8) * (rng.random((53, 47)) > 0.985)
    m[0, 0] = m[-1, -1] = m[0, -1] = m[-1, 0] = 200            # corners: the window runs outside the image
    m[26, 0] = 103
    m[10, 20] = 102
    ref = cv2.dilate(np.where(m > 0.4 * 255, np.uint8(255), np.uint8(0)), np.ones((10, 10), np.uint8), iterations=1)
    np.testing.assert_array_equal(OI.dilate10(m >= 103), ref > 0)


def test_to_tensor_product_matches_torchvision():
    from torchvision.transforms.functional import to_tensor
    rng = np.random.default_rng(3)
    clean = rng.integers(0, 256, (32, 40, 3), dtype=np.uint8)
    hole = rng.random((32, 40)) > 0.7
    mask_t = to_tensor(np.expand_dims(np.where(hole, np.uint8(255), np.uint8(0)), -1))
    binary = (1 - mask_t).expand(3, -1, -1)
    clean_t = to_tensor(clean)
    corrupted, b, c = OI.to_tensors(clean, hole)
    np.testing.assert_array_equal(c, clean_t.numpy())
    np.testing.assert_array_equal(b, binary.numpy())
    np.testing.assert_array_equal(corrupted, (clean_t * binary).numpy())


@needs_ref
@pytest.mark.parametrize("seed,H,W,out", [(0, 300, 220, 128), (1, 140, 400, 96), (2, 512, 512, 64)])
def test_process_images_without_strokes_is_the_restatement(seed, H, W, out):
    rgb, mask = R.sources(seed, H, W)
    random.seed(seed)
    torch.manual_seed(seed)
    for _ in range(4):
        (corr, binary, clean), p = R.run_reference(rgb, mask, out, add_random_masks=False)
        c8, hole = OI.process(rgb, mask, p, out, strokes=False)
        oc, ob, ocl = OI.to_tensors(c8, hole)
        np.testing.assert_array_equal(ocl, clean)
        np.testing.assert_array_equal(ob, binary)
        np.testing.assert_array_equal(oc, corr)


class _Draws:
    """Stands in for the reference's random sources, serving the sampler's uniforms in the order the reference draws."""

    def __init__(self, u):
        self.u = list(u)

    def next(self):
        return float(self.u.pop(0))


def test_crop_mapping_matches_get_params():
    from torchvision.transforms import RandomResizedCrop
    rng = np.random.default_rng(4)
    for trial in range(400):
        H, W = (int(v) for v in rng.integers(20, 1600, 2))
        u = OI.uniforms(1000 + trial, trial, 1)[0]
        if trial % 7 == 0:
            W = H * 5                                   # no attempt fits: the fallback branch
            u[0:40:4] = np.float32(0.999)
        # the sampler gives every attempt four fixed slots (scale, log-aspect, top, left); the reference draws top / left only
        # when an attempt fits, so an attempt that does not fit skips its two unused slots
        d = _Draws(u[:40])
        calls = [0]

        class FakeEmpty:
            def uniform_(self, lo, hi):
                lo, hi = np.float32(float(lo)), np.float32(float(hi))
                return torch.tensor([lo + (hi - lo) * np.float32(d.next())], dtype=torch.float32)

        def fake_empty(*a, **k):
            calls[0] += 1
            if calls[0] % 2 == 1 and calls[0] > 1:
                d.next()
                d.next()
            return FakeEmpty()

        def fake_randint(lo, hi, size):
            return torch.tensor([lo + int(np.float64(d.next()) * (hi - lo))])

        with um.patch.object(torch, "empty", fake_empty), um.patch.object(torch, "randint", fake_randint):
            ref = RandomResizedCrop.get_params(torch.zeros(1, H, W), scale=(0.5, 2.0), ratio=(3. / 4., 4. / 3.))
        assert tuple(ref) == OI.crop_from_uniforms(H, W, u), (H, W, trial)


@needs_ref
def test_stroke_mapping_matches_random_masks():
    from PIL import Image
    dl = R.dataloader()
    for trial in range(200):
        size = (512, 256, 96)[trial % 3]
        u = OI.uniforms(7, trial, 1)[0]
        p = np.zeros(OI.PARAM_INTS, np.int32)
        OI.strokes_from_uniforms(size, u, p)
        # the reference's draw order: nlines, then per line 4 coordinates + width, nell, then per ellipse 2 corners + 2 extents;
        # the sampler's fixed slots for strokes that are not drawn are skipped
        order = [u[41]]
        for k in range(int(p[5])):
            order += [u[42 + 5 * k + t] for t in range(5)]
        order.append(u[67])
        for k in range(int(p[6])):
            order += [u[68 + 4 * k + t] for t in range(4)]
        d = _Draws(order)

        class FakeRandom:
            @staticmethod
            def randint(lo, hi):
                return lo + int(np.float64(d.next()) * (hi - lo + 1))

            @staticmethod
            def choices(pop, k):
                return [pop[int(np.float64(d.next()) * len(pop))] for _ in range(k)]

        with um.patch.object(dl, "random", FakeRandom), R.recording() as rec:
            rec["box"] = (0, 0, 1, 1)
            dl.random_masks(Image.new("L", (size, size)), size=size, offset=10)
        np.testing.assert_array_equal(R.params_of(rec)[5:], p[5:])


@needs_ref
def test_stroke_rule_is_within_two_percent_of_pillow_after_dilation():
    from PIL import Image, ImageDraw
    size, diff, holes = 512, 0, 0
    for p in OI.sample(11, 0, [(1024, 1448)] * 50, size):
        im = Image.new("L", (size, size), 0)
        d = ImageDraw.Draw(im)
        for k in range(int(p[5])):
            q = [int(v) for v in p[OI.LINE0 + 5 * k:OI.LINE0 + 5 * k + 5]]
            d.line(q[:4], width=q[4], fill=255)
        for k in range(int(p[6])):
            d.ellipse([int(v) for v in p[OI.ELL0 + 4 * k:OI.ELL0 + 4 * k + 4]], fill=255)
        pil = OI.dilate10(np.array(im) >= 103)
        rule = OI.dilate10(OI.strokes_px(size, p))
        diff += int((pil != rule).sum())
        holes += int(pil.sum())
    assert diff / holes < 0.02, diff / holes


def test_golden_fixture_is_the_restatement():
    import os
    from conftest import GOLDEN
    g = np.load(os.path.join(GOLDEN, "inpaint_data.npz"))
    for k, (seed, H, W, size, strokes, gray) in enumerate(g["cases"]):
        rgb, mask = R.sources(int(seed), int(H), int(W))
        p = g[f"params{k}"]
        assert p[4] == gray
        clean, hole = OI.process(rgb, mask, p, int(size), strokes=bool(strokes))
        ref_hole = np.unpackbits(g[f"hole{k}"])[:size * size].reshape(size, size).astype(bool)
        np.testing.assert_array_equal(clean, g[f"clean{k}"].transpose(1, 2, 0))
        if strokes:
            assert (hole != ref_hole).sum() <= 0.02 * ref_hole.sum()
        else:
            np.testing.assert_array_equal(hole, ref_hole)

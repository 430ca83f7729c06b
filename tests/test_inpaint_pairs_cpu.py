"""The numpy restatement of the raw/clean pair path (tests/inpaint_pair_ref.py) against the reference's own code on the CPU:
Pillow's `L` conversion over every RGB triplet, ImageChops.difference, `TestDataset.process_images` without strokes, and the
golden fixture (tests/golden/inpaint_pairs.npz) against the restatement."""
import os
import random

import numpy as np
import pytest
import torch

import inpaint_pair_ref as P
from conftest import GOLDEN
from oracle import inpaint_data as OI

needs_ref = pytest.mark.skipif(P.R.dataloader() is None, reason="reference not staged in oracle/_ref")


def test_l_conversion_matches_pillow_for_every_rgb_triplet():
    from PIL import Image
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([v >> 16, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    np.testing.assert_array_equal(P.to_l(rgb), np.array(Image.fromarray(rgb).convert("L")))


def test_difference_matches_imagechops():
    from PIL import Image, ImageChops
    rng = np.random.default_rng(5)
    a, b = (rng.integers(0, 256, (97, 131), dtype=np.uint8) for _ in range(2))
    a[0, :256 % 131], b[0, :256 % 131] = 255, 0
    ref = np.array(ImageChops.difference(Image.fromarray(a), Image.fromarray(b)))
    np.testing.assert_array_equal(P.difference(a, b), ref)


@needs_ref
@pytest.mark.parametrize("seed,H,W,out", [(0, 300, 220, 128), (1, 140, 400, 96), (2, 60, 50, 64), (3, 900, 700, 256)])
def test_process_images_without_strokes_is_the_restatement(seed, H, W, out):
    raw, clean = P.pair(seed, H, W)
    random.seed(seed)
    torch.manual_seed(seed)
    for _ in range(3):
        (corr, binary, clean_t), p = P.run_reference(raw, clean, out, add_random_masks=False)
        assert p[4] == 0 and p[5] == 0 and p[6] == 0
        c8, hole = P.process_pair(raw, clean, p, out, strokes=False)
        oc, ob, ocl = OI.to_tensors(c8, hole)
        np.testing.assert_array_equal(ocl, clean_t)
        np.testing.assert_array_equal(ob, binary)
        np.testing.assert_array_equal(oc, corr)


@needs_ref
def test_a_page_paired_with_itself_has_no_text_mask():
    raw, _ = P.pair(7, 120, 160)
    random.seed(7)
    (corr, binary, clean_t), p = P.run_reference(raw, raw, 64, add_random_masks=False)
    assert (binary == 1).all()
    assert not P.process_pair(raw, raw, p, 64, strokes=False)[1].any()


def test_golden_fixture_is_the_restatement():
    g = np.load(os.path.join(GOLDEN, "inpaint_pairs.npz"))
    assert {bool(c[4]) for c in g["cases"]} == {False, True}
    diff = holes = 0
    for k, (seed, H, W, size, strokes) in enumerate(g["cases"]):
        raw, clean = P.pair(int(seed), int(H), int(W))
        p = g[f"params{k}"]
        assert p[4] == 0
        c8, hole = P.process_pair(raw, clean, p, int(size), strokes=bool(strokes))
        ref_hole = np.unpackbits(g[f"hole{k}"])[:size * size].reshape(size, size).astype(bool)
        np.testing.assert_array_equal(P.digest(c8.transpose(2, 0, 1)), g[f"clean_sha256_{k}"])
        if strokes:
            diff, holes = diff + int((hole != ref_hole).sum()), holes + int(ref_hole.sum())
        else:
            np.testing.assert_array_equal(hole, ref_hole)
    # the stroke rule's bound against Pillow's rasteriser holds over many images (test_inpaint_data_cpu), not for every one
    assert diff <= 0.02 * holes, (diff, holes)

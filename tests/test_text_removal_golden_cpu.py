"""The text-removal restatement (tests/text_removal_ref.py) against the golden fixture (tests/golden/text_removal.npz) recorded
from the reference's own statements: the demo's mask, cv2's 10x10 dilation (anchor and border rules) and the corrupted image,
bit for bit.  A second test re-runs the reference's statements from the staged Dataloader.py (oracle/_ref) when that copy and
the packages it imports (cv2, PIL, torchvision) are there."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import text_removal_ref as R
from conftest import GOLDEN, ROOT


def _golden():
    return np.load(os.path.join(GOLDEN, "text_removal.npz"))


def _names(g):
    return sorted({k.split(".")[0] for k in g.files})


def test_fixture_covers_the_cases():
    g = _golden()
    names = _names(g)
    assert len(names) >= 5
    sizes = [g[k + ".page"].shape for k in names]
    assert any(s[0] > 1 for s in sizes)                                              # batch > 1
    assert all(s[2] % 8 and s[3] % 8 for s in sizes)                                  # padding on the right and bottom
    holes = [g[k + ".hole"].mean() for k in names]
    assert min(holes) == 0.0 and max(holes) == 1.0                                    # an all-background and an all-text page
    for k in names:
        logits = torch.from_numpy(g[k + ".logits"])
        assert bool((logits.abs() >= 1e-6).all()) and torch.equal(logits, logits.to(torch.bfloat16).float())
        hole = g[k + ".hole"]
        if "borders" in k:                                                            # text touching every border
            assert hole[:, 0].any() and hole[:, -1].any() and hole[:, :, 0].any() and hole[:, :, -1].any(), k


def test_restatement_matches_golden():
    g = _golden()
    for k in _names(g):
        logits, page = torch.from_numpy(g[k + ".logits"]), torch.from_numpy(g[k + ".page"])
        n, _, h, w = page.shape
        pad = tuple(int(v) for v in g[k + ".pad"])
        assert pad == (0, logits.shape[3] - w, 0, logits.shape[2] - h)
        mask = R.text_mask(logits, h, w)
        assert torch.equal(mask, torch.from_numpy(g[k + ".mask"])), k
        assert torch.equal(R.holes(mask).to(torch.uint8), torch.from_numpy(g[k + ".hole"])), k
        for hu, wu in ((h, w), (h + 11, w + 5)):
            valid, corrupted = R.unet_input(mask, page, hu, wu)
            assert torch.equal(valid[:, :h, :w], 1 - torch.from_numpy(g[k + ".hole"])), k
            assert not bool(valid[:, h:].any()) and not bool(valid[:, :, w:].any())
            assert torch.equal(corrupted[:, :, :h, :w], torch.from_numpy(g[k + ".corrupted"])), k
            assert not bool(corrupted[:, :, h:].any()) and not bool(corrupted[:, :, :, w:].any())
            fill = torch.full((n, 3, hu, wu), -7.0)
            comp = R.composite(fill, page, valid)
            hole = torch.from_numpy(g[k + ".hole"]).bool()[:, None].expand(n, 3, h, w)
            assert torch.equal(comp[~hole], page[~hole]) and bool((comp[hole] == -7.0).all())


def test_golden_matches_reference_dataloader():
    for pkg in ("cv2", "PIL", "torchvision"):
        pytest.importorskip(pkg)
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "Dataloader.py")):
        pytest.skip("the reference is not staged at oracle/_ref")
    spec = importlib.util.spec_from_file_location("make_golden_text_removal", os.path.join(GOLDEN, "make_golden_text_removal.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    dl = gen.load_dataloader()
    g = _golden()
    torch.set_num_threads(8)
    assert sorted(gen.CASES) == _names(g)
    for name, (n, h, w, style) in gen.CASES.items():
        logits, page = gen.case_logits(name, n, h, w, style), gen.case_page(name, n, h, w)
        assert torch.equal(logits, torch.from_numpy(g[name + ".logits"])) and torch.equal(page, torch.from_numpy(g[name + ".page"]))
        demo, hole, corrupted = gen.reference_stages(dl, logits, page)
        assert np.array_equal(demo.numpy(), g[name + ".mask"]), name
        assert np.array_equal(hole.numpy(), g[name + ".hole"]), name
        assert np.array_equal(corrupted.numpy(), g[name + ".corrupted"]), name

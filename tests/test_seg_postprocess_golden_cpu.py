"""The post-processing golden (tests/golden/seg_postprocess.npz) against a fresh run of the reference's own code: the demo's
sigmoid / threshold / max-pool statements and EvaluateSet.resize_mask from the staged Dataloader.py (oracle/_ref).  Skips when
that copy, or one of the packages Dataloader.py imports (cv2, PIL, torchvision), is missing."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_seg_postprocess", os.path.join(GOLDEN, "make_golden_seg_postprocess.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_golden_matches_reference_dataloader():
    for pkg in ("cv2", "PIL", "torchvision"):
        pytest.importorskip(pkg)
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "Dataloader.py")):
        pytest.skip("the reference is not staged at oracle/_ref")
    gen = _generator()
    dl = gen.load_dataloader()
    g = np.load(os.path.join(GOLDEN, "seg_postprocess.npz"))
    torch.set_num_threads(8)
    for name, (n, h, w, pad, out_hw) in gen.CASES.items():
        logits = torch.from_numpy(g[name + ".logits"])
        assert tuple(logits.shape) == (n, 1, h, w)
        assert torch.equal(logits, gen.case_logits(name, n, h, w))
        assert bool((logits.abs() >= 1e-6).all()) and torch.equal(logits, logits.to(torch.bfloat16).float())
        assert tuple(g[name + ".pad"]) == pad and tuple(g[name + ".out_hw"]) == out_hw
        m = gen.reference_postprocess(dl, logits, pad, out_hw)
        assert tuple(m.shape) == (n, 3) + out_hw
        assert np.array_equal(m[:, :1].numpy().astype(np.uint8), g[name + ".mask"]), name

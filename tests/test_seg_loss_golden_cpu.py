"""Pins oracle/seg_loss.py (fp64) to goldens that the reference's own BinaryFocalLoss and SoftBootstrapCrossEntropy produced
(tests/golden/make_golden_seg_loss.py), and the bootstrap indicator rule to torch's CPU sigmoid.  CPU only."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import seg_loss as OL

FOCAL = np.load(os.path.join(GOLDEN, "seg_loss_focal.npz"))
BOOT = np.load(os.path.join(GOLDEN, "seg_loss_bootstrap.npz"))


def _close(got, ref, what):
    """fp64 oracle against the reference's fp32 computation: a few fp32 roundings per element."""
    ref = np.asarray(ref, np.float64)
    np.testing.assert_allclose(got, ref, rtol=2e-6, atol=2e-6 * np.abs(ref).max(), err_msg=what)


@pytest.mark.parametrize("k", range(len(FOCAL["focal_cases"])))
def test_focal_oracle_matches_the_reference(k):
    gamma, _ = FOCAL["focal_cases"][k]
    loss, grad = OL.focal(FOCAL[f"x{k}"], FOCAL[f"t{k}"], gamma=int(gamma))
    _close(loss, FOCAL[f"loss{k}"], "loss")
    _close(grad, FOCAL[f"grad{k}"], "grad")


@pytest.mark.parametrize("k", range(len(BOOT["bootstrap_cases"])))
def test_bootstrap_oracle_matches_the_reference(k):
    size_average, reduce, _ = BOOT["bootstrap_cases"][k]
    reduction = "none" if not reduce else ("mean" if size_average else "sum")
    loss, grad = OL.bootstrap(BOOT[f"x{k}"], BOOT[f"t{k}"], reduction=reduction)
    ref = BOOT[f"loss{k}"]
    if reduction == "none":
        assert ref.shape == (BOOT[f"x{k}"].size, 1)
        loss = loss.reshape(-1, 1)
    _close(loss, ref, "loss")
    _close(grad * BOOT[f"g{k}"].reshape(-1)[0] if reduction != "none" else grad * BOOT[f"g{k}"].reshape(grad.shape),
           BOOT[f"grad{k}"], "grad")


def test_goldens_cover_the_cases():
    assert {tuple(c) for c in FOCAL["focal_cases"]} == {(0, 0), (0, 1), (2, 0), (2, 1)}
    assert {(a, b) for a, b, _ in BOOT["bootstrap_cases"]} == {(1, 1), (0, 1), (1, 0)}
    x = np.concatenate([FOCAL[f"x{k}"].ravel() for k in range(4)])
    assert (x > 0).any() and (x < 0).any() and (np.abs(x) < 1e-7).sum() >= 10


def test_indicator_rule_is_torch_cpu_sigmoid():
    # every bf16 pattern but NaN, and a dense fp32 sweep of all floats of magnitude below 2^-20
    b = torch.arange(0, 65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    b = b[~torch.isnan(b)]
    assert torch.equal(torch.sigmoid(b) > 0.5, torch.from_numpy(OL.indicator(b.numpy())))
    bits = np.arange(0, 0x35800000, 97, dtype=np.int64).astype(np.int32)
    x = np.concatenate([bits.view(np.float32), -bits.view(np.float32)])
    edge = np.array([OL.BOOT_THRESHOLD, np.nextafter(OL.BOOT_THRESHOLD, np.float32(1)), np.nextafter(OL.BOOT_THRESHOLD, np.float32(0))],
                    np.float32)
    x = np.concatenate([x, edge, -edge])
    t = torch.from_numpy(x)
    assert torch.equal(torch.sigmoid(t) > 0.5, torch.from_numpy(OL.indicator(x)))

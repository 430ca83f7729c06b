"""Generate tests/golden/seg_loss_focal.npz and seg_loss_bootstrap.npz: the reference's own `BinaryFocalLoss` and
`SoftBootstrapCrossEntropy` (the staged, unmodified loss.py) on seeded fp32 logits of both signs, near 0 and large, with soft
and hard targets.  Recorded per case: the loss and d loss / d input (for reduce=False: of sum(loss * g) with the seeded g
stored alongside).

    python tests/golden/make_golden_seg_loss.py
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.stage_reference import reference_dir  # noqa: E402

SHAPE = (2, 1, 16, 24)
# focal: (gamma, hard targets); bootstrap: (size_average, reduce, hard targets)
FOCAL = [(0, False), (0, True), (2, False), (2, True)]
BOOTSTRAP = [(True, True, False), (True, True, True), (False, True, False), (True, False, False), (True, False, True)]


def inputs(seed, hard):
    """Logits: N(0, 3) with every 7th element near 0 (around sigmoid's 0.5 rounding edge) and a few at +-20; targets soft in
    [0, 1] with exact 0s and 1s, or hard {0, 1}."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(SHAPE) * 3).astype(np.float32)
    flat = x.reshape(-1)
    near = np.array([0.0, 1e-9, -1e-9, 8.9e-8, 8.940697e-08, 8.9407e-08, 1.2e-7, -1.2e-7, 3e-8, -3e-8], np.float32)
    flat[::7] = near[np.arange(flat[::7].size) % near.size]
    flat[3::41] = 20.0
    flat[5::43] = -20.0
    if hard:
        t = (rng.random(SHAPE) < 0.3).astype(np.float32)
    else:
        t = rng.random(SHAPE).astype(np.float32)
        t.reshape(-1)[::5] = 0.0
        t.reshape(-1)[2::9] = 1.0
    return x, t


def main():
    ref = reference_dir()
    if ref is None:
        raise SystemExit("stage the reference first (oracle/stage_reference.py)")
    sys.path.insert(0, ref)
    import loss as L  # the reference's loss.py
    out = {"focal_cases": np.array(FOCAL, np.int64)}
    for k, (gamma, hard) in enumerate(FOCAL):
        x, t = inputs(10 + k, hard)
        xi = torch.from_numpy(x).requires_grad_(True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            loss = L.BinaryFocalLoss(gamma=gamma)(xi, torch.from_numpy(t))
        loss.backward()
        out.update({f"x{k}": x, f"t{k}": t, f"loss{k}": loss.detach().numpy(), f"grad{k}": xi.grad.numpy()})
    np.savez_compressed(os.path.join(HERE, "seg_loss_focal.npz"), **out)
    out = {"bootstrap_cases": np.array(BOOTSTRAP, np.int64)}
    for k, (size_average, reduce, hard) in enumerate(BOOTSTRAP):
        x, t = inputs(20 + k, hard)
        xi = torch.from_numpy(x).requires_grad_(True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            loss = L.SoftBootstrapCrossEntropy(size_average=size_average, reduce=reduce)(xi, torch.from_numpy(t))
        g = np.random.default_rng(30 + k).uniform(0.5, 1.5, loss.shape).astype(np.float32)
        (loss * torch.from_numpy(g)).sum().backward()
        out.update({f"x{k}": x, f"t{k}": t, f"g{k}": g, f"loss{k}": loss.detach().numpy(), f"grad{k}": xi.grad.numpy()})
    np.savez_compressed(os.path.join(HERE, "seg_loss_bootstrap.npz"), **out)


if __name__ == "__main__":
    main()

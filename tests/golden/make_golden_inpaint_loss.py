"""Generate tests/golden/inpaint_loss_*.npz: the reference's own `loss.InpaintingLoss(VggExtractor(pretrained=False))` (the
staged, unmodified loss.py) with the seeded VGG weights of `oracle.inpaint_loss.vgg_state_dict`, on seeded images and stroke
masks (oracle/masks.py) plus an all-valid case.  Recorded: the total loss, the five unweighted terms (computed with the
reference module's own pieces in its order) and d loss / d output.  8 intra-op threads, as the other goldens.

    python tests/golden/make_golden_inpaint_loss.py
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.inpaint_loss import TERMS, vgg_state_dict  # noqa: E402
from oracle.masks import random_hole_masks  # noqa: E402
from oracle.stage_reference import reference_dir  # noqa: E402

# name -> (batch, size, mask seed or None for all valid, image seed)
CASES = {"inpaint_loss_b2_64": (2, 64, 11, 1), "inpaint_loss_b1_128": (1, 128, 12, 2), "inpaint_loss_valid_b2_64": (2, 64, None, 3)}
VGG_SEED = 0


def inputs(n, s, mask_seed, seed):
    """(clean, mask, output) float32 NCHW: a smooth image with edges, a stroke mask (1 = valid), an output that differs from
    the clean image everywhere."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:s, 0:s] / s
    clean = np.stack([np.stack([0.5 + 0.4 * np.sin(6 * xx * (c + 1) + 3 * yy + k) for c in range(3)]) for k in range(n)])
    clean = np.clip(clean + rng.uniform(-0.05, 0.05, clean.shape), 0, 1).astype(np.float32)
    mask = np.ones((n, 3, s, s), np.float32) if mask_seed is None else random_hole_masks(n, s, s, seed=mask_seed)
    output = np.clip(clean + rng.normal(0, 0.2, clean.shape), -0.2, 1.2).astype(np.float32)
    return clean, mask, output


def main():
    ref = reference_dir()
    if ref is None:
        raise SystemExit("stage the reference first (oracle/stage_reference.py)")
    sys.path.insert(0, ref)
    import loss as L  # the reference's loss.py
    torch.set_num_threads(8)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        crit = L.InpaintingLoss(L.VggExtractor(pretrained=False))
    crit.feature_encoder.layers.load_state_dict({k[len("features."):]: v for k, v in vgg_state_dict(VGG_SEED).items()})
    for name, (n, s, mseed, seed) in CASES.items():
        clean, mask, output = inputs(n, s, mseed, seed)
        origin = torch.from_numpy(clean)
        m = torch.from_numpy(mask)
        raw = origin * m
        out = torch.from_numpy(output).requires_grad_(True)
        loss = crit(raw, m, out, origin)
        loss.backward()
        with torch.no_grad():   # the terms, from the module's own pieces in forward's order
            comp = m * raw + (1 - m) * out
            fc, fo, fr = crit.feature_encoder(comp), crit.feature_encoder(out), crit.feature_encoder(origin)
            terms = [crit.l1(m * out, m * origin), crit.l1((1 - m) * out, (1 - m) * origin), L.total_variation_loss(comp),
                     sum(map(crit.l1, fc, fr)) + sum(map(crit.l1, fo, fr)),
                     sum(map(lambda x, y: crit.l1(L.gram_matrix(x), L.gram_matrix(y)), fo, fr))
                     + sum(map(lambda x, y: crit.l1(L.gram_matrix(x), L.gram_matrix(y)), fc, fr))]
        np.savez_compressed(os.path.join(HERE, name + ".npz"), cfg=np.array([n, s, VGG_SEED], np.int64), clean=clean,
                            hole=np.packbits(mask[:, 0] == 0), output=output, loss=loss.detach().numpy(),
                            terms=np.array([float(t) for t in terms], np.float32), term_names=np.array(TERMS),
                            grad=out.grad.numpy())
        print(name, float(loss), [float(t) for t in terms])


if __name__ == "__main__":
    main()

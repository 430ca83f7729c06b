"""Generate tests/golden/seg_data.npz: the reference's own `TextSegmentationData.process_images` (staged Dataloader.py, with
Pillow and torchvision) on sources regenerated from a numpy seed (tests/seg_ref.CASES), with the parameters it drew recorded
(crop box, ColorJitter's order and factors) or forced where a case needs them.

The outputs are stored losslessly as uint8: page = page_u8 / 255.f and mask = mask_u8 / 255.f exactly (checked here).

    python tests/golden/make_golden_seg_data.py
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import inpaint_ref as R  # noqa: E402
import seg_ref as S  # noqa: E402


def main():
    if R.dataloader() is None:
        raise SystemExit("stage the reference first (oracle/stage_reference.py)")
    out = {"cases": np.array([c[:4] for c in S.CASES], dtype=np.int64)}
    for k, (seed, H, W, size, force) in enumerate(S.CASES):
        page, mask = S.case_sources(k)
        random.seed(seed)
        torch.manual_seed(seed)
        (pg, m), p = S.run_reference(page, mask, size, **force)
        pg_u8, m_u8 = np.rint(pg[0] * 255).astype(np.uint8), np.rint(m[0] * 255).astype(np.uint8)
        assert np.array_equal(pg_u8.astype(np.float32)[None] / np.float32(255), pg)
        assert np.array_equal(m_u8.astype(np.float32)[None] / np.float32(255), m)
        out[f"params{k}"] = p
        out[f"page{k}"] = pg_u8
        out[f"mask{k}"] = m_u8
    np.savez_compressed(os.path.join(HERE, "seg_data.npz"), **out)


if __name__ == "__main__":
    main()

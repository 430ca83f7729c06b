"""Generate tests/golden/inpaint_pairs.npz: the reference's own `TestDataset.process_images` (staged Dataloader.py, with Pillow,
cv2 and torchvision) on raw/clean page pairs regenerated from a numpy seed (tests/inpaint_pair_ref.pair), with the crop box and
the stroke arguments it drew recorded.

The outputs are stored losslessly, as in make_golden_inpaint_data.py: clean = clean_u8 / 255.f and binary =
1 - 255 * hole / 255.f exactly (checked here), corrupted = clean * binary.  The hole masks, what this path adds, are kept as
packed bits; of clean_u8 (the resize that tests/golden/inpaint_data.npz pins pixel for pixel) the fixture keeps its SHA-256
(inpaint_pair_ref.digest), which pins it as exactly and keeps the file small.

    python tests/golden/make_golden_inpaint_pairs.py
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import inpaint_pair_ref as P  # noqa: E402

# (source seed, source height, width, output size, random strokes): sources larger and smaller than the output
CASES = [
    (0, 300, 220, 128, False),
    (1, 140, 400, 96, False),
    (2, 1448, 1024, 512, False),
    (3, 50, 60, 64, False),
    (4, 600, 450, 128, True),
    (5, 257, 700, 256, True),
    (6, 200, 180, 256, True),
]


def main():
    if P.R.dataloader() is None:
        raise SystemExit("stage the reference first (oracle/stage_reference.py)")
    out = {"cases": np.array(CASES, dtype=np.int64)}
    for k, (seed, H, W, size, strokes) in enumerate(CASES):
        raw, clean = P.pair(seed, H, W)
        random.seed(seed)
        torch.manual_seed(seed)
        (corr, binary, clean_t), p = P.run_reference(raw, clean, size, bool(strokes))
        assert p[4] == 0
        clean_u8 = np.rint(clean_t * 255).astype(np.uint8)
        hole = binary[0] == 0
        assert np.array_equal(clean_u8.astype(np.float32) / np.float32(255), clean_t)
        assert np.array_equal(np.float32(1) - hole.astype(np.float32) * np.float32(255) / np.float32(255), binary[0])
        assert np.array_equal(clean_t * binary, corr)
        assert hole.any() and not hole.all()
        out[f"params{k}"] = p
        out[f"clean_sha256_{k}"] = P.digest(clean_u8)
        out[f"hole{k}"] = np.packbits(hole)
    np.savez_compressed(os.path.join(HERE, "inpaint_pairs.npz"), **out)


if __name__ == "__main__":
    main()

"""Generate tests/golden/inpaint_data.npz: the reference's own `ImageInpaintingData.process_images` (staged Dataloader.py, with
Pillow, cv2 and torchvision) on sources regenerated from a numpy seed (tests/inpaint_ref.sources), with the parameters it drew
recorded (crop box, grayscale draw, ImageDraw.line / ellipse arguments).

The outputs are stored losslessly as uint8: clean = clean_u8 / 255.f and binary = 1 - 255 * hole / 255.f exactly (checked here),
corrupted = clean * binary.

    python tests/golden/make_golden_inpaint_data.py
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import inpaint_ref as R  # noqa: E402

# (source seed, source height, width, output size, random strokes, grayscale wanted)
CASES = [
    (0, 300, 220, 128, False, 0),
    (1, 140, 400, 96, False, 1),
    (2, 1448, 1024, 512, False, 0),
    (3, 600, 450, 128, True, 0),
    (4, 257, 700, 128, True, 1),
    (5, 90, 120, 64, False, 0),
]


def main():
    if R.dataloader() is None:
        raise SystemExit("stage the reference first (oracle/stage_reference.py)")
    out = {"cases": np.array(CASES, dtype=np.int64)}
    for k, (seed, H, W, size, strokes, gray) in enumerate(CASES):
        rgb, mask = R.sources(seed, H, W)
        random.seed(seed)
        torch.manual_seed(seed)
        while True:
            (corr, binary, clean), p = R.run_reference(rgb, mask, size, bool(strokes))
            if p[4] == gray:
                break
        clean_u8 = np.rint(clean * 255).astype(np.uint8)
        hole = binary[0] == 0
        assert np.array_equal(clean_u8.astype(np.float32) / np.float32(255), clean)
        assert np.array_equal(np.float32(1) - hole.astype(np.float32) * np.float32(255) / np.float32(255), binary[0])
        assert np.array_equal(clean * binary, corr)
        out[f"params{k}"] = p
        out[f"clean{k}"] = clean_u8
        out[f"hole{k}"] = np.packbits(hole)
    np.savez_compressed(os.path.join(HERE, "inpaint_data.npz"), **out)


if __name__ == "__main__":
    main()

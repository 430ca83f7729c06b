"""The raw/clean pair path (`TestDataset.process_images` + `get_mask`, Dataloader.py:201-222): a helper that runs the staged
reference's own code and records what it drew, the numpy restatement that `csrc/inpaint_data.cu` implements for pair sources
(built from oracle/inpaint_data.py), and seeded page pairs.  Shared by the CPU tests, the GPU tests and the golden generator."""
import hashlib

import numpy as np

import inpaint_ref as R
from oracle import inpaint_data as OI


# ------------------------------------------------------------------------------------------------------- restatement
def to_l(rgb):
    """PIL Image.convert("L") of uint8 [..., 3]: (19595 R + 38470 G + 7471 B + 0x8000) >> 16."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    return ((19595 * r + 38470 * g + 7471 * b + 0x8000) >> 16).astype(np.uint8)


def difference(a, b):
    """ImageChops.difference of two `L` images: |a - b|."""
    return np.abs(a.astype(np.int16) - b.astype(np.int16)).astype(np.uint8)


def process_pair(raw, clean, p, out, strokes=True):
    """One pair: (clean uint8 [out, out, 3] after the resize, hole bool [out, out] after the dilation).  Both pages are cropped
    and resized with the box of `p`; the mask is |L(raw) - L(clean)| with the strokes drawn at 255 on it, > 0.4 * 255, dilated
    10x10.  The tensors follow as in OI.to_tensors (no grayscale draw)."""
    box = [int(v) for v in p[:4]]
    raw_r, clean_r = OI.resized_crop(raw, box, out), OI.resized_crop(clean, box, out)
    hole = difference(to_l(raw_r), to_l(clean_r)) >= 103
    if strokes:
        hole |= OI.strokes_px(out, p)
    return clean_r, OI.dilate10(hole)


def digest(clean_u8):
    """SHA-256 of a uint8 [3, s, s] (CHW) clean image, as uint8 [32]: what the golden fixture keeps of the reference's clean
    images.  The image itself is the resize pinned pixel for pixel by tests/golden/inpaint_data.npz; a digest pins it here as
    exactly at a fraction of the size."""
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(clean_u8, np.uint8).tobytes()).digest(), np.uint8)


# ------------------------------------------------------------------------------------------------------- the reference
def dataset(size, add_random_masks):
    """A TestDataset without a folder scan (process_images only needs these attributes)."""
    dl = R.dataloader()
    from torchvision.transforms import Compose, ToTensor
    ds = dl.TestDataset.__new__(dl.TestDataset)
    ds.img_size = (size, size)
    ds.add_random_masks = add_random_masks
    ds.transformer = Compose([ToTensor()])
    return ds


def run_reference(raw, clean, size, add_random_masks):
    """TestDataset.process_images on PIL images of the uint8 arrays: ((corrupted, binary, clean) numpy fp32 CHW, params row)."""
    from PIL import Image
    ds = dataset(size, add_random_masks)
    with R.recording() as rec:
        out = ds.process_images(Image.fromarray(raw), Image.fromarray(clean))
    return tuple(t.numpy() for t in out), R.params_of(rec)


# ------------------------------------------------------------------------------------------------------- sources
def pair(seed, H, W):
    """A clean page (inpaint_ref.sources) and its raw copy: the clean page with seeded dark text-like blocks."""
    clean, _ = R.sources(seed, H, W)
    rng = np.random.default_rng(10_000 + seed)
    raw = clean.copy()
    for _ in range(max(2, H * W // 3000)):
        y, x = int(rng.integers(0, H)), int(rng.integers(0, W))
        raw[y:y + int(rng.integers(2, 10)), x:x + int(rng.integers(2, 24))] = rng.integers(0, 70, 3)
    return raw, clean

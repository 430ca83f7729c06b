"""Helpers that run the reference's own `ImageInpaintingData.process_images` (the staged, unmodified Dataloader.py) and
record the parameters it drew: the crop box (RandomResizedCrop.get_params), the grayscale draw (F.rgb_to_grayscale) and the
stroke arguments (ImageDraw.line / ImageDraw.ellipse).  Shared by the CPU tests, the GPU tests and the golden generator."""
import contextlib
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import inpaint_data as OI  # noqa: E402
from oracle.stage_reference import reference_dir  # noqa: E402

_DL = None


def dataloader():
    """The staged reference Dataloader module, or None when build() staged nothing."""
    global _DL
    if _DL is None:
        ref = reference_dir()
        path = os.path.join(ref, "Dataloader.py") if ref else None
        if not path or not os.path.exists(path):
            return None
        spec = importlib.util.spec_from_file_location("pcb_ref_dataloader", path)
        mod = importlib.util.module_from_spec(spec)
        with contextlib.redirect_stdout(None):
            spec.loader.exec_module(mod)
        _DL = mod
    return _DL


def dataset(size, add_random_masks):
    """An ImageInpaintingData without a folder scan (process_images only needs these attributes)."""
    dl = dataloader()
    from torchvision.transforms import Compose, RandomGrayscale, ToTensor
    ds = dl.ImageInpaintingData.__new__(dl.ImageInpaintingData)
    ds.img_size = (size, size)
    ds.add_random_masks = add_random_masks
    ds.transformer = Compose([RandomGrayscale(p=0.4), ToTensor()])
    return ds


@contextlib.contextmanager
def recording():
    """Patch the reference's draw sites; yields a dict that fills with box / gray / lines / ellipses."""
    import torchvision.transforms.functional as F
    from PIL import ImageDraw
    from torchvision.transforms import RandomResizedCrop
    rec = {"gray": 0, "lines": [], "ellipses": []}
    orig_gp, orig_gray = RandomResizedCrop.get_params, F.rgb_to_grayscale
    orig_line, orig_ell = ImageDraw.ImageDraw.line, ImageDraw.ImageDraw.ellipse

    def gp(*a, **k):
        rec["box"] = orig_gp(*a, **k)
        return rec["box"]

    def gray(*a, **k):
        rec["gray"] = 1
        return orig_gray(*a, **k)

    def line(self, xy, *a, **k):
        rec["lines"].append([int(v) for v in xy] + [int(k["width"])])
        return orig_line(self, xy, *a, **k)

    def ell(self, xy, *a, **k):
        rec["ellipses"].append([int(v) for v in xy])
        return orig_ell(self, xy, *a, **k)

    RandomResizedCrop.get_params = staticmethod(gp)
    F.rgb_to_grayscale = gray
    ImageDraw.ImageDraw.line, ImageDraw.ImageDraw.ellipse = line, ell
    try:
        yield rec
    finally:
        RandomResizedCrop.get_params = staticmethod(orig_gp)
        F.rgb_to_grayscale = orig_gray
        ImageDraw.ImageDraw.line, ImageDraw.ImageDraw.ellipse = orig_line, orig_ell


def params_of(rec):
    """Recorded draws -> the int32 parameter row of oracle.inpaint_data."""
    p = np.zeros(OI.PARAM_INTS, np.int32)
    p[0:4] = rec["box"]
    p[4] = rec["gray"]
    p[5], p[6] = len(rec["lines"]), len(rec["ellipses"])
    for k, ln in enumerate(rec["lines"]):
        p[OI.LINE0 + 5 * k:OI.LINE0 + 5 * k + 5] = ln
    for k, el in enumerate(rec["ellipses"]):
        p[OI.ELL0 + 4 * k:OI.ELL0 + 4 * k + 4] = el
    return p


def run_reference(rgb, mask, size, add_random_masks):
    """process_images on PIL images of the uint8 arrays: ((corrupted, binary, clean) numpy fp32 CHW, params row)."""
    from PIL import Image
    ds = dataset(size, add_random_masks)
    with recording() as rec:
        out = ds.process_images(Image.fromarray(rgb), Image.fromarray(mask))
    return tuple(t.numpy() for t in out), params_of(rec)


def sources(seed, H, W):
    """A smooth RGB page with sharp edges plus a sparse text-like mask, regenerated from a numpy seed."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    base = np.stack([(xx * (1 + c) * 255 // max(W, 1) + yy * (3 - c) * 255 // max(H, 1)) % 256 for c in range(3)], -1)
    rgb = (base + rng.integers(0, 24, (H, W, 3))).clip(0, 255).astype(np.uint8)
    mask = np.zeros((H, W), np.uint8)
    for _ in range(max(1, H * W // 4000)):
        y, x = int(rng.integers(0, H)), int(rng.integers(0, W))
        mask[y:y + int(rng.integers(2, 12)), x:x + int(rng.integers(2, 30))] = rng.integers(60, 256)
    return rgb, mask

"""Helpers that run the reference's own `TextSegmentationData.process_images` (the staged, unmodified Dataloader.py) and
record the parameters it drew: the crop box (RandomResizedCrop.get_params) and ColorJitter's order and factors
(ColorJitter.get_params).  Any of them can be forced instead.  Shared by the CPU tests, the GPU tests and the golden generator."""
import contextlib

import numpy as np

import inpaint_ref as R
from oracle import seg_data as OS


def dataset(size):
    """A TextSegmentationData without a folder scan (process_images only needs these attributes)."""
    dl = R.dataloader()
    from torchvision.transforms import ColorJitter, Compose
    ds = dl.TextSegmentationData.__new__(dl.TextSegmentationData)
    ds.img_size = (size, size)
    ds.transformer = Compose([ColorJitter(brightness=0.2, contrast=0.2, saturation=0.2, hue=0.2)])
    return ds


@contextlib.contextmanager
def recording(box=None, brightness_first=None, b=None, c=None):
    """Patch the reference's draw sites; yields a dict that fills with box / brightness_first / b / c.  Arguments that are not
    None replace the corresponding draw."""
    import torch
    from torchvision.transforms import ColorJitter, RandomResizedCrop
    rec = {}
    orig_gp, orig_cj = RandomResizedCrop.get_params, ColorJitter.get_params

    def gp(*a, **k):
        drawn = orig_gp(*a, **k)
        rec["box"] = tuple(int(v) for v in (box if box is not None else drawn))
        return rec["box"]

    def cj(*a, **k):
        fn_idx, fb, fc, fs, fh = orig_cj(*a, **k)
        if brightness_first is not None:
            fn_idx = torch.tensor([0, 1, 2, 3] if brightness_first else [1, 0, 2, 3])
        idx = [int(v) for v in fn_idx]
        rec["brightness_first"] = int(idx.index(0) < idx.index(1))
        rec["b"] = float(fb if b is None else b)
        rec["c"] = float(fc if c is None else c)
        return fn_idx, rec["b"], rec["c"], fs, fh

    RandomResizedCrop.get_params = staticmethod(gp)
    ColorJitter.get_params = staticmethod(cj)
    try:
        yield rec
    finally:
        RandomResizedCrop.get_params = staticmethod(orig_gp)
        ColorJitter.get_params = staticmethod(orig_cj)


def params_of(rec):
    return OS.params_row(rec["box"], rec["brightness_first"], rec["b"], rec["c"])


def run_reference(page, mask, size, **force):
    """process_images on `L` PIL images of the uint8 arrays: ((page, mask) numpy fp32 [1, s, s], params row)."""
    from PIL import Image
    ds = dataset(size)
    with recording(**force) as rec:
        out = ds.process_images(Image.fromarray(page, "L"), Image.fromarray(mask, "L"))
    return tuple(t.numpy() for t in out), params_of(rec)


def sources(seed, H, W):
    """A gray page (the green channel of inpaint_ref's smooth page) and a sparse text-like mask, regenerated from a numpy seed."""
    rgb, mask = R.sources(seed, H, W)
    return np.ascontiguousarray(rgb[..., 1]), mask


def half_page(H, W, lo=100):
    """A page whose mean is exactly lo + 0.5 (half the pixels lo, half lo + 1): ImageEnhance.Contrast's int(mean + 0.5) sits on
    the .5 boundary."""
    page = np.full((H, W), lo, np.uint8)
    page.reshape(-1)[: H * W // 2] = lo + 1
    return page, (np.arange(H * W).reshape(H, W) % 7 == 0).astype(np.uint8) * 255


# (seed, H, W, out, forced parameters): natural draws, an upscaling box (scale near 0.1), the centre-crop fallback box, both
# orders with factors at 0.8 and 1.2, and the .5 contrast-mean boundary (source == box == output: the resize is the identity)
CASES = [
    (0, 300, 220, 64, {}),
    (1, 181, 240, 96, {"box": (30, 40, 60, 72)}),
    (2, 60, 300, 64, {"box": (0, 110, 60, 80)}),
    (3, 140, 400, 96, {"brightness_first": 1, "b": 0.8, "c": 1.2}),
    (4, 240, 200, 64, {"brightness_first": 0, "b": 1.2, "c": 0.8}),
    (5, 64, 64, 64, {"box": (0, 0, 64, 64), "brightness_first": 0, "b": 1.0, "c": 1.2}),
]


def case_sources(k):
    seed, H, W, _, _ = CASES[k]
    return half_page(H, W) if k == 5 else sources(seed, H, W)


_LOSS = None


def reference_loss_module():
    """The staged reference loss.py (its `models.BaseModels` import resolved to this package's mirror), or None."""
    global _LOSS
    if _LOSS is None:
        import importlib.util
        import warnings

        from ref_inject import reference_dir, reference_l2
        if reference_dir() is None:
            return None
        import os
        with reference_l2("text_segmentation.py"):
            spec = importlib.util.spec_from_file_location("pcb_ref_loss", os.path.join(reference_dir(), "loss.py"))
            mod = importlib.util.module_from_spec(spec)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                spec.loader.exec_module(mod)
        _LOSS = mod
    return _LOSS

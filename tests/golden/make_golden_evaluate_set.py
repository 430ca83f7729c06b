"""Golden fixture of EvaluateSet's page preparation (Dataloader.py:285-305: the resize, Normalize and one-sided pad the
segmentation demo applies, Examples/demo_segmentation.py:59-62), produced on CPU by the reference's own
EvaluateSet.resize_pad_tensor, imported from the staged reference copy oracle/_ref (needs cv2, PIL and torchvision, which
Dataloader.py imports):

    python tests/golden/make_golden_evaluate_set.py

Per page case: the uint8 RGB page [H, W, 3], the resized uint8 image [rh, rw, 3] (the PIL image EvaluateSet hands its
transformer), the normalized padded fp32 tensor [1, 3, hs, ws] and border_pad (left, right, top, bottom).  The pages are
synthetic and compressible: flat colour panels with dark strokes and a patch of noise.

`geometry`: int32 rows (W, H, resize, rh, rw, left, right, top, bottom) of blank pages: every long side in 281..8000 whose
resized long side rounds down to 592 at resize 600, in both orientations, and a spread of ordinary sizes and resizes."""
import contextlib
import importlib.util
import io
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.stage_reference import reference_dir  # noqa: E402

MEAN_STD = ((0.4935, 0.4563, 0.4544), (0.3769, 0.3615, 0.3566))      # the demo's Normalize

# name: (W, H, resize)
CASES = {
    "r600_1109x800": (1109, 800, 600),            # landscape, width rounds to 592: 8 columns of right padding
    "r600_800x1109": (800, 1109, 600),            # portrait, height rounds to 592
    "r64_1024x896": (1024, 896, 64),              # a 16x reduction on both axes
    "r96_1530x1405": (1530, 1405, 96),            # just under 16x on both axes
    "r128_2040x1915": (2040, 1915, 128),
    "r600_300x400": (300, 400, 600),              # upscaling
    "r600_700x700": (700, 700, 600),              # square
    "r600_1203x857": (1203, 857, 600),            # a short side that is not a multiple of 8
}


def quirk_long_sides(fix_len=600, lo=281, hi=8000):
    """long sides L whose int(L * (fix_len / L)) falls below fix_len"""
    return [L for L in range(lo, hi + 1) if int(L * (fix_len / L)) < fix_len]


def geometry_sizes():
    sizes = []
    for L in quirk_long_sides():
        s = L // 7 + 3
        sizes += [(L, s, 600), (s, L, 600)]
    for L in (281, 300, 512, 600, 601, 640, 777, 1000, 1200, 1700, 2480, 3508, 4000, 7999, 8000):
        for s in (L, L * 3 // 4 + 1):
            sizes += [(L, s, 600), (s, L, 600)]
    for W, H, r in ((1024, 1000, 64), (1700, 1200, 512), (1700, 1200, 1024), (640, 480, 96), (333, 2000, 128)):
        sizes += [(W, H, r), (H, W, r)]
    return sorted(set(sizes))


def _seed(name):
    return sum(ord(ch) * (i + 1) for i, ch in enumerate(name))


def case_page(name, W, H):
    """uint8 [H, W, 3]: flat panels, dark text-like strokes and one patch of noise"""
    rng = np.random.Generator(np.random.PCG64(_seed(name)))
    img = np.empty((H, W, 3), np.uint8)
    img[:] = rng.integers(180, 256, 3, dtype=np.uint8)
    for _ in range(6):                                                      # panels
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        img[y0:y0 + int(rng.integers(H // 8, H // 2 + 1)), x0:x0 + int(rng.integers(W // 8, W // 2 + 1))] = \
            rng.integers(0, 256, 3, dtype=np.uint8)
    for _ in range(40):                                                     # strokes
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        img[y0:y0 + max(1, H // 60), x0:x0 + max(2, W // 12)] = rng.integers(0, 60, 3, dtype=np.uint8)
    y0, x0 = int(rng.integers(0, H - H // 16)), int(rng.integers(0, W - W // 16))   # noise
    patch = img[y0:y0 + H // 16, x0:x0 + W // 16]
    patch[:] = rng.integers(0, 256, patch.shape, dtype=np.uint8)
    return img


def load_dataloader():
    path = os.path.join(reference_dir(), "Dataloader.py")
    spec = importlib.util.spec_from_file_location("reference_Dataloader", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_prepare(dl, img, resize):
    """(resized uint8 [rh, rw, 3], normalized padded fp32 [1, 3, hs, ws], border_pad) by EvaluateSet.resize_pad_tensor"""
    from PIL import Image
    with tempfile.TemporaryDirectory() as empty, contextlib.redirect_stdout(io.StringIO()):
        ev = dl.EvaluateSet(MEAN_STD[0], MEAN_STD[1], img_folder=empty, resize=resize)
    seen = []
    transformer = ev.transformer

    def recording(pil_img):                                                 # the resized image, as the transformer gets it
        seen.append(np.array(pil_img, dtype=np.uint8))
        return transformer(pil_img)
    ev.transformer = recording
    x, _, unpadder = ev.resize_pad_tensor(Image.fromarray(img, "RGB"))
    pad = tuple(-int(v) for v in unpadder.transforms[0].padding)
    return seen[0], x.numpy(), np.asarray(pad, np.int32)


def main():
    import torch
    torch.set_num_threads(8)
    dl = load_dataloader()
    arrs = {}
    for name, (W, H, resize) in CASES.items():
        img = case_page(name, W, H)
        resized, x, pad = reference_prepare(dl, img, resize)
        arrs[name + ".page"] = img
        arrs[name + ".resize"] = np.asarray(resize, np.int32)
        arrs[name + ".resized"] = resized
        arrs[name + ".input"] = x
        arrs[name + ".pad"] = pad
        print(f"{name}: {W}x{H} -> {resized.shape[1]}x{resized.shape[0]}, pad {tuple(pad.tolist())}, input {x.shape[3]}x{x.shape[2]}")
    rows = []
    for W, H, resize in geometry_sizes():
        resized, _, pad = reference_prepare(dl, np.zeros((H, W, 3), np.uint8), resize)
        rows.append((W, H, resize, resized.shape[0], resized.shape[1], *pad))
    arrs["geometry"] = np.asarray(rows, np.int32)
    print(f"geometry: {len(rows)} sizes, {sum(1 for r in rows if max(r[3], r[4]) == 592)} with a 592 long side")
    path = os.path.join(HERE, "evaluate_set.npz")
    np.savez_compressed(path, **arrs)
    print(f"evaluate_set: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()

"""Golden fixture of the text-removal glue (engine.TextRemovalStep stages 3-5, ops.removal_holes), produced on CPU by the
reference's own code, imported from the staged reference copy oracle/_ref (needs cv2, PIL and torchvision, which Dataloader.py
imports):

  * the demo's statements (Examples/demo_segmentation.py:33-36: sigmoid, > 0.5, 3x3 max-pool, the unpadder) with the unpadder
    built by EvaluateSet.resize_mask (Dataloader.py:308-316) for the page's own size;
  * the demo's mask image (demo_segmentation.py:41-42: to_pil_image(mask[0]).convert("L"));
  * the threshold and dilation lines of ImageInpaintingData.process_images (Dataloader.py:120-121);
  * binary_mask and corrupted_img as there (:128-131), on the page.

    python tests/golden/make_golden_text_removal.py

Per case: logits [n, 1, hs, ws] (bf16-representable, |x| >= 1e-6, so sigmoid(x) > 0.5 does not hinge on how a sigmoid
rounds next to 0), pad (left, right, top, bottom), page fp32 [n, 3, h, w] (uint8 / 255, as to_tensor makes it), the demo's mask
uint8 [n, 1, h, w], the hole mask uint8 [n, h, w] and the corrupted image fp32 [n, 3, h, w]."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.stage_reference import reference_dir  # noqa: E402

# name: (batch, page h, page w, logit style); the logits cover the page padded on the right and bottom to multiples of 8
CASES = {
    "b1_37x53_blobs": (1, 37, 53, "blobs"),
    "b2_45x30_borders": (2, 45, 30, "borders"),
    "b1_20x27_background": (1, 20, 27, "background"),
    "b1_19x26_text": (1, 19, 26, "text"),
    "b3_61x44_blobs": (3, 61, 44, "blobs"),
}


def padded(v):
    return (v + 7) // 8 * 8


def _seed(name):
    return sum(ord(ch) * (i + 1) for i, ch in enumerate(name))


def case_logits(name, n, h, w, style):
    """[n, 1, hs, ws] logits: smooth blobs plus noise ("blobs"), blobs centred on the four borders and corners ("borders"),
    all negative ("background") or all positive ("text"); rounded to bf16, |x| >= 1e-6."""
    hs, ws = padded(h), padded(w)
    rng = np.random.Generator(np.random.PCG64(_seed(name)))
    yy, xx = np.meshgrid(np.arange(hs, dtype=np.float32), np.arange(ws, dtype=np.float32), indexing="ij")
    out = np.empty((n, 1, hs, ws), np.float32)
    for i in range(n):
        if style == "background":
            f = -rng.uniform(0.5, 4.0, (hs, ws)).astype(np.float32)
        elif style == "text":
            f = rng.uniform(0.5, 4.0, (hs, ws)).astype(np.float32)
        else:
            f = np.full((hs, ws), -3.0, np.float32)
            if style == "borders":
                centres = [(0, rng.uniform(0, w)), (h - 1, rng.uniform(0, w)), (rng.uniform(0, h), 0), (rng.uniform(0, h), w - 1),
                           (0, 0), (h - 1, w - 1)]
            else:
                centres = [(rng.uniform(0, h), rng.uniform(0, w)) for _ in range(3)]
            for cy, cx in centres:
                r = rng.uniform(1.0, 3.0)
                f += 6.0 * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))
            f += rng.normal(0, 0.5, (hs, ws)).astype(np.float32)
        out[i, 0] = f
    x = torch.from_numpy(out).to(torch.bfloat16).float()
    return torch.where(x.abs() < 1e-6, torch.full_like(x, -0.5), x)


def case_page(name, n, h, w):
    """fp32 [n, 3, h, w] in [0, 1] as to_tensor makes it from an 8-bit RGB page."""
    rng = np.random.Generator(np.random.PCG64(_seed(name) + 1))
    return torch.from_numpy(rng.integers(0, 256, (n, 3, h, w), dtype=np.uint8)).float().div(255)


def load_dataloader():
    path = os.path.join(reference_dir(), "Dataloader.py")
    spec = importlib.util.spec_from_file_location("reference_Dataloader", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_stages(dl, logits, page):
    """(demo mask uint8 [n, 1, h, w], hole mask uint8 [n, h, w], corrupted fp32 [n, 3, h, w]) by the reference's statements."""
    import cv2
    from torch.nn import functional as F
    from torchvision.transforms.functional import to_pil_image, to_tensor
    n, _, h, w = page.shape
    hs, ws = logits.shape[2:]
    unpadder = dl.EvaluateSet.resize_mask((0, ws - w, 0, hs - h), (w, h))
    prob = F.sigmoid(logits)                                                    # demo_segmentation.py:33-36
    mask = prob > 0.5
    mask = torch.nn.MaxPool2d(kernel_size=(3, 3), padding=(1, 1), stride=1)(mask.float()).byte()
    mask = unpadder(mask)
    mask = mask.float().cpu()
    demo, hole, corrupted = [], [], []
    for i in range(n):
        mask_np = to_pil_image(mask[i]).convert("L")                           # demo_segmentation.py:41-42
        mask_np = np.array(mask_np, dtype='uint8')
        m = np.where(np.array(mask_np) > dl.brightness_difference * 255, np.uint8(255), np.uint8(0))   # Dataloader.py:120-121
        m = cv2.dilate(m, np.ones((10, 10), np.uint8), iterations=1)
        m = np.expand_dims(m, -1)
        mask_t = to_tensor(m)                                                   # Dataloader.py:128-131
        binary_mask = (1 - mask_t)
        binary_mask = binary_mask.expand(3, -1, -1)
        corrupted.append(page[i] * binary_mask)
        demo.append(mask[i, :1].to(torch.uint8))
        hole.append(torch.from_numpy((m[:, :, 0] != 0).astype(np.uint8)))
    return torch.stack(demo), torch.stack(hole), torch.stack(corrupted)


def main():
    torch.set_num_threads(8)
    dl = load_dataloader()
    arrs = {}
    for name, (n, h, w, style) in CASES.items():
        logits, page = case_logits(name, n, h, w, style), case_page(name, n, h, w)
        demo, hole, corrupted = reference_stages(dl, logits, page)
        arrs[name + ".logits"] = logits.numpy()
        arrs[name + ".pad"] = np.asarray((0, logits.shape[3] - w, 0, logits.shape[2] - h), np.int32)
        arrs[name + ".page"] = page.numpy()
        arrs[name + ".mask"] = demo.numpy()
        arrs[name + ".hole"] = hole.numpy()
        arrs[name + ".corrupted"] = corrupted.numpy()
        print(f"{name}: text {float(demo.float().mean()):.3f}, holes {float(hole.float().mean()):.3f}")
    path = os.path.join(HERE, "text_removal.npz")
    np.savez_compressed(path, **arrs)
    print(f"text_removal: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()

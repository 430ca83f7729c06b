"""Golden fixture of the text-mask post-processing (ops.text_mask_postprocess), produced on CPU by the reference's own code:
the demo's statements (Examples/demo_segmentation.py:33-36: sigmoid, > 0.5, 3x3 max-pool) followed by the resizer of
EvaluateSet.resize_mask (Dataloader.py:308-316: unpad, bilinear resize to the original size, > 0), imported from the staged
reference copy oracle/_ref (needs cv2, PIL and torchvision, which Dataloader.py imports).

    python tests/golden/make_golden_seg_postprocess.py

The logits are bf16-representable (the kernel reads bf16 and fp32 logits) and keep |x| >= 1e-6, so sigmoid(x) > 0.5 does not
hinge on how a particular sigmoid implementation rounds next to 0."""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle.stage_reference import reference_dir  # noqa: E402

# name: (batch, padded h, padded w, border pad (left, right, top, bottom) as EvaluateSet builds it, original (h, w))
CASES = {
    "crop_right_upscale": (1, 48, 48, (0, 12, 0, 0), (100, 75)),
    "crop_bottom_downscale": (1, 64, 64, (0, 0, 0, 20), (30, 40)),
    "batch3_crop_right": (3, 40, 40, (0, 8, 0, 0), (57, 41)),
    "batch2_same_size": (2, 32, 32, (0, 0, 0, 0), (32, 32)),
}


def case_logits(name, n, h, w):
    """Smooth blobs plus noise, rounded to bf16, |x| >= 1e-6."""
    seed = sum(ord(ch) * (i + 1) for i, ch in enumerate(name))
    rng = np.random.Generator(np.random.PCG64(seed))
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    out = np.empty((n, 1, h, w), np.float32)
    for i in range(n):
        f = np.full((h, w), -2.0, np.float32)
        for _ in range(4):
            cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, max(3, h / 5))
            f += 5.0 * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))
        out[i, 0] = f + rng.normal(0, 0.8, (h, w)).astype(np.float32)
    x = torch.from_numpy(out).to(torch.bfloat16).float()
    return torch.where(x.abs() < 1e-6, torch.full_like(x, 0.5), x)


def load_dataloader():
    path = os.path.join(reference_dir(), "Dataloader.py")
    spec = importlib.util.spec_from_file_location("reference_Dataloader", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_postprocess(dl, logits, border_pad, out_hw):
    """demo_segmentation.py:33-36 with `unpadder` = EvaluateSet.resize_mask(border_pad, origin PIL size (w, h))."""
    from torch.nn import functional as F
    unpadder = dl.EvaluateSet.resize_mask(border_pad, (out_hw[1], out_hw[0]))
    prob = F.sigmoid(logits)
    mask = prob > 0.5
    mask = torch.nn.MaxPool2d(kernel_size=(3, 3), padding=(1, 1), stride=1)(mask.float()).byte()
    mask = unpadder(mask)
    return mask                                            # bool [n, 3, oh, ow]


def main():
    torch.set_num_threads(8)
    dl = load_dataloader()
    arrs = {}
    for name, (n, h, w, pad, out_hw) in CASES.items():
        logits = case_logits(name, n, h, w)
        m = reference_postprocess(dl, logits, pad, out_hw)
        assert bool((m == m[:, :1]).all())
        arrs[name + ".logits"] = logits.numpy()
        arrs[name + ".pad"] = np.asarray(pad, np.int32)
        arrs[name + ".out_hw"] = np.asarray(out_hw, np.int32)
        arrs[name + ".mask"] = m[:, :1].numpy().astype(np.uint8)
        print(f"{name}: {tuple(m.shape)}, {float(m[:, :1].float().mean()):.3f} set")
    path = os.path.join(HERE, "seg_postprocess.npz")
    np.savez_compressed(path, **arrs)
    print(f"seg_postprocess: {os.path.getsize(path) / 1024:.1f} KiB")


if __name__ == "__main__":
    main()

"""Golden fixture of the segmentation demo's region image (ops.text_region_hulls), produced on CPU by the reference's own
draw_bounding_box (Examples/demo_segmentation.py:17-25): its FunctionDef is taken from the file with `ast` and executed with
cv2 -- the module itself is never imported, since it loads a checkpoint at import.  Applied as the demo applies it
(:40-45): to np.array(to_pil_image(page)) and the mask image to_pil_image(mask.float()).convert("L").

    python tests/golden/make_golden_text_regions.py         # reads $PCB_REFERENCE (default /root/reference)

Per case: mask uint8 [n, 1, h, w] (1 = text), page fp32 [n, 3, h, w] (uint8 / 255, as to_tensor makes it), threshold
(float64) and out uint8 [n, h, w, 3]; `cv2_version` records the OpenCV that drew them."""
import ast
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = os.environ.get("PCB_REFERENCE", "/root/reference")


def _seed(name):
    return sum(ord(ch) * (i + 1) for i, ch in enumerate(name))


def load_draw_bounding_box():
    import cv2
    path = os.path.join(REFERENCE, "Examples", "demo_segmentation.py")
    tree = ast.parse(open(path).read(), path)
    fdef = next(node for node in tree.body if isinstance(node, ast.FunctionDef) and node.name == "draw_bounding_box")
    scope = {"cv2": cv2}
    exec(compile(ast.Module(body=[fdef], type_ignores=[]), path, "exec"), scope)
    return scope["draw_bounding_box"]


def _rect(m, y0, x0, y1, x1, v=1):
    m[max(y0, 0):max(y1, 0), max(x0, 0):max(x1, 0)] = v


def glyphs(rng, h, w):
    """rings and nested islands in their holes, like 口, 回 and 日, at random places"""
    m = np.zeros((h, w), np.uint8)
    for _ in range(4):
        s = int(rng.integers(9, 16))
        y, x = int(rng.integers(0, h - s)), int(rng.integers(0, w - s))
        _rect(m, y, x, y + s, x + s)
        _rect(m, y + 2, x + 2, y + s - 2, x + s - 2, 0)
        kind = int(rng.integers(0, 3))
        if kind == 0:                                                   # 回: an island in the hole
            _rect(m, y + 4, x + 4, y + s - 4, x + s - 4)
            _rect(m, y + 5, x + 5, y + s - 5, x + s - 5, 0)
        elif kind == 1:                                                 # 日: a bar splitting the hole
            _rect(m, y + s // 2, x + 2, y + s // 2 + 1, x + s - 2)
        else:                                                           # 口 with a dot inside
            m[y + s // 2, x + s // 2] = 1
    return m


def borders(rng, h, w):
    """blobs on each border and corner"""
    m = np.zeros((h, w), np.uint8)
    for cy, cx in ((0, w // 2), (h - 1, w // 3), (h // 2, 0), (h // 3, w - 1), (0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)):
        r = int(rng.integers(2, 6))
        yy, xx = np.ogrid[:h, :w]
        m[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = 1
    return m


def lines(rng, h, w):
    """single pixels, horizontal, vertical and 1-px diagonal lines"""
    m = np.zeros((h, w), np.uint8)
    for _ in range(5):
        m[rng.integers(0, h), rng.integers(0, w)] = 1
    m[3, 5:5 + w // 2] = 1
    m[6:6 + h // 2, w - 4] = 1
    for i in range(min(h, w) // 2):
        m[h // 3 + i, 2 + i] = 1
        m[h - 3 - i, w // 2 + i] = 1
    return m


def noise(rng, h, w):
    return (rng.random((h, w)) < 0.2).astype(np.uint8)


def serpent(rng, h, w):
    """a serpentine text component, and a serpentine background corridor inside a block that opens to the outside at one end"""
    m = np.zeros((h, w), np.uint8)
    half = w // 2
    for i, y in enumerate(range(1, h - 1, 4)):
        _rect(m, y, 1, y + 2, half - 2)
        c = 1 if i % 2 else half - 4
        _rect(m, y, c, y + 4, c + 2)
    _rect(m, 0, half, h, w)                                             # a block carved by a corridor that reaches the border
    for i, y in enumerate(range(2, h - 2, 4)):
        _rect(m, y, half + 2, y + 2, w - 2, 0)
        c = half + 2 if i % 2 else w - 4
        _rect(m, y, c, y + 4, c + 2, 0)
    _rect(m, 2, w - 4, 4, w, 0)                                         # the corridor's mouth on the right border
    return m


def at_threshold(rng, h, w, t):
    """rectangles of contourArea exactly t, t - 0.5 (a corner cut), t + 0.5 (cut plus a bump) and t + 1 (a bump)"""
    a, b = (11, 11) if t == 100 else (21, 26)
    m = np.zeros((h, w), np.uint8)
    for k, (y, x) in enumerate(((2, 2), (2, 4 + b + 2), (4 + a + 2, 2), (4 + a + 2, 4 + b + 2))):
        _rect(m, y, x, y + a, x + b)
        if k in (1, 2):
            m[y, x] = 0                                                 # a corner cut: -0.5
        if k in (2, 3):
            m[y + a // 2, x + b] = 1                                    # a bump on the right side: +1
    return m


def full(rng, h, w):
    return np.ones((h, w), np.uint8)


def empty(rng, h, w):
    return np.zeros((h, w), np.uint8)


# name: (batch, h, w, threshold, mask styles per page)
CASES = {
    "glyphs_b1_47x61_t0": (1, 47, 61, 0, ("glyphs",)),
    "glyphs_b2_47x61_t100": (2, 47, 61, 100, ("glyphs", "glyphs")),
    "borders_b1_33x45_t0": (1, 33, 45, 0, ("borders",)),
    "borders_b1_33x45_tm1": (1, 33, 45, -1, ("borders",)),
    "lines_b1_37x41_tm1": (1, 37, 41, -1, ("lines",)),
    "lines_b1_37x41_t0": (1, 37, 41, 0, ("lines",)),
    "empty_full_b2_19x23_tm1": (2, 19, 23, -1, ("empty", "full")),
    "full_b1_31x29_t500": (1, 31, 29, 500, ("full",)),
    "full_b1_31x29_t100": (1, 31, 29, 100, ("full",)),
    "noise_b1_53x67_tm1": (1, 53, 67, -1, ("noise",)),
    "noise_b3_29x31_t0": (3, 29, 31, 0, ("noise", "noise", "noise")),
    "serpent_b1_45x64_t100": (1, 45, 64, 100, ("serpent",)),
    "serpent_b1_45x64_t500": (1, 45, 64, 500, ("serpent",)),
    "threshold_b1_33x33_t100": (1, 33, 33, 100, ("at_threshold",)),
    "threshold_b1_53x63_t500": (1, 53, 63, 500, ("at_threshold",)),
    "mixed_b3_41x39_t20": (3, 41, 39, 20, ("glyphs", "lines", "borders")),
}


def case_inputs(name):
    n, h, w, t, styles = CASES[name]
    rng = np.random.Generator(np.random.PCG64(_seed(name)))
    gen = {"glyphs": glyphs, "borders": borders, "lines": lines, "noise": noise, "serpent": serpent, "full": full, "empty": empty}
    masks = []
    for s in styles:
        masks.append(at_threshold(rng, h, w, t) if s == "at_threshold" else gen[s](rng, h, w))
    mask = np.stack(masks)[:, None].astype(np.uint8)
    page = torch.from_numpy(rng.integers(0, 256, (n, 3, h, w), dtype=np.uint8)).float().div(255)
    return mask, page, float(t)


def reference_out(draw, mask, page, threshold):
    from torchvision.transforms.functional import to_pil_image
    outs = []
    for i in range(mask.shape[0]):
        origin_np = np.array(to_pil_image(page[i]))                                     # demo_segmentation.py:40-43
        mask_np = to_pil_image(torch.from_numpy(mask[i]).float()).convert("L")
        mask_np = np.array(mask_np, dtype='uint8')
        outs.append(draw(origin_np, mask_np, threshold))
    return np.stack(outs)


def main():
    import cv2
    draw = load_draw_bounding_box()
    arrs = {"cv2_version": np.asarray(cv2.__version__)}
    for name in CASES:
        mask, page, t = case_inputs(name)
        out = reference_out(draw, mask, page, t)
        arrs[name + ".mask"] = mask
        arrs[name + ".page"] = page.numpy()
        arrs[name + ".threshold"] = np.asarray(t, np.float64)
        arrs[name + ".out"] = out
        painted = (out == np.asarray((50, 128, 30), np.uint8)).all(-1).mean()
        print(f"{name}: text {mask.mean():.3f}, painted {painted:.3f}")
    path = os.path.join(HERE, "text_regions.npz")
    np.savez_compressed(path, **arrs)
    print(f"text_regions: {os.path.getsize(path) / 1024:.1f} KiB, cv2 {cv2.__version__}")


if __name__ == "__main__":
    main()

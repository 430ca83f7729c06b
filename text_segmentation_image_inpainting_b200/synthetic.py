"""Synthetic benchmark inputs: seeded free-form hole masks (thick lines + ellipses + square dilation) in the
style of the reference's training data (Dataloader.py:142-162 random_masks, :119-121 10x10 dilation,
:128-129 one plane repeated over RGB).  numpy only; mask convention 1 = valid, 0 = hole."""
import numpy as np


def _draw_line(canvas, x0, y0, x1, y1, width):
    h, w = canvas.shape
    yy, xx = np.mgrid[0:h, 0:w]
    dx, dy = x1 - x0, y1 - y0
    L2 = float(dx * dx + dy * dy) or 1.0
    t = np.clip(((xx - x0) * dx + (yy - y0) * dy) / L2, 0.0, 1.0)
    d2 = (xx - (x0 + t * dx)) ** 2 + (yy - (y0 + t * dy)) ** 2
    canvas[d2 <= (width / 2.0) ** 2] = 0


def _draw_ellipse(canvas, cx, cy, ax, ay):
    h, w = canvas.shape
    yy, xx = np.mgrid[0:h, 0:w]
    canvas[((xx - cx) / ax) ** 2 + ((yy - cy) / ay) ** 2 <= 1.0] = 0


def _dilate_holes(canvas, k):
    hole = (canvas == 0)
    h, w = hole.shape
    pad = k // 2
    p = np.pad(hole, ((pad, k - 1 - pad), (pad, k - 1 - pad)))
    out = np.zeros_like(hole)
    for dy in range(k):
        for dx in range(k):
            out |= p[dy:dy + h, dx:dx + w]
    res = np.ones_like(canvas)
    res[out] = 0
    return res


def random_hole_plane(h, w, rng: np.random.Generator, dilate=10):
    canvas = np.ones((h, w), dtype=np.uint8)
    s = min(h, w) / 512.0
    for _ in range(int(rng.integers(1, 6))):
        x0, x1 = rng.integers(0, w, size=2)
        y0, y1 = rng.integers(0, h, size=2)
        _draw_line(canvas, int(x0), int(y0), int(x1), int(y1), max(2.0, float(rng.integers(15, 21)) * s))
    for _ in range(int(rng.integers(1, 6))):
        cx, cy = int(rng.integers(0, w)), int(rng.integers(0, h))
        ax, ay = rng.integers(20, 71, size=2)
        _draw_ellipse(canvas, cx, cy, max(2.0, float(ax) * s), max(2.0, float(ay) * s))
    if dilate:
        canvas = _dilate_holes(canvas, max(1, int(round(dilate * s))))
    return canvas


def random_hole_masks(n, h, w, seed=0, channels=3):
    """[n, channels, h, w] float32 {0,1} masks, one plane per image repeated over channels."""
    rng = np.random.Generator(np.random.PCG64(seed))
    planes = np.stack([random_hole_plane(h, w, rng) for _ in range(n)]).astype(np.float32)
    return np.repeat(planes[:, None], channels, axis=1)


def manga_text_mask(h, w, seed=0):
    """uint8 [h, w] text mask (1 = text) of a manga-like page: speech-bubble rings (ellipse outlines a few pixels thick),
    each holding columns of glyph-sized blobs (small filled rectangles, some with a hole, some split in two); bubbles cut by
    the page border leave their glyphs as regions of their own."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = np.zeros((h, w), np.uint8)
    s = max(1.0, min(h, w) / 1200.0)
    yy, xx = np.ogrid[0:h, 0:w]
    for _ in range(int(12 * s * s)):
        ay, ax = int(rng.integers(90, 200) * s), int(rng.integers(60, 140) * s)
        cy, cx = int(rng.integers(0, h)), int(rng.integers(0, w))
        y0, y1, x0, x1 = max(cy - ay - 4, 0), min(cy + ay + 5, h), max(cx - ax - 4, 0), min(cx + ax + 5, w)
        if y0 >= y1 or x0 >= x1:
            continue
        r = ((yy[y0:y1] - cy) / ay) ** 2 + ((xx[:, x0:x1] - cx) / ax) ** 2
        m[y0:y1, x0:x1][(r <= 1.0) & (r >= (1 - 3.0 / min(ax, ay)) ** 2)] = 1              # the bubble's ring
        g = int(rng.integers(9, 15) * s)                                                   # glyph pitch
        for col in range(cx + ax // 2 - g, cx - ax // 2, -g - 2):
            for row in range(cy - ay // 2, cy + ay // 2 - g, g + 1):
                if not (0 <= row and row + g <= h and 0 <= col and col + g <= w) or rng.random() < 0.15:
                    continue
                gh, gw = int(rng.integers(g // 2, g)), int(rng.integers(g // 2, g))
                m[row:row + gh, col:col + gw] = 1
                kind = rng.random()
                if kind < 0.3 and gh > 4 and gw > 4:
                    m[row + 2:row + gh - 2, col + 2:col + gw - 2] = 0                      # a glyph with a hole
                elif kind < 0.5 and gw > 3:
                    m[row:row + gh, col + gw // 2] = 0                                     # a glyph in two strokes
    return m

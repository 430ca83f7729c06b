"""numpy / scipy restatement of the segmentation demo's text-region drawing (Examples/demo_segmentation.py:17-25, 40-45:
findContours RETR_TREE, contourArea > threshold, convexHull, drawContours filled in (50, 128, 30)), written as the parallel
formulation ops.text_region_hulls computes (DESIGN 4.14), with no cv2:

  F1  only the outermost components are drawn;
  F2  exterior = background 4-connected to a virtual ring of zeros around the page; each 8-connected component of the other
      pixels is one outer contour's region (the component, its holes and whatever is nested in them);
  F3  contourArea of that contour is Q4 + Q3 / 2 over the 2x2 windows of the zero-padded (h + 1) x (w + 1) grid, so the test
      is ``(2 Q4 + Q3) * 0.5 > threshold`` in double;
  F4  the hull is taken over the region's pixels (per row, its leftmost and rightmost pixel);
  F5  the filled hull is cv2.fillPoly with LINE_8: each edge's 8-connected Bresenham line plus the 16-bit fixed-point
      scanline fill (fill_poly below)."""
import numpy as np
from scipy import ndimage

COLOR = (50, 128, 30)
XY_SHIFT = 16


def page_bytes(page: np.ndarray) -> np.ndarray:
    """np.array(to_pil_image(page)) of fp32 [3, h, w]: mul(255) in fp32, truncated, clamped to [0, 255] (NaN as 0)."""
    v = np.nan_to_num(page.astype(np.float32) * np.float32(255), nan=0.0)
    return np.clip(v, 0, 255).astype(np.uint8).transpose(1, 2, 0).copy()


def line_pixels(p0, p1):
    """cv2.line(LINE_8)'s pixels from p0 to p1 ((x, y) integers): Bresenham started at the left end (LineIterator with
    leftToRight), the major axis stepping every pixel and the minor one when the error term is negative."""
    (x0, y0), (x1, y1) = p0, p1
    if x1 < x0:
        x0, y0, x1, y1 = x1, y1, x0, y0
    dx, dy = x1 - x0, abs(y1 - y0)
    sy = -1 if y1 < y0 else 1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err, x, y, out = dx - 2 * dy, x0, y0, []
    for _ in range(dx + 1):
        out.append((x, y))
        step = err < 0
        err += -2 * dy + (2 * dx if step else 0)
        if vert:
            y += sy
            x += 1 if step else 0
        else:
            x += 1
            y += sy if step else 0
    return out


def fill_poly(img: np.ndarray, pts, color=COLOR):
    """cv2.fillPoly(img, [pts], color, LINE_8) for one polygon of integer vertices inside the image: every edge's line, then
    per scanline y (from the top vertex, bottom vertex excluded) the active edges (y0 <= y < y1, horizontal ones skipped) at
    16-bit fixed point -- x starts at x_top << 16 and steps by ((x1 - x0) << 16) / (y1 - y0) truncated -- sorted, and filled
    pairwise from the lower x rounded up to the higher x rounded down."""
    pts = [(int(x), int(y)) for x, y in pts]
    h, w = img.shape[:2]
    edges = []
    for i in range(len(pts)):
        p0, p1 = pts[i - 1], pts[i]
        for x, y in line_pixels(p0, p1):
            if 0 <= x < w and 0 <= y < h:
                img[y, x] = color
        if p0[1] == p1[1]:
            continue
        a, b = (p0, p1) if p0[1] < p1[1] else (p1, p0)
        num = (p1[0] - p0[0]) << XY_SHIFT
        den = p1[1] - p0[1]
        dx = abs(num) // abs(den) * (1 if (num >= 0) == (den > 0) else -1)     # C division: truncated towards zero
        edges.append((a[1], b[1], a[0] << XY_SHIFT, dx))
    if len(edges) < 2:
        return img
    for y in range(min(e[0] for e in edges), min(max(e[1] for e in edges), h)):
        xs = sorted(x + (y - y0) * dx for y0, y1, x, dx in edges if y0 <= y < y1)
        for k in range(0, len(xs) - 1, 2):
            x1, x2 = (xs[k] + (1 << XY_SHIFT) - 1) >> XY_SHIFT, xs[k + 1] >> XY_SHIFT
            if x1 < w and x2 >= 0:
                img[y, max(x1, 0):min(x2, w - 1) + 1] = color
    return img


def regions(mask: np.ndarray):
    """(labels int32 [h, w], count): F2's regions, labelled 1..count (0 = exterior)."""
    fg = mask != 0
    bg = np.pad(~fg, 1, constant_values=True)
    lab, _ = ndimage.label(bg, structure=ndimage.generate_binary_structure(2, 1))
    exterior = lab[1:-1, 1:-1] == lab[0, 0]
    return ndimage.label(~exterior, structure=np.ones((3, 3), bool))


def doubled_areas(labels: np.ndarray, count: int) -> np.ndarray:
    """int64 [count + 1]: A2 = 2 Q4 + Q3 per label (F3).  Two regions are never 8-adjacent, so the labelled pixels of a window
    belong to one region, the window's largest label."""
    p = np.pad(labels, 1)
    win = np.stack([p[:-1, :-1], p[:-1, 1:], p[1:, :-1], p[1:, 1:]])
    s = (win != 0).sum(0)
    add = np.where(s == 4, 2, np.where(s == 3, 1, 0))
    return np.bincount(win.max(0).ravel(), weights=add.ravel(), minlength=count + 1).astype(np.int64)


def _chain(pts, left):
    """Monotone chain over points already sorted by y (one per row): the left (x convex in y) or right boundary of their hull,
    collinear points dropped."""
    out = []
    for p in pts:
        while len(out) >= 2:
            (ax, ay), (bx, by) = out[-2], out[-1]
            cross = (bx - ax) * (p[1] - ay) - (by - ay) * (p[0] - ax)
            if (cross >= 0) if left else (cross <= 0):
                out.pop()
            else:
                break
        out.append(p)
    return out


def hull(rows_lo, rows_hi, ymin):
    """The convex hull polygon of a region from each row's leftmost and rightmost pixel: the left chain top to bottom, then
    the right chain bottom to top (F4)."""
    ys = range(ymin, ymin + len(rows_lo))
    left = _chain(list(zip(rows_lo, ys)), True)
    right = _chain(list(zip(rows_hi, ys)), False)
    return left + right[::-1]


def text_region_hulls(mask: np.ndarray, page: np.ndarray, area_threshold=500) -> np.ndarray:
    """The demo's draw_bounding_box(np.array(to_pil_image(page)), mask image, area_threshold) for one page: mask uint8
    [h, w] (nonzero = text), page fp32 [3, h, w].  Returns uint8 [h, w, 3]."""
    out = page_bytes(page)
    labels, count = regions(mask)
    if count == 0:
        return out
    keep = doubled_areas(labels, count) * 0.5 > float(area_threshold)
    keep[0] = False
    ys, xs = np.nonzero(keep[labels])
    if len(ys) == 0:
        return out
    lab = labels[ys, xs]
    order = np.lexsort((xs, ys, lab))
    ys, xs, lab = ys[order], xs[order], lab[order]
    key = lab.astype(np.int64) * mask.shape[0] + ys
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]])
    ends = np.r_[starts[1:], len(key)] - 1
    row_lab, row_y, row_lo, row_hi = lab[starts], ys[starts], xs[starts], xs[ends]
    comp = np.flatnonzero(np.r_[True, row_lab[1:] != row_lab[:-1]])
    for a, b in zip(comp, np.r_[comp[1:], len(row_lab)]):
        fill_poly(out, hull(row_lo[a:b].tolist(), row_hi[a:b].tolist(), int(row_y[a])))
    return out


def text_region_hulls_batch(mask: np.ndarray, page: np.ndarray, area_threshold=500) -> np.ndarray:
    """text_region_hulls of every page: mask uint8 [n, 1, h, w], page fp32 [n, 3, h, w] -> uint8 [n, h, w, 3]."""
    return np.stack([text_region_hulls(m[0], p, area_threshold) for m, p in zip(mask, page)])

"""CPU checks of the segmentation demo's region image (ops.text_region_hulls, DESIGN 4.14): the numpy restatement
(tests/text_regions_ref.py) equals the fixture drawn by the reference's own draw_bounding_box (tests/golden/text_regions.npz),
and, where cv2 imports, seeded sweeps check each finding the GPU formulation rests on against OpenCV itself."""
import os

import numpy as np
import pytest

import text_regions_ref as R
from conftest import GOLDEN


def _golden():
    return np.load(os.path.join(GOLDEN, "text_regions.npz"))


def _names(g):
    return sorted({k.split(".")[0] for k in g.files if "." in k})


def test_restatement_matches_golden():
    g = _golden()
    assert str(g["cv2_version"]).startswith("4.")
    names = _names(g)
    assert len(names) >= 12
    thresholds = set()
    for name in names:
        mask, page, t = g[name + ".mask"], g[name + ".page"], float(g[name + ".threshold"])
        thresholds.add(t)
        got = R.text_region_hulls_batch(mask, page, t)
        assert got.dtype == np.uint8 and got.shape == g[name + ".out"].shape, name
        assert np.array_equal(got, g[name + ".out"]), name
    assert {-1.0, 0.0, 100.0, 500.0} <= thresholds


def test_threshold_cases_sit_on_the_boundary():
    """the at-threshold rectangles have doubled areas 2t - 1, 2t, 2t + 1, 2t + 2: only the last two are painted"""
    g = _golden()
    for name in ("threshold_b1_33x33_t100", "threshold_b1_53x63_t500"):
        t = float(g[name + ".threshold"])
        labels, count = R.regions(g[name + ".mask"][0, 0])
        a2 = sorted(R.doubled_areas(labels, count)[1:].tolist())
        assert a2 == [2 * t - 1, 2 * t, 2 * t + 1, 2 * t + 2], (name, a2)


try:
    import cv2
except ImportError:                      # the sweeps against OpenCV itself run where it is installed
    cv2 = None
needs_cv2 = pytest.mark.skipif(cv2 is None, reason="cv2 not installed")


def _demo(img, mask, thr):
    contours, _ = cv2.findContours(mask, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
    for cnt in contours:
        if cv2.contourArea(cnt) > thr:
            cv2.drawContours(img, [cv2.convexHull(cnt)], 0, R.COLOR, -1)
    return img


def _random_mask(rng, h, w):
    m = np.zeros((h, w), np.uint8)
    for _ in range(int(rng.integers(1, 6))):
        cy, cx = int(rng.integers(-5, h + 5)), int(rng.integers(-5, w + 5))
        ax = (int(rng.integers(1, max(2, w // 2))), int(rng.integers(1, max(2, h // 2))))
        thick = -1 if rng.random() < 0.5 else int(rng.integers(1, 4))
        cv2.ellipse(m, (cx, cy), ax, float(rng.uniform(0, 180)), 0, 360, 255, thick)
    noise = rng.random((h, w)) < rng.choice([0.0, 0.02, 0.1, 0.2])
    m[noise] = 255 - m[noise]
    return m


@needs_cv2
def test_fill_poly_matches_cv2():
    """F5: the restated fillPoly (LINE_8 edges plus the fixed-point scanline fill) equals cv2.fillPoly on random hulls"""
    rng = np.random.default_rng(5)
    for t in range(1500):
        h, w = (int(v) for v in rng.integers(3, 200 if t % 3 == 0 else 40, 2))
        k = int(rng.integers(1, 13))
        pts = np.stack([rng.integers(0, w, k), rng.integers(0, h, k)], 1).astype(np.int32)
        hull = cv2.convexHull(pts)
        a = np.zeros((h, w, 3), np.uint8)
        cv2.fillPoly(a, [hull], R.COLOR)
        b = R.fill_poly(np.zeros((h, w, 3), np.uint8), hull[:, 0].tolist())
        assert np.array_equal(a, b), (t, hull[:, 0].tolist())
        # drawContours(thickness=-1) of the hull paints the same pixels, whatever vertex it starts from
        c = cv2.drawContours(np.zeros((h, w, 3), np.uint8), [np.roll(hull, int(rng.integers(0, len(hull))), 0)], 0, R.COLOR, -1)
        assert np.array_equal(a, c), t


@needs_cv2
def test_windowed_area_matches_contour_area():
    """F2 + F3: per outer contour, cv2.contourArea equals (2 Q4 + Q3) / 2 of its region"""
    rng = np.random.default_rng(6)
    for t in range(200):
        h, w = (int(v) for v in rng.integers(4, 90, 2))
        m = _random_mask(rng, h, w)
        labels, count = R.regions(m)
        a2 = R.doubled_areas(labels, count)
        contours, _ = cv2.findContours(m, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)
        assert len(contours) == count, t
        for cnt in contours:
            x, y = cnt[0, 0]
            assert cv2.contourArea(cnt) == a2[labels[y, x]] * 0.5, t


@needs_cv2
def test_restatement_matches_cv2_pipeline():
    """F1-F5 together: the restatement equals findContours / contourArea / convexHull / drawContours on random masks"""
    rng = np.random.default_rng(7)
    for t in range(150):
        h, w = (int(v) for v in rng.integers(3, 100, 2))
        m = _random_mask(rng, h, w)
        page = rng.integers(0, 256, (3, h, w)).astype(np.float32) / 255
        for thr in (-1, 0, 20, 100, 500):
            want = _demo(R.page_bytes(page), m, thr)
            assert np.array_equal(R.text_region_hulls(m, page, thr), want), (t, thr)

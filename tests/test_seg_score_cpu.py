"""The numpy restatement of the pixel average precision (seg_score_ref.py) against the recorded sklearn fixture
(tests/golden/seg_ap.npz), against sklearn itself where it is installed, and its independence of how pixels are batched."""
import os
import warnings

import numpy as np
import pytest

import seg_score_ref as R
from conftest import GOLDEN


def _golden():
    g = np.load(os.path.join(GOLDEN, "seg_ap.npz"))
    return [(g[f"bits_{k}"], g[f"labels_{k}"].astype(np.float32), float(g["ap"][k])) for k in range(len(g["ap"]))]


def test_restatement_matches_the_recorded_sklearn_scores():
    cases = _golden()
    assert len(cases) == 10
    for bits, labels, ap in cases:
        hist, counts = R.score_counts(bits, labels, bf16=True)
        got = R.average_precision(hist, counts)
        assert abs(got - ap) <= 1e-12 * max(abs(ap), 1e-300), (got, ap)
        assert float(R.average_precision_exact(hist)) == pytest.approx(ap, rel=1e-14, abs=0)
    assert {ap for _, _, ap in cases} >= {0.0, 1.0}


def test_restatement_matches_sklearn_on_random_ties_and_signed_zeros():
    metrics = pytest.importorskip("sklearn.metrics")
    rng = np.random.default_rng(5)
    for case in range(60):
        n = int(rng.integers(1, 3000))
        pool = np.concatenate([rng.normal(0, 2.0 ** rng.integers(-30, 30), int(rng.integers(1, 40))), [0.0, -0.0, np.inf, -np.inf]])
        x = rng.choice(pool, n).astype(np.float32)
        t = rng.random(n).astype(np.float32)
        hist, counts = R.score_counts(x, t)
        y, s = R.sklearn_inputs(x, t)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = float(metrics.average_precision_score(y, s))
        got = R.average_precision(hist, counts)
        assert abs(got - ref) <= 1e-12 * max(abs(ref), 1e-300), (case, got, ref)


def test_rounding_keys_and_threshold_definitions():
    # round to nearest-even at the bf16 midpoints, +-0 folded, +-inf at the ends of the key order
    x = np.array([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, np.float32(1.0 + 2 ** -8) + np.float32(2 ** -20), 3.4e38, -0.0, np.inf, -np.inf],
                 np.float32)
    assert R.bf16_bits(x).tolist() == [0x3F80, 0x3F82, 0x3F81, 0x7F80, 0x8000, 0x7F80, 0xFF80]
    k = R.keys(np.array([0xFF80, 0xBF80, 0x8001, 0x8000, 0x0000, 0x0001, 0x3F80, 0x7F80], np.uint16))
    assert k[3] == k[4] and np.all(np.diff(np.delete(k, 3)) > 0)
    # the threshold is applied to the unrounded logit; the label is target > 0.5 in fp32
    x = np.array([2 ** -25, 2 ** -24, 1.5 * 2 ** -24, np.nextafter(np.float32(1.5 * 2 ** -24), np.float32(1)), -2 ** -24], np.float32)
    t = np.array([0.5, np.nextafter(np.float32(0.5), np.float32(1)), 1.0, 0.0, 1.0], np.float32)
    hist, counts = R.score_counts(x, t)
    # predicted: only the value above 1.5 * 2^-24; labels: entries 1, 2, 4
    assert dict(zip(R.COUNTS, counts.tolist())) == {"tp": 0, "fp": 1, "fn": 3, "tn": 1, "nan": 0}
    hist, counts = R.score_counts(np.array([1.0, np.nan], np.float32), np.ones(2, np.float32))
    assert counts[4] == 1 and hist.sum() == 2 and np.isnan(R.average_precision(hist, counts))


def test_histogram_is_independent_of_the_partition():
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.normal(-4, 3, 20000), [np.nan] * 3, [0.0, -0.0, np.inf]]).astype(np.float32)
    t = rng.random(x.size).astype(np.float32)
    perm = rng.permutation(x.size)
    x, t = x[perm], t[perm]
    whole = R.score_counts(x, t)
    for parts in (2, 8, 37):
        cuts = np.sort(rng.choice(np.arange(1, x.size), parts - 1, replace=False))
        hs = [R.score_counts(a, b) for a, b in zip(np.split(x, cuts), np.split(t, cuts))]
        assert np.array_equal(sum(h for h, _ in hs), whole[0])
        assert np.array_equal(sum(c for _, c in hs), whole[1])
    finite = ~np.isnan(x)
    h, c = R.score_counts(x[finite], t[finite])
    assert R.average_precision(h, c) == R.average_precision(*R.score_counts(x[finite][::-1], t[finite][::-1]))

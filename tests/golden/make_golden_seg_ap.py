"""Record tests/golden/seg_ap.npz: sklearn's average_precision_score on seeded cases of bf16 scores and binary labels.

Per case `k`: `bits_k` (uint16 bf16 bit patterns, no NaN), `labels_k` (uint8) and `ap` [k] (fp64, from
sklearn.metrics.average_precision_score on the fp64 values of the scores, +-inf passed as +-1e300 since sklearn refuses
infinities).  Cases: heavy ties, +-0 mixed, a single pixel (positive and negative), no positives, all positives, scores drawn
from every bf16 binade (subnormals and +-inf included), and clustered logits like a network's.

    python tests/golden/make_golden_seg_ap.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import seg_score_ref as R  # noqa: E402


def cases():
    rng = np.random.default_rng(20261017)
    out = []
    # heavy ties: a handful of distinct scores over many pixels
    for n, distinct in ((1000, 3), (5000, 17), (20000, 200)):
        vals = R.bf16_bits(rng.normal(0, 4, distinct).astype(np.float32))
        out.append((vals[rng.integers(0, distinct, n)], rng.random(n) < 0.3))
    # +-0 among a few other values, labels unrelated to sign
    z = np.array([0x0000, 0x8000, 0x3F80, 0xBF80, 0x0001, 0x8001], np.uint16)
    out.append((z[rng.integers(0, len(z), 3000)], rng.random(3000) < 0.5))
    # a single pixel, positive and negative
    out.append((np.array([0x4000], np.uint16), np.array([True])))
    out.append((np.array([0xC000], np.uint16), np.array([False])))
    # no positives, all positives
    out.append((R.bf16_bits(rng.normal(0, 3, 4000).astype(np.float32)), np.zeros(4000, bool)))
    out.append((R.bf16_bits(rng.normal(0, 3, 4000).astype(np.float32)), np.ones(4000, bool)))
    # every bf16 binade: random mantissa and sign under each of the 256 exponents (0: zeros and subnormals, 255: +-inf only)
    e = np.repeat(np.arange(256, dtype=np.uint32), 40)
    m = rng.integers(0, 128, e.size).astype(np.uint32)
    m[e == 255] = 0
    s = rng.integers(0, 2, e.size).astype(np.uint32)
    bits = ((s << 15) | (e << 7) | m).astype(np.uint16)
    out.append((bits, rng.random(bits.size) < 0.4))
    # clustered logits with labels that depend on them (a network's output)
    lab = rng.random(15000) < 0.1
    x = np.where(lab, rng.normal(3, 2.5, lab.size), rng.normal(-6, 3, lab.size)).astype(np.float32)
    out.append((R.bf16_bits(x), lab))
    return out


def main():
    from sklearn.metrics import average_precision_score
    data, aps = {}, []
    for k, (bits, labels) in enumerate(cases()):
        y, s = R.sklearn_inputs(bits, labels.astype(np.float32), bf16=True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")           # no positives: sklearn warns and returns 0
            aps.append(float(average_precision_score(y, s)))
        data[f"bits_{k}"] = bits.astype(np.uint16)
        data[f"labels_{k}"] = labels.astype(np.uint8)
    data["ap"] = np.array(aps, np.float64)
    np.savez_compressed(os.path.join(HERE, "seg_ap.npz"), **data)
    print(len(aps), "cases:", aps)


if __name__ == "__main__":
    main()

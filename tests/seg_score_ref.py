"""numpy restatement of the pixel average precision of metrics.PixelAveragePrecision (csrc/seg_loss.cu, pcb_seg_score_*).

  * score: the logit rounded to bf16 (fp32 to nearest-even as torch's .to(torch.bfloat16); bf16 logits as they are), -0 as +0,
    +-inf the largest and smallest scores;
  * label: target > 0.5 in fp32;
  * AP:    sklearn.metrics.average_precision_score(labels, scores) over the 65,536 bf16 values in descending order,
           AP = (1 / P) sum_k pos_k TP_k / N_k, 0 without positives, NaN when any logit is NaN;
  * tp, fp, fn, tn at sigmoid(x) > 0.5 of the unrounded logit (x > 1.5 * 2^-24, pcb_common.cuh's sigmoid_above_half).

Everything but the final sum is an integer count, so the histogram of a set of pixels is the sum of the histograms of any
partition of it."""
from fractions import Fraction

import numpy as np

KEYS = 65536
THRESHOLD = np.float32(8.940696716308594e-08)
COUNTS = ("tp", "fp", "fn", "tn", "nan")


def bf16_bits(x):
    """uint16 bf16 bit patterns of fp32 values, rounded to nearest-even (NaN stays NaN, as a quiet pattern)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, dtype=np.float32))
    r[nan] = ((u[nan] >> 16) | 0x40).astype(np.uint16)
    return r


def bf16_value(bits):
    """fp32 values of uint16 bf16 bit patterns."""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def keys(bits):
    """Order-preserving 16-bit keys of non-NaN bf16 bit patterns (-0 as +0)."""
    b = np.asarray(bits, dtype=np.uint32).copy()
    b[b == 0x8000] = 0
    return np.where(b & 0x8000, ~b & 0xFFFF, b | 0x8000).astype(np.int64)


def score_counts(logits, target, bf16=False):
    """(hist int64 [2, 65536], counts int64 [5]) of logits (fp32 values, or uint16 bf16 bit patterns with bf16=True) against
    fp32 targets of the same shape."""
    if bf16:
        bits = np.asarray(logits, dtype=np.uint16).reshape(-1)
        x = bf16_value(bits)
    else:
        x = np.asarray(logits, dtype=np.float32).reshape(-1)
        bits = bf16_bits(x)
    label = np.asarray(target, dtype=np.float32).reshape(-1) > np.float32(0.5)
    nan = np.isnan(x)
    ok = ~nan
    k = keys(bits[ok])
    hist = np.zeros((2, KEYS), np.int64)
    hist[0] = np.bincount(k, minlength=KEYS)
    hist[1] = np.bincount(k[label[ok]], minlength=KEYS)
    pred = x[ok] > THRESHOLD
    lab = label[ok]
    counts = np.array([np.sum(pred & lab), np.sum(pred & ~lab), np.sum(~pred & lab), np.sum(~pred & ~lab), np.sum(nan)], np.int64)
    return hist, counts


def average_precision(hist, counts=None):
    """AP of a histogram in fp64: the terms in descending score order, summed left to right."""
    if counts is not None and counts[4] > 0:
        return float("nan")
    n = hist[0][::-1].astype(np.int64)
    p = hist[1][::-1].astype(np.int64)
    total = int(p.sum())
    if total == 0:
        return 0.0
    N, TP = np.cumsum(n), np.cumsum(p)
    sel = p > 0
    terms = p[sel].astype(np.float64) * (TP[sel].astype(np.float64) / N[sel].astype(np.float64))
    s = 0.0
    for t in terms:
        s += float(t)
    return s / total


def average_precision_exact(hist):
    """The same AP as an exact rational (Python integers: counts beyond 2^53 stay exact)."""
    total = sum(int(v) for v in hist[1])
    if total == 0:
        return Fraction(0)
    acc, N, TP = Fraction(0), 0, 0
    for k in range(KEYS - 1, -1, -1):
        nk, pk = int(hist[0][k]), int(hist[1][k])
        N += nk
        TP += pk
        if pk:
            acc += Fraction(pk * TP, N)
    return acc / total


def sklearn_inputs(logits, target, bf16=False):
    """(labels, scores) as sklearn sees them: the scores as fp64 values of the rounded bf16 scores, +-inf replaced by +-1e300
    (sklearn refuses infinities; no finite bf16 comes near 1e300, so the order is kept).  NaN logits are dropped."""
    bits = np.asarray(logits, dtype=np.uint16).reshape(-1) if bf16 else bf16_bits(np.asarray(logits, np.float32).reshape(-1))
    x = bf16_value(bits).astype(np.float64)
    ok = ~np.isnan(x)
    x = np.clip(x[ok], -1e300, 1e300)
    return np.asarray(target, dtype=np.float32).reshape(-1)[ok] > np.float32(0.5), x

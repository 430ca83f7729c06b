"""fp64 restatement of the reference's segmentation losses (loss.py:58-121) and their gradients, the yardstick of
`csrc/seg_loss.cu`.  Inputs are the [N*H*W] flattening of [n, 1, h, w] logits x and targets t; w = words weight where t > 0,
background weight elsewhere; s = 2t - 1; bce(x, y) = max(x, 0) - x y + log1p(exp(-|x|)).

  BinaryFocalLoss:            mean(exp(gamma logsigmoid(-x s)) w bce(x, t)), gradient through pt as well
  SoftBootstrapCrossEntropy:  w bce(x, beta t + (1 - beta) [sigmoid(x) > 0.5]), reduced by mean, sum or not at all; the
                              indicator carries no gradient
"""
import numpy as np

# torch's CPU float32 sigmoid(x) > 0.5 holds exactly for float32 x > 1.5 * 2^-24 (below it 1 + exp(-x) rounds to 2)
BOOT_THRESHOLD = np.float32(1.5 * 2.0 ** -24)


def sigmoid(x):
    x = np.asarray(x, np.float64)
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1 / (1 + e), e / (1 + e))


def bce(x, y):
    return np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))


def log_sigmoid(z):
    return np.minimum(z, 0) - np.log1p(np.exp(-np.abs(z)))


def indicator(x32):
    """torch.sigmoid(x.float()) > 0.5 on the CPU, for float32 logits."""
    return np.asarray(x32, np.float32) > BOOT_THRESHOLD


def _weights(t, background, words):
    return np.where(t > 0, float(words), float(background))


def focal(x, t, gamma=0, background_weights=1, words_weights=2):
    """(loss, d loss / d x) in fp64 for BinaryFocalLoss."""
    x, t = np.asarray(x, np.float64), np.asarray(t, np.float64)
    w, s = _weights(t, background_weights, words_weights), 2 * t - 1
    b = bce(x, t)
    f = np.exp(gamma * log_sigmoid(-x * s))
    n = x.size
    loss = (f * w * b).sum() / n
    grad = w * f * (-gamma * s * sigmoid(x * s) * b + sigmoid(x) - t) / n
    return loss, grad


def bootstrap(x, t, beta=0.95, background_weight=1, words_weight=2, reduction="mean", x32=None):
    """(loss, d loss / d x) in fp64 for SoftBootstrapCrossEntropy; reduction "mean", "sum" or "none" (then the loss is per
    element and the gradient is that of the sum).  x32: the float32 logits the indicator is taken on (default: x)."""
    x, t = np.asarray(x, np.float64), np.asarray(t, np.float64)
    ind = indicator(x if x32 is None else x32)
    w = _weights(t, background_weight, words_weight)
    tb = beta * t + (1 - beta) * ind
    le = w * bce(x, tb)
    ge = w * (sigmoid(x) - tb)
    if reduction == "mean":
        return le.sum() / x.size, ge / x.size
    if reduction == "sum":
        return le.sum(), ge
    return le, ge

"""Validation metrics on the GPU.

`PixelAveragePrecision`: the pixel-level average precision of segmentation logits against their targets, the score the
reference's README picks its loss settings by (an AP table on validation images).  Over every pixel since the last reset:

  * score: the logit rounded to bf16.  bf16 logits (the networks' bf16 output) are used as they are; fp32 logits are rounded
    to nearest-even as torch's ``.to(torch.bfloat16)``.  -0 counts as +0 (sklearn ties them); +-inf are the largest and
    smallest scores.  Logits rather than probabilities: fp32 sigmoid saturates (sigmoid(17) == sigmoid(30) == 1.0), so
    ranking by probability would tie pixels that the network ranks apart;
  * label: target > 0.5 in fp32 (SegBatcher's targets are bicubic-resampled masks, soft at the edges);
  * AP: ``sklearn.metrics.average_precision_score(labels, scores)``: over the 65,536 bf16 values in descending order, with
    pos_k the positives at value k, TP_k and N_k the positives and pixels at values >= k and P all positives,
    AP = (1 / P) sum_k pos_k TP_k / N_k; 0 when P = 0 (as sklearn returns);
  * at the demo's threshold, tp / fp / fn / tn with predicted = sigmoid(x) > 0.5 of the unrounded logit (the test the bootstrap
    loss and ops.text_mask_postprocess use);
  * NaN logits are counted in `nan` and nowhere else; the AP is NaN whenever `nan > 0`, so a diverged model gets no score.

The state is integer counts (csrc/seg_loss.cu, pcb_seg_score_update): a histogram of pixels and positives per score, and the
five counts.  The AP of a pass is therefore bit-identical however its pixels are split into batches and in whatever order the
device's atomics land.  Data parallel: all-reduce `hist` and `counts_tensor` (SUM) across ranks before `average_precision()`
(not done here).
"""
from __future__ import annotations

import ctypes

import torch

from . import _lib, ops

KEYS = 65536
COUNTS = ("tp", "fp", "fn", "tn", "nan")


def _strides(t):
    return (ctypes.c_longlong * 4)(*t.stride())


class PixelAveragePrecision:
    """Pixel average precision of [n, 1, h, w] segmentation logits on `device` (see the module docstring for the definition).

    ``update(logits, target)`` adds a batch: `logits` fp32 or bf16 on the device, dense or the channel-padded NHWC view the
    networks return (read in place through its strides); `target` a contiguous fp32 tensor of the same shape.  One launch, no
    host synchronisation: it can be captured in a CUDA graph.  Wrong devices, dtypes or shapes raise before anything is
    launched.  ``reset()`` zeroes the state.  ``average_precision()`` finalises on the device and returns a Python float
    (it synchronises); `counts` returns tp, fp, fn, tn, nan and pixels as Python ints.  `hist` (int64 [2, 65536]: pixels and
    positives per score key) and `counts_tensor` (int64 [5]) are the raw state, at fixed addresses."""

    def __init__(self, device=None):
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if self.device.type != "cuda":
            raise ValueError("PixelAveragePrecision runs on a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        _lib.load()
        self.hist = torch.zeros((2, KEYS), dtype=torch.int64, device=self.device)
        self.counts_tensor = torch.zeros((5,), dtype=torch.int64, device=self.device)
        self._out = torch.zeros((1,), dtype=torch.float64, device=self.device)

    def reset(self):
        self.hist.zero_()
        self.counts_tensor.zero_()

    def _check(self, logits, target):
        name = type(self).__name__
        if not isinstance(logits, torch.Tensor) or not isinstance(target, torch.Tensor):
            raise TypeError(f"{name}.update takes two tensors")
        if logits.device != self.device or target.device != self.device:
            raise _lib.PcbError(f"{name}: logits ({logits.device}) and target ({target.device}) must be on {self.device}")
        if logits.dim() != 4 or logits.size(1) != 1:
            raise _lib.PcbError(f"{name}: logits must be [n, 1, h, w], got {tuple(logits.shape)}")
        if logits.dtype not in (torch.float32, torch.bfloat16):
            raise _lib.PcbError(f"{name}: logits must be float32 or bfloat16, got {logits.dtype}")
        if logits.numel() == 0:
            raise _lib.PcbError(f"{name}: empty logits {tuple(logits.shape)}")
        if tuple(target.shape) != tuple(logits.shape) or target.dtype != torch.float32 or not target.is_contiguous():
            raise _lib.PcbError(f"{name}: target must be a contiguous float32 tensor of shape {tuple(logits.shape)}, got "
                                f"{target.dtype} {tuple(target.shape)}")

    def update(self, logits: torch.Tensor, target: torch.Tensor):
        """Add the pixels of one batch (see the class docstring)."""
        self._check(logits, target)
        n, _, h, w = logits.shape
        _lib.check(_lib.load().pcb_seg_score_update(logits.data_ptr(), ops._dtype_code(logits), _strides(logits), target.data_ptr(),
                                                    n, h, w, self.hist.data_ptr(), self.counts_tensor.data_ptr(), ops._stream()))

    def finalize(self) -> torch.Tensor:
        """Launch the AP pass; returns the device fp64 [1] result buffer (overwritten by the next call) without synchronising."""
        _lib.check(_lib.load().pcb_seg_score_finalize(self.hist.data_ptr(), self.counts_tensor.data_ptr(), self._out.data_ptr(),
                                                      ops._stream()))
        return self._out

    def average_precision(self) -> float:
        return float(self.finalize().item())

    @property
    def counts(self) -> dict:
        c = dict(zip(COUNTS, (int(v) for v in self.counts_tensor.tolist())))
        c["pixels"] = sum(c.values())
        return c

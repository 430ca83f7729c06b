"""Measure held-out segmentation evaluation (engine.SegEvalStep) and its pixel average precision (metrics.PixelAveragePrecision)
on one GPU, bf16, for XceptionTextSegment 512^2 batch 16 and TextSegament 512^2 batch 8, and print one JSON line per network
with the card's name and power limit:

  * update_ms:  device time of PixelAveragePrecision.update() alone on the network's [n, 1, 512, 512] channel-padded bf16 logits
                (CUDA events over many launches, mean); finalize_ms likewise for average_precision()'s device pass;
  * run_ms:     SegEvalStep.run() (prepare + eval forward + BinaryFocalLoss + score in one graph), the same without the loss,
                the same without loss and score, and SegInferStep.run() on a device-resident batch (CUDA events, medians of
                rounds, the variants alternating within each round);
  * score_share: update_ms over the run without loss and score;
  * host_sklearn_ms: copying one batch's logits and targets to the host and sklearn's average_precision_score over its pixels
                (host clock), when sklearn is installed; null otherwise.

    python tools/bench_seg_eval.py [--rounds 5 --steps 10]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = [("XceptionTextSegment", 16), ("TextSegament", 8)]


def _timed(fn, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--update-iters", type=int, default=200)
    args = ap.parse_args()

    import torch

    import seg_ref as S
    from bench_inpaint_data import card
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegEvalStep, SegInferStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    from text_segmentation_image_inpainting_b200.metrics import PixelAveragePrecision
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS

    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_eval.py needs a CUDA device")
    try:
        from sklearn.metrics import average_precision_score
    except ImportError:
        average_precision_score = None

    class _NoScore(SegEvalStep):
        """The same graph without the score (and without a loss when constructed without one)."""

        def _forward(self):
            x, target = self.batcher.prepare()
            out = self.net(x)
            if self.criterion is not None:
                self._keep_loss(self.criterion(out, target))
            return out

    dev = torch.device("cuda")
    name_card, power = card()
    S_, H, W = 512, 1024, 768
    for name, batch in CONFIGS:
        res = {"card": name_card, "power_limit": power, "net": name, "batch": batch, "image_size": S_, "dtype": "bf16"}
        torch.manual_seed(0)
        net = getattr(TS, name)().to(dev)
        src = [S.sources(i, H, W) for i in range(batch)]
        b = SegBatcher(batch, (H, W), image_size=S_, seed=0)
        b.stage(src)

        steps = {"loss_and_score": SegEvalStep(net, b, BinaryFocalLoss(gamma=2)), "score": SegEvalStep(net, b),
                 "neither": _NoScore(net, b)}
        for st in steps.values():
            st.warmup_and_capture()
        x_dev = b.x.float().contiguous()
        infer = SegInferStep(net)
        infer.run(x_dev)
        net.train()

        # update() alone, on the [n, 1, 512, 512] view of the channel-padded bf16 buffer the network returns
        net.eval()
        with torch.no_grad():
            logits = net(b.prepare()[0])
        net.train()
        target = b.target
        sc = PixelAveragePrecision(dev)
        _timed(lambda: sc.update(logits, target), 10)
        res["logits_strides"] = list(logits.stride())
        res["update_ms"] = _timed(lambda: sc.update(logits, target), args.update_iters)
        res["finalize_ms"] = _timed(sc.finalize, args.update_iters)

        times = {k: [] for k in list(steps) + ["infer"]}
        for _ in range(args.rounds):
            for k, st in steps.items():
                times[k].append(_timed(st.run, args.steps))
            times["infer"].append(_timed(lambda: infer.run(x_dev), args.steps))
        res["run_ms"] = {k: statistics.median(v) for k, v in times.items()}
        res["score_share"] = res["update_ms"] / res["run_ms"]["neither"]

        res["host_sklearn_ms"] = None
        if average_precision_score is not None:
            out = steps["score"].run()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            x = out.cpu().numpy().reshape(-1)
            y = target.cpu().numpy().reshape(-1) > 0.5
            average_precision_score(y, x)
            res["host_sklearn_ms"] = (time.perf_counter() - t0) * 1e3
        print(json.dumps(res), flush=True)
        del steps, infer


if __name__ == "__main__":
    main()

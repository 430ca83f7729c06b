"""Measure the segmentation training path on the reference's data and losses (data.SegBatcher, loss.BinaryFocalLoss,
engine.SegLossTrainStep) on one GPU, on the BASELINE shapes (TextSegament 512^2 batch 8, XceptionTextSegment 512^2 batch 16,
bf16), and print one JSON line per network:

  * pipeline_ms:   device time of prepare() from 1024 x 768 gray sources (CUDA events, mean),
  * loss_ms:       BinaryFocalLoss forward + backward on the network's [n, 1, 512, 512] padded bf16 output view,
  * step_ms:       SegLossTrainStep (data + network + loss + SGD in one graph) against SegTrainStep (out.abs().mean()) fed a
                   device-resident batch of the same shape, alternating rounds,
  * host_ms_per_image: the reference's process_images on one host core (staged oracle/_ref/Dataloader.py, when present) next
                   to this path's host work (stage(): copy into pinned memory and enqueue the upload).

Every line carries the card's name and power limit.

    python tools/bench_seg_train.py [--rounds 5 --steps 20]
"""
import argparse
import contextlib
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_inpaint_data import card  # noqa: E402

CONFIGS = [("TextSegament", 8), ("XceptionTextSegment", 16)]


def timed(fn, iters):
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=100)
    args = ap.parse_args()

    import numpy as np
    import torch

    import inpaint_ref as R
    import seg_ref as S
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep, SegTrainStep
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS

    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_train.py needs a CUDA device")
    dev = torch.device("cuda")
    size, H, W = 512, 1024, 768
    name_, power = card()
    for net_name, B in CONFIGS:
        srcs = [S.sources(i, H, W) for i in range(B)]
        res = {"card": name_, "power_limit": power, "network": net_name, "batch": B, "image_size": size, "source": [H, W],
               "dtype": "bf16"}
        b = SegBatcher(B, (H, W), image_size=size, seed=0)
        b.stage(srcs)
        for _ in range(10):
            b.prepare()
        res["pipeline_ms"] = timed(b.prepare, args.iters)

        t0 = time.perf_counter()
        for _ in range(20):
            b.stage(srcs)
        torch.cuda.synchronize()
        res["host_ms_per_image_stage"] = (time.perf_counter() - t0) / (20 * B) * 1e3
        if R.dataloader() is not None:
            from PIL import Image
            threads = torch.get_num_threads()
            torch.set_num_threads(1)
            ds = S.dataset(size)
            pil = [(Image.fromarray(p, "L"), Image.fromarray(m, "L")) for p, m in srcs[:2]]
            t0 = time.perf_counter()
            for i in range(10):
                ds.process_images(*pil[i % 2])
            res["host_ms_per_image_reference"] = (time.perf_counter() - t0) / 10 * 1e3
            torch.set_num_threads(threads)
        else:
            res["host_ms_per_image_reference"] = None

        def net():
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                return getattr(TS, net_name)().to(dev)

        # ---- the loss alone, on the output layout of the network
        crit = BinaryFocalLoss()
        buf = torch.empty((B, 8, size, size), dtype=torch.bfloat16, device=dev, memory_format=torch.channels_last).zero_()
        buf[:, :1].copy_(torch.randn(B, 1, size, size, device=dev))
        logits = buf[:, :1].detach().requires_grad_(True)
        target = b.target

        def loss_fwd_bwd():
            crit(logits, target).backward()
        for _ in range(10):
            loss_fwd_bwd()
        res["loss_ms"] = timed(loss_fwd_bwd, args.iters)

        # ---- training step: SegLossTrainStep vs SegTrainStep fed a device-resident batch
        x_dev = b.prepare()[0].float().contiguous()
        plain = SegTrainStep(net(), compute_dtype=torch.bfloat16)
        plain.warmup_and_capture(x_dev, None, eager_warmup=2)
        fused = SegLossTrainStep(net(), b, crit)
        fused.warmup_and_capture(eager_warmup=2)
        times = {"seg_train_step": [], "seg_loss_train_step": []}
        for r in range(args.rounds):
            for name in ("seg_train_step", "seg_loss_train_step") if r % 2 == 0 else ("seg_loss_train_step", "seg_train_step"):
                fn = (lambda: plain.step(x_dev)) if name == "seg_train_step" else fused.step
                times[name].append(timed(fn, args.steps))
        res["step_ms"] = {k: float(np.median(v)) for k, v in times.items()}
        res["step_ms_all"] = times
        res["data_and_loss_share_of_step"] = (res["pipeline_ms"] + res["loss_ms"]) / res["step_ms"]["seg_loss_train_step"]
        print(json.dumps(res), flush=True)
        del plain, fused
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

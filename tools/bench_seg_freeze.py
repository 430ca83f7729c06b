"""Measure the first stage of the reference's two-stage segmentation recipe (encoder frozen) against the all-trainable step on
one GPU: the captured SegTrainStep (bf16, out.abs().mean()) on a device-resident batch, the two steps replayed alternately one
step at a time, each step timed by CUDA events.  Prints one JSON line per workload with the median and the spread (min, max)
of the per-step times of both steps, this library's launches per step of both, and the card's name and power limit:

  * TextSegament 512^2, batch 8, with MobileNetV2.freeze_params(k), k = 0, 1 and 2, and k = -1 (nothing frozen: the baseline timed
    against itself, which shows the spread of the alternation);
  * XceptionTextSegment 512^2, batch 16, with the encoder frozen.

For TextSegament it also times, in one eager step of each with the convolution profile on (ops.set_profile), the data
gradients of the convolutions that read the RFB's concatenated input (features[3:], 1344 channels at width 2): `rfb_dgrad_ms`,
the channels of that input that want a gradient, and `rfb_unwanted_ms`, the share of that time spent on the channels of frozen
stages (time x unwanted / all channels), which is what restricting those launches to the wanted channels could save at most.

    python tools/bench_seg_freeze.py [--steps 60 --warmup 10]
"""
import argparse
import contextlib
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_inpaint_data import card  # noqa: E402

WORKLOADS = [("TextSegament", 8, 0), ("TextSegament", 8, 1), ("TextSegament", 8, 2), ("TextSegament", 8, -1),
             ("XceptionTextSegment", 16, None)]
SIZE = 512


def build(net_name, batch, k, dev):
    """the captured step of `net_name` frozen as k says (MobileNetV2.freeze_params(k); None: the whole encoder; -1: nothing)"""
    import torch

    from text_segmentation_image_inpainting_b200.engine import SegTrainStep
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        net = getattr(TS, net_name)()
        if k is None:
            net.encoder.requires_grad_(False)
        elif k >= 0:
            net.encoder.freeze_params(k)
    x = torch.rand(batch, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(1)).to(dev)
    ts = SegTrainStep(net.to(dev), compute_dtype=torch.bfloat16, lr=1e-4)
    ts.warmup_and_capture(x, None, eager_warmup=2)
    return ts, x


def rfb_dgrad(ts, x, rounds=5):
    """(median ms of the data gradients of the convolutions reading the RFB input over `rounds` eager steps, channels of that
    input, channels that want a gradient)"""
    import numpy as np
    import torch

    from text_segmentation_image_inpainting_b200 import ops
    stages = ts.net.encoder.features[3:]
    cin = sum(stage[0].out_channels for stage in stages)
    wanted = sum(stage[0].out_channels for stage in stages if any(p.requires_grad for p in stage.parameters()))
    per_step = []
    for _ in range(rounds):
        rec = []
        ops.set_profile(rec)
        try:
            ts._step(x, None, False)
        finally:
            ops.set_profile(None)
        torch.cuda.synchronize()
        per_step.append(sum(s.elapsed_time(e) for kind, g, s, e in rec if kind == "dgrad" and g.cin == cin))
    return float(np.median(per_step)), cin, wanted


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_seg_freeze.py needs a CUDA device")
    dev = torch.device("cuda")
    name_, power = card()
    for net_name, batch, k in WORKLOADS:
        steps = {"frozen": build(net_name, batch, k, dev), "all_trainable": build(net_name, batch, -1, dev)}
        for ts, x in steps.values():
            for _ in range(args.warmup):
                ts.step(x)
        times = {n: [] for n in steps}
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(2 * args.steps)]
        order = []
        torch.cuda.synchronize()
        for i in range(args.steps):
            for n in (("frozen", "all_trainable") if i % 2 == 0 else ("all_trainable", "frozen")):
                e0, e1 = ev[len(order)]
                ts, x = steps[n]
                e0.record()
                ts.step(x)
                e1.record()
                order.append((n, e0, e1))
        torch.cuda.synchronize()
        for n, e0, e1 in order:
            times[n].append(e0.elapsed_time(e1))
        res = {"card": name_, "power_limit": power, "network": net_name, "batch": batch, "image_size": SIZE, "dtype": "bf16",
               "free_last_blocks": k if k is not None else "encoder frozen", "steps": args.steps}
        for n, (ts, _) in steps.items():
            t = np.asarray(times[n])
            res[n] = {"median_ms": float(np.median(t)), "min_ms": float(t.min()), "max_ms": float(t.max()),
                      "launches_per_step": ts.launches_per_step,
                      "trainable_params": sum(p.numel() for p in ts.net.parameters() if p.requires_grad)}
        res["frozen_over_all"] = res["frozen"]["median_ms"] / res["all_trainable"]["median_ms"]
        if net_name == "TextSegament":
            ms, cin, wanted = rfb_dgrad(*steps["frozen"])
            res["rfb_input_channels"], res["rfb_wanted_channels"], res["rfb_dgrad_ms"] = cin, wanted, ms
            res["rfb_unwanted_ms"] = ms * (cin - wanted) / cin
            res["rfb_unwanted_share_of_step"] = res["rfb_unwanted_ms"] / res["frozen"]["median_ms"]
        print(json.dumps(res), flush=True)
        for ts, _ in steps.values():
            ts.close()
        del steps, ts
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

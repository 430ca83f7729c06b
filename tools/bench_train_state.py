"""Measure what the cyclical learning rate and the training-state checkpoint cost on bench.py's workload (ImageFillOrigin 512^2,
batch 8, bf16, one GPU) and print one JSON line:

  * step_ms:  the captured constant-rate TrainStep (bench.py's step) against the captured TrainStep with
              lr_schedule=CyclicLR(1e-4, 4e-4) (one extra single-thread kernel node; the SGD kernel reads its rate from device
              memory), alternating one step of each, every step between its own pair of CUDA events; medians;
  * state_dict_ms / load_state_dict_ms: host wall time of TrainStep.state_dict() (device-to-host copy of the parameters,
              buffers and momentum) and of load_state_dict() of that dict (host-to-device, in place), each ending in a device
              synchronise; medians.

The line carries the card's name and power limit, read in the same run.

    python tools/bench_train_state.py [--steps 30 --warmup 5 --reps 5]
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_inpaint_data import card  # noqa: E402

HW, B = 512, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per variant (>= 20)")
    ap.add_argument("--warmup", type=int, default=5, help="untimed replays per variant after capture")
    ap.add_argument("--reps", type=int, default=5, help="state_dict / load_state_dict repetitions")
    args = ap.parse_args()

    import torch

    from text_segmentation_image_inpainting_b200 import _lib
    from text_segmentation_image_inpainting_b200.engine import CyclicLR, TrainStep
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks

    if not torch.cuda.is_available():
        raise SystemExit("bench_train_state.py: no CUDA device -- the GPU path has no CPU fallback")
    dev = torch.device("cuda", 0)
    _lib.load()
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(B, 3, HW, HW, generator=g).to(dev)
    m = torch.from_numpy(random_hole_masks(B, HW, HW, seed=0)).to(dev)

    def make(schedule):
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):     # the reference's constructors print ("No check point ...")
            net = ImageFillOrigin().to(dev)
        ts = TrainStep(net, compute_dtype=torch.bfloat16, lr_schedule=schedule)
        ts.warmup_and_capture(x, m, eager_warmup=2)
        return ts

    steps = {"constant": make(None), "cyclic": make(CyclicLR(1e-4, 4e-4, step_size=2000, mode="triangular2"))}
    for ts in steps.values():
        for _ in range(args.warmup):
            ts.step(x, m)
    torch.cuda.synchronize()
    times = {k: [] for k in steps}
    for _ in range(args.steps):
        for k, ts in steps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ts.step(x, m)
            e1.record()
            times[k].append((e0, e1))
    torch.cuda.synchronize()
    ms = {k: [a.elapsed_time(b) for a, b in v] for k, v in times.items()}

    ts = steps["cyclic"]
    save, load = [], []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sd = ts.state_dict()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ts.load_state_dict(sd)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        save.append((t1 - t0) * 1e3)
        load.append((t2 - t1) * 1e3)
    loss = float(ts.step(x, m))
    name, power = card()
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": f"ImageFillOrigin {HW}x{HW}, batch {B}, bf16, fwd+bwd+SGD(nesterov) graph replay",
        "card": name, "power_limit": power,
        "step_ms_constant_median": round(med["constant"], 3),
        "step_ms_cyclic_median": round(med["cyclic"], 3),
        "step_ms_cyclic_minus_constant": round(med["cyclic"] - med["constant"], 3),
        "step_ms_constant_min_max": [round(min(ms["constant"]), 3), round(max(ms["constant"]), 3)],
        "step_ms_cyclic_min_max": [round(min(ms["cyclic"]), 3), round(max(ms["cyclic"]), 3)],
        "steps_each": args.steps,
        "arena_mb": round(ts.flat.numel * 4 / 1e6, 1),
        "state_dict_ms_median": round(statistics.median(save), 1),
        "load_state_dict_ms_median": round(statistics.median(load), 1),
        "reps": args.reps,
        "iteration_after": ts.iteration,
        "loss_after_resume_finite": bool(loss == loss and abs(loss) != float("inf")),
    }), flush=True)
    for t in steps.values():
        t.close()


if __name__ == "__main__":
    main()

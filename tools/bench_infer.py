"""Inference benchmark: ms per forward of today's eager eval path (``net.eval()`` under no_grad, two-pass BatchNorm) and of the
graph-captured engines (engine.InferStep / SegInferStep, BatchNorm + activation fused into the convolution epilogues), per
workload.  Prints one JSON line with the card's name, power limit and max SM clock (read in the same run).

    python tools/bench_infer.py [--iters 30] [--warmup 5] [--only NAME]

Times are medians over CUDA-event-timed forwards after warm-up, the two paths alternating forward by forward.  Weights are
deterministic; BatchNorm running statistics come from one training-mode forward on the benchmark batch (momentum 1), so the
eval activations are O(1).  `max_rel_diff` = max |engine - eager| / max |eager| over the outputs."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch import nn  # noqa: E402

# name: (network module, class, image size, batch, with the demo's post-processing)
WORKLOADS = {
    "ImageFillOrigin_512_b1": ("image_inpainting", "ImageFillOrigin", 512, 1, False),
    "ImageFillOrigin_512_b8": ("image_inpainting", "ImageFillOrigin", 512, 8, False),
    "XceptionTextSegment_600_b1": ("text_segmentation", "XceptionTextSegment", 600, 1, False),
    "XceptionTextSegment_600_b1_post": ("text_segmentation", "XceptionTextSegment", 600, 1, True),
    "XceptionTextSegment_512_b16": ("text_segmentation", "XceptionTextSegment", 512, 16, False),
    "TextSegament_512_b8": ("text_segmentation", "TextSegament", 512, 8, False),
}
# the demo's crop and original size for the post-processed workload: a 800 x 600 photo resized to 600 x 448, padded to 600 x 600
POST_PAD, POST_HW = (0, 0, 0, 152), (600, 800)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": str(exc)}


def bench(name, iters, warmup):
    from oracle.detfill import det_fill_state_dict, det_tensor
    from text_segmentation_image_inpainting_b200 import _lib, ops
    from text_segmentation_image_inpainting_b200.engine import InferStep, SegInferStep
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    mod, cls, hw, batch, post = WORKLOADS[name]
    import importlib
    torch.manual_seed(0)
    net = getattr(importlib.import_module(f"text_segmentation_image_inpainting_b200.models.{mod}"), cls)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.cuda()
    dev = torch.device("cuda")
    x = det_tensor("bench_infer.x", (batch, 3, hw, hw)).to(dev)
    if mod == "image_inpainting":
        mask = torch.from_numpy(random_hole_masks(batch, hw, hw, seed=3)).to(dev)
        step = InferStep(net)
        args = (x, mask)
        eager_fwd = lambda: net(step._prepare(x, mask))  # noqa: E731
    else:
        step = SegInferStep(net)
        args = (x,)
        eager_fwd = lambda: step._forward(x)  # noqa: E731
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    for m in bns:
        m.momentum = 1.0
    net.train()
    with torch.no_grad():
        eager_fwd()
    for m in bns:
        m.momentum = 0.1
    net.eval()

    def eager():
        with torch.no_grad():
            out = eager_fwd()
            return ops.text_mask_postprocess(out, POST_PAD, POST_HW) if post else out

    def engine():
        out = step.run(*args)
        return ops.text_mask_postprocess(out, POST_PAD, POST_HW) if post else out

    before = _lib.launch_count()
    ref = eager()
    eager_launches = _lib.launch_count() - before
    got = engine()
    torch.cuda.synchronize()
    if post:
        diff = float((got.float() - ref.float()).abs().mean())               # fraction of differing mask pixels
    else:
        diff = float((got.float() - ref.float()).abs().max() / ref.float().abs().max())
    times = {"eager": [], "engine": []}
    for i in range(warmup + iters):
        for kind, fn in (("eager", eager), ("engine", engine)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            if i >= warmup:
                times[kind].append(s.elapsed_time(e))
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"workload": name, "batch": batch, "eager_ms": round(med["eager"], 3), "engine_ms": round(med["engine"], 3),
            "eager_images_per_s": round(batch * 1000 / med["eager"], 1), "engine_images_per_s": round(batch * 1000 / med["engine"], 1),
            "eager_launches": eager_launches, "engine_launches": step.launches_per_run + (1 if post else 0),
            "fused_sites": step.fused_sites, "unfused_sites": step.unfused_sites,
            ("mask_pixels_differing" if post else "max_rel_diff"): diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer.py needs a CUDA device")
    names = a.only.split(",") if a.only else list(WORKLOADS)
    res = {"card": card(), "workloads": []}
    for n in names:
        res["workloads"].append(bench(n, a.iters, a.warmup))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

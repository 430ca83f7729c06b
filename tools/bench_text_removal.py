"""Text-removal benchmark: ms per batch of engine.TextRemovalStep.run (segmentation, mask, holes, inpainting and composite in
one CUDA graph) against the same pipeline composed from the other public engines and torch ops:

    SegInferStep.run(normalized, padded page) -> ops.text_mask_postprocess -> torch 10x10 dilation (F.pad + max_pool2d)
    -> InferStep.run(padded page, dense 3-channel valid mask) -> torch.where, cropped

Prints one JSON line with the card's name, power limit and max SM clock (read in the same run).

    python tools/bench_text_removal.py [--iters 30] [--warmup 5] [--only NAME]

Times are medians over CUDA-event-timed calls after warm-up, the two paths alternating call by call.  Weights are
deterministic; BatchNorm running statistics come from one training-mode forward on the benchmark page (momentum 1), and the
segmentation output bias is shifted so that about 0.5 % of the logits are positive.  `bitwise_equal`: the two composites are
identical.  XceptionTextSegment is run-to-run deterministic, so both paths feed the U-Net the same bf16 input and mask and
must agree bit for bit; TextSegament's float atomics can flip a few mask pixels between runs, so for it
`mask_pixels_differing` reports the fraction of valid-plane pixels that differ.  Launches are this library's kernels per call;
the composed path also runs torch kernels (padding, dilation, mask expansion, the input copies and the select), not counted."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch import nn  # noqa: E402

# name: (segmentation network, inpainting U-Net, page height, page width, batch)
WORKLOADS = {
    "Xception_ImageFillOrigin_1700x1200_b1": ("XceptionTextSegment", "ImageFillOrigin", 1700, 1200, 1),
    "Xception_ImageFillOrigin_1024_b1": ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 1),
    "Xception_ImageFillOrigin_1024_b4": ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 4),
    "TextSegament_ImageFill_1024_b1": ("TextSegament", "ImageFill", 1024, 1024, 1),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": str(exc)}


def _calibrate(net, run_train):
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm2d)]
    for m in bns:
        m.momentum = 1.0
    net.train()
    with torch.no_grad():
        run_train()
    for m in bns:
        m.momentum = 0.1
    net.eval()


def bench(name, iters, warmup):
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import DEMO_MEAN_STD, InferStep, SegInferStep, TextRemovalStep
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    seg_name, fill_name, h, w, n = WORKLOADS[name]
    dev = torch.device("cuda")
    torch.manual_seed(0)
    seg, fill = getattr(TS, seg_name)(), getattr(II, fill_name)()
    seg.load_state_dict(det_fill_state_dict(seg.state_dict()))
    fill.load_state_dict(det_fill_state_dict(fill.state_dict()))
    seg, fill = seg.to(dev), fill.to(dev)
    g = torch.Generator().manual_seed(1)
    base = F.interpolate(torch.rand((n, 3, h // 16 + 2, w // 16 + 2), generator=g), size=(h, w), mode="bilinear", align_corners=False)
    page = (0.8 * base + 0.2 * torch.rand((n, 3, h, w), generator=g)).clamp(0, 1).to(dev)

    step = TextRemovalStep(seg, fill)
    (hs, ws), (hu, wu) = step.padded_sizes(h, w)
    mean, std = (torch.tensor(v, device=dev)[:, None, None] for v in DEMO_MEAN_STD)
    x32 = F.pad((page - mean) / std, (0, ws - w, 0, hs - h))
    xin = ops.removal_seg_input(page, DEMO_MEAN_STD, hs, ws, torch.bfloat16)
    _calibrate(seg, lambda: seg(xin))
    with torch.no_grad():
        logits = seg(xin).float()
    with torch.no_grad():
        [m for m in seg.modules() if getattr(m, "out_channels", None) == 1 and getattr(m, "bias", None) is not None][-1].bias.sub_(
            float(torch.quantile(logits.flatten()[::97], 0.995)))
    ops.bump_weight_epoch()
    with torch.no_grad():
        mask = ops.text_mask_postprocess(seg(xin), (0, ws - w, 0, hs - h), (h, w))
    corrupted, valid = ops.removal_holes(mask, page, hu, wu, torch.bfloat16)
    _calibrate(fill, lambda: fill((corrupted, HoleMask.from_plane(valid, 3))))

    seg_step, fill_step = SegInferStep(seg), InferStep(fill)
    page_pad = F.pad(page, (0, wu - w, 0, hu - h))
    state = {}

    def composed():
        lg = seg_step.run(x32)
        tm = ops.text_mask_postprocess(lg, (0, ws - w, 0, hs - h), (h, w))
        hole = F.max_pool2d(F.pad(tm.float(), (5, 4, 5, 4)), 10, stride=1) > 0          # cv2.dilate(10x10), anchor 5
        v = torch.zeros((n, 1, hu, wu), dtype=torch.float32, device=dev)
        v[:, :, :h, :w] = (~hole).float()
        out = fill_step.run(page_pad, v.expand(n, 3, hu, wu))
        state["valid"] = v
        return torch.where(v[:, :, :h, :w] > 0, page, out[:, :, :h, :w])

    def engine():
        return step.run(page)

    composed(), engine()                                  # captures both paths' graphs
    ref, got = composed(), engine()
    # this library's kernels per call (the engines count them in their eager warm-up); the composed path's torch ops come on top
    composed_launches = seg_step.launches_per_run + 1 + fill_step.launches_per_run
    torch.cuda.synchronize()
    equal = bool(torch.equal(got, ref))
    valid_ref = state["valid"][:, 0].to(torch.uint8)
    differing = float((valid_ref != step.valid).float().mean())
    holes = 1.0 - float(step.valid[:, :h, :w].float().mean())
    times = {"composed": [], "engine": []}
    for i in range(warmup + iters):
        for kind, fn in (("composed", composed), ("engine", engine)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            if i >= warmup:
                times[kind].append(s.elapsed_time(e))
    med = {k: statistics.median(v) for k, v in times.items()}
    return {"workload": name, "page_hw": [h, w], "batch": n, "unet_hw": [hu, wu], "hole_fraction": round(holes, 4),
            "composed_ms": round(med["composed"], 3), "engine_ms": round(med["engine"], 3),
            "composed_pages_per_s": round(n * 1000 / med["composed"], 2), "engine_pages_per_s": round(n * 1000 / med["engine"], 2),
            "composed_launches": composed_launches, "engine_launches": step.launches_per_run,
            "bitwise_equal": equal, "mask_pixels_differing": differing}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_removal.py needs a CUDA device")
    names = a.only.split(",") if a.only else list(WORKLOADS)
    res = {"card": card(), "workloads": []}
    for n in names:
        res["workloads"].append(bench(n, a.iters, a.warmup))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

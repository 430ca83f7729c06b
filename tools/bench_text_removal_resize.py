"""Text removal with and without EvaluateSet's page resize: ms per batch of engine.TextRemovalStep.run with seg_resize=600 (the
segmentation demo's scale) against the same step segmenting at page size, the two alternating call by call, medians of
CUDA-event times; the resize stage alone (ops.page_resize_bicubic, CUDA events around the call); the library's launches per
run of each; and, where Pillow is importable, the host's own EvaluateSet-style preparation of the same pages (PIL bicubic
resize, to_tensor, Normalize, pad, upload to the device), timed on the host clock to a device synchronise.

Prints one JSON line with the card's name, power limit and max SM clock (read in the same run).

    python tools/bench_text_removal_resize.py [--iters 20] [--warmup 3] [--only NAME]

Networks and pages as tools/bench_text_removal.py makes them (deterministic weights, BatchNorm statistics from one training
forward on the page at its own size, segmentation bias shifted to about 0.5 % positive logits)."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_text_removal import _calibrate, card  # noqa: E402

RESIZE = 600
# name: (segmentation network, inpainting U-Net, page height, page width, batch)
WORKLOADS = {
    "Xception_ImageFillOrigin_1700x1200_b1": ("XceptionTextSegment", "ImageFillOrigin", 1700, 1200, 1),
    "Xception_ImageFillOrigin_3508x2480_b1": ("XceptionTextSegment", "ImageFillOrigin", 3508, 2480, 1),     # A4 at 300 dpi
    "Xception_ImageFillOrigin_1024_b4": ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 4),
}


def _event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def host_prepare_ms(page_u8, resize, iters, dev):
    """EvaluateSet.resize_pad_tensor's statements for each page of the batch, then the upload: median ms per batch"""
    try:
        from PIL import Image
    except ImportError:
        return None
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import DEMO_MEAN_STD
    mean, std = (torch.tensor(v)[:, None, None] for v in DEMO_MEAN_STD)
    imgs = [Image.fromarray(p) for p in page_u8]
    times = []
    for _ in range(iters + 1):
        t0 = time.perf_counter()
        for img in imgs:
            (rh, rw), pad = ops.evaluate_set_geometry(img.size[1], img.size[0], resize)
            x = torch.from_numpy(np.asarray(img.resize((rw, rh), Image.BICUBIC), dtype=np.uint8))
            x = x.permute(2, 0, 1).float().div(255).sub_(mean).div_(std)
            x = F.pad(x[None], pad, value=0).to(dev, non_blocking=False)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1000)
    return statistics.median(times[1:])


def bench(name, iters, warmup):
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import DEMO_MEAN_STD, TextRemovalStep
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
    page_u8 = (0.8 * base + 0.2 * torch.rand((n, 3, h, w), generator=g)).clamp(0, 1).mul(255).to(torch.uint8)
    page = page_u8.float().div(255).to(dev)                                   # to_tensor of an 8-bit page

    plain, resized = TextRemovalStep(seg, fill), TextRemovalStep(seg, fill, seg_resize=RESIZE)
    (hs, ws), (hu, wu) = plain.padded_sizes(h, w)
    (rs, rws), _ = resized.padded_sizes(h, w)
    (rh, rw), pad = ops.evaluate_set_geometry(h, w, RESIZE)
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
    del xin, logits, mask, corrupted, valid

    plain.run(page), resized.run(page)                                        # captures both graphs
    torch.cuda.synchronize()
    holes = {k: 1.0 - float(s.valid[:, :h, :w].float().mean()) for k, s in (("plain", plain), ("resized", resized))}
    times = {"plain": [], "resized": [], "resize_stage": []}
    for i in range(warmup + iters):
        for kind, fn in (("plain", lambda: plain.run(page)), ("resized", lambda: resized.run(page)),
                         ("resize_stage", lambda: ops.page_resize_bicubic(page, rh, rw))):
            t = _event_ms(fn)
            if i >= warmup:
                times[kind].append(t)
    med = {k: statistics.median(v) for k, v in times.items()}
    host = host_prepare_ms(page_u8.permute(0, 2, 3, 1).numpy(), RESIZE, max(3, iters // 4), dev)
    return {"workload": name, "page_hw": [h, w], "batch": n, "seg_grid_page_size": [hs, ws], "seg_grid_resized": [rs, rws],
            "resized_hw": [rh, rw], "unet_hw": [hu, wu], "hole_fraction": {k: round(v, 4) for k, v in holes.items()},
            "run_ms_page_size": round(med["plain"], 3), "run_ms_seg_resize": round(med["resized"], 3),
            "resize_stage_ms": round(med["resize_stage"], 4),
            "launches_page_size": plain.launches_per_run, "launches_seg_resize": resized.launches_per_run,
            "host_evaluate_set_prepare_ms": None if host is None else round(host, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_removal_resize.py needs a CUDA device")
    names = a.only.split(",") if a.only else list(WORKLOADS)
    res = {"card": card(), "resize": RESIZE, "workloads": []}
    for n in names:
        res["workloads"].append(bench(n, a.iters, a.warmup))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

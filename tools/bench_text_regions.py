"""Region-image benchmark: the segmentation demo's ``_contour`` image (draw_bounding_box(page, mask, 500),
Examples/demo_segmentation.py:17-25, 40-45) drawn on the GPU by ops.text_region_hulls, against the demo's host path for the
same pages, and the cost of adding it to engine.TextRemovalStep.

Per workload (page size and batch) and mask:
  * `op_ms`: ops.text_region_hulls alone, median of CUDA-event-timed calls;
  * `host_ms`: the demo's host path, median by host clock: the mask and page copied to the host, to_pil_image of both
    (the mask as its "L" image) and draw_bounding_box's statements with cv2, page by page ("not measured" without cv2);
  * `step_ms` / `step_regions_ms`: TextRemovalStep(seg_resize=600).run() without and with region_hulls=500 (XceptionTextSegment
    + ImageFillOrigin set up as tools/bench_text_removal.py does), alternating call by call, CUDA events;
  * launches of the op and of both steps, the regions and painted fraction, and whether the op's bytes equal the host path's.
Masks: "manga" (synthetic.manga_text_mask: speech-bubble rings holding columns of glyphs) and "step" (the text mask the step
itself produces on the benchmark page).  Prints one JSON line with the card's name, power limit and max SM clock (read in the
same run).

    python tools/bench_text_regions.py [--iters 30] [--warmup 5] [--only NAME]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_text_removal import _calibrate, card  # noqa: E402

# name: (page height, page width, batch)
WORKLOADS = {
    "1700x1200_b1": (1700, 1200, 1),
    "3508x2480_b1": (3508, 2480, 1),          # A4 at 300 dpi
    "1024x1024_b4": (1024, 1024, 4),
}
THRESHOLD = 500                                # the demo's call


def _events(fn, iters, warmup):
    times = []
    for i in range(warmup + iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        if i >= warmup:
            times.append(s.elapsed_time(e))
    return statistics.median(times)


def _host_path(mask, page):
    """the demo's statements after its network: copies, to_pil_image, draw_bounding_box with cv2 (None without cv2)"""
    try:
        import cv2
        from torchvision.transforms.functional import to_pil_image
    except ImportError:
        return None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m, p = mask.float().cpu(), page.cpu()
    outs = []
    for i in range(m.shape[0]):
        origin_np = np.array(to_pil_image(p[i]))
        mask_np = np.array(to_pil_image(m[i]).convert("L"), dtype="uint8")
        contours, _ = cv2.findContours(mask_np, cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)
        for cnt in contours:
            if cv2.contourArea(cnt) > THRESHOLD:
                cv2.drawContours(origin_np, [cv2.convexHull(cnt)], 0, (50, 128, 30), -1)
        outs.append(origin_np)
    return (time.perf_counter() - t0) * 1000, np.stack(outs)


def _nets(page):
    """XceptionTextSegment + ImageFillOrigin with deterministic weights, calibrated on the page as tools/bench_text_removal.py
    does (about 0.5 % of the segmentation logits positive), for the step with seg_resize=600"""
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import DEMO_MEAN_STD
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models import image_inpainting as II
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    torch.manual_seed(0)
    seg, fill = TS.XceptionTextSegment(), II.ImageFillOrigin()
    seg.load_state_dict(det_fill_state_dict(seg.state_dict()))
    fill.load_state_dict(det_fill_state_dict(fill.state_dict()))
    seg, fill = seg.to(page.device), fill.to(page.device)
    n, _, h, w = page.shape
    (rh, rw), pad = ops.evaluate_set_geometry(h, w, 600)
    xin = ops.removal_seg_input(ops.page_resize_bicubic(page, rh, rw), DEMO_MEAN_STD, rh + pad[3], rw + pad[1], torch.bfloat16)
    _calibrate(seg, lambda: seg(xin))
    with torch.no_grad():
        logits = seg(xin).float()
        [m for m in seg.modules() if getattr(m, "out_channels", None) == 1 and getattr(m, "bias", None) is not None][-1].bias.sub_(
            float(torch.quantile(logits.flatten()[::97], 0.995)))
    ops.bump_weight_epoch()
    with torch.no_grad():
        mask = ops.text_mask_postprocess(seg(xin), pad, (h, w))
    mult = 2 ** len(fill.decoder)
    corrupted, valid = ops.removal_holes(mask, page, (h + mult - 1) // mult * mult, (w + mult - 1) // mult * mult, torch.bfloat16)
    _calibrate(fill, lambda: fill((corrupted, HoleMask.from_plane(valid, 3))))
    return seg, fill


def bench(name, iters, warmup):
    from text_segmentation_image_inpainting_b200 import _lib, ops
    from text_segmentation_image_inpainting_b200.engine import TextRemovalStep
    from text_segmentation_image_inpainting_b200.synthetic import manga_text_mask
    from scipy import ndimage
    h, w, n = WORKLOADS[name]
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(1)
    base = F.interpolate(torch.rand((n, 3, h // 16 + 2, w // 16 + 2), generator=g), size=(h, w), mode="bilinear", align_corners=False)
    page = (0.8 * base + 0.2 * torch.rand((n, 3, h, w), generator=g)).clamp(0, 1).to(dev)
    seg, fill = _nets(page)
    plain = TextRemovalStep(seg, fill, seg_resize=600)
    drawn = TextRemovalStep(seg, fill, seg_resize=600, region_hulls=THRESHOLD)
    plain.run(page), drawn.run(page)                                           # captures both graphs
    steps = {"plain": [], "regions": []}
    for i in range(warmup + iters):
        for kind, st in (("plain", plain), ("regions", drawn)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            st.run(page)
            e.record()
            e.synchronize()
            if i >= warmup:
                steps[kind].append(s.elapsed_time(e))
    masks = {"manga": torch.from_numpy(np.stack([manga_text_mask(h, w, 7 + i) for i in range(n)])[:, None]).to(dev),
             "step": drawn.text_mask.clone()}
    rows = []
    for mname, mask in masks.items():
        out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
        before = _lib.launch_count()
        ops.text_region_hulls(mask, page, THRESHOLD, out=out)
        launches = _lib.launch_count() - before
        op_ms = _events(lambda: ops.text_region_hulls(mask, page, THRESHOLD, out=out), iters, warmup)
        host = [_host_path(mask, page) for _ in range(max(3, iters // 5))]
        mh = mask.cpu().numpy()
        regions = 0
        for i in range(n):
            fg = mh[i, 0] != 0
            lab, _ = ndimage.label(np.pad(~fg, 1, constant_values=True))
            regions += ndimage.label(lab[1:-1, 1:-1] != lab[0, 0], structure=np.ones((3, 3), bool))[1]
        painted = float((out == torch.tensor((50, 128, 30), dtype=torch.uint8, device=dev)).all(-1).float().mean())
        rows.append({"mask": mname, "text_fraction": round(float(mask.float().mean()), 4), "regions": int(regions),
                     "painted_fraction": round(painted, 4), "op_ms": round(op_ms, 3), "op_launches": launches,
                     "host_ms": "not measured" if host[0] is None else round(statistics.median(t for t, _ in host), 2),
                     "equal_to_host": None if host[0] is None else bool(np.array_equal(out.cpu().numpy(), host[0][1]))})
    med = {k: statistics.median(v) for k, v in steps.items()}
    return {"workload": name, "page_hw": [h, w], "batch": n, "threshold": THRESHOLD, "masks": rows,
            "step_ms": round(med["plain"], 3), "step_regions_ms": round(med["regions"], 3),
            "step_launches": plain.launches_per_run, "step_regions_launches": drawn.launches_per_run}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_text_regions.py needs a CUDA device")
    names = a.only.split(",") if a.only else list(WORKLOADS)
    res = {"card": card(), "workloads": []}
    for n in names:
        res["workloads"].append(bench(n, a.iters, a.warmup))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

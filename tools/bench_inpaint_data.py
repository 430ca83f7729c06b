"""Measure the GPU inpainting data path (data.InpaintBatcher, engine.InpaintTrainStep) on one GPU and print one JSON line:

  * pipeline_ms:  device time of prepare() for 8 x 512^2 from 1448 x 1024 sources with random strokes (CUDA events, mean),
  * step_ms:      InpaintTrainStep (pipeline + training step in one graph) against TrainStep fed device-resident batches,
                  ImageFillOrigin, bf16, alternating rounds, same seeds,
  * host_ms_per_image: the reference's process_images on one host core (staged oracle/_ref/Dataloader.py, when present) next
                  to this path's host work (stage(): copy into pinned memory and enqueue the upload).

    python tools/bench_inpaint_data.py [--rounds 5 --steps 20]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in q.split(","))
        return name, power
    except Exception:  # noqa: BLE001
        import torch
        return torch.cuda.get_device_name(), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--pipeline-iters", type=int, default=200)
    args = ap.parse_args()

    import numpy as np
    import torch

    import inpaint_ref as R
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintTrainStep, TrainStep
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin

    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint_data.py needs a CUDA device")
    dev = torch.device("cuda")
    B, S, H, W = 8, 512, 1448, 1024
    srcs = [R.sources(i, H, W) for i in range(B)]
    res = {"card": None, "power_limit": None, "batch": B, "image_size": S, "source": [H, W]}
    res["card"], res["power_limit"] = card()

    # ---- pipeline alone
    b = InpaintBatcher(B, (H, W), image_size=S, add_random_masks=True, seed=0)
    b.stage(srcs)
    for _ in range(10):
        b.prepare()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.pipeline_iters):
        b.prepare()
    e1.record()
    torch.cuda.synchronize()
    res["pipeline_ms"] = e0.elapsed_time(e1) / args.pipeline_iters

    # ---- host work per image
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        b.stage(srcs)
    torch.cuda.synchronize()
    res["host_ms_per_image_stage"] = (time.perf_counter() - t0) / (reps * B) * 1e3
    if R.dataloader() is not None:
        from PIL import Image
        torch.set_num_threads(1)
        ds = R.dataset(S, True)
        pil = [(Image.fromarray(r), Image.fromarray(m)) for r, m in srcs[:2]]
        t0 = time.perf_counter()
        for i in range(10):
            ds.process_images(*pil[i % 2])
        res["host_ms_per_image_reference"] = (time.perf_counter() - t0) / 10 * 1e3
    else:
        res["host_ms_per_image_reference"] = None

    # ---- training step: InpaintTrainStep vs TrainStep fed device-resident batches
    def net():
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            return ImageFillOrigin().to(dev)

    b.stage(srcs)
    _, hm, clean = b.prepare()
    x_dev, m_dev = clean.clone(), hm.dense().clone()
    plain = TrainStep(net(), compute_dtype=torch.bfloat16)
    plain.warmup_and_capture(x_dev, m_dev, eager_warmup=2)
    fused = InpaintTrainStep(net(), b)
    fused.warmup_and_capture(eager_warmup=2)
    times = {"train_step": [], "inpaint_train_step": []}
    for r in range(args.rounds):
        for name in ("train_step", "inpaint_train_step") if r % 2 == 0 else ("inpaint_train_step", "train_step"):
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                if name == "train_step":
                    plain.step(x_dev, m_dev)
                else:
                    fused.step()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    res["step_ms"] = {k: float(np.median(v)) for k, v in times.items()}
    res["step_ms_all"] = times
    res["pipeline_share_of_step"] = res["pipeline_ms"] / res["step_ms"]["train_step"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()

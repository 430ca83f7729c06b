"""Measure the inpainting loss (loss.InpaintingLoss, engine.InpaintLossTrainStep) on one GPU and print one JSON line:

  * step_ms:   InpaintLossTrainStep against InpaintTrainStep (same net, batcher and seeds; L1 stand-in loss), ImageFillOrigin,
               bf16, 512^2, batch 8, graph replay, alternating rounds (CUDA events, medians);
  * loss_ms:   forward + backward of the loss alone on the network-shaped bf16 output (CUDA events, mean), and the achieved
               rate against the FLOPs of its VGG convolutions and Gram products computed from the shapes;
  * parts_ms:  CUDA events around each part of the loss (loss.set_part_timing, eager calls, mean): VGG forward (convolutions
               and pools), VGG data gradient (pool backward, convolutions with the ReLU backward, conv1_1 in kernel-to-row form),
               Gram products and Gram backward, and the fused pixel / L1 kernels.

    python tools/bench_inpaint_loss.py [--rounds 4 --steps 20]
"""
import argparse
import contextlib
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

STAGES = (((3, 64), (64, 64)), ((64, 128), (128, 128)), ((128, 256), (256, 256), (256, 256)))


def loss_flops(n, s):
    """(VGG forward FLOPs over 3n images, VGG data-gradient FLOPs over 2n images, Gram forward + backward FLOPs)."""
    fwd = dg = gram = 0
    for convs in STAGES:
        for cin, cout in convs:
            f = 2 * s * s * cin * cout * 9
            fwd += 3 * n * f
            dg += 2 * n * f
        s //= 2
        c = convs[-1][1]
        gram += 3 * n * 2 * s * s * c * c + 2 * n * 2 * s * s * c * c
    return fwd, dg, gram


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--loss-iters", type=int, default=20)
    args = ap.parse_args()

    import numpy as np
    import torch

    import inpaint_ref as R
    from bench_inpaint_data import card
    from oracle.inpaint_loss import vgg_state_dict
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintLossTrainStep, InpaintTrainStep
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin

    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint_loss.py needs a CUDA device")
    dev = torch.device("cuda")
    B, S, H, W = 8, 512, 1448, 1024
    res = {"batch": B, "image_size": S}
    res["card"], res["power_limit"] = card()
    fwd, dg, gram = loss_flops(B, S)
    res["loss_tflop"] = {"vgg_forward": fwd / 1e12, "vgg_dgrad": dg / 1e12, "gram": gram / 1e12}
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(vgg_state_dict(0))
    vgg = vgg.to(dev)
    srcs = [R.sources(i, H, W) for i in range(B)]
    b = InpaintBatcher(B, (H, W), image_size=S, add_random_masks=True, seed=0)
    b.stage(srcs)

    # ---- the loss alone
    crit = InpaintingLoss(vgg)
    _, hm, clean = b.prepare()
    torch.manual_seed(0)
    out = ops.padded_empty(B, 3, S, S, torch.bfloat16, dev)
    with torch.no_grad():
        out.copy_((clean + 0.1 * torch.randn_like(clean)).to(torch.bfloat16))
    out.requires_grad_(True)

    def once():
        out.grad = None
        crit(clean, hm, out, clean).backward()

    for _ in range(3):
        once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.loss_iters):
        once()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.loss_iters
    res["loss_ms"] = ms
    res["loss_tflops_achieved"] = (fwd + dg + gram) / (ms * 1e-3) / 1e12

    from text_segmentation_image_inpainting_b200 import loss as L
    parts = {}
    for _ in range(args.loss_iters):
        sink = []
        L.set_part_timing(sink)
        once()
        L.set_part_timing(None)
        torch.cuda.synchronize()
        for name, s0, s1 in sink:
            parts[name] = parts.get(name, 0.0) + s0.elapsed_time(s1) / args.loss_iters
    res["parts_ms"] = parts

    # ---- training step with and without the loss
    def net():
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            return ImageFillOrigin().to(dev)

    plain = InpaintTrainStep(net(), b)
    plain.warmup_and_capture(eager_warmup=2)
    full = InpaintLossTrainStep(net(), b, vgg)
    full.warmup_and_capture(eager_warmup=2)
    times = {"inpaint_train_step": [], "inpaint_loss_train_step": []}
    for r in range(args.rounds):
        order = ("inpaint_train_step", "inpaint_loss_train_step") if r % 2 == 0 else ("inpaint_loss_train_step", "inpaint_train_step")
        for name in order:
            ts = plain if name == "inpaint_train_step" else full
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                ts.step()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    res["step_ms"] = {k: float(np.median(v)) for k, v in times.items()}
    res["step_ms_all"] = times
    res["last_terms"] = [float(v) for v in full.last_terms.cpu()]
    plain.close()
    full.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

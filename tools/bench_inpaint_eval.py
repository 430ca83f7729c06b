"""Measure the raw/clean pair data path (data.InpaintPairBatcher) and held-out evaluation (engine.InpaintEvalStep) on one GPU and
print one JSON line:

  * pipeline_ms:  prepare() of 8 x 512^2 from 1448 x 1024 sources (CUDA events over many calls, mean): the pair path with and
                  without strokes, and the mask-file path (data.InpaintBatcher) with strokes for comparison;
  * host_ms_per_image: stage() of the pairs, and the reference's TestDataset.process_images on one host core (staged
                  oracle/_ref/Dataloader.py, when present);
  * eval_ms:      InpaintEvalStep.run() against the same prepare + fused eval forward (+ InpaintingLoss) run eagerly, without and
                  with the VGG16 extractor: ImageFillOrigin, bf16, batch 8 (CUDA events, medians of rounds);
  * refresh_ms:   run() right after an InpaintTrainStep replay on the same network (operand buffers and BatchNorm coefficients
                  rewritten once) minus a run() without one.

    python tools/bench_inpaint_eval.py [--rounds 5 --steps 10]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _timed(fn, iters):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
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
    ap.add_argument("--pipeline-iters", type=int, default=200)
    args = ap.parse_args()

    import torch

    import inpaint_pair_ref as P
    from bench_inpaint_data import card
    from oracle import inpaint_loss as OL
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher, InpaintPairBatcher
    from text_segmentation_image_inpainting_b200.engine import InpaintEvalStep, InpaintTrainStep
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor
    from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin

    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint_eval.py needs a CUDA device")
    dev = torch.device("cuda")
    B, S, H, W = 8, 512, 1448, 1024
    pairs = [P.pair(i, H, W) for i in range(B)]
    res = {"card": None, "power_limit": None, "batch": B, "image_size": S, "source": [H, W]}
    res["card"], res["power_limit"] = card()

    # ---- pipelines alone
    res["pipeline_ms"] = {}
    for name, cls, src, strokes in (("pair_strokes", InpaintPairBatcher, pairs, True), ("pair_no_strokes", InpaintPairBatcher, pairs, False),
                                    ("mask_file_strokes", InpaintBatcher, [(c, P.R.sources(i, H, W)[1]) for i, (_, c) in enumerate(pairs)],
                                     True)):
        b = cls(B, (H, W), image_size=S, add_random_masks=strokes, seed=0)
        b.stage(src)
        _timed(b.prepare, 10)
        res["pipeline_ms"][name] = _timed(b.prepare, args.pipeline_iters)
        del b

    # ---- host work per image
    b = InpaintPairBatcher(B, (H, W), image_size=S, add_random_masks=True, seed=0)
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        b.stage(pairs)
    torch.cuda.synchronize()
    res["host_ms_per_image"] = {"stage": (time.perf_counter() - t0) / (reps * B) * 1e3, "reference": None}
    if P.R.dataloader() is not None:
        from PIL import Image
        threads = torch.get_num_threads()
        torch.set_num_threads(1)
        ds = P.dataset(S, True)
        pil = [(Image.fromarray(r), Image.fromarray(c)) for r, c in pairs[:2]]
        t0 = time.perf_counter()
        for i in range(10):
            ds.process_images(*pil[i % 2])
        res["host_ms_per_image"]["reference"] = (time.perf_counter() - t0) / 10 * 1e3
        torch.set_num_threads(threads)

    # ---- evaluation: graph against eager
    def net():
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            return ImageFillOrigin().to(dev)

    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(OL.vgg_state_dict(0))
    vgg = vgg.to(dev)
    res["eval_ms"] = {}
    for label, extractor in (("no_loss", None), ("loss", vgg)):
        n = net()
        b.stage(pairs)
        ev = InpaintEvalStep(n, b, extractor)
        ev.warmup_and_capture()
        crit = InpaintingLoss(extractor) if extractor is not None else None
        scope = ops.StepScope(dev, training=False)

        def eager():
            n.eval()
            try:
                with scope, torch.no_grad():
                    xin, hm, clean = b.prepare()
                    out = n((xin, hm))
                    if crit is not None:
                        crit(clean, hm, out, clean)
            finally:
                n.train()
        eager()
        graph_ms, eager_ms = [], []
        for _ in range(args.rounds):
            graph_ms.append(_timed(ev.run, args.steps))
            eager_ms.append(_timed(eager, args.steps))
        res["eval_ms"][label] = {"graph": statistics.median(graph_ms), "eager": statistics.median(eager_ms),
                                 "fused_sites": ev.fused_sites, "launches_per_run": ev.launches_per_run}
        del ev

    # ---- refresh after a training replay
    n = net()
    tb = InpaintPairBatcher(B, (H, W), image_size=S, add_random_masks=True, seed=1)
    tb.stage(pairs)
    ts = InpaintTrainStep(n, tb, lr=1e-4)
    ts.warmup_and_capture()
    b.stage(pairs)
    ev = InpaintEvalStep(n, b, vgg)
    ev.warmup_and_capture()
    after, steady = [], []
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    for _ in range(args.rounds * args.steps):
        tb.stage(pairs)
        ts.step()
        e[0].record()
        ev.run()
        e[1].record()
        ev.run()
        e[2].record()
        torch.cuda.synchronize()
        after.append(e[0].elapsed_time(e[1]))
        steady.append(e[1].elapsed_time(e[2]))
    res["refresh_ms"] = {"run_after_train_step": statistics.median(after), "run_steady": statistics.median(steady),
                         "refresh": statistics.median(after) - statistics.median(steady)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Generate tests/golden/elementwise_sites.json: every distinct call site of the BatchNorm, concat / upsample, mask-format,
pooling, bilinear, GAP, scSE, L1-loss and SGD entry points that the workloads make, for tests/test_gpu_batchnorm.py and
tests/test_gpu_glue_ops.py.

On a GPU, wrap those attributes of the loaded library with recorders and run what make_golden_conv_dispatch.py --record runs:
  * one eager forward + backward of ImageFillOrigin 512^2 b8, TextSegament 512^2 b8 and XceptionTextSegment 512^2 b16 (bf16),
  * the eager eval forward of XceptionTextSegment at 600^2 b1,
  * one optimiser step of TrainStep (ImageFillOrigin),
  * the inference runs (make_golden_conv_dispatch.inference_runs): the eager forward of TextRemovalStep on every page of
    TEXT_REMOVAL_RUNS (the rows of tools/bench_text_removal.py and tools/bench_text_removal_resize.py, the A4 page segmented at
    page size, TextSegament + ImageFill at 1700 x 1200 with and without seg_resize=600) and of InferStep(ImageFillOriginV2) at
    the 1700 x 1200 page's U-Net grid: bilinear resampling at unequal, non-integer ratios, pooling and GAP on odd grids, concat
    and the unfused residual BatchNorm at page sizes.
Each call is recorded by its non-pointer arguments, which of its optional pointers were null, whether the two sums of the
statistics / backward reduction were one [2][c] buffer (one memset instead of two), and the part table of a concat.  Sites
the fixture does not hold yet are appended to it, sorted; the entries already there stay as they are:
    python tests/golden/make_golden_elementwise_sites.py [fixture.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), HERE]
FIXTURE = os.path.join(HERE, "elementwise_sites.json")

# argument names per entry point (include/pconv_b200.h).  "?name": a pointer recorded as null / non-null; "-": a pointer or
# stream not recorded; anything else: a value recorded as is.
ARGS = {
    "pcb_bn_stats": ["-", "dtype", "count", "c", "-", "-", "-"],
    "pcb_bn_stats_acc": ["-", "dtype", "count", "c", "-", "-"],
    "pcb_bn_forward_fused": ["-", "dtype", "count", "c", "-", "?gamma", "?beta", "?running", "-", "?nbt", "momentum", "eps", "act",
                             "slope", "?residual", "-", "-", "-"],
    "pcb_bn_finalize": ["?sum", "-", "count", "c", "?gamma", "?beta", "?running", "-", "?nbt", "momentum", "eps", "training", "-", "-",
                        "?save_mean", "?save_invstd", "-"],
    "pcb_bn_act_forward": ["-", "dtype", "count", "c", "?scale", "-", "act", "slope", "?residual", "-", "-"],
    "pcb_bn_act_backward_reduce": ["-", "-", "dtype", "count", "c", "?scale", "?shift", "?mean", "?invstd", "act", "slope", "-", "-", "-"],
    "pcb_bn_act_backward_reduce_acc": ["-", "-", "dtype", "count", "c", "?scale", "?shift", "?mean", "?invstd", "act", "slope", "-", "-"],
    "pcb_bn_act_backward_small": ["-", "-", "dtype", "count", "c", "-", "act", "slope", "?msum", "-", "?dgamma", "?dbeta", "-"],
    "pcb_bn_act_backward_apply": ["-", "-", "dtype", "count", "c", "?scale", "?shift", "?mean", "?invstd", "act", "slope", "?sum_g",
                                  "?sum_gx", "training", "-", "?dgamma", "?dbeta", "-"],
    "pcb_bn_act_backward_apply_renorm": ["-", "-", "dtype", "count", "c", "?scale", "?shift", "?mean", "?invstd", "act", "slope",
                                         "?sum_g", "?sum_gx", "training", "?msum", "-", "?dgamma", "?dbeta", "-"],
    "pcb_upsample2x_forward": ["-", "dtype", "n", "h", "w", "c", "-", "-"],
    "pcb_upsample2x_backward": ["-", "dtype", "n", "h", "w", "c", "-", "-"],
    "pcb_concat_forward": ["-", "nparts", "dtype", "n", "h", "w", "-", "-"],
    "pcb_concat_backward": ["-", "-", "-", "nparts", "dtype", "n", "h", "w", "-", "-"],
    "pcb_mask_planes_from_dense": ["-", "n", "c", "h", "w", "-", "-"],
    "pcb_mask_plane_to_dense": ["-", "n", "h", "w", "up", "-", "ctot", "c0", "c", "-"],
    "pcb_avgpool_forward": ["-", "-", "dtype", "n", "h", "w", "c", "k", "stride", "pad", "-"],
    "pcb_avgpool_backward": ["-", "-", "dtype", "n", "h", "w", "c", "k", "stride", "pad", "-"],
    "pcb_bilinear_forward": ["-", "-", "dtype", "n", "h", "w", "c", "scale", "-"],
    "pcb_bilinear_backward": ["-", "-", "dtype", "n", "h", "w", "c", "scale", "-"],
    "pcb_gap_forward": ["-", "dtype", "n", "hw", "c", "-", "-"],
    "pcb_gap_backward": ["-", "-", "dtype", "n", "hw", "c", "accumulate", "-"],
    "pcb_scse_forward": ["-", "-", "-", "-", "-", "dtype", "n", "hw", "c", "-"],
    "pcb_scse_backward": ["-", "-", "-", "-", "-", "-", "-", "-", "dtype", "n", "hw", "c", "-"],
    "pcb_l1_mean_forward": ["-", "dtype", "numel", "-", "-", "-"],
    "pcb_l1_mean_backward": ["-", "dtype", "numel", "gscale", "-", "-"],
    "pcb_sgd_step": ["-", "-", "-", "numel", "lr", "momentum", "weight_decay", "nesterov", "first_step", "-"],
    "pcb_sgd_step_scaled": ["-", "-", "-", "numel", "lr", "momentum", "weight_decay", "nesterov", "first_step", "grad_scale", "-"],
}


def _ptr(v):
    return 0 if v is None else int(v.value if hasattr(v, "value") else v)


def describe(fn, args):
    site = {"fn": fn}
    for name, v in zip(ARGS[fn], args):
        if name == "-":
            continue
        if name.startswith("?"):
            site["null_" + name[1:]] = int(_ptr(v) == 0)
        elif isinstance(v, float):
            site[name] = float(f"{v:.7g}")                   # the float32 the C ABI receives, printed compactly
        else:
            site[name] = int(v)
    if fn == "pcb_bn_stats":
        site["aliased"] = int(_ptr(args[5]) == _ptr(args[4]) + 8 * args[3])
    if fn == "pcb_bn_act_backward_reduce":
        site["aliased"] = int(_ptr(args[12]) == _ptr(args[11]) + 8 * args[4])
    if fn == "pcb_concat_forward":
        parts = args[0]
        site["parts"] = [[int(parts[i].c), int(parts[i].x_cstride), int(parts[i].x_up)] for i in range(args[1])]
    if fn == "pcb_concat_backward":
        site["parts"] = [[int(args[1][i]), int(args[2][i]), int(_ptr(args[8][i]) == 0)] for i in range(args[3])]
    return site


def record(path):
    import torch

    from make_golden_conv_dispatch import inference_runs
    from oracle.detfill import det_fill_state_dict, det_tensor
    from text_segmentation_image_inpainting_b200 import _lib
    from text_segmentation_image_inpainting_b200.engine import SegInferStep, SegTrainStep, TrainStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting, text_segmentation
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks

    dev = torch.device("cuda")
    lib = _lib.load()
    rec = []
    originals = {fn: getattr(lib, fn) for fn in ARGS}

    def recorder(fn, f):
        def call(*args):
            rec.append(describe(fn, args))
            return f(*args)
        return call
    for fn, f in originals.items():
        setattr(lib, fn, recorder(fn, f))
    try:
        torch.manual_seed(0)
        for mod, cls, batch, masks in ((image_inpainting, "ImageFillOrigin", 8, True), (text_segmentation, "TextSegament", 8, False),
                                       (text_segmentation, "XceptionTextSegment", 16, False)):
            net = getattr(mod, cls)().to(dev)
            ts = (TrainStep if masks else SegTrainStep)(net, compute_dtype=torch.bfloat16, use_graph=False)
            x = torch.randn(batch, 3, 512, 512, device=dev)
            m = torch.from_numpy(random_hole_masks(batch, 512, 512, seed=0)).to(dev) if masks else None
            ts._fwd_bwd(x, m)
            if masks:
                ts._update(True)
            torch.cuda.synchronize()
            del net, ts
        net = text_segmentation.XceptionTextSegment()
        net.load_state_dict(det_fill_state_dict(net.state_dict()))
        net = net.to(dev).eval()
        with torch.no_grad():
            SegInferStep(net)._forward(det_tensor("conv_dispatch.x", (1, 3, 600, 600)).to(dev))
        torch.cuda.synchronize()
        for run in inference_runs(dev):
            print(run)
    finally:
        for fn, f in originals.items():
            setattr(lib, fn, f)
    with open(path) as f:
        known = [json.dumps(s, sort_keys=True) for s in json.load(f)]
    new = sorted({json.dumps(s, sort_keys=True) for s in rec} - set(known))
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(known + new) + "\n]\n")
    print(f"{len(rec)} calls, {len(new)} new sites appended, {len(known) + len(new)} in all -> {path}")


if __name__ == "__main__":
    record(sys.argv[1] if len(sys.argv) > 1 else FIXTURE)

"""Generate tests/golden/seg_loss_sites.json: every distinct call site of the segmentation-loss kernels (csrc/seg_loss.cu) and of
the text-mask post-processing kernel (csrc/seg_ops.cu) that training and inference make, for
tests/test_gpu_seg_loss_kernels.py.

On a GPU, wrap pcb_seg_loss_forward, pcb_seg_loss_backward and pcb_seg_mask_postprocess on the loaded library with recorders
and run
  * one eager SegLossTrainStep step each for TextSegament (batch 8) and XceptionTextSegment (batch 16) at 512^2, bf16, with
    BinaryFocalLoss(), BinaryFocalLoss(gamma=2) and SoftBootstrapCrossEntropy() (the logits reach the loss as the networks
    return them, the [n, 1, h, w] view of a channel-padded NHWC buffer),
  * forward + backward of the same three losses on dense NCHW fp32 logits at 256^2, batch 2 (the layout of the reference's
    goldens),
  * SegInferStep (XceptionTextSegment) at 600^2 with the post-processing call of tools/bench_infer.py.
Each call is recorded by its non-pointer arguments (float parameters as the float32 values the kernel receives) and the four
entries of each stride array:
    python tests/golden/make_golden_seg_loss_sites.py [out.json]
"""
import ctypes
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
FIXTURE = os.path.join(HERE, "seg_loss_sites.json")

# argument names per entry point (include/pconv_b200.h).  "@name": an array of 4 host values recorded as a list; "-": a pointer
# or stream not recorded; anything else: a value (the names of FLOAT_ARGS are float parameters of the C ABI).
_LOSS = ["-", "dtype", "@x_strides", "-", "n", "h", "w", "loss", "reduction", "p0", "one_minus_beta", "background_weight",
         "words_weight"]
ARGS = {
    "pcb_seg_loss_forward": _LOSS + ["-", "-", "-", "-"],
    "pcb_seg_loss_backward": _LOSS + ["-", "-", "@dx_strides", "-"],
    "pcb_seg_mask_postprocess": ["-", "dtype", "n", "h", "w", "cstride", "h_valid", "w_valid", "oh", "ow", "-", "-"],
}
FLOAT_ARGS = {"p0", "one_minus_beta", "background_weight", "words_weight"}
# the demo's crop and original size of tools/bench_infer.py's post-processed workload
POST_PAD, POST_HW = (0, 0, 0, 152), (600, 800)


def _num(v):
    """ints as they are; floats by the shortest repr that reads back as the same double"""
    return v if isinstance(v, int) else float(repr(float(v)))


def _arg(name, v):
    """the value the kernel receives: the recorder sees the Python number before ctypes converts it, so a float parameter is
    rounded to float32 here as the conversion does (loss.py passes 0.95 and 1 - 0.95 as doubles)"""
    return _num(ctypes.c_float(v).value) if name in FLOAT_ARGS else _num(v)


def describe(fn, args):
    site = {"fn": fn}
    for name, v in zip(ARGS[fn], args):
        if name == "-":
            continue
        site[name[1:] if name.startswith("@") else name] = [_num(v[i]) for i in range(4)] if name.startswith("@") else _arg(name, v)
    return site


def recording(lib, rec):
    """context manager: the entry points of ARGS on lib append describe(...) of each call to rec"""
    import contextlib

    @contextlib.contextmanager
    def ctx():
        originals = {fn: getattr(lib, fn) for fn in ARGS}

        def recorder(fn, f):
            def call(*args):
                rec.append(describe(fn, args))
                return f(*args)
            return call
        for fn, f in originals.items():
            setattr(lib, fn, recorder(fn, f))
        try:
            yield rec
        finally:
            for fn, f in originals.items():
                setattr(lib, fn, f)
    return ctx()


def criteria():
    from text_segmentation_image_inpainting_b200.loss import BinaryFocalLoss, SoftBootstrapCrossEntropy
    return [BinaryFocalLoss(), BinaryFocalLoss(gamma=2), SoftBootstrapCrossEntropy()]


def _net(name):
    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.models import text_segmentation as TS
    net = getattr(TS, name)()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    return net.cuda()


def run_train(name, batch, size, crit, seed):
    """one eager SegLossTrainStep step of network `name` on a staged batch of `batch` pages, bf16, at size^2"""
    import torch

    import seg_ref
    from text_segmentation_image_inpainting_b200.data import SegBatcher
    from text_segmentation_image_inpainting_b200.engine import SegLossTrainStep
    b = SegBatcher(batch, (2 * size, 2 * size), image_size=size, seed=seed)
    b.stage([seg_ref.sources(seed + i, 2 * size - 37 * (i % 3), 2 * size - 53 * (i % 2)) for i in range(batch)])
    step = SegLossTrainStep(_net(name), b, crit, use_graph=False, lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False)
    step.step()
    torch.cuda.synchronize()


def run_dense(batch, size, crit, seed):
    """forward + backward of crit on dense NCHW fp32 logits"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(batch, 1, size, size, device="cuda", generator=g) * 3).requires_grad_(True)
    t = (torch.rand(batch, 1, size, size, device="cuda", generator=g) < 0.2).float()
    crit(x, t).backward()
    torch.cuda.synchronize()


def run_infer(name, size, pad, out_hw):
    """SegInferStep at size^2, batch 1, and the demo's post-processing of its logits"""
    import torch

    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import SegInferStep
    net = _net(name).eval()
    x = torch.rand(1, 3, size, size, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    ops.text_mask_postprocess(SegInferStep(net).run(x), pad, out_hw)
    torch.cuda.synchronize()


def record(path):
    from text_segmentation_image_inpainting_b200 import _lib
    rec = []
    with recording(_lib.load(), rec):
        for name, batch in (("TextSegament", 8), ("XceptionTextSegment", 16)):
            for k, crit in enumerate(criteria()):
                run_train(name, batch, 512, crit, 10 + k)
        for k, crit in enumerate(criteria()):
            run_dense(2, 256, crit, 20 + k)
        run_infer("XceptionTextSegment", 600, POST_PAD, POST_HW)
    uniq = {json.dumps(s, sort_keys=True) for s in rec}
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(sorted(uniq)) + "\n]\n")
    print(f"{len(rec)} calls, {len(uniq)} distinct sites -> {path}")


if __name__ == "__main__":
    record(sys.argv[1] if len(sys.argv) > 1 else FIXTURE)

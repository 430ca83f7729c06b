"""Generate tests/golden/inpaint_loss_sites.json: every distinct call site of the inpainting-loss kernels (csrc/inpaint_loss.cu)
that the loss makes, for tests/test_gpu_inpaint_loss_kernels.py.

On a GPU, wrap the eleven entry points of inpaint_loss.cu on the loaded library with recorders and run
  * one forward + backward of InpaintingLoss at 512^2, batch 8, bf16, with the networks' 8-channel-padded NHWC output (the
    run make_golden_conv_dispatch.py --record makes),
  * the same at 256^2, batch 2, fp32, with a dense NCHW output (the path of the reference's goldens),
  * total_variation_loss on a 512^2 batch-8 fp32 image, and gram_matrix on a stage-3 feature map (its products are the
    convolution weight-gradient problem, so it makes no call recorded here).
Each call is recorded by its non-pointer arguments, the four entries of each stride array, the host coef[4] and inv[16] values
and which of its optional pointers were null:
    python tests/golden/make_golden_inpaint_loss_sites.py [out.json]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
FIXTURE = os.path.join(HERE, "inpaint_loss_sites.json")

# argument names per entry point (include/pconv_b200.h).  "?name": a pointer recorded as null / non-null; "@name": an array of
# 4 (strides, coef) or 16 (inv) host values recorded as a list; "-": a pointer or stream not recorded; anything else: a value.
ARGS = {
    "pcb_inpaint_loss_pixel_forward": ["-", "-", "-", "out_dtype", "@out_strides", "-", "n", "h", "w", "-", "dtype", "-", "-"],
    "pcb_inpaint_loss_pixel_backward": ["-", "-", "-", "out_dtype", "@out_strides", "-", "n", "h", "w", "?dvgg_in", "dtype", "@coef", "-",
                                        "-", "@grad_strides", "-"],
    "pcb_maxpool2x2_forward": ["-", "-", "dtype", "n", "h", "w", "c", "-"],
    "pcb_maxpool2x2_backward": ["-", "-", "-", "dtype", "n", "h", "w", "c", "relu_mask", "-"],
    "pcb_feature_l1_forward": ["-", "dtype", "n", "hw", "c", "-", "-"],
    "pcb_feature_loss_backward": ["-", "dtype", "n", "hw", "c", "?g_next", "?g_gram", "l1_coef", "gram_coef", "-", "-", "-"],
    "pcb_gram_l1_forward": ["-", "n", "c", "norm", "-", "-"],
    "pcb_gram_sign_sym": ["-", "n", "c", "norm", "-", "-"],
    "pcb_k2r_image_weight": ["-", "cout", "-", "-"],
    "pcb_k2r_image_dgrad": ["-", "dtype", "n", "h", "w", "-", "-"],
    "pcb_inpaint_loss_finalize": ["-", "@inv", "-", "-", "-"],
}
SIZES = {"@out_strides": 4, "@grad_strides": 4, "@coef": 4, "@inv": 16}


def _ptr(v):
    return 0 if v is None else int(v.value if hasattr(v, "value") else v)


def _num(v):
    """ints as they are; floats by the shortest repr that reads back as the same double (a float32 argument arrives as the
    double of its float32 value, so it is kept exactly too)"""
    return v if isinstance(v, int) else float(repr(float(v)))


def describe(fn, args):
    site = {"fn": fn}
    for name, v in zip(ARGS[fn], args):
        if name == "-":
            continue
        if name.startswith("?"):
            site["null_" + name[1:]] = int(_ptr(v) == 0)
        elif name.startswith("@"):
            site[name[1:]] = [_num(v[i]) for i in range(SIZES[name])]
        else:
            site[name] = _num(v)
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


def run_loss(crit, n, size, dtype, nhwc, seed):
    """one forward + backward of crit at [n, 3, size, size] with random holes; output in dtype, NHWC-padded or dense NCHW"""
    import torch

    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    clean = torch.rand(n, 3, size, size, device=dev, generator=g)
    mask = torch.from_numpy(random_hole_masks(n, size, size, seed=seed)).to(dev)
    out = ops.padded_empty(n, 3, size, size, dtype, dev) if nhwc else torch.empty(n, 3, size, size, dtype=dtype, device=dev)
    with torch.no_grad():
        out.copy_(torch.rand(n, 3, size, size, device=dev, generator=g))
    out.requires_grad_(True)
    crit(clean * mask, mask, out, clean).backward()
    torch.cuda.synchronize()


def record(path):
    import torch

    from oracle.inpaint_loss import vgg_state_dict
    from text_segmentation_image_inpainting_b200 import _lib
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor, gram_matrix, total_variation_loss

    dev = torch.device("cuda")
    lib = _lib.load()
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(vgg_state_dict(0))
    crit = InpaintingLoss(vgg.to(dev))
    rec = []
    with recording(lib, rec):
        run_loss(crit, 8, 512, torch.bfloat16, True, 1)
        run_loss(crit, 2, 256, torch.float32, False, 2)
        total_variation_loss(torch.rand(8, 3, 512, 512, device=dev))
        gram_matrix(torch.relu(torch.randn(2, 256, 128, 128, device=dev)).to(torch.bfloat16))
        torch.cuda.synchronize()
    uniq = {json.dumps(s, sort_keys=True) for s in rec}
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(sorted(uniq)) + "\n]\n")
    print(f"{len(rec)} calls, {len(uniq)} distinct sites -> {path}")


if __name__ == "__main__":
    record(sys.argv[1] if len(sys.argv) > 1 else FIXTURE)

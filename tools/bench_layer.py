"""Time single partial-conv layers of the bench network (forward + backward) with CUDA events.  Development tool."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from text_segmentation_image_inpainting_b200 import ops
from text_segmentation_image_inpainting_b200.masks import HoleMask
from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
dev = torch.device("cuda:0")
LAYERS = {  # name: (parts [(c, up)], cout, k, s, p, hw_out_res_in, same_holes)
    "dec6_192_64": ([(128, 1), (64, 0)], 64, 3, 1, 1, 256, False),
    "dec5_384_128": ([(256, 1), (128, 0)], 128, 3, 1, 1, 128, False),
    "dec4_768_256": ([(512, 1), (256, 0)], 256, 3, 1, 1, 64, False),
    "dec3_1024_512": ([(512, 1), (512, 0)], 512, 3, 1, 1, 32, False),
    "enc1_64_128": ([(64, 0)], 128, 5, 2, 2, 256, True),
    "enc2_128_256": ([(128, 0)], 256, 5, 2, 2, 128, True),
    "enc3_256_512": ([(256, 0)], 512, 3, 2, 1, 64, True),
    "tail_67_3": ([(64, 1), (8, 0)], 8, 3, 1, 1, 512, False),
    # pointwise convolutions of the segmentation family (XceptionTextSegment middle flow at batch 16 = 65536 pixels)
    "pw_512_512": ([(512, 0)], 512, 1, 1, 0, 64, False, 16),
    "pw_256_256": ([(256, 0)], 256, 1, 1, 0, 128, False, 16),
}
ONCE = "--once" in sys.argv
names = [a for a in sys.argv[1:] if not a.startswith("--")] or list(LAYERS)
for name in names:
    parts, cout, k, s, p, hw, sh = LAYERS[name][:7]
    n = LAYERS[name][7] if len(LAYERS[name]) > 7 else 8
    xs, ms = [], []
    for c, up in parts:
        r = hw >> up
        xs.append(torch.randn(n, c, r, r, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True))
        ms.append(HoleMask.from_plane((torch.rand(n, r, r, device=dev) > 0.1).to(torch.uint8), c, up))
    mod = PC.PartialConv(sum(c for c, _ in parts), cout, k, s, p, 1, 1, False, sh).to(dev)
    x = ops.LazyCat(xs, [u for _, u in parts]) if len(xs) > 1 else xs[0]
    m = torch.cat(ms, 1) if len(ms) > 1 else ms[0]
    if name.startswith("pw_"):                     # plain nn.Conv2d semantics (no masks, no fixer warps), as the segmentation nets run them
        wgt = mod.feature_conv.weight
        def fwd():
            return ops.conv2d(x, wgt, None, s, p, 1, 1)
    else:
        def fwd():
            return mod((x, m))[0]
    y = fwd(); gy = torch.randn_like(y)
    y.backward(gy); torch.cuda.synchronize()
    if ONCE:
        continue
    for tag, fn in (("fwd", lambda: fwd()), ("fwd+bwd", lambda: fwd().backward(gy))):
        for _ in range(3): fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(10): fn()
        e1.record(); torch.cuda.synchronize()
        print(f"{name:16s} {tag:8s} {e0.elapsed_time(e1) / 10:8.3f} ms", flush=True)

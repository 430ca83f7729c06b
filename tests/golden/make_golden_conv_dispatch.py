"""Generate tests/golden/conv_dispatch.json for tests/test_conv_dispatch_cpu.py, in two steps:

  1. on a GPU, record the `pcb_conv` descriptor (geometry and parts, no pointers) of every distinct convolution of the following
     runs -- every descriptor `ops.ConvGeom.struct` hands to the library, so also the calls loss.py's VGG16 makes directly --
       * one eager forward + backward of ImageFillOrigin 512^2 b8, TextSegament 512^2 b8 and XceptionTextSegment 512^2 b16 (bf16),
       * the eager eval forward of XceptionTextSegment at 600^2 b1 (non-power-of-two grids: the gather kernels),
       * one forward + backward of InpaintingLoss at 512^2 b8: the VGG16 forward over 3n = 24 images, its data gradient over
         the 16 images the loss differentiates, and the 1x1 problem of conv1_1's data gradient,
       * the cases of tests/gpu_cases.py and the tile cases of test_gpu_conv_routes.py (TILE_CASES),
       * the inference runs (inference_runs): the eager forward of TextRemovalStep (bf16, no_grad, deterministic weights) on
         every page of TEXT_REMOVAL_RUNS -- every row of tools/bench_text_removal.py and tools/bench_text_removal_resize.py, the
         A4 page also segmented at page size, TextSegament + ImageFill at 1700 x 1200 with and without seg_resize=600 -- and
         InferStep(ImageFillOriginV2) at the U-Net grid of the 1700 x 1200 page.  Each network runs at the grids of the step's
         padded_sizes(): U-Nets on non-square grids padded to 2 ** len(decoder) (1792 x 1280, 3584 x 2560, 1712 x 1200), the
         segmentation networks at the page padded to a multiple of 8 (up to 3512 x 2480), at 600^2 and at b4;
         python tests/golden/make_golden_conv_dispatch.py --record descriptors.json
  2. on any machine, evaluate every host query of the library on the descriptors the fixture does not hold yet and append them
     to it (the entries already there stay as they are):
         python tests/golden/make_golden_conv_dispatch.py descriptors.json

A descriptor that only the inference runs reach carries "forward_only": 1: no workload runs its backward, so the kernel suites
check its forward alone (test_gpu_conv_routes.py, test_gpu_dwconv.py).  Entries without the key are tested in every direction.

The queries depend on the SM count; without a visible device the library assumes 132 (H100 SXM), which is what the fixture
holds.  Step 2 was first run with the library of the commit before the dispatch was gathered into one plan per problem, so the
test pins that the refactor kept every choice.  One descriptor came later: the tile case two_parts_one_upsampled moved from
batch 1 to batch 6 (where it reaches the sub-pixel data gradient), and its batch-1 descriptor, which no other run records,
was replaced by the batch-6 one with its host queries evaluated by the library of that change.  The inference runs' entries
were appended last, their host queries evaluated by the library of that change."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from test_conv_dispatch_cpu import FIELDS, FIXTURE, PART_FIELDS, conv_of, host_queries  # noqa: E402


def describe(c):
    d = {k: getattr(c, k) for k in FIELDS}
    d["parts"] = [dict({k: getattr(c.parts[i], k) for k in PART_FIELDS}, mask=int(bool(c.parts[i].mask))) for i in range(c.nparts)]
    return d


# (segmentation network, inpainting U-Net, page height, page width, batch, seg_resize) of the recorded TextRemovalStep runs
TEXT_REMOVAL_RUNS = (
    ("XceptionTextSegment", "ImageFillOrigin", 1700, 1200, 1, None),         # tools/bench_text_removal.py
    ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 1, None),
    ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 4, None),
    ("TextSegament", "ImageFill", 1024, 1024, 1, None),
    ("XceptionTextSegment", "ImageFillOrigin", 1700, 1200, 1, 600),          # tools/bench_text_removal_resize.py
    ("XceptionTextSegment", "ImageFillOrigin", 3508, 2480, 1, 600),          # A4 at 300 dpi
    ("XceptionTextSegment", "ImageFillOrigin", 1024, 1024, 4, 600),
    ("XceptionTextSegment", "ImageFillOrigin", 3508, 2480, 1, None),         # its page-size arm
    ("TextSegament", "ImageFill", 1700, 1200, 1, None),
    ("TextSegament", "ImageFill", 1700, 1200, 1, 600),
)
V2_PAGE = (1700, 1200)        # InferStep(ImageFillOriginV2) runs at this page's U-Net grid


def inference_runs(dev):
    """The eager forward of every TextRemovalStep run of TEXT_REMOVAL_RUNS and of InferStep(ImageFillOriginV2) at the U-Net grid
    of a V2_PAGE page: bf16, no_grad, deterministic weights, fused eval epilogues as the steps run them.  Yields the name of
    each run after it has finished."""
    import torch

    from oracle.detfill import det_fill_state_dict
    from text_segmentation_image_inpainting_b200.engine import InferStep, TextRemovalStep
    from text_segmentation_image_inpainting_b200.models import image_inpainting, text_segmentation
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks

    def det(net):
        net.load_state_dict(det_fill_state_dict(net.state_dict()))
        return net.to(dev).eval()
    nets = {}
    gen = torch.Generator(device=dev).manual_seed(0)
    for seg_name, fill_name, h, w, n, resize in TEXT_REMOVAL_RUNS:
        for mod, name in ((text_segmentation, seg_name), (image_inpainting, fill_name)):
            if name not in nets:
                nets[name] = det(getattr(mod, name)())
        step = TextRemovalStep(nets[seg_name], nets[fill_name], seg_resize=resize)
        step._run_forward(torch.rand((n, 3, h, w), generator=gen, device=dev))
        torch.cuda.synchronize()
        (hs, ws), (hu, wu) = step.padded_sizes(h, w)
        yield f"TextRemovalStep({seg_name}, {fill_name}, seg_resize={resize}) {h}x{w} b{n}: segmentation {hs}x{ws}, U-Net {hu}x{wu}"
        del step
    v2 = det(image_inpainting.ImageFillOriginV2())
    _, (hu, wu) = TextRemovalStep(nets["XceptionTextSegment"], v2).padded_sizes(*V2_PAGE)
    mask = torch.from_numpy(random_hole_masks(1, hu, wu, seed=2)).to(dev)
    InferStep(v2)._run_forward(torch.rand((1, 3, hu, wu), generator=gen, device=dev), mask)
    torch.cuda.synchronize()
    yield f"InferStep(ImageFillOriginV2) {hu}x{wu} b1"


def _tile_case_descs(cases):
    from text_segmentation_image_inpainting_b200 import _lib
    out = []
    for case in cases.values():
        n, h, w, parts, cout, k, s, d = case[:8]
        pad = d * (k - 1) // 2
        c = _lib.Conv()
        c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw = n, h, w, sum(p[0] for p in parts), cout, k, k
        c.stride, c.pad_h, c.pad_w, c.dil, c.groups = s, pad, pad, d, 1
        c.ho, c.wo = (h + 2 * pad - d * (k - 1) - 1) // s + 1, (w + 2 * pad - d * (k - 1) - 1) // s + 1
        c.dtype, c.nparts, c.no_guard = _lib.PCB_BF16, len(parts), int(case[8:] == ("no_guard",))
        for i, (ch, up, masked) in enumerate(parts):
            c.parts[i].c, c.parts[i].x_cstride, c.parts[i].x_up, c.parts[i].mask_up = ch, ch, up, up
            c.parts[i].mask = 1 if masked else None
        out.append(describe(c))
    return out


def record(path):
    import torch

    import gpu_cases as G
    from test_gpu_conv_routes import TILE_CASES
    from oracle.detfill import det_fill_state_dict, det_tensor
    from oracle.inpaint_loss import vgg_state_dict
    from text_segmentation_image_inpainting_b200 import ops
    from text_segmentation_image_inpainting_b200.engine import SegInferStep, SegTrainStep, TrainStep
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss, VggExtractor
    from text_segmentation_image_inpainting_b200.models import image_inpainting, text_segmentation
    from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks

    dev = torch.device("cuda")
    rec = []
    struct = ops.ConvGeom.struct

    def recording_struct(self, xs, force_generic=False):
        c = struct(self, xs, force_generic)
        rec.append(describe(c))
        return c
    ops.ConvGeom.struct = recording_struct
    torch.manual_seed(0)
    for mod, cls, batch, masks in ((image_inpainting, "ImageFillOrigin", 8, True), (text_segmentation, "TextSegament", 8, False),
                                   (text_segmentation, "XceptionTextSegment", 16, False)):
        net = getattr(mod, cls)().to(dev)
        ts = (TrainStep if masks else SegTrainStep)(net, compute_dtype=torch.bfloat16, use_graph=False)
        x = torch.randn(batch, 3, 512, 512, device=dev)
        m = torch.from_numpy(random_hole_masks(batch, 512, 512, seed=0)).to(dev) if masks else None
        ts._fwd_bwd(x, m)
        torch.cuda.synchronize()
        del net, ts
    net = text_segmentation.XceptionTextSegment()
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(dev).eval()
    with torch.no_grad():
        SegInferStep(net)._forward(det_tensor("conv_dispatch.x", (1, 3, 600, 600)).to(dev))
    torch.cuda.synchronize()
    del net
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(vgg_state_dict(0))
    crit = InpaintingLoss(vgg.to(dev))
    clean = torch.rand(8, 3, 512, 512, device=dev)
    mask = torch.from_numpy(random_hole_masks(8, 512, 512, seed=1)).to(dev)
    out = ops.padded_empty(8, 3, 512, 512, torch.bfloat16, dev)
    with torch.no_grad():
        out.copy_(clean.to(torch.bfloat16))
    out.requires_grad_(True)
    crit(clean * mask, mask, out, clean).backward()
    torch.cuda.synchronize()
    for tag in G.CONV_CASES:
        G.conv_case(tag, dev)
    for tag in G.LAZYCAT_CASES:
        G.lazycat_case(tag, dev)
    torch.cuda.synchronize()
    trained = {json.dumps(d, sort_keys=True) for d in rec + _tile_case_descs(TILE_CASES)}
    rec.clear()
    for run in inference_runs(dev):
        print(run)
    ops.ConvGeom.struct = struct
    uniq = {k: json.loads(k) for k in trained}
    for d in rec:
        k = json.dumps(d, sort_keys=True)
        if k not in uniq:
            uniq[k] = dict(d, forward_only=1)
    with open(path, "w") as f:
        json.dump([uniq[k] for k in sorted(uniq)], f)
    print(f"{len(uniq)} distinct descriptors, {sum('forward_only' in d for d in uniq.values())} forward only -> {path}")


def expect(path):
    """append the recorded descriptors the fixture does not hold, with their host queries; the fixture's entries stay as they are"""
    from text_segmentation_image_inpainting_b200 import _lib
    lib = _lib.load()
    with open(path) as f:
        descs = json.load(f)
    with open(FIXTURE) as f:
        cases = json.load(f)["cases"]
    known = {json.dumps(c["conv"], sort_keys=True) for c in cases}
    added = 0
    for d in descs:
        fwd_only = d.pop("forward_only", 0)
        if json.dumps(d, sort_keys=True) in known:
            continue
        cases.append(dict({"conv": d, "expect": host_queries(lib, conv_of(d))}, **({"forward_only": 1} if fwd_only else {})))
        added += 1
    with open(FIXTURE, "w") as f:
        f.write('{"cases": [\n' + ",\n".join(json.dumps(c, sort_keys=True) for c in cases) + "\n]}\n")
    print(f"{added} cases appended, {len(cases)} in all -> {FIXTURE}")


if __name__ == "__main__":
    if sys.argv[1] == "--record":
        record(sys.argv[2])
    else:
        expect(sys.argv[1])

"""Drop-in boundary on the GPU (SURVEY 8b, BASELINE north_star: "the new layers drop into the existing model files unchanged"):
the reference's OWN models/image_inpainting.py and models/text_segmentation.py -- byte-for-byte, imported from the copy build()
staged in oracle/_ref -- run forward + backward on cuda:0 on top of this repo's layer library and must reproduce the goldens that
the same files produced on top of the reference's layer library on CPU (tests/golden/*.npz)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from gpu_cases import BF, F32, ROOT, rel_l2, relerr
from oracle.detfill import det_fill_state_dict, det_tensor
from ref_inject import reference_dir, reference_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if reference_dir() is None:
        pytest.skip("reference not staged (run __graft_entry__.build() in the build container)")
    return torch.device("cuda:0")


def test_staged_reference_is_verbatim():
    """The staged copy must be byte-identical to the reference files the goldens were made from (SHA-256 in tests/golden)."""
    ref = reference_dir()
    if ref is None:
        pytest.skip("reference not staged in oracle/_ref")
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_sha256.json")))
    for f, digest in want.items():
        with open(os.path.join(ref, f), "rb") as fh:
            assert hashlib.sha256(fh.read()).hexdigest() == digest, f


def _run_inpainting(mod, cls_name, dev, dtype, tag=""):
    from text_segmentation_image_inpainting_b200 import ops
    g = np.load(os.path.join(ROOT, "tests", "golden", f"net_{cls_name}{tag}.npz"))
    n, hw, step = int(g["n"]), int(g["hw"]), int(g["step"])
    net = getattr(mod, cls_name)()                                   # the reference's class, built from THIS repo's L1 factories
    net.load_state_dict(det_fill_state_dict(net.state_dict()))
    net = net.to(dev).train()
    plane = np.unpackbits(g["mask_bits"])[: n * hw * hw].reshape(n, 1, hw, hw).astype(np.float32)
    mask = torch.from_numpy(np.repeat(plane, 3, 1))
    x = det_tensor(cls_name + ".x", (n, 3, hw, hw))
    xin = (x * mask).to(dev).to(dtype).contiguous(memory_format=torch.channels_last)
    before = ops.LAZYCAT_MATERIALIZED
    out = net((xin, mask.to(dev)))                                   # the reference's forward(): its own torch.cat / double_upscale
    loss = out.float().abs().mean()
    loss.backward()
    torch.cuda.synchronize()
    errs = {"out": relerr(out[..., ::step, ::step], torch.from_numpy(g["out_sub"])),
            "loss": abs(float(loss.detach()) - float(g["loss"])) / abs(float(g["loss"]))}
    params = dict(net.named_parameters())
    if dtype == F32:
        for k in g.files:
            if k.startswith("g."):
                errs[k] = relerr(params[k[2:]].grad, torch.from_numpy(g[k]))
    return errs, ops.LAZYCAT_MATERIALIZED - before, net


@pytest.mark.parametrize("cls_name", ["ImageFillOrigin", "ImageFillOriginV2", "ImageFill"])
def test_reference_image_inpainting_py_runs_unchanged_fp32(cls_name, dev):
    from text_segmentation_image_inpainting_b200.models import partial_convolution as PC
    with reference_l2("image_inpainting.py") as mod:
        assert os.path.basename(os.path.dirname(os.path.dirname(mod.__reference_file__))) in ("reference", "_ref")
        errs, materialized, net = _run_inpainting(mod, cls_name, dev, F32)
    assert isinstance(net.encoder[0][0], PC.PartialConv)
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    assert errs["out"] <= 1e-3 and errs["loss"] <= 1e-5 and max(errs.values()) <= 2e-3, worst
    # its `torch.cat([x_up, skip], dim=1)` of features and `self.double_upscale(...)` stayed lazy: no upsample / concat pass ran
    assert materialized == 0, materialized


def test_reference_image_inpainting_py_runs_unchanged_bf16_tensor_cores(dev):
    with reference_l2("image_inpainting.py") as mod:
        errs, materialized, _ = _run_inpainting(mod, "ImageFillOrigin", dev, BF)
    assert errs["out"] <= 2e-2 and errs["loss"] <= 2e-3 and materialized == 0, (errs, materialized)


@pytest.mark.parametrize("cls_name,tag", [("TextSegament", ""), ("XceptionTextSegment", ""), ("TextSegament", "_256")])
def test_reference_text_segmentation_py_runs_unchanged_fp32(cls_name, tag, dev):
    g = np.load(os.path.join(ROOT, "tests", "golden", f"segnet_{cls_name}{tag}.npz"))
    n, hw, step = int(g["n"]), int(g["hw"]), int(g["step"])
    with reference_l2("text_segmentation.py") as mod:
        net = getattr(mod, cls_name)()
        net.load_state_dict(det_fill_state_dict(net.state_dict()))
        net = net.to(dev).train()
        x = det_tensor(cls_name + ".x", (n, 3, hw, hw)).to(dev).contiguous(memory_format=torch.channels_last)
        out = net(x)                                                 # the reference's forward(): F.interpolate / torch.cat / AvgPool2d glue
        loss = out.abs().mean()
        loss.backward()
        torch.cuda.synchronize()
    errs = {"out": relerr(out[..., ::step, ::step], torch.from_numpy(g["out_sub"])),
            "loss": abs(float(loss.detach()) - float(g["loss"])) / abs(float(g["loss"]))}
    params = dict(net.named_parameters())
    for k in g.files:
        if k.startswith("g."):
            errs[k] = relerr(params[k[2:]].grad, torch.from_numpy(g[k]))
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:4]
    # forward: the north_star bar.  Gradients: fp32 re-association noise (here also ATen's own avg-pool / bilinear / cat kernels
    # instead of this repo's) amplified through ~70 BatchNorm'd layers of a randomly initialised net -- the late layers agree
    # to 1e-3, the very first convolution to a few percent
    assert errs["out"] <= 1e-3 and errs["loss"] <= 1e-4, worst
    assert all(v <= (8e-2 if "encoder.features.0" in k or "entry_flow_1" in k else 2e-2) for k, v in errs.items()), worst

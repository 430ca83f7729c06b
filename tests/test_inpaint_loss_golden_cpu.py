"""Pins oracle/inpaint_loss.py bit for bit to the reference's own InpaintingLoss (tests/golden/make_golden_inpaint_loss.py):
total loss, the five unweighted terms and d loss / d output.  CPU only."""
import os

import numpy as np
import pytest
import torch

from oracle import inpaint_loss as OL
from oracle import pconv_torch as O

from conftest import GOLDEN

CASES = ("inpaint_loss_b2_64", "inpaint_loss_b1_128", "inpaint_loss_valid_b2_64")


@pytest.fixture(autouse=True, scope="module")
def _golden_thread_count():
    before = torch.get_num_threads()
    torch.set_num_threads(8)       # the goldens were recorded with 8 intra-op threads (oneDNN splits reductions by count)
    yield
    torch.set_num_threads(before)


def load_case(name):
    """(golden dict, clean, mask, output) with the fp32 NCHW tensors the reference consumed."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    g = {k: z[k] for k in z.files}
    n, s, _ = (int(v) for v in g["cfg"])
    hole = np.unpackbits(g["hole"])[:n * s * s].reshape(n, 1, s, s).astype(bool)
    mask = torch.from_numpy(np.repeat(~hole, 3, axis=1).astype(np.float32))
    return g, torch.from_numpy(g["clean"]), mask, torch.from_numpy(g["output"])


def oracle_run(clean, mask, output, sd):
    out = output.clone().requires_grad_(True)
    terms = OL.inpainting_loss_terms(clean * mask, mask, out, clean, sd)
    loss = OL.combine(terms)
    loss.backward()
    return loss.detach(), {k: v.detach() for k, v in terms.items()}, out.grad


@pytest.mark.parametrize("name", CASES)
def test_inpaint_loss_oracle_bit_exact(name):
    g, clean, mask, output = load_case(name)
    sd = OL.vgg_state_dict(int(g["cfg"][2]))
    loss, terms, grad = oracle_run(clean, mask, output, sd)
    assert np.array_equal(loss.numpy(), g["loss"])
    assert [str(t) for t in g["term_names"]] == list(OL.TERMS)
    assert np.array_equal(np.array([float(terms[k]) for k in OL.TERMS], np.float32), g["terms"])
    assert np.array_equal(grad.numpy(), g["grad"])


def test_inpaint_loss_storage_emulation():
    """storage(None) is the exact path; storage(bf16) rounds and lands near the fp32 result (and is not the same)."""
    g, clean, mask, output = load_case("inpaint_loss_b2_64")
    sd = OL.vgg_state_dict(0)
    with O.storage(None):
        loss, _, grad = oracle_run(clean, mask, output, sd)
    assert np.array_equal(loss.numpy(), g["loss"]) and np.array_equal(grad.numpy(), g["grad"])
    with O.storage(torch.bfloat16):
        lb, _, gb = oracle_run(clean, mask, output, sd)
    assert not torch.equal(gb, grad)
    assert abs(float(lb) - float(loss)) <= 1e-2 * abs(float(loss))
    assert float((gb - grad).norm() / grad.norm()) < 5e-2


def test_vgg_state_dict_keys_match_torchvision():
    """The seeded weights use VggExtractor's keys and shapes (vgg16.features[:17] split into three stages)."""
    torchvision = pytest.importorskip("torchvision")
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        vgg = torchvision.models.vgg16(weights=None)
    feats = [torch.nn.Sequential(*vgg.features[a:b]) for a, b in ((0, 5), (5, 10), (10, 17))]
    ref = {f"features.{i}.{k}": v for i, f in enumerate(feats) for k, v in f.state_dict().items()}
    sd = OL.vgg_state_dict(0)
    assert sorted(sd) == sorted(ref)
    assert all(sd[k].shape == ref[k].shape for k in ref)
    assert all(float(sd[k].abs().min()) > 0 for k in sd if k.endswith("bias"))

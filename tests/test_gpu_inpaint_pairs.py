"""The raw/clean pair path on the device (csrc/inpaint_data.cu for pair sources, data.InpaintPairBatcher) and held-out
evaluation (engine.InpaintEvalStep): bit-exact against the reference's recorded `TestDataset.process_images` without strokes and
against the numpy restatement with them, the pair sampler against the mask-file sampler, graph replays and validation, the
training steps on pairs, and the evaluation step against eager evaluation, interleaved with training and across passes."""
import ctypes
import os

import numpy as np
import pytest
import torch

import inpaint_pair_ref as P
from conftest import GOLDEN
from oracle import inpaint_data as OI
from oracle import inpaint_loss as OL
from test_gpu_inpaint_data import _small_net

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN, "inpaint_pairs.npz"))
STROKE_FREE = [k for k, c in enumerate(G["cases"]) if not c[4]]
STROKED = [k for k, c in enumerate(G["cases"]) if c[4]]


def _batcher(*a, **k):
    from text_segmentation_image_inpainting_b200.data import InpaintPairBatcher
    return InpaintPairBatcher(*a, **k)


def _case(k):
    seed, H, W, size, strokes = (int(v) for v in G["cases"][k])
    raw, clean = P.pair(seed, H, W)
    hole = np.unpackbits(G[f"hole{k}"])[:size * size].reshape(size, size).astype(bool)
    return raw, clean, size, bool(strokes), G[f"params{k}"], G[f"clean_sha256_{k}"], hole


def _clean_u8(c):
    """fp32 [3, s, s] device clean image -> uint8 CHW, checking that it is exactly ToTensor's u8 / 255.f."""
    u8 = torch.round(c.cpu() * 255).to(torch.uint8)
    assert torch.equal(u8.float() / 255, c.cpu())
    return u8.numpy()


def _prepare_one(raw, clean, size, strokes, params, dtype):
    b = _batcher(1, raw.shape[:2], image_size=size, add_random_masks=strokes, compute_dtype=dtype)
    b.stage([(raw, clean)])
    x, hm, c = b.prepare(params[None])
    torch.cuda.synchronize()
    return b, x, hm, c


def _pairs(sizes, seed):
    return [P.pair(seed + i, h, w) for i, (h, w) in enumerate(sizes)]


def _vgg():
    from text_segmentation_image_inpainting_b200.loss import VggExtractor
    vgg = VggExtractor(pretrained=False)
    vgg.load_state_dict(OL.vgg_state_dict(0))
    return vgg.cuda()


# ------------------------------------------------------------------------------------------------ the batch
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", STROKE_FREE)
def test_stroke_free_cases_are_bit_exact_against_the_reference(k, dtype):
    raw, clean, size, strokes, p, clean_sha, hole = _case(k)
    b, x, hm, c = _prepare_one(raw, clean, size, strokes, p, dtype)
    got = _clean_u8(c[0])
    np.testing.assert_array_equal(P.digest(got), clean_sha)                 # the reference's clean image, byte for byte
    ref_clean = torch.from_numpy(got).float() / 255
    binary = 1 - torch.from_numpy(hole).float() * 255 / 255
    assert torch.equal(c[0].cpu(), ref_clean)
    assert torch.equal(b.plane[0].cpu(), torch.from_numpy(~hole).to(torch.uint8))
    assert torch.equal(hm.dense()[0].cpu(), binary.expand(3, -1, -1))
    assert torch.equal(x[0].cpu(), (ref_clean * binary).to(dtype))
    assert not bool(b._xbuf[:, 3:].any())


def test_stroke_cases_match_the_restatement_exactly_and_pillow_within_two_percent():
    diff = holes = 0
    for k in STROKED:
        raw, clean, size, strokes, p, clean_sha, hole = _case(k)
        b, x, hm, c = _prepare_one(raw, clean, size, strokes, p, torch.bfloat16)
        rule_clean, rule_hole = P.process_pair(raw, clean, p, size, strokes=True)
        got_hole = b.plane[0].cpu().numpy() == 0
        np.testing.assert_array_equal(got_hole, rule_hole)
        assert torch.equal(c[0].cpu(), torch.from_numpy(rule_clean).permute(2, 0, 1).float() / 255)
        np.testing.assert_array_equal(P.digest(_clean_u8(c[0])), clean_sha)
        diff, holes = diff + int((got_hole != hole).sum()), holes + int(hole.sum())
    assert diff <= 0.02 * holes, (diff, holes)            # over the cases together, as the rule's bound is stated


def test_pair_path_with_identical_pages_is_the_mask_file_path_with_an_empty_mask():
    from text_segmentation_image_inpainting_b200.data import InpaintBatcher
    sizes, size = [(300, 420), (700, 380)], 256
    pages = [P.R.sources(60 + i, h, w)[0] for i, (h, w) in enumerate(sizes)]
    params = OI.sample(8, 2, sizes, size)
    params[:, 4] = 0
    a = _batcher(2, (700, 420), image_size=size, add_random_masks=True)
    a.stage([(pg, pg) for pg in pages])
    a.prepare(params)
    m = InpaintBatcher(2, (700, 420), image_size=size, add_random_masks=True)
    m.stage([(pg, np.zeros(pg.shape[:2], np.uint8)) for pg in pages])
    m.prepare(params)
    torch.cuda.synchronize()
    assert torch.equal(a.plane, m.plane) and torch.equal(a.clean, m.clean) and torch.equal(a._xbuf, m._xbuf)


# ------------------------------------------------------------------------------------------------ sampler, replays, validation
def _device_draws(entry, seed, counter, sizes, out, strokes=True):
    from text_segmentation_image_inpainting_b200 import _lib
    n = len(sizes)
    table = np.zeros(n, dtype=[("a", "<u8"), ("b", "<u8"), ("h", "<i4"), ("w", "<i4"), ("sa", "<i4"), ("sb", "<i4")])
    table["a"] = table["b"] = 1
    table["h"], table["w"] = [s[0] for s in sizes], [s[1] for s in sizes]
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    rng = torch.tensor([seed, counter], dtype=torch.int64, device="cuda")
    params = torch.empty((n, OI.PARAM_INTS), dtype=torch.int32, device="cuda")
    _lib.check(getattr(_lib.load(), entry)(tab.data_ptr(), n, out, int(strokes), rng.data_ptr(), params.data_ptr(),
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert int(rng[1]) == counter + 1
    return params.cpu().numpy()


def test_pair_sampler_draws_the_mask_file_boxes_and_strokes_without_grayscale():
    rng = np.random.default_rng(1)
    sizes = [(int(h), int(w)) for h, w in rng.integers(40, 2000, (300, 2))] + [(100, 900), (900, 100)]
    for seed, counter, out, strokes in ((0, 0, 512, True), (123456789012, 7, 256, True), (5, 2 ** 33 + 1, 128, False)):
        pair = _device_draws("pcb_inpaint_pair_sample", seed, counter, sizes, out, strokes)
        mask_file = _device_draws("pcb_inpaint_sample", seed, counter, sizes, out, strokes)
        assert not pair[:, 4].any() and mask_file[:, 4].any()
        ref = OI.sample(seed, counter, sizes, out, strokes)
        ref[:, 4] = 0
        np.testing.assert_array_equal(pair, ref)
        mask_file[:, 4] = 0
        np.testing.assert_array_equal(pair, mask_file)


def test_graph_replays_draw_fresh_batches_take_new_sizes_and_reject_bad_input():
    from text_segmentation_image_inpainting_b200._lib import PcbError
    from text_segmentation_image_inpainting_b200.engine import InpaintTrainStep
    seed, size = 17, 256
    sizes_a, sizes_b = [(300, 420), (512, 380)], [(260, 261), (400, 512)]
    b = _batcher(2, (512, 512), image_size=size, add_random_masks=True, seed=seed)
    src_a, src_b = _pairs(sizes_a, 20), _pairs(sizes_b, 30)
    b.stage(src_a)
    ts = InpaintTrainStep(_small_net().cuda(), b, lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    counter = int(b.rng[1])
    seen = []
    for step, (sizes, src) in enumerate([(sizes_a, src_a), (sizes_b, src_b), (sizes_a, src_a)]):
        b.stage(src)
        assert np.isfinite(float(ts.step()))
        p = b.params.cpu().numpy()
        ref = OI.sample(seed, counter + step, sizes, size)
        ref[:, 4] = 0
        np.testing.assert_array_equal(p, ref)
        clean_u8, hole = P.process_pair(*src[1], p[1], size)
        assert torch.equal(b.clean[1].cpu(), torch.from_numpy(clean_u8).permute(2, 0, 1).float() / 255)
        np.testing.assert_array_equal(b.plane[1].cpu().numpy() == 0, hole)
        seen.append(b.plane.clone())
    assert not torch.equal(seen[0], seen[2])
    raw, clean = src_a[0]
    with pytest.raises(ValueError):
        b.stage([(raw, clean[:-1]), src_a[1]])                                  # unequal sizes
    with pytest.raises(ValueError):
        b.stage([(raw.astype(np.int16), clean), src_a[1]])                      # not uint8
    with pytest.raises(ValueError):
        b.stage([(raw[..., 0], clean[..., 0]), src_a[1]])                       # not RGB
    eager = _batcher(2, (512, 512), image_size=size)
    eager.stage(src_a)
    bad = OI.sample(1, 0, sizes_a, size)
    bad[:, 4] = 1
    with pytest.raises(PcbError, match="grayscale"):
        eager.prepare(bad)
    from text_segmentation_image_inpainting_b200 import _lib
    table = eager._host_table.copy()
    table["sb"][0] = 3 * table["w"][0] - 1
    assert _lib.load().pcb_inpaint_pair_validate(table.ctypes.data, None, 2, 2, 512, 512, size) != 0
    assert b"strides" in _lib.load().pcb_last_error()


# ------------------------------------------------------------------------------------------------ training on pairs
@pytest.mark.parametrize("with_loss", [False, True])
def test_training_steps_on_pairs_replay_equals_eager(with_loss):
    from text_segmentation_image_inpainting_b200.engine import InpaintLossTrainStep, InpaintTrainStep
    seed = 5
    b = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=seed)
    b.stage(_pairs([(300, 420), (512, 380)], 40))
    kw = dict(lr=0.0, momentum=0.0, weight_decay=0.0, nesterov=False)

    def make(use_graph):
        if with_loss:
            return InpaintLossTrainStep(_small_net().cuda(), b, _vgg(), use_graph=use_graph, **kw)
        return InpaintTrainStep(_small_net().cuda(), b, use_graph=use_graph, **kw)
    ts = make(True)
    ts.warmup_and_capture(eager_warmup=2)
    counter = int(b.rng[1])
    loss = float(ts.step())
    terms = ts.last_terms.clone() if with_loss else None
    plane = b.plane.clone()
    torch.cuda.synchronize()
    b.reseed(seed, counter)                                   # the eager step draws what the replay drew
    eager = make(False)
    le = float(eager.step())
    torch.cuda.synchronize()
    assert torch.equal(b.plane, plane)
    assert np.isfinite(loss) and abs(loss - le) <= 1e-5 * abs(le), (loss, le)
    if with_loss:
        assert torch.allclose(terms, eager.last_terms, rtol=1e-5, atol=0)


# ------------------------------------------------------------------------------------------------ evaluation
def _eager_eval(net, b, crit):
    """prepare + eval-mode forward with the fused epilogues + InpaintingLoss, eagerly under no_grad."""
    from text_segmentation_image_inpainting_b200 import ops
    training = net.training
    net.eval()
    try:
        with ops.StepScope(b.device, training=False), torch.no_grad():
            xin, hm, clean = b.prepare()
            out = net((xin, hm))
            loss = crit(clean, hm, out, clean) if crit is not None else None
    finally:
        net.train(training)
    torch.cuda.synchronize()
    return out.float(), loss, (crit.last_terms.clone() if crit is not None else None)


@pytest.mark.parametrize("with_loss", [False, True])
def test_eval_step_matches_eager_evaluation(with_loss):
    from text_segmentation_image_inpainting_b200.engine import InpaintEvalStep
    from text_segmentation_image_inpainting_b200.loss import InpaintingLoss
    seed = 9
    b = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=seed)
    b.stage(_pairs([(300, 420), (512, 380)], 50))
    net = _small_net().cuda()
    vgg = _vgg() if with_loss else None
    ev = InpaintEvalStep(net, b, vgg)
    assert net.training
    ev.warmup_and_capture()
    assert int(b.rng[1]) == 0 and net.training
    out = ev.run().clone()
    loss, terms = (ev.last_loss.clone(), ev.last_terms.clone()) if with_loss else (None, None)
    torch.cuda.synchronize()
    assert net.training and ev.fused_sites > 0
    b.reseed(seed)
    e_out, e_loss, e_terms = _eager_eval(net, b, InpaintingLoss(vgg) if with_loss else None)
    assert torch.equal(out, e_out)
    if with_loss:
        # the loss sums are fp64 atomics: their order may differ in the last bits
        assert torch.allclose(loss, e_loss, rtol=1e-6, atol=0) and torch.allclose(terms, e_terms, rtol=1e-6, atol=0)
        assert float(terms[3]) > 0 and float(terms[4]) > 0


def test_eval_step_fp32_against_the_oracle():
    from oracle import pconv_torch as O
    from text_segmentation_image_inpainting_b200.engine import InpaintEvalStep
    b = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=4, compute_dtype=torch.float32)
    b.stage(_pairs([(300, 200), (256, 380)], 70))
    net = _small_net().cuda()
    ev = InpaintEvalStep(net, b, _vgg(), compute_dtype=torch.float32)
    out = ev.run().clone()
    loss, terms = float(ev.last_loss), ev.last_terms.cpu().double()
    clean, mask = b.clean.cpu(), b.plane.cpu().float()[:, None].expand(-1, 3, -1, -1).contiguous()
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    with torch.no_grad():
        ref = O.image_fill_origin(O.clone_state_dict(sd), clean * mask, mask, training=False)
        ref_terms = OL.inpainting_loss_terms(clean, mask, ref, clean, OL.vgg_state_dict(0))
    rel = float((out.cpu() - ref).norm() / ref.norm())
    assert rel <= 2e-2, rel
    ref_loss = float(OL.combine(ref_terms))
    ref_terms = torch.tensor([float(ref_terms[t]) for t in OL.TERMS], dtype=torch.float64)
    assert torch.allclose(terms, ref_terms, rtol=2e-2, atol=1e-6), (terms, ref_terms)
    assert abs(loss - ref_loss) <= 2e-2 * abs(ref_loss), (loss, ref_loss)


def _state(ts):
    net = ts.net
    return [ts.flat.flat_p.clone(), ts.flat.flat_m.clone()] + [t.clone() for t in net.buffers()]


def _operand_bits(ts):
    """The bytes of the training graph's captured operand buffers (compared as bytes, so that NaN patterns compare equal)."""
    return [t.view(torch.uint8).clone() for v in ts._captured_operands if v is not None for t in v if t is not None]


def test_eval_interleaved_with_training_changes_nothing_and_sees_every_update():
    from text_segmentation_image_inpainting_b200.engine import InpaintEvalStep, InpaintTrainStep
    tb = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=1)
    train_src = _pairs([(300, 420), (512, 380)], 80)
    tb.stage(train_src)
    ts = InpaintTrainStep(_small_net().cuda(), tb, lr=1e-3, use_graph=True)
    ts.warmup_and_capture(eager_warmup=2)
    captured = _operand_bits(ts)
    eb = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=2)
    eval_src = _pairs([(400, 300), (350, 500)], 90)
    eb.stage(eval_src)
    ev = InpaintEvalStep(ts.net, eb, _vgg())
    ev.warmup_and_capture()
    outs = []
    for k in range(3):
        tb.stage(train_src)
        ts.step()
        torch.cuda.synchronize()
        before = _state(ts)
        ops_before = _operand_bits(ts)
        for _ in range(2):                                      # a pass of two batches: one refresh
            eb.reseed(2)
            eb.stage(eval_src)
            outs.append((ev.run().clone(), ev.last_loss.clone()))
        torch.cuda.synchronize()
        assert ts.net.training
        # nothing the training graph reads changed: parameters, momentum, running statistics, its captured operand buffers
        for a, c in zip(before, _state(ts)):
            assert torch.equal(a, c)
        for a, c in zip(ops_before, _operand_bits(ts)):
            assert torch.equal(a, c)
        assert torch.equal(outs[-1][0], outs[-2][0])            # reseeded passes repeat
        # a fresh evaluation step on a copy of the state at this point
        copy = _small_net().cuda()
        copy.load_state_dict(ts.net.state_dict())
        eb2 = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=2)
        eb2.stage(eval_src)
        fresh = InpaintEvalStep(copy, eb2, _vgg())
        fresh.warmup_and_capture()
        assert torch.equal(fresh.run(), outs[-1][0])
        assert torch.allclose(fresh.last_loss, outs[-1][1], rtol=1e-6, atol=0)
    assert not torch.equal(outs[0][0], outs[-1][0])             # the evaluations followed the updates
    assert len(captured) > 0


def test_reseeded_validation_passes_are_identical():
    from text_segmentation_image_inpainting_b200.engine import InpaintEvalStep
    sizes = [[(300, 420), (512, 380)], [(260, 261), (400, 512)], [(512, 512), (333, 444)]]
    sources = [_pairs(s, 100 + 10 * i) for i, s in enumerate(sizes)]
    b = _batcher(2, (512, 512), image_size=256, add_random_masks=True, seed=3)
    b.stage(sources[0])
    ev = InpaintEvalStep(_small_net().cuda(), b, _vgg())
    ev.warmup_and_capture()
    passes = []
    for _ in range(2):
        b.reseed(3)
        outs = []
        for src in sources:
            b.stage(src)
            outs.append((ev.run().clone(), b.plane.clone(), ev.last_terms.clone()))
        torch.cuda.synchronize()
        passes.append(outs)
    for (o1, p1, t1), (o2, p2, t2) in zip(*passes):
        assert torch.equal(o1, o2) and torch.equal(p1, p2) and torch.allclose(t1, t2, rtol=1e-6, atol=0)
    assert not torch.equal(passes[0][0][1], passes[0][2][1])

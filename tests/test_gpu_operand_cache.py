"""GPU tests of the operand cache (ops.OperandCache): when it hands back the operands it holds, when it rewrites them in place,
when it lays out new ones, what a frozen cache ignores, the prefetch stream's refresh and the refresh of a pinned record.

One 64 -> 64 3x3 bf16 convolution on the tensor-core kernels.  "Fresh" operands are a new ops.Operands of the same weight and
problem; buffers are compared as bytes."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _mods():
    from text_segmentation_image_inpainting_b200 import _lib, ops
    return _lib, ops


def _problem(seed=0):
    _, ops = _mods()
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = ops.padded_empty(2, 64, 16, 16, torch.bfloat16, DEV)
    geom = ops.ConvGeom([x], [0], 64, 3, 1, 1, 1, 1, False, False, [(None, 64, 0)], plain=True)
    w = torch.randn(64, 64, 3, 3, generator=g, device=DEV).contiguous(memory_format=torch.channels_last)
    return geom, w


def _bits(rec):
    return [t.view(torch.uint8).clone() for t in (rec.w_fwd, rec.w_dg) if t is not None]


def _fresh_bits(w, geom):
    _, ops = _mods()
    return _bits(ops.Operands(w, geom))


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _update_behind_version(w, seed):
    """Change the weight's values the way a raw-pointer optimiser step does: its version counter stays as it was."""
    v = w._version
    w.data.copy_(torch.randn(w.shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV))
    assert w._version == v


@pytest.fixture
def inplace():
    """a training scope: in-place operand refresh and prefetch_weights are on"""
    _, ops = _mods()
    with ops.StepScope(DEV, training=True):
        yield


def test_hit_returns_the_same_buffers_and_launches_nothing():
    _lib, ops = _mods()
    geom, w = _problem()
    cache = ops.OperandCache()
    before = _lib.launch_count()
    rec = cache.get(w, geom)
    assert _lib.launch_count() > before                   # the miss laid the weight out
    before = _lib.launch_count()
    again = cache.get(w, geom)
    assert _lib.launch_count() == before
    assert again is rec and again.w_fwd.data_ptr() == rec.w_fwd.data_ptr()
    torch.cuda.synchronize()
    assert _same(_bits(rec), _fresh_bits(w, geom))


def test_epoch_bump_with_inplace_refresh_rewrites_the_same_storage(inplace):
    _, ops = _mods()
    geom, w = _problem()
    cache = ops.OperandCache()
    rec = cache.get(w, geom)
    ptrs = [t.data_ptr() for t in (rec.w_fwd, rec.w_dg) if t is not None]
    _update_behind_version(w, 1)
    ops.bump_weight_epoch()
    new = cache.get(w, geom)
    assert new is rec and [t.data_ptr() for t in (new.w_fwd, new.w_dg) if t is not None] == ptrs
    torch.cuda.synchronize()
    assert _same(_bits(new), _fresh_bits(w, geom))


def test_epoch_bump_without_inplace_refresh_lays_out_new_buffers_and_spares_a_pinned_record():
    _, ops = _mods()
    geom, w = _problem()
    cache = ops.OperandCache()
    pinned = cache.get(w, geom)
    torch.cuda.synchronize()
    old = _bits(pinned)
    _update_behind_version(w, 2)
    ops.bump_weight_epoch()
    new = cache.get(w, geom)
    assert new is not pinned and cache.current is new
    assert new.w_fwd.data_ptr() != pinned.w_fwd.data_ptr()
    torch.cuda.synchronize()
    assert _same(_bits(pinned), old)
    assert _same(_bits(new), _fresh_bits(w, geom))
    assert not _same(_bits(new), old)


def test_frozen_cache_ignores_the_epoch_and_follows_the_weight():
    _lib, ops = _mods()
    geom, w = _problem()
    cache = ops.OperandCache(frozen=True)
    rec = cache.get(w, geom)
    ops.bump_weight_epoch()
    before = _lib.launch_count()
    assert cache.get(w, geom) is rec
    assert _lib.launch_count() == before
    with torch.no_grad():
        w.add_(1.0)
    new = cache.get(w, geom)
    assert new is not rec
    torch.cuda.synchronize()
    assert _same(_bits(new), _fresh_bits(w, geom))


def test_prefetch_refreshes_ahead_and_the_lookup_waits_for_it(inplace):
    _, ops = _mods()
    geom, w = _problem()
    cache, frozen = ops.OperandCache(), ops.OperandCache(frozen=True)
    rec = cache.get(w, geom)
    frozen_rec = frozen.get(w, geom)
    _update_behind_version(w, 3)
    ops.bump_weight_epoch()
    ops.prefetch_weights([cache, frozen, ops.OperandCache()])
    assert cache.ready is not None
    assert frozen.ready is None and frozen.current is frozen_rec          # frozen caches are not prefetched
    got = cache.get(w, geom)
    assert got is rec and cache.ready is None
    torch.cuda.synchronize()
    assert _same(_bits(got), _fresh_bits(w, geom))


def test_refreshed_pinned_record_marked_current_makes_the_next_lookup_hit():
    _lib, ops = _mods()
    geom, w = _problem()
    cache = ops.OperandCache()
    rec = cache.get(w, geom)
    _update_behind_version(w, 4)
    ops.bump_weight_epoch()
    cache.refresh(rec)
    before = _lib.launch_count()
    assert cache.get(w, geom) is rec
    assert _lib.launch_count() == before
    torch.cuda.synchronize()
    assert _same(_bits(rec), _fresh_bits(w, geom))

"""GPU tests of ops.StepScope, the execution mode of one engine step: scopes do not nest, and leaving one (on an exception
too) restores the behaviour outside any scope -- the two-pass eval path and fresh zero buffers."""
import pytest
import torch
from torch import nn

from gpu_cases import blob
from test_gpu_inference import _feature, _randomise_bn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _ops():
    from text_segmentation_image_inpainting_b200 import ops
    return ops


def test_nesting_is_refused():
    ops = _ops()
    outer = ops.StepScope(DEV, training=True)
    with outer:
        for inner in (ops.StepScope(DEV, training=False), outer):
            with pytest.raises(ops._lib.PcbError, match="already current"):
                with inner:
                    pass
            assert ops.current_scope() is outer
    assert ops.current_scope() is None


def _eval_block():
    from text_segmentation_image_inpainting_b200.masks import HoleMask
    from text_segmentation_image_inpainting_b200.models.partial_convolution import partial_convolution_block
    torch.manual_seed(7)
    block = partial_convolution_block(64, 64, 3, 1, 1, 1, BN=True, activation=nn.LeakyReLU(0.2))
    _randomise_bn(block, 3)
    block = block.to(DEV).eval()
    hm = HoleMask.from_dense(blob(2, 1, 8, 128, 5).expand(2, 64, 8, 128).contiguous().to(DEV), channel_uniform=True)
    return block, (_feature(2, 64, 8, 128, 1), hm)


def _affine_act_calls(monkeypatch):
    """counts of the fused-epilogue forward launches"""
    from text_segmentation_image_inpainting_b200 import _lib
    lib, calls = _lib.load(), []
    fused = lib.pcb_pconv_forward_affine_act
    monkeypatch.setattr(lib, "pcb_pconv_forward_affine_act", lambda *a: calls.append(1) or fused(*a))
    return calls


def test_after_an_exception_an_eval_forward_runs_the_two_pass_path(monkeypatch):
    ops = _ops()
    block, args = _eval_block()
    bn, act = block[1].bn_act[0], block[1].bn_act[1]
    calls = _affine_act_calls(monkeypatch)
    scope = ops.StepScope(DEV, training=False)
    with torch.no_grad():
        with scope:                                       # positive control: inside the scope the epilogue is fused
            block(args)
        assert scope.fused_sites == 1 and len(calls) == 1
        with pytest.raises(RuntimeError, match="inside the scope"):
            with scope:
                raise RuntimeError("inside the scope")
        assert ops.current_scope() is None
        assert ops.eval_epilogue(bn, act) is None
        block(args)
    torch.cuda.synchronize()
    assert len(calls) == 1 and scope.fused_sites == 0


def test_after_an_exception_zeros_f64_returns_fresh_zeros():
    ops = _ops()
    scope = ops.StepScope(DEV, training=True)
    arena = scope._arena.data_ptr()
    with pytest.raises(RuntimeError, match="inside the scope"):
        with scope:
            z = ops.zeros_f64(64, DEV)                    # positive control: a slice of the scope's arena
            assert z.untyped_storage().data_ptr() == arena
            raise RuntimeError("inside the scope")
    z = ops.zeros_f64(64, DEV)
    assert z.untyped_storage().data_ptr() != arena
    assert z.dtype == torch.float64 and z.shape == (64,) and not bool(z.any())

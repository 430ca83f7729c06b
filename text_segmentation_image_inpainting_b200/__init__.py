"""text_segmentation_image_inpainting_b200 -- H100-native (sm_90a) partial-convolution hot path.

Drop-in for the layer library of yu45020/Text_Segmentation_Image_Inpainting (models/partial_convolution.py,
the blocks of models/MobileNetV2.py / models/BaseModels.py that its networks are built from): same module
names, constructor signatures, ``forward((x, mask)) -> (y, new_mask)`` convention and ``state_dict()`` keys,
backed by hand-written CUDA (wgmma / TMA implicit-GEMM + vectorised HBM-bound kernels) behind the
C ABI in ``include/pconv_b200.h``.  No CPU path: ops raise on non-CUDA tensors.
"""
from . import _lib  # noqa: F401
from .masks import HoleMask  # noqa: F401

__all__ = ["HoleMask", "build_extension", "load_extension"]


def build_extension(force=False, verbose=False):
    from . import build as _b
    return _b.build(force=force, verbose=verbose)


def load_extension():
    return _lib.load()

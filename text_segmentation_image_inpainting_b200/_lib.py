"""ctypes binding of libpconv_b200.so (C ABI: include/pconv_b200.h).

The product path has NO fallback: if the shared library is missing (and cannot be built because nvcc is
absent) importing an op raises; calling an op with non-CUDA tensors raises."""
import ctypes
import os
import threading

from . import build as _build

PCB_F32, PCB_BF16 = 0, 1
ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_RELU6 = 0, 1, 2, 3
MAX_PARTS = 8
SEG_FOCAL, SEG_BOOTSTRAP = 0, 1
SEG_NONE, SEG_MEAN, SEG_SUM = 0, 1, 2
CLR_TRIANGULAR, CLR_TRIANGULAR2, CLR_EXP_RANGE = 0, 1, 2
# PCB_ROUTE_* of pcb_debug_conv_routes, by code
ROUTES = ("none", "generic", "depthwise", "stem", "k2r", "smallco", "tma", "tma_s2", "gather")

c_int, c_ll, c_float, c_void_p, c_size_t = ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t


class Part(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("mask", c_void_p), ("c", ctypes.c_int32), ("x_cstride", ctypes.c_int32),
                ("x_up", ctypes.c_int32), ("mask_up", ctypes.c_int32)]


class Conv(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in
                ("n", "h", "w", "cin", "cout", "kh", "kw", "stride", "pad_h", "pad_w", "dil", "groups", "ho", "wo",
                 "dtype", "same_holes", "no_guard", "plain", "force_generic", "nparts")] + [("parts", Part * MAX_PARTS)]


_SIGS = {
    "pcb_last_error": (ctypes.c_char_p, []),
    "pcb_version": (c_int, []),
    "pcb_launch_count": (ctypes.c_ulonglong, []),
    "pcb_conv_uses_tensor_cores": (c_int, [ctypes.POINTER(Conv)]),
    "pcb_conv_dgrad_at_source_resolution": (c_int, [ctypes.POINTER(Conv)]),
    "pcb_pconv_workspace": (c_size_t, [ctypes.POINTER(Conv)]),
    "pcb_conv_weight_layout": (None, [ctypes.POINTER(Conv), ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t)]),
    "pcb_conv_weight_prepare": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_conv_weight_refresh": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_pconv_forward": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_pconv_forward_premasked": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_conv_fuses_bn_stats": (c_int, [ctypes.POINTER(Conv)]),
    "pcb_pconv_forward_bn": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "pcb_conv_fuses_affine_act": (c_int, [ctypes.POINTER(Conv)]),
    "pcb_pconv_forward_affine_act": (c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                             c_void_p, c_void_p, c_int, c_float, c_void_p]),
    "pcb_seg_mask_postprocess": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_pconv_mask_pass":(c_int, [ctypes.POINTER(Conv), c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_pconv_renorm_backward": (c_int, [ctypes.POINTER(Conv), c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "pcb_pconv_backward_data": (c_int, [ctypes.POINTER(Conv), c_void_p, c_int, c_void_p, c_void_p, ctypes.POINTER(c_void_p),
                                        ctypes.POINTER(ctypes.c_int32), c_void_p]),
    "pcb_pconv_backward_weight": (c_int, [ctypes.POINTER(Conv), c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_pconv_backward_weight_acc": (c_int, [ctypes.POINTER(Conv), c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_debug_pipeline_status": (c_int, [ctypes.POINTER(c_int)]),
    "pcb_debug_conv_routes": (c_int, [ctypes.POINTER(Conv), ctypes.POINTER(ctypes.c_int32)]),
    "pcb_mask_planes_from_dense": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_mask_plane_to_dense": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pcb_bn_stats": (c_int, [c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_stats_acc": (c_int, [c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p]),
    "pcb_bn_forward_fused": (c_int, [c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_float, c_float, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_act_backward_reduce_acc": (c_int, [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_int, c_float, c_void_p, c_void_p]),
    "pcb_bn_act_backward_small": (c_int, [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_finalize": (c_int, [c_void_p, c_void_p, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_act_forward": (c_int, [c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_act_backward_reduce": (c_int, [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_act_backward_apply": (c_int, [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_int, c_float, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_bn_act_backward_apply_renorm": (c_int, [c_void_p, c_void_p, c_int, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                 c_int, c_float, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_upsample2x_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_upsample2x_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_concat_forward": (c_int, [ctypes.POINTER(Part), c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_concat_backward": (c_int, [c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int32), c_int, c_int,
                                    c_int, c_int, c_int, ctypes.POINTER(c_void_p), c_void_p]),
    "pcb_avgpool_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_avgpool_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_bilinear_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_bilinear_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_gap_forward": (c_int, [c_void_p, c_int, c_int, c_ll, c_int, c_void_p, c_void_p]),
    "pcb_gap_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_ll, c_int, c_int, c_void_p]),
    "pcb_scse_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_ll, c_int, c_void_p]),
    "pcb_scse_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_ll,
                                  c_int, c_void_p]),
    "pcb_inpaint_validate": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "pcb_inpaint_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_inpaint_prepare": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                    c_void_p]),
    "pcb_inpaint_pair_validate": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "pcb_inpaint_pair_sample": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_inpaint_pair_prepare": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                         c_void_p, c_void_p]),
    "pcb_page_resize_workspace": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "pcb_page_resize_bicubic": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_removal_seg_input": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]),
    "pcb_removal_holes": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "pcb_removal_composite": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_seg_validate": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "pcb_seg_sample": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_seg_prepare": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                c_void_p, c_void_p]),
    "pcb_seg_loss_partials": (c_int, [c_ll]),
    "pcb_seg_loss_forward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_float,
                                     c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_seg_loss_backward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_float,
                                      c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_seg_score_update": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "pcb_seg_score_finalize": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_inpaint_loss_pixel_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                               c_int, c_void_p, c_void_p]),
    "pcb_inpaint_loss_pixel_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                                c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_maxpool2x2_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_maxpool2x2_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pcb_feature_l1_forward": (c_int, [c_void_p, c_int, c_int, c_ll, c_int, c_void_p, c_void_p]),
    "pcb_feature_loss_backward": (c_int, [c_void_p, c_int, c_int, c_ll, c_int, c_void_p, c_void_p, c_float, c_float, c_void_p, c_void_p,
                                          c_void_p]),
    "pcb_gram_l1_forward": (c_int, [c_void_p, c_int, c_int, c_float, c_void_p, c_void_p]),
    "pcb_gram_sign_sym": (c_int, [c_void_p, c_int, c_int, c_float, c_void_p, c_void_p]),
    "pcb_inpaint_loss_finalize": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pcb_k2r_image_weight": (c_int, [c_void_p, c_int, c_void_p, c_void_p]),
    "pcb_k2r_image_dgrad": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pcb_conv_dgrad_fuses_relu": (c_int, [ctypes.POINTER(Conv)]),
    "pcb_pconv_backward_data_relu": (c_int, [ctypes.POINTER(Conv), c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p]),
    "pcb_l1_mean_forward": (c_int, [c_void_p, c_int, c_ll, c_void_p, c_void_p, c_void_p]),
    "pcb_l1_mean_backward": (c_int, [c_void_p, c_int, c_ll, c_float, c_void_p, c_void_p]),
    "pcb_sgd_step": (c_int, [c_void_p, c_void_p, c_void_p, c_ll, c_float, c_float, c_float, c_int, c_int, c_void_p]),
    "pcb_sgd_step_scaled": (c_int, [c_void_p, c_void_p, c_void_p, c_ll, c_float, c_float, c_float, c_int, c_int, c_float, c_void_p]),
    "pcb_sgd_step_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_float, c_float, c_int, c_float, c_void_p]),
    "pcb_lr_cyclic": (c_int, [c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_double, c_int, ctypes.c_double, c_void_p, c_void_p,
                              c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGS)

_lib = None
_lock = threading.Lock()


class PcbError(RuntimeError):
    pass


def lib_path():
    return _build.LIB


def load():
    """Load (building in-tree first if sources are newer and nvcc exists) the shared library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = _build.LIB
        # stale or missing library -> rebuild (content fingerprint, file-locked: safe under torchrun); raises if nvcc is
        # missing: no silent fallback, and never a silently stale .so
        if os.environ.get("PCB_REBUILD") == "1":
            path = _build.build(force=True)
        elif _build.needs_build():
            path = _build.build()
        lib = ctypes.CDLL(path)
        for name, (res, args) in _SIGS.items():
            fn = getattr(lib, name)    # AttributeError if the .so does not export what the header declares
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        raise PcbError(load().pcb_last_error().decode(errors="replace"))


def launch_count():
    return int(load().pcb_launch_count())

"""Pins the kernel dispatch of the convolutions the workloads actually run: for every descriptor in
tests/golden/conv_dispatch.json (the distinct convolutions of the training steps, the 600^2 segmentation inference, the
InpaintingLoss VGG16 and the GPU test cases; see make_golden_conv_dispatch.py) every host query of the C ABI must answer
what it answered when the fixture was generated.  The queries are host code, so this runs without a GPU; the answers depend
on the SM count, which the library takes as 132 (H100 SXM) when no device is visible."""
import ctypes
import json
import os

import pytest

from text_segmentation_image_inpainting_b200 import _lib

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_dispatch.json")
FIELDS = ("n", "h", "w", "cin", "cout", "kh", "kw", "stride", "pad_h", "pad_w", "dil", "groups", "ho", "wo", "dtype",
          "same_holes", "no_guard", "plain", "force_generic")
PART_FIELDS = ("c", "x_cstride", "x_up", "mask_up")
MASK_PTR = 1 << 12            # stands for "this part has a hole plane": the queries only test the pointer for null
FIXTURE_SMS = 132


def conv_of(desc):
    c = _lib.Conv()
    for k in FIELDS:
        setattr(c, k, desc[k])
    c.nparts = len(desc["parts"])
    for i, p in enumerate(desc["parts"]):
        for k in PART_FIELDS:
            setattr(c.parts[i], k, p[k])
        c.parts[i].x = None
        c.parts[i].mask = MASK_PTR if p["mask"] else None
    return c


def host_queries(lib, c):
    ref = ctypes.byref(c)
    fe, de = ctypes.c_size_t(), ctypes.c_size_t()
    lib.pcb_conv_weight_layout(ref, ctypes.byref(fe), ctypes.byref(de))
    routes = (ctypes.c_int32 * 3)()
    _lib.check(lib.pcb_debug_conv_routes(ref, routes))
    return {"uses_tensor_cores": lib.pcb_conv_uses_tensor_cores(ref), "workspace": lib.pcb_pconv_workspace(ref),
            "routes": [_lib.ROUTES[r] for r in routes],
            "weight_fwd_elems": fe.value, "weight_dgrad_elems": de.value, "fuses_bn_stats": lib.pcb_conv_fuses_bn_stats(ref),
            "fuses_affine_act": lib.pcb_conv_fuses_affine_act(ref),
            "dgrad_at_source_resolution": lib.pcb_conv_dgrad_at_source_resolution(ref),
            "dgrad_fuses_relu": lib.pcb_conv_dgrad_fuses_relu(ref)}


def _visible_sms():
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:  # noqa: BLE001
        pass
    return None


def test_host_queries_match_fixture():
    sms = _visible_sms()
    if sms is not None and sms != FIXTURE_SMS:
        pytest.skip(f"the fixture's expected values assume {FIXTURE_SMS} SMs, the visible device has {sms}")
    lib = _lib.load()
    with open(FIXTURE) as f:
        fixture = json.load(f)
    assert len(fixture["cases"]) > 100
    bad = []
    for case in fixture["cases"]:
        got = host_queries(lib, conv_of(case["conv"]))
        if got != case["expect"]:
            bad.append((case["conv"], {k: (v, got[k]) for k, v in case["expect"].items() if got[k] != v}))
    assert not bad, f"{len(bad)} of {len(fixture['cases'])} descriptors dispatch differently; first: {bad[0]}"

"""Page geometries in the kernel fixtures, and the 32-bit bounds of the convolution plan.  Host code and fixture reads only: no
GPU.

Fixtures.  tests/golden/conv_dispatch.json and elementwise_sites.json hold, besides the training runs, the inference runs of
make_golden_conv_dispatch.inference_runs (TextRemovalStep and InferStep at page sizes); the descriptors only those runs reach
carry "forward_only": 1 and are checked forward-only by the fp64 kernel suites.  These tests pin that the fixtures still reach
the geometries that no training run makes, so that a regeneration cannot quietly drop them: a 2x-upsampled decoder input
read from an odd, non-square source grid; a tensor-core forward over 2^21 output pixels or more; ImageFillOrigin's
full-resolution RGB tail on the A4 U-Net grid (3584 x 2560); depthwise layers on odd grids (stride 2 with an odd output
grid, stride 1 on an odd input grid); a segmentation layer at b4 whose routes change with the page's grid; bilinear
resampling on an odd, non-square grid.

Bounds.  The tensor-core kernels address their operands with 32-bit element offsets, so the plan keeps a problem off them
(conv_tc.cu common_ok, conv_stem.cu pcb_stem_plan) once n ho wo rup(cout, 64) output elements, or n (h >> up) (w >> up)
x_cstride elements of a part, pass 2^31 - 1.  Each bound is tested at 2^31 elements and one pixel below it (the largest count
the geometry can make below 2^31: the counts are multiples of 64 or of the channel stride): the tensor-core route below, the
shape-general kernels at the bound, and at both the workspace and weight-layout queries must report sizes that did not wrap.
The stem's `cells * 32` bound is implied by its `cells * rup64(cout)` one (rup64(cout) >= 64), so the latter is the one tested.
"""
import ctypes
import json
import os

import pytest

from test_conv_dispatch_cpu import FIELDS, conv_of, host_queries
from text_segmentation_image_inpainting_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LIM = 2 ** 31 - 1
TC_ROUTES = {"stem", "k2r", "smallco", "tma", "tma_s2", "gather"}


def _rup(v, m):
    return (v + m - 1) // m * m


def _desc(n, h, w, parts, cout, k=3, s=1, pad=None):
    """a bf16 descriptor in the fixture's format; parts: (channels, x_up, masked[, x_cstride])"""
    pad = (k - 1) // 2 if pad is None else pad
    return dict(n=n, h=h, w=w, cin=sum(p[0] for p in parts), cout=cout, kh=k, kw=k, stride=s, pad_h=pad, pad_w=pad, dil=1, groups=1,
                ho=(h + 2 * pad - k) // s + 1, wo=(w + 2 * pad - k) // s + 1, dtype=_lib.PCB_BF16, same_holes=0, no_guard=0, plain=0,
                force_generic=0,
                parts=[dict(c=p[0], x_cstride=p[3] if len(p) > 3 else _rup(p[0], 8), x_up=p[1], mask_up=p[1], mask=p[2]) for p in parts])


def _out_elems(d):
    return d["n"] * d["ho"] * d["wo"] * _rup(d["cout"], 64)


def _part_elems(d, i):
    p = d["parts"][i]
    return d["n"] * (d["h"] >> p["x_up"]) * (d["w"] >> p["x_up"]) * p["x_cstride"]


def _queries(d):
    return host_queries(_lib.load(), conv_of(d))


def _assert_sane(tag, d, q):
    """workspace and operand sizes that did not wrap: the operands hold at least the weights, and nothing reaches 2^40"""
    weights = d["cout"] * d["kh"] * d["kw"] * d["cin"] // d["groups"]
    assert weights <= q["weight_fwd_elems"] < 2 ** 40, f"{tag}: forward operand of {q['weight_fwd_elems']} elements"
    assert 0 <= q["weight_dgrad_elems"] < 2 ** 40, f"{tag}: data-gradient operand of {q['weight_dgrad_elems']} elements"
    assert 0 <= q["workspace"] < 2 ** 40, f"{tag}: workspace of {q['workspace']} bytes"
    if set(q["routes"]) <= {"generic"}:
        assert q["workspace"] == 0 and q["weight_fwd_elems"] == weights and q["weight_dgrad_elems"] == 0, f"{tag}: {q}"
    else:
        assert q["workspace"] > 0, f"{tag}: a tensor-core problem without workspace"


# (below, at): descriptors one pixel below the bound and at 2^31 elements, and which count each one bounds
BOUNDS = {
    # outputs: n ho wo rup(cout, 64) with cout 128, the input part at half of that
    "outputs": (_desc(1, 4095, 4097, [(64, 0, 1)], 128), _desc(1, 4096, 4096, [(64, 0, 1)], 128), _out_elems),
    # a full-resolution part: 1x1 at stride 2, so the outputs stay at a quarter
    "part": (_desc(1, 18631, 1801, [(64, 0, 1)], 64, 1, 2), _desc(1, 8192, 4096, [(64, 0, 1)], 64, 1, 2),
             lambda d: _part_elems(d, 0)),
    # a 2x-upsampled part, counted at its source resolution, with a channel stride of 512 so that it binds first
    "upsampled_part": (_desc(1, 4094, 4098, [(64, 1, 1, 512), (32, 0, 1)], 64), _desc(1, 4096, 4096, [(64, 1, 1, 512), (32, 0, 1)], 64),
                       lambda d: _part_elems(d, 0)),
    # the space-to-depth stem: cells rup64(cout), cout 32 and 96
    "stem_cout32": (_desc(1, 37262, 3602, [(3, 0, 1, 8)], 32, 7, 2), _desc(1, 16384, 8192, [(3, 0, 1, 8)], 32, 7, 2), _out_elems),
    "stem_cout96": (_desc(1, 8190, 8194, [(3, 0, 1, 8)], 96, 7, 2), _desc(1, 8192, 8192, [(3, 0, 1, 8)], 96, 7, 2), _out_elems),
}


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_tensor_core_routes_end_at_the_32bit_bound(name):
    below, at, count = BOUNDS[name]
    assert count(below) <= LIM < count(at) == 2 ** 31, f"{name}: {count(below)}, {count(at)}"
    for d in (below, at):              # the bound named is the one that binds: every other count stays below it
        others = [_out_elems(d)] + [_part_elems(d, i) for i in range(len(d["parts"]))]
        assert sorted(others)[-2 if count(d) in others else -1] <= LIM, f"{name}: another count passes the bound too"
    qb, qa = _queries(below), _queries(at)
    assert qb["routes"][0] in TC_ROUTES and qb["uses_tensor_cores"] == 1, f"{name}: below the bound the plan routes {qb['routes']}"
    if name.startswith("stem"):
        assert qb["routes"][0] == "stem", f"{name}: {qb['routes']}"
    assert qa["routes"] == ["generic"] * 3 and qa["uses_tensor_cores"] == 0, f"{name}: at 2^31 elements the plan routes {qa['routes']}"
    _assert_sane(f"{name} below", below, qb)
    _assert_sane(f"{name} at", at, qa)


def test_a4_rgb_tail_at_b4_leaves_the_tensor_cores():
    """ImageFillOrigin's full-resolution RGB tail on the A4 U-Net grid (3584 x 2560): at b1 the kernel-to-row route, at b4 its
    outputs are 4 x 2560 x 3584 x 64 > 2^31 elements and the plan must take the shape-general kernels"""
    tails = [c["conv"] for c in _fixture()["cases"] if (c["conv"]["h"], c["conv"]["w"]) == (3584, 2560) and c["expect"]["routes"][0] == "k2r"]
    assert tails, "the fixture holds no kernel-to-row tail on the A4 U-Net grid"
    for d in tails:
        assert d["n"] == 1 and _out_elems(d) <= LIM
        d4 = dict(d, n=4)
        assert _out_elems(d4) > LIM
        q = _queries(d4)
        assert q["routes"] == ["generic"] * 3 and q["uses_tensor_cores"] == 0, f"A4 tail at b4: {q['routes']}"
        _assert_sane("A4 tail at b4", d4, q)
        _assert_sane("A4 tail at b1", d, _queries(d))


# ------------------------------------------------------------------------------------------------ what the fixtures reach
def _fixture():
    with open(os.path.join(GOLDEN, "conv_dispatch.json")) as f:
        return json.load(f)


def _forward_only():
    return [c for c in _fixture()["cases"] if c.get("forward_only")]


def _key(d, **drop):
    return json.dumps({k: v for k, v in d.items() if k not in drop}, sort_keys=True)


def test_forward_only_marks_only_new_descriptors():
    cases = _fixture()["cases"]
    fo = [c for c in cases if c.get("forward_only")]
    assert len(fo) >= 20, f"{len(fo)} forward-only descriptors"
    assert all(c["forward_only"] == 1 and set(c) == {"conv", "expect", "forward_only"} for c in fo)
    assert len({_key(c["conv"]) for c in cases}) == len(cases), "a descriptor appears twice"
    first = next(i for i, c in enumerate(cases) if c.get("forward_only"))
    assert all(c.get("forward_only") for c in cases[first:]), "the inference runs' entries are appended after the others"


def test_forward_only_reaches_an_upsampled_part_on_an_odd_non_square_source_grid():
    hits = [c["conv"] for c in _forward_only() for p in c["conv"]["parts"] if p["x_up"]
            and (c["conv"]["h"] >> 1) != (c["conv"]["w"] >> 1) and ((c["conv"]["h"] >> 1) % 2 or (c["conv"]["w"] >> 1) % 2)]
    assert hits, "no forward-only decoder layer reads a 2x-upsampled part from an odd, non-square source grid"
    assert any(c["expect"]["routes"][0] in TC_ROUTES for c in _forward_only() if c["conv"] in hits)


def test_forward_only_reaches_a_tensor_core_forward_over_2_21_outputs():
    assert any(c["expect"]["routes"][0] in TC_ROUTES and c["conv"]["n"] * c["conv"]["ho"] * c["conv"]["wo"] >= 2 ** 21
               for c in _forward_only())


def test_forward_only_reaches_the_a4_rgb_tail():
    assert any(c["expect"]["routes"][0] == "k2r" and (c["conv"]["h"], c["conv"]["w"]) == (3584, 2560) for c in _forward_only())


def test_forward_only_reaches_depthwise_layers_on_odd_grids():
    """no workload runs a stride-2 layer on an odd input grid (every one of them halves an even grid); what the pages add are
    depthwise stride-2 layers with an odd, non-square output grid and depthwise layers on odd, non-square input grids"""
    dw = [c["conv"] for c in _forward_only() if c["expect"]["routes"][0] == "depthwise"]
    assert any(d["stride"] == 2 and d["ho"] != d["wo"] and (d["ho"] % 2 or d["wo"] % 2) for d in dw)
    assert any(d["stride"] == 1 and d["h"] != d["w"] and (d["h"] % 2 or d["w"] % 2) for d in dw)


def test_forward_only_reaches_b4_layers_whose_routes_change_with_the_grid():
    """the segmentation networks at b4 (no hole planes): the same layer on the 600^2 and 1024^2 pages' grids takes different
    routes (the launch count of the b4 segmentation changes with seg_resize, DESIGN 5.2), and the 600^2 b4 layers have their b1
    counterparts in the fixture too"""
    def key(d, *drop):
        return json.dumps({k: v for k, v in d.items() if k not in drop}, sort_keys=True)
    b4 = [c for c in _forward_only() if c["conv"]["n"] == 4 and not any(p["mask"] for p in c["conv"]["parts"])]
    routes = {}
    for c in b4:
        routes.setdefault(key(c["conv"], "h", "w", "ho", "wo"), set()).add(tuple(c["expect"]["routes"]))
    assert any(len(r) > 1 for r in routes.values()), "no b4 segmentation layer changes its routes with the grid"
    b1 = {key(c["conv"], "n") for c in _fixture()["cases"] if c["conv"]["n"] == 1}
    assert any(c["conv"]["h"] == 75 and key(c["conv"], "n") in b1 for c in b4), "no 600^2 b4 layer has its b1 counterpart"


def _sites():
    with open(os.path.join(GOLDEN, "elementwise_sites.json")) as f:
        return json.load(f)


def test_elementwise_sites_reach_bilinear_on_odd_non_square_grids():
    """pcb_bilinear_* take one integer scale factor for both axes (the segmentation networks upsample by 2 and 4), so every
    site resamples at equal, integer ratios; what the page geometries add is the source grid: non-square with an odd side,
    where the last source row or column is clamped on one axis and not on the other"""
    hits = [s for s in _sites() if s["fn"] == "pcb_bilinear_forward" and s["h"] != s["w"] and (s["h"] % 2 or s["w"] % 2)]
    assert hits, "no bilinear site on a non-square source grid with an odd side"


def test_bound_descriptors_are_valid():
    """every descriptor above passes the library's own validation (a refused descriptor would make the route test vacuous)"""
    lib = _lib.load()
    for below, at, _ in BOUNDS.values():
        for d in (below, at):
            assert set(FIELDS) <= set(d)
            r = (ctypes.c_int32 * 3)()
            assert lib.pcb_debug_conv_routes(ctypes.byref(conv_of(d)), r) == 0, lib.pcb_last_error()

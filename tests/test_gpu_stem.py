"""The space-to-depth stem kernels (conv_stem.cu: stem_fwd_kernel, stem_wgrad_kernel) against fp64, through the full route
check of test_gpu_conv_routes.py (bit-exact integer regime, fp64 bounds, the kernel trace, the weight refresh and the
two-call forward), at shapes its fixture list does not reach: the production stem (3 -> 64 at 512^2, batch 8, holes),
every image width 1 / 3 / 4 / 5 / 8 across the 16- / 32-channel cell boundary, cout that is not a multiple of 64 or spans
two N tiles, grids that are not a whole number of tiles, and holes placed on purpose in the first and last two rows and columns
of the image, at even and odd sub-pixel offsets (the space-to-depth masking and the padding-2 edge of the im2row gather)."""
import pytest

import kernel_harness
import test_gpu_conv_routes as R

pytestmark = pytest.mark.gpu

STEM = ("stem", "none", "stem")
P_, C_ = R._part, R._case

STEM_CASES = {
    "stem_prod_c3_o64_512_b8_holes": C_(8, 512, 512, [P_(3, mask=True)], 64, 7, 2, route=STEM),
    "stem_c1_o64_holes": C_(2, 64, 96, [P_(1, mask=True)], 64, 7, 2, route=STEM),
    "stem_c3_o64_plain": C_(1, 128, 64, [P_(3)], 64, 7, 2, plain=True, route=STEM),
    "stem_c4_o48_ragged_holes": C_(3, 30, 46, [P_(4, mask=True)], 48, 7, 2, route=STEM),
    "stem_c5_o64_holes": C_(2, 64, 64, [P_(5, mask=True)], 64, 7, 2, route=STEM),
    "stem_c8_o40_ragged_noguard": C_(2, 38, 54, [P_(8, mask=True)], 40, 7, 2, no_guard=True, route=STEM),
    "stem_c3_o96_two_ntiles_holes": C_(2, 64, 64, [P_(3, mask=True)], 96, 7, 2, route=STEM),
    "stem_c8_o128_two_ntiles": C_(1, 32, 256, [P_(8, mask=True)], 128, 7, 2, route=STEM),
}
BORDER_CASES = {
    "stem_c3_o64_border_holes": C_(2, 40, 72, [P_(3, mask=True)], 64, 7, 2, route=STEM),
    "stem_c8_o40_ragged_border_holes": C_(1, 34, 50, [P_(8, mask=True)], 40, 7, 2, route=STEM),
}


def border_holes(n, h, w, gen):
    """kernel_harness.holes plus holes in the two outermost rows and columns on every side, at even and odd positions, so
    both sub-pixels (a, b) of the border cells are holes in some cells and valid in others"""
    m = kernel_harness.holes(n, h, w, gen)
    m[:, 0, 0::2] = 0
    m[:, 1, 1::2] = 0
    m[:, h - 1, 0::3] = 0
    m[:, h - 2, 1::4] = 0
    m[:, 0::2, 0] = 0
    m[:, 1::2, 1] = 0
    m[:, 1::3, w - 1] = 0
    m[:, 0::4, w - 2] = 0
    return m


@pytest.mark.parametrize("name", sorted(STEM_CASES))
def test_stem_vs_fp64(name, monkeypatch):
    monkeypatch.setitem(R.CASES, name, STEM_CASES[name])
    R.test_conv_route_vs_fp64(name)


@pytest.mark.parametrize("name", sorted(BORDER_CASES))
def test_stem_border_holes_vs_fp64(name, monkeypatch):
    monkeypatch.setitem(R.CASES, name, BORDER_CASES[name])
    monkeypatch.setattr(R, "holes", border_holes)
    R.test_conv_route_vs_fp64(name)

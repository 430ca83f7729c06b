"""Weight gradient of the TMA-fed tensor-core kernel (pcb_pconv_backward_weight through the C ABI) against an fp64 CPU
weight gradient of the same masked bf16 input and bf16 output gradient, one case per tile configuration:

  * 128-wide output-channel tiles, with and without row-halo A blocks;
  * a 64-channel input block shared by both consumer warpgroups: output channels split (128-wide tile) or K blocks split
    (64-wide tile, cout <= 64);
  * ragged output-channel tiles, an input-channel tile straddling two parts, a 2x-upsampled part;
  * row-halo blocks taller than 128 rows (dilation 48) with holes over large input values.

Error bound.  Every product x*m * dc of two bf16 values is exact in fp32, so the kernel differs from the exact sum only in how
it adds the products of each weight: fp32 tensor-core accumulation plus fp32 red.global.add of the split-K partials, in an
order the test does not know.  Adding an exact zero is exact, so only the n nonzero products of an element count.  Any order
of n - 1 additions with unit roundoff u is off by at most (n - 1) u / (1 - (n - 1) u) * S, S = sum |x*m| |dc| (Higham,
Accuracy and Stability of Numerical Algorithms, 4.2).  The tensor cores' fp32 adder is not guaranteed to round to nearest,
so u = 2^-23 (one ulp) instead of 2^-24, and 1 / (1 - (n - 1) u) < 2 here:   |dw - dw_exact| <= n * 2^-22 * S   per element.
dc is nonzero on a quarter of the pixels, which keeps that bound well below what one 64-pixel K block contributes.
The 128-wide cases have 8192 output pixels, the fewest for which pcb_tc_wgrad picks 128-wide tiles.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from text_segmentation_image_inpainting_b200 import _lib

pytestmark = pytest.mark.gpu

# name: (n, h, w, parts [(channels, upsampled, masked)], cout, k, stride, dilation)
#   an upsampled part is stored at (h/2, w/2) with its hole plane at that resolution; padding keeps "same" geometry
CASES = {
    "halo_n128_holes": (2, 32, 128, [(128, 0, 1)], 128, 3, 1, 1),
    "decoder_upsampled_two_parts_n128": (1, 64, 128, [(128, 1, 1), (64, 0, 1)], 128, 3, 1, 1),
    "enc1_like_k5_s2_64_128_split_n": (2, 128, 128, [(64, 0, 1)], 128, 5, 2, 1),
    "k3_s2_256_512": (2, 128, 128, [(256, 0, 1)], 512, 3, 2, 1),
    "dec7_like_192_64_split_k": (1, 16, 128, [(128, 1, 1), (64, 0, 1)], 64, 3, 1, 1),
    "ragged_cout192_halo": (1, 64, 128, [(128, 0, 1)], 192, 3, 1, 1),
    "ragged_cout320_split_n": (8, 32, 32, [(64, 0, 1)], 320, 3, 1, 1),
    "ci_tile_straddles_parts": (1, 128, 64, [(64, 0, 1), (128, 0, 1)], 128, 3, 1, 1),
    "short_reduction_n64_tiles": (2, 8, 64, [(256, 0, 1)], 256, 3, 1, 1),
    "halo_d48_holes_over_large_x": (1, 64, 128, [(128, 0, 1)], 128, 3, 1, 48),
}
HOLE_VALUE = 64.0            # x under the holes in the dilation-48 case: a row left unmasked is far outside the bound


def _holes(n, h, w, gen):
    """uint8 plane, 1 = valid: a few rectangles plus scattered single pixels"""
    m = (torch.rand(n, h, w, generator=gen) > 0.15).to(torch.uint8)
    for i in range(n):
        y0, x0 = int(torch.randint(0, max(1, h // 2), (1,), generator=gen)), int(torch.randint(0, max(1, w // 2), (1,), generator=gen))
        m[i, y0:y0 + max(1, h // 3), x0:x0 + max(2, w // 3)] = 0
    return m


@pytest.mark.parametrize("name", sorted(CASES))
def test_wgrad_tma_tiles_vs_fp64(name):
    n, h, w, parts, cout, k, s, d = CASES[name]
    dev = torch.device("cuda:0")
    lib = _lib.load()
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    pad = d * (k - 1) // 2
    ho, wo = (h + 2 * pad - d * (k - 1) - 1) // s + 1, (w + 2 * pad - d * (k - 1) - 1) // s + 1
    cin = sum(p[0] for p in parts)

    c = _lib.Conv()
    c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw = n, h, w, cin, cout, k, k
    c.stride, c.pad_h, c.pad_w, c.dil, c.groups, c.ho, c.wo = s, pad, pad, d, 1, ho, wo
    c.dtype, c.nparts = _lib.PCB_BF16, len(parts)
    keep = []                                   # device buffers the struct points into
    xm_full = []                                # fp64 x * m at the logical input resolution
    for i, (ch, up, masked) in enumerate(parts):
        hs, ws = h >> up, w >> up
        x = torch.randn(n, hs, ws, ch, generator=gen).to(torch.bfloat16)
        m = _holes(n, hs, ws, gen) if masked else torch.ones(n, hs, ws, dtype=torch.uint8)
        if name == "halo_d48_holes_over_large_x":
            x = torch.where(m[..., None] == 0, torch.full_like(x, HOLE_VALUE), x)
        xd, md = x.to(dev).contiguous(), m.to(dev).contiguous()
        keep += [xd, md]
        c.parts[i].x, c.parts[i].mask = xd.data_ptr(), (md.data_ptr() if masked else None)
        c.parts[i].c, c.parts[i].x_cstride, c.parts[i].x_up, c.parts[i].mask_up = ch, ch, up, up
        xm = (x.double() * m.double()[..., None]).permute(0, 3, 1, 2)
        if up:
            xm = F.interpolate(xm, scale_factor=2, mode="nearest")
        xm_full.append(xm)
    assert lib.pcb_conv_uses_tensor_cores(ctypes.byref(c)) == 1

    dc = torch.randn(n, ho, wo, cout, generator=gen).to(torch.bfloat16)
    dc = dc * (torch.rand(n, ho, wo, 1, generator=gen) < 0.25).to(dc.dtype)
    dcd = dc.to(dev).contiguous()
    dw = torch.full((cout, k, k, cin), float("nan"), device=dev)
    ws_bytes = lib.pcb_pconv_workspace(ctypes.byref(c))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.pcb_pconv_backward_weight(ctypes.byref(c), dcd.data_ptr(), cout, dw.data_ptr(), ws.data_ptr(), stream))
    torch.cuda.synchronize()
    got = dw.cpu().double().permute(0, 3, 1, 2)                     # KRSC -> [cout][cin][kh][kw]

    xm = torch.cat(xm_full, 1)
    g = dc.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xm, (cout, cin, k, k), g, stride=s, padding=pad, dilation=d)
    mag = torch.nn.grad.conv2d_weight(xm.abs(), (cout, cin, k, k), g.abs(), stride=s, padding=pad, dilation=d)
    nonzero = torch.nn.grad.conv2d_weight((xm != 0).double(), (cout, cin, k, k), (g != 0).double(), stride=s, padding=pad, dilation=d)
    bound = nonzero * 2.0 ** -22 * mag
    assert torch.isfinite(got).all(), "weight gradient left unwritten"
    assert float(ref.abs().max()) > 0
    excess = (got - ref).abs() - bound
    worst = int(excess.argmax())
    assert float(excess.max()) <= 0.0, (f"{name}: |err| exceeds n * 2^-22 * S at flat index {worst}: "
                                       f"err {float((got - ref).abs().flatten()[worst]):.3e}, bound {float(bound.flatten()[worst]):.3e}")

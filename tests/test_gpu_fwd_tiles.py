"""Forward (with the fused BatchNorm sums, or the eval-mode affine + activation epilogue) and data gradient of the TMA-fed
tensor-core kernels, through the C ABI, against fp64 references on the same bf16 operands, one case per tile configuration:

  * 256-wide forward and data-gradient tiles (dec1-like 1024 -> 512 at 32x32, two parts), and the eval epilogue at 256;
  * ragged output channels (cout 320, 384);
  * two parts, one of them 2x-upsampled (sub-pixel kernels);
  * holes without the zero guard (no_guard: 0 * inf = NaN exactly where the mask box is empty);
  * the stride-2 data gradient as four parity classes at Cin 256;
  * a 64-wide row-halo tile with dilation 48 (halo rows up to 224, past the fixers' third row at 192) and large values under
    the holes, so a hole row left unzeroed is far outside the bound.

Error bounds.  Every product of two bf16 values is exact in fp32; the tensor cores add the n nonzero products of an element in
an order the test does not know, which is off by at most n * 2^-22 * S, S = sum of |products| (Higham 4.2, one-ulp adds; see
test_gpu_wgrad_tiles.py).  Sub-pixel launches sum taps of the weight in fp32 and round them to bf16 once: a further
2^-8 * S.  The forward then multiplies by fl(1 / s) and adds the bias in one fma (two more roundings of the result, 2^-22
relative covers both), the eval epilogue one more fma (2^-23) and a 1-Lipschitz activation; the stored value is rounded to
bf16 once (half an ulp, 2^-9 relative; 2^-8 is used).  The BatchNorm sums are checked against the stored values: M fp32
additions of terms bounded by |y| are off by at most M * 2^-23 * sum |y|.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from text_segmentation_image_inpainting_b200 import _lib

pytestmark = pytest.mark.gpu

# name: (n, h, w, parts [(channels, upsampled, masked)], cout, k, stride, dilation, mode)
#   mode: "bn" = training forward with fused BatchNorm sums, "eval" = affine + LeakyReLU epilogue, "no_guard" = NaN at empty
#   boxes; an upsampled part is stored at (h/2, w/2) with its hole plane at that resolution
CASES = {
    "n256_two_parts_1024_512": (8, 32, 32, [(512, 0, 1), (512, 0, 1)], 512, 3, 1, 1, "bn"),
    "eval_affine_leaky_n256": (8, 32, 32, [(256, 0, 1)], 512, 3, 1, 1, "eval"),
    "ragged_cout320": (2, 32, 64, [(128, 0, 1)], 320, 3, 1, 1, "bn"),
    "ragged_cout384": (2, 32, 64, [(128, 0, 1)], 384, 3, 1, 1, "bn"),
    "two_parts_one_upsampled": (1, 64, 64, [(128, 1, 1), (64, 0, 1)], 64, 3, 1, 1, "bn"),
    "holes_no_guard_nan": (2, 32, 128, [(128, 0, 1)], 128, 3, 1, 1, "no_guard"),
    "s2_parity_dgrad_cin256": (2, 64, 64, [(256, 0, 1)], 512, 3, 2, 1, "bn"),
    "halo_n64_d48_holes_over_large_x": (2, 64, 128, [(64, 0, 1)], 64, 3, 1, 48, "bn"),
}
HOLE_VALUE = 64.0
SLOPE = 0.2


def _holes(n, h, w, gen):
    """uint8 plane, 1 = valid: a few rectangles plus scattered single pixels"""
    m = (torch.rand(n, h, w, generator=gen) > 0.15).to(torch.uint8)
    for i in range(n):
        y0, x0 = int(torch.randint(0, max(1, h // 2), (1,), generator=gen)), int(torch.randint(0, max(1, w // 2), (1,), generator=gen))
        m[i, y0:y0 + max(1, h // 3), x0:x0 + max(2, w // 3)] = 0
    return m


def _rup(v, m):
    return (v + m - 1) // m * m


@pytest.mark.parametrize("name", sorted(CASES))
def test_fwd_dgrad_tma_tiles_vs_fp64(name):
    n, h, w, parts, cout, k, s, d, mode = CASES[name]
    dev = torch.device("cuda:0")
    lib = _lib.load()
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    pad = d * (k - 1) // 2
    ho, wo = (h + 2 * pad - d * (k - 1) - 1) // s + 1, (w + 2 * pad - d * (k - 1) - 1) // s + 1
    cin = sum(p[0] for p in parts)
    wround = any(p[1] for p in parts)                 # sub-pixel launches round summed weight taps to bf16

    c = _lib.Conv()
    c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw = n, h, w, cin, cout, k, k
    c.stride, c.pad_h, c.pad_w, c.dil, c.groups, c.ho, c.wo = s, pad, pad, d, 1, ho, wo
    c.dtype, c.nparts, c.no_guard = _lib.PCB_BF16, len(parts), int(mode == "no_guard")
    keep, xm_full, m_full = [], [], []
    for i, (ch, up, masked) in enumerate(parts):
        hs, ws = h >> up, w >> up
        x = torch.randn(n, hs, ws, ch, generator=gen).to(torch.bfloat16)
        m = _holes(n, hs, ws, gen) if masked else torch.ones(n, hs, ws, dtype=torch.uint8)
        if name.startswith("halo"):
            x = torch.where(m[..., None] == 0, torch.full_like(x, HOLE_VALUE), x)
        xd, md = x.to(dev).contiguous(), m.to(dev).contiguous()
        keep += [xd, md]
        c.parts[i].x, c.parts[i].mask = xd.data_ptr(), (md.data_ptr() if masked else None)
        c.parts[i].c, c.parts[i].x_cstride, c.parts[i].x_up, c.parts[i].mask_up = ch, ch, up, up
        mf = m.to(dev).double()[:, None].expand(n, ch, hs, ws)
        xm = x.to(dev).double().permute(0, 3, 1, 2) * mf
        if up:
            xm, mf = F.interpolate(xm, scale_factor=2, mode="nearest"), F.interpolate(mf, scale_factor=2, mode="nearest")
        xm_full.append(xm)
        m_full.append(mf)
    assert lib.pcb_conv_uses_tensor_cores(ctypes.byref(c)) == 1
    stream = torch.cuda.current_stream().cuda_stream

    wm = (torch.randn(cout, k, k, cin, generator=gen) / (cin * k * k) ** 0.5).to(dev)
    fe, de = ctypes.c_size_t(), ctypes.c_size_t()
    lib.pcb_conv_weight_layout(ctypes.byref(c), ctypes.byref(fe), ctypes.byref(de))
    w_fwd = torch.zeros(max(fe.value, 1), dtype=torch.bfloat16, device=dev)
    w_dg = torch.zeros(max(de.value, 1), dtype=torch.bfloat16, device=dev)
    _lib.check(lib.pcb_conv_weight_prepare(ctypes.byref(c), wm.data_ptr(), w_fwd.data_ptr(), w_dg.data_ptr(), stream))
    W = wm.to(torch.bfloat16).double().permute(0, 3, 1, 2).contiguous()          # [cout][cin][k][k]
    bias = (torch.randn(cout, generator=gen) * 0.1).to(dev)

    # ---------------- forward
    ycs = _rup(cout, 8)
    y = torch.full((n, ho, wo, ycs), float("nan"), dtype=torch.bfloat16, device=dev)
    msum = torch.empty(n, ho, wo, device=dev)
    newmask = torch.empty(n, ho, wo, dtype=torch.uint8, device=dev)
    ws_buf = torch.empty(max(lib.pcb_pconv_workspace(ctypes.byref(c)), 1), dtype=torch.uint8, device=dev)
    sums = torch.zeros(2, cout, dtype=torch.float64, device=dev)
    if mode == "eval":
        scale = (torch.rand(cout, generator=gen) + 0.5).to(dev)
        shift = (torch.randn(cout, generator=gen) * 0.1).to(dev)
        assert lib.pcb_conv_fuses_affine_act(ctypes.byref(c)) == 1
        _lib.check(lib.pcb_pconv_forward_affine_act(ctypes.byref(c), w_fwd.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                                    newmask.data_ptr(), ws_buf.data_ptr(), 0, scale.data_ptr(), shift.data_ptr(), 2, SLOPE, stream))
    else:
        assert lib.pcb_conv_fuses_bn_stats(ctypes.byref(c)) == 1
        _lib.check(lib.pcb_pconv_forward_bn(ctypes.byref(c), w_fwd.data_ptr(), bias.data_ptr(), y.data_ptr(), ycs, msum.data_ptr(),
                                            newmask.data_ptr(), ws_buf.data_ptr(), 0, sums.data_ptr(), stream))
    torch.cuda.synchronize()

    XM, M = torch.cat(xm_full, 1), torch.cat(m_full, 1)
    box = F.conv2d(M, torch.ones(1, cin, k, k, dtype=torch.float64, device=dev), stride=s, padding=pad, dilation=d)[:, 0]
    assert torch.equal(msum.double(), box), f"{name}: mask sums"
    conv = lambda a, b: F.conv2d(a, b, stride=s, padding=pad, dilation=d)
    acc = conv(XM, W)
    mag = conv(XM.abs(), W.abs())
    nz = conv((XM != 0).double(), (W != 0).double())
    e_acc = nz * 2.0 ** -22 * mag + (2.0 ** -8 * mag if wround else 0.0)
    sb = box[:, None]
    empty = (sb == 0).expand_as(acc)
    safe = torch.where(sb == 0, torch.ones_like(sb), sb)
    v_ref = torch.where(empty, torch.zeros_like(acc), acc / safe + bias.double()[None, :, None, None])
    e = torch.where(empty, torch.zeros_like(acc), e_acc / safe + 2.0 ** -22 * (acc.abs() / safe + v_ref.abs()))
    if mode == "eval":
        sc, sh = scale.double()[None, :, None, None], shift.double()[None, :, None, None]
        z = v_ref * sc + sh
        e = sc * e + 2.0 ** -23 * (z.abs() + sh.abs())
        v_ref = torch.where(z > 0, z, z * SLOPE)
    bound = e + 2.0 ** -8 * (v_ref.abs() + e)
    got = y.double().permute(0, 3, 1, 2)
    assert torch.all(got[:, cout:] == 0), f"{name}: channels past cout must be zeros"
    got = got[:, :cout]
    if mode == "no_guard":
        assert bool(empty.any()), "case needs empty mask boxes"
        assert torch.isnan(got[empty]).all(), f"{name}: empty boxes must give NaN without the zero guard"
        got, v_ref, bound = got[~empty], v_ref[~empty], bound[~empty]
    assert torch.isfinite(got).all(), f"{name}: forward output left unwritten or not finite"
    excess = (got - v_ref).abs() - bound
    worst = int(excess.argmax())
    assert float(excess.max()) <= 0.0, (f"{name}: forward |err| exceeds the bound at flat index {worst}: "
                                       f"err {float((got - v_ref).abs().flatten()[worst]):.3e}, bound {float(bound.flatten()[worst]):.3e}")
    if mode == "bn":                                  # the sums are of the stored bf16 values
        yv = y.double()[..., :cout].reshape(-1, cout)
        for row, vals in ((0, yv), (1, yv * yv)):
            tol = yv.shape[0] * 2.0 ** -23 * vals.abs().sum(0)
            assert torch.all((sums[row] - vals.sum(0)).abs() <= tol), f"{name}: BatchNorm {'sums' if row == 0 else 'squares'}"

    # ---------------- data gradient
    dcs = _rup(cout, 8)
    dc = torch.randn(n, ho, wo, dcs, generator=gen).to(torch.bfloat16)
    dc[..., cout:] = 0
    dcd = dc.to(dev).contiguous()
    at_src = lib.pcb_conv_dgrad_at_source_resolution(ctypes.byref(c)) == 1
    dxs, ptrs, strides = [], [], []
    for ch, up, _m in parts:
        r = up if at_src else 0
        buf = torch.full((n, h >> r, w >> r, ch), float("nan"), dtype=torch.bfloat16, device=dev)
        dxs.append(buf); ptrs.append(buf.data_ptr()); strides.append(ch)
    _lib.check(lib.pcb_pconv_backward_data(ctypes.byref(c), dcd.data_ptr(), dcs, w_fwd.data_ptr(), w_dg.data_ptr(),
                                           (ctypes.c_void_p * len(parts))(*ptrs), (ctypes.c_int32 * len(parts))(*strides), stream))
    torch.cuda.synchronize()
    g = dcd.double()[..., :cout].permute(0, 3, 1, 2)
    shape = (n, cin, h, w)
    tconv = lambda a, b: torch.nn.grad.conv2d_input(shape, b, a, stride=s, padding=pad, dilation=d)
    gref = tconv(g, W)
    gmag = tconv(g.abs(), W.abs())
    gnz = tconv((g != 0).double(), (W != 0).double())
    ge = gnz * 2.0 ** -22 * gmag + (2.0 ** -8 * gmag if wround else 0.0)
    c0 = 0
    for i, (ch, up, _m) in enumerate(parts):
        mf = m_full[i]
        ref, err = gref[:, c0:c0 + ch] * mf, ge[:, c0:c0 + ch] * mf
        if up and at_src:
            ref, err = F.avg_pool2d(ref, 2) * 4, F.avg_pool2d(err, 2) * 4
        c0 += ch
        gb = err + 2.0 ** -8 * (ref.abs() + err)
        gg = dxs[i].double().permute(0, 3, 1, 2)
        assert torch.isfinite(gg).all(), f"{name}: dx of part {i} left unwritten or not finite"
        excess = (gg - ref).abs() - gb
        worst = int(excess.argmax())
        assert float(excess.max()) <= 0.0, (f"{name}: dx part {i} |err| exceeds the bound at flat index {worst}: "
                                           f"err {float((gg - ref).abs().flatten()[worst]):.3e}, bound {float(gb.flatten()[worst]):.3e}")

"""BatchNorm kernels of elementwise.cu through the C ABI, every element against an fp64 reference of the same stored operands
computed on the device.  Cases:

  * one per distinct BatchNorm call site of tests/golden/elementwise_sites.json (dtype, rows, channels, activation, residual:
    the layers the three training workloads and the eval forward run), at the recorded size; rows are capped only where x
    would exceed 2^27 elements, which keeps the channel route and stays far above the grid-cap threshold of ew_grid_red;
  * hand cases for what production never reaches: c 8 / 24 / 1544 / 2048 (one vector per row, an idle thread, one row per
    block with 63 idle threads, the widest vector route), the scalar routes (c 12, 2056), 2 rows, ragged row counts around
    rpb * 16, a c = 8 tensor of 2^24 rows (about 166 grid-stride sweeps per thread), the one-launch small backward at 1, 1023,
    1025, 16384 and 2^20 rows, every activation with and without a residual, and ill-conditioned channels.

Routes (kernel names asserted from one complete torch.profiler trace per case, see kernel_harness.traced):
    vector  (c % 8 == 0, c <= 2048)  bn_stats_kernel, bn_fwd_fused_kernel, bn_finalize_kernel, bn_act_fwd_kernel,
                                     bn_bwd_reduce_kernel, bn_bwd_apply_kernel               every case with such c
    small   (vector, rows <= 2^20)   bn_bwd_small_kernel                                    every vector case of <= 2^20 rows
    scalar  (any other c)            bn_stats_scalar_kernel, bn_finalize_kernel, bn_act_fwd_scalar_kernel,
                                     bn_bwd_reduce_scalar_kernel, bn_bwd_apply_scalar_kernel, bn_param_grad_kernel
                                                                                             scalar_c12*, scalar_c2056*
Every case runs every entry point that applies: pcb_bn_stats (separate and aliased [2][c] sums), pcb_bn_stats_acc onto
non-zero sums, pcb_bn_forward_fused (coef, running statistics, num_batches_tracked +1), pcb_bn_finalize (training and eval)
+ pcb_bn_act_forward, the activation-only forward, pcb_bn_act_backward_reduce (separate and aliased) / _reduce_acc onto
non-zero sums, _apply (training, eval, activation only, with dgamma / dbeta), _apply_renorm and _small (with and without a
mask-sum plane holding holes and renormalisers that are not powers of two).  On the scalar route pcb_bn_forward_fused,
_reduce_acc and _apply_renorm must refuse, launch nothing and leave every output untouched.  Outputs are prefilled with NaN.

Integer regime (case dtype).  x, gy and the residual are integers of magnitude <= 4; the backward is handed its own dyadic
scale (k/8), shift (k/8), mean (k/4) and invstd (2^-k), and LeakyReLU's slope is 1/4, so every gz = gy * act'(x * scale +
shift) and every gz * (x - mean) * invstd is a multiple of 2^-7 of magnitude <= 20.  A sum of such terms is exact in fp32 in
any order while the sum of their magnitudes stays below 2^24 units; the statistics are bounded per fp32 chain (the rows of
one block: at most 42496 rows * 16 < 2^24 here), the backward terms are thinned where needed so that the sum of |term| over
all rows stays below 2^24 units (asserted).  Then the statistics, both backward sums, dgamma and dbeta are bit-identical to
the exact sums (fp64, or their fp32 rounding where the kernel converts), and dx is bit-identical to the kernel's own fp32
sequence evaluated on exact sums: B = ((-scale * invstd) * fl(sum_gx)) * fl(1/count), C = (-scale * fl(sum_g)) * fl(1/count),
fma(scale, gz, fma(B, x - mean, C)), times fl(1/s) (0 at holes), stored in the case's type.  The fma results are taken as the
exact fp64 value rounded to fp32 (exact in fp64: at most 24 + 3 + 24 significant bits).  A multiply-add that nvcc may
contract (x * scale + shift in the forwards, the scalar backward's two updates) is accepted in either its fused or its
unfused rounding, element by element.  The forward's coefficients are computed by the kernels from exact sums and are held
to the Gaussian bounds below with dS = dQ = 0; y must then be exact given the kernel's own coefficients.

Gaussian regime (fp32 storage, the forward's own coefficients).  Higham (Accuracy and Stability of Numerical Algorithms,
4.2): a chain of L fp32 additions of terms t is off by at most L * 2^-24 * sum |t|; a product adds one rounding per term.
  * statistics: L = rows per thread + rows per block (vector: block_flush adds rpb partials), or rows per thread + 5 + 8
    (scalar: warp shuffle tree, 8 warps); dS = (L + 1) u sum |x|, dQ = (L + 2) u sum x^2, u = 2^-24;
  * mean = fl(S / n): dm = dS / n + u |m|;  var = Q / n - (S / n)^2 in fp64: dv = dQ / n + (2 |m| + dS / n) dS / n;
    invstd = 1 / sqrtf(fl(var) + eps): relative error <= (dv + u (2 var + eps + 2 dv)) / (2 (var + eps)) + 2u (sqrt and
    division, correctly rounded: no fast math); scale = g * invstd adds u; shift = b - (m g) invstd adds
    |g invstd| dm + |m g invstd| (rel + 2u) + u |shift|;  running statistics: (1 - mom) r + mom v adds 3u of each term;
  * y against x * scale + shift of the kernel's coefficients: 2u (|x scale| + |shift|), the residual add u |y|;
  * backward sums against fp64 of the kernel's coefficients: (L + 1) u sum |gz| and (L + 4) u sum |gz (x - mean) invstd|
    (gz's product, the subtraction, the product, the final invstd multiply); an element whose pre-activation lies within 2u (|x scale| +
    |shift|) of a kink may take either derivative and adds its |gy| (times |x - mean| invstd) to the bound;
  * dx = scale gz + B (x - mean) + C from those sums: |x - mean| dB + dC + u (|x - mean| |B| + 2 |B (x - mean) + C| + 2 |dx|),
    dB = |scale invstd / n| (d sum_gx + 4u |sum_gx|), dC = |scale / n| (d sum_g + 3u |sum_g|); times fl(1/s) adds 2u |dx|.
Ill-conditioned channels (mean >= 64 x spread, the "spread below one bf16 ulp of its mean" case) run through the same bounds:
E[x^2] - m^2 from fp32 partials loses about (L + 2) u m^2 / var of relative variance, which dv carries.
"""
import math

import pytest
import torch

from kernel_harness import act_ref, assert_bitwise, assert_within, elementwise_sites, nan, traced
from text_segmentation_image_inpainting_b200 import _lib

MAX_ELEMS = 1 << 27
SMALL_MAX = 1 << 20               # the row limit of pcb_bn_act_backward_small
U = 2.0 ** -24
EPS, MOM = 1e-5, 0.1
EPS_F, MOM_F = (float(torch.tensor(v, dtype=torch.float32)) for v in (EPS, MOM))   # what the C ABI receives
SLOPE_INT, SLOPE = 0.25, 0.2      # LeakyReLU slope: dyadic in the integer regime, the networks' 0.2 in the Gaussian one
ACTS = (_lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_LEAKY, _lib.ACT_RELU6)
DTYPES = {_lib.PCB_BF16: ("bf16", torch.bfloat16), _lib.PCB_F32: ("f32", torch.float32)}
VEC_KERNELS = {"bn_stats_kernel", "bn_fwd_fused_kernel", "bn_finalize_kernel", "bn_act_fwd_kernel", "bn_bwd_reduce_kernel",
               "bn_bwd_apply_kernel"}
SCALAR_KERNELS = {"bn_stats_scalar_kernel", "bn_finalize_kernel", "bn_act_fwd_scalar_kernel", "bn_bwd_reduce_scalar_kernel",
                  "bn_bwd_apply_scalar_kernel", "bn_param_grad_kernel"}


def _spec(dtype, count, c, act=_lib.ACT_NONE, res=False, illcond=False):
    return dict(dtype=dtype, count=count, c=c, act=act, res=res, illcond=illcond)


def _site_case(site):
    """(case name, spec) of a BatchNorm call site: sites that differ only in the entry point share one case"""
    dt = site.get("dtype", _lib.PCB_F32)
    count, c, act = site["count"], site["c"], site.get("act", _lib.ACT_NONE)
    res = not site.get("null_residual", 1)
    name = f"fx_{DTYPES[dt][0]}_r{count}_c{c}_a{act}" + ("_res" if res else "")
    return name, _spec(dt, max(2, min(count, MAX_ELEMS // c)), c, act, res)


def _fixture_cases():
    return dict(_site_case(s) for s in elementwise_sites() if s["fn"].startswith("pcb_bn_"))


BF, F32 = _lib.PCB_BF16, _lib.PCB_F32
HAND_CASES = {
    "c8_r4095": _spec(BF, 4095, 8), "c8_r4096": _spec(BF, 4096, 8), "c8_r4097_f32": _spec(F32, 4097, 8),
    "c8_r2p24_sweeps": _spec(BF, 1 << 24, 8),
    "c24_idle_thread": _spec(BF, 3 * 85 * 16 + 7, 24), "c1544_one_row_per_block": _spec(BF, 5000, 1544),
    "c2048": _spec(BF, 3001, 2048), "c2048_f32_relu": _spec(F32, 777, 2048, _lib.ACT_RELU),
    "c64_r2": _spec(BF, 2, 64), "c64_r2048_ragged": _spec(BF, 32 * 16 * 4 - 1, 64), "c64_r2049": _spec(F32, 32 * 16 * 4 + 1, 64),
    "scalar_c12": _spec(BF, 3000, 12, _lib.ACT_LEAKY, True), "scalar_c12_f32": _spec(F32, 513, 12),
    "scalar_c2056": _spec(BF, 700, 2056, _lib.ACT_RELU),
    "small_r1": _spec(BF, 1, 256), "small_r1023": _spec(BF, 1023, 256, _lib.ACT_RELU), "small_r1025": _spec(F32, 1025, 512),
    "small_r16384": _spec(BF, 16384, 256, _lib.ACT_LEAKY), "small_r2p20": _spec(BF, 1 << 20, 64, _lib.ACT_RELU6),
    **{f"act{a}{'_res' if r else ''}": _spec(BF, 3000, 64, a, r) for a in ACTS for r in (False, True)},
    "illcond_f32": _spec(F32, 200003, 64, illcond=True), "illcond_bf16": _spec(BF, 65536, 128, illcond=True),
}


def _cases():
    return {**_fixture_cases(), **HAND_CASES}


def test_fixture_sites_map_to_cases():
    """every BatchNorm site of the fixture names exactly one case, and every case name is distinct from the hand cases"""
    sites = [s for s in elementwise_sites() if s["fn"].startswith("pcb_bn_")]
    assert sites, "the fixture holds no BatchNorm site"
    names = [_site_case(s)[0] for s in sites]
    assert all(n.startswith("fx_") for n in names) and not set(names) & set(HAND_CASES)
    for s, n in zip(sites, names):
        assert _site_case(s)[0] == n and n in _cases()


# ------------------------------------------------------------------------------------------------ helpers
def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _vec(c):
    return c % 8 == 0 and c <= 2048


def _chain(count, c, per_thread_rows):
    """L of the statistics / backward-sum chains: rows per thread + rows summed per block (vector), or + warp tree (scalar)"""
    if not _vec(c):
        return math.ceil(count / 256) + 13
    rpb = 256 // (c // 8)
    grid = max(1, min(math.ceil(count / (rpb * per_thread_rows)), 3 * _nsm()))
    return math.ceil(count / (grid * rpb)) + rpb


def _rows_per_block(count, c, per_thread_rows):
    rpb = 256 // (c // 8)
    grid = max(1, min(math.ceil(count / (rpb * per_thread_rows)), 3 * _nsm()))
    return rpb * math.ceil(count / (grid * rpb))


def _act_grad(z, act, slope):
    one = torch.ones_like(z)
    if act == _lib.ACT_RELU:
        return torch.where(z > 0, one, 0 * one)
    if act == _lib.ACT_LEAKY:
        return torch.where(z > 0, one, float(torch.tensor(slope, dtype=torch.float32)) * one)
    if act == _lib.ACT_RELU6:
        return torch.where((z > 0) & (z < 6), one, 0 * one)
    return one


def _p(t):
    return None if t is None else t.data_ptr()


def _fl(x):
    """fp64 -> nearest fp32, back in fp64"""
    return x.float().double()


def _fwd_candidates(x64, sc, sh, act, slope, res):
    """the two roundings of act(x * scale + shift) [+ residual] in fp32: unfused and contracted"""
    x32 = x64.float()
    outs = []
    for z in ((x32 * sc.float()) + sh.float(), (x64 * sc.double() + sh.double()).float()):
        z = act_ref(z, act, slope, f32_slope=True)
        if res is not None:
            z = z + res.float()
        outs.append(z)
    return outs


def _coef_ref(S, Q, dS, dQ, count, g, b):
    """fp64 mean / var / invstd / scale / shift from (S, Q) and their bounds (module docstring)"""
    n = float(count)
    m = S / n
    var = (Q / n - m * m).clamp_min(0)
    EPS, MOM = EPS_F, MOM_F
    dm = dS / n + U * m.abs() + 2.0 ** -50 * m.abs()
    dv = dQ / n + (2 * m.abs() + dS / n) * dS / n + 2.0 ** -50 * (Q.abs() / n + m * m)
    inv = 1 / torch.sqrt(var + EPS)
    rel = (dv + U * (2 * var + EPS + 2 * dv)) / (2 * (var + EPS)) * 1.01 + 2 * U
    sc = g * inv
    sh = b - m * g * inv
    d_sc = (g * inv).abs() * rel + U * sc.abs()
    d_sh = (g * inv).abs() * dm + (m * g * inv).abs() * (rel + 2 * U) + U * sh.abs() + U * b.abs()
    return dict(m=m, var=var, inv=inv, sc=sc, sh=sh, dm=dm, dv=dv, d_inv=inv * rel, d_sc=d_sc, d_sh=d_sh)


def _check_coef(name, R, mean, invstd, scale, shift):
    for tag, got, ref, bd in (("mean", mean, R["m"], R["dm"]), ("invstd", invstd, R["inv"], R["d_inv"]),
                              ("scale", scale, R["sc"], R["d_sc"]), ("shift", shift, R["sh"], R["d_sh"])):
        assert_within(f"{name}: {tag}", got, ref, bd)


def _check_running(name, R, rm0, rv0, rm, rv, count):
    MOM = MOM_F
    unb = R["var"] * count / (count - 1) if count > 1 else R["var"]
    d_unb = (R["dv"] + 2 * U * R["var"]) * (count / (count - 1) if count > 1 else 1) + 3 * U * unb
    rm_ref = (1 - MOM) * rm0.double() + MOM * R["m"]
    rv_ref = (1 - MOM) * rv0.double() + MOM * unb
    assert_within(f"{name}: running mean", rm, rm_ref, MOM * R["dm"] + 3 * U * ((1 - MOM) * rm0.double().abs() + MOM * R["m"].abs()) + 1e-7 * MOM * R["m"].abs())
    assert_within(f"{name}: running var", rv, rv_ref, MOM * d_unb + 3 * U * ((1 - MOM) * rv0.double().abs() + MOM * unb) + 1e-7 * MOM * unb)


# ------------------------------------------------------------------------------------------------ the test
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(_cases()))
def test_batchnorm_vs_fp64(name):
    sp = _cases()[name]
    dev = torch.device("cuda:0")
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    dcode, count, c, act = sp["dtype"], sp["count"], sp["c"], sp["act"]
    dt = DTYPES[dcode][1]
    vec, small = _vec(c), _vec(c) and count <= SMALL_MAX
    gen = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))

    def ints(*shape, lo=-4, hi=4):
        return torch.randint(lo, hi + 1, shape, generator=gen, device=dev).double()

    # ================= integer regime
    x = ints(count, c).to(dt)
    x64 = x.double()
    res = ints(count, c).to(dt) if sp["res"] else None
    rows = _rows_per_block(count, c, 16) if vec else math.ceil(count / 8)
    assert rows * 16 < 2 ** 24, f"{name}: statistics partials could round: not an exact case"
    S, Q = x64.sum(0), (x64 * x64).sum(0)
    gamma = (ints(c, lo=1, hi=16) / 8 * torch.where(ints(c) >= 0, 1.0, -1.0)).float()
    beta = (ints(c, lo=-16, hi=16) / 8).float()
    rm0, rv0 = torch.randn(c, generator=gen, device=dev), torch.rand(c, generator=gen, device=dev) + 0.5
    # the backward's own dyadic coefficients, and the thinned gradient
    bsc = (ints(c, lo=1, hi=8) / 8 * torch.where(ints(c) >= 0, 1.0, -1.0)).float()
    bsh = (ints(c, lo=-8, hi=8) / 8).float()
    bmu = (ints(c, lo=-4, hi=4) / 4).float()
    binv = (2.0 ** -ints(c, lo=0, hi=3)).float()
    keep = min(1.0, 2 ** 23 / (count * 4 * 128))      # E|term| < 4: the sum stays near 2^22 units, asserted below
    gy = ints(count, c)
    if keep < 1:
        gy = gy * (torch.rand(count, c, generator=gen, device=dev) < keep)
    gy = gy.to(dt)
    g64 = gy.double()
    z = x64 * bsc.double() + bsh.double()
    gz = g64 * _act_grad(z, act, SLOPE_INT)
    t_gx = gz * (x64 - bmu.double()) * binv.double()
    assert float(t_gx.abs().sum(0).max()) * 128 < 2 ** 24 and float(gz.abs().sum(0).max()) * 128 < 2 ** 24, \
        f"{name}: backward partials could round: not an exact case"
    SG, SGX = gz.sum(0), t_gx.sum(0)
    msum = torch.randint(0, 10, (count,), generator=gen, device=dev).float()           # 0 = hole; 3, 5, 6, 7, 9: not 2^k
    coef_b = torch.stack([bsc, bsh, bmu, binv]).contiguous()

    sum_a, sq_a = nan(c, dtype=torch.float64), nan(c, dtype=torch.float64)
    sums_al = nan(2, c, dtype=torch.float64)
    acc0 = ints(2, c, lo=-1000, hi=1000)
    sums_acc = acc0.clone()
    y_fused, coef = nan(count, c, dtype=dt), nan(4, c)
    rm_f, rv_f, nbt_f = rm0.clone(), rv0.clone(), torch.tensor([5], dtype=torch.int64, device=dev)
    scale_t, shift_t, mean_t, inv_t = nan(c), nan(c), nan(c), nan(c)
    rm_t, rv_t, nbt_t = rm0.clone(), rv0.clone(), torch.tensor([7], dtype=torch.int64, device=dev)
    y_t = nan(count, c, dtype=dt)
    scale_e, shift_e = nan(c), nan(c)
    y_e, y_a = nan(count, c, dtype=dt), nan(count, c, dtype=dt)
    sg_a, sgx_a, red_al = nan(c, dtype=torch.float64), nan(c, dtype=torch.float64), nan(2, c, dtype=torch.float64)
    red_acc = acc0.clone()
    exact = torch.stack([SG, SGX])
    dx_t, dx_r, dx_e, dx_a = (nan(count, c, dtype=dt) for _ in range(4))
    dg_t, db_t, dg_r, db_r = nan(c), nan(c), nan(c), nan(c)
    dx_s, dx_sm, dg_s, db_s, dg_sm, db_sm = nan(count, c, dtype=dt), nan(count, c, dtype=dt), nan(c), nan(c), nan(c), nan(c)
    exact_sums = torch.stack([S, Q]).contiguous()
    bargs = (bsc.data_ptr(), bsh.data_ptr(), bmu.data_ptr(), binv.data_ptr(), act, SLOPE_INT)
    ex = exact.contiguous()
    state = [(t, float("nan")) for t in (sum_a, sq_a, sums_al, y_fused, coef, scale_t, shift_t, mean_t, inv_t, y_t, scale_e, shift_e,
                                         y_e, y_a, sg_a, sgx_a, red_al, dx_t, dx_r, dx_e, dx_a, dg_t, db_t, dg_r, db_r, dx_s, dx_sm,
                                         dg_s, db_s, dg_sm, db_sm)]
    state += [(sums_acc, acc0), (red_acc, acc0), (rm_f, rm0), (rv_f, rv0), (nbt_f, 5), (rm_t, rm0), (rv_t, rv0), (nbt_t, 7)]

    def run():
        _lib.check(lib.pcb_bn_stats(x.data_ptr(), dcode, count, c, sum_a.data_ptr(), sq_a.data_ptr(), st))
        _lib.check(lib.pcb_bn_stats(x.data_ptr(), dcode, count, c, sums_al[0].data_ptr(), sums_al[1].data_ptr(), st))
        _lib.check(lib.pcb_bn_stats_acc(x.data_ptr(), dcode, count, c, sums_acc.data_ptr(), st))
        if vec:
            _lib.check(lib.pcb_bn_forward_fused(x.data_ptr(), dcode, count, c, exact_sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                rm_f.data_ptr(), rv_f.data_ptr(), nbt_f.data_ptr(), MOM, EPS, act, SLOPE_INT, _p(res),
                                                y_fused.data_ptr(), coef.data_ptr(), st))
        _lib.check(lib.pcb_bn_finalize(exact_sums[0].data_ptr(), exact_sums[1].data_ptr(), count, c, gamma.data_ptr(), beta.data_ptr(),
                                       rm_t.data_ptr(), rv_t.data_ptr(), nbt_t.data_ptr(), MOM, EPS, 1, scale_t.data_ptr(),
                                       shift_t.data_ptr(), mean_t.data_ptr(), inv_t.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_forward(x.data_ptr(), dcode, count, c, scale_t.data_ptr(), shift_t.data_ptr(), act, SLOPE_INT,
                                          _p(res), y_t.data_ptr(), st))
        _lib.check(lib.pcb_bn_finalize(None, None, count, c, gamma.data_ptr(), beta.data_ptr(), rm0.data_ptr(), rv0.data_ptr(), None,
                                       MOM, EPS, 0, scale_e.data_ptr(), shift_e.data_ptr(), None, None, st))
        _lib.check(lib.pcb_bn_act_forward(x.data_ptr(), dcode, count, c, scale_e.data_ptr(), shift_e.data_ptr(), act, SLOPE_INT,
                                          _p(res), y_e.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_forward(x.data_ptr(), dcode, count, c, None, None, act, SLOPE_INT, _p(res), y_a.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_backward_reduce(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, sg_a.data_ptr(),
                                                  sgx_a.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_backward_reduce(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, red_al[0].data_ptr(),
                                                  red_al[1].data_ptr(), st))
        if vec:
            _lib.check(lib.pcb_bn_act_backward_reduce_acc(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, red_acc.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, ex[0].data_ptr(), ex[1].data_ptr(),
                                                 1, dx_t.data_ptr(), dg_t.data_ptr(), db_t.data_ptr(), st))
        if vec:
            _lib.check(lib.pcb_bn_act_backward_apply_renorm(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, ex[0].data_ptr(),
                                                            ex[1].data_ptr(), 1, msum.data_ptr(), dx_r.data_ptr(), dg_r.data_ptr(),
                                                            db_r.data_ptr(), st))
        _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), dcode, count, c, bsc.data_ptr(), bsh.data_ptr(), None, None,
                                                 act, SLOPE_INT, None, None, 0, dx_e.data_ptr(), None, None, st))
        _lib.check(lib.pcb_bn_act_backward_apply(gy.data_ptr(), x.data_ptr(), dcode, count, c, None, None, None, None, act, SLOPE_INT,
                                                 None, None, 0, dx_a.data_ptr(), None, None, st))
        if small:
            _lib.check(lib.pcb_bn_act_backward_small(gy.data_ptr(), x.data_ptr(), dcode, count, c, coef_b.data_ptr(), act, SLOPE_INT,
                                                     None, dx_s.data_ptr(), dg_s.data_ptr(), db_s.data_ptr(), st))
            _lib.check(lib.pcb_bn_act_backward_small(gy.data_ptr(), x.data_ptr(), dcode, count, c, coef_b.data_ptr(), act, SLOPE_INT,
                                                     msum.data_ptr(), dx_sm.data_ptr(), dg_sm.data_ptr(), db_sm.data_ptr(), st))

    want = (VEC_KERNELS | ({"bn_bwd_small_kernel"} if small else set())) if vec else SCALAR_KERNELS

    def check(records):
        ran = {k for k, _ in records if k.startswith("bn_")}
        assert ran == want, f"{name}: ran {sorted(ran)}, the case covers {sorted(want)}"
    traced(name, run, check, state)

    # statistics: exact
    for tag, a, b in (("separate", sum_a, sq_a), ("aliased", sums_al[0], sums_al[1])):
        assert_bitwise(f"{name}: sum ({tag})", a, S)
        assert_bitwise(f"{name}: sum of squares ({tag})", b, Q)
    assert_bitwise(f"{name}: accumulated sums", sums_acc, acc0 + torch.stack([S, Q]))

    # forward: coefficients within the bounds, y exact given them
    R = _coef_ref(S, Q, 0 * S, 0 * Q, count, gamma.double(), beta.double())
    if vec:
        _check_coef(f"{name}: fused forward", R, coef[2], coef[3], coef[0], coef[1])
        _check_running(f"{name}: fused forward", R, rm0, rv0, rm_f, rv_f, count)
        assert int(nbt_f) == 6, f"{name}: num_batches_tracked must grow by exactly 1 per call, got {int(nbt_f) - 5}"
        assert_bitwise(f"{name}: fused forward y", y_fused, *(v.to(dt) for v in _fwd_candidates(x64, coef[0], coef[1], act, SLOPE_INT, res)))
    _check_coef(f"{name}: finalize", R, mean_t, inv_t, scale_t, shift_t)
    _check_running(f"{name}: finalize", R, rm0, rv0, rm_t, rv_t, count)
    assert int(nbt_t) == 8, f"{name}: pcb_bn_finalize must bump num_batches_tracked by 1"
    assert_bitwise(f"{name}: finalize + apply y", y_t, *(v.to(dt) for v in _fwd_candidates(x64, scale_t, shift_t, act, SLOPE_INT, res)))
    inv_e = 1 / torch.sqrt(rv0.double() + EPS)
    assert_within(f"{name}: eval scale", scale_e, gamma.double() * inv_e, (gamma.double() * inv_e).abs() * 4 * U)
    assert_within(f"{name}: eval shift", shift_e, beta.double() - rm0.double() * gamma.double() * inv_e,
                   (rm0.double() * gamma.double() * inv_e).abs() * 6 * U + U * beta.double().abs() * 2)
    assert_bitwise(f"{name}: eval forward y", y_e, *(v.to(dt) for v in _fwd_candidates(x64, scale_e, shift_e, act, SLOPE_INT, res)))
    ya = act_ref(x64.float(), act, SLOPE_INT, f32_slope=True) + (res.float() if res is not None else 0)
    assert_bitwise(f"{name}: activation-only forward y", y_a, ya.to(dt))

    # backward: exact
    for tag, a, b in (("separate", sg_a, sgx_a), ("aliased", red_al[0], red_al[1])):
        assert_bitwise(f"{name}: sum gz ({tag})", a, SG)
        assert_bitwise(f"{name}: sum gz xhat ({tag})", b, SGX)
    if vec:
        assert_bitwise(f"{name}: accumulated backward sums", red_acc, acc0 + exact)
    inv_n = torch.tensor(1.0, dtype=torch.float32, device=dev) / torch.tensor(float(count), dtype=torch.float32, device=dev)
    sc32, mu64 = bsc, bmu.double()
    B = ((-sc32 * binv) * SGX.float()) * inv_n
    C = (-sc32 * SG.float()) * inv_n
    inner = (B.double() * (x64 - mu64) + C.double()).float()
    d = (sc32.double() * gz + inner.double()).float()
    rs = torch.where(msum == 0, torch.zeros_like(msum), (1 / msum.double()).float())
    d_r = d * rs[:, None]
    if vec:
        assert_bitwise(f"{name}: apply dx", dx_t, d.to(dt))
        assert_bitwise(f"{name}: apply_renorm dx", dx_r, d_r.to(dt))
        for tag, dg, db in (("apply", dg_t, db_t), ("apply_renorm", dg_r, db_r)):
            assert_bitwise(f"{name}: {tag} dgamma", dg, SGX.float())
            assert_bitwise(f"{name}: {tag} dbeta", db, SG.float())
    else:
        # sc * ((gz - sg * ic) - (xhat * sgx) * ic): either subtraction may be contracted with its product
        xhat = (x64 - mu64) * binv.double()
        ic = inv_n.double()
        p1, q = SG.float().double() * ic, _fl(xhat * SGX.float().double())
        outs = [_fl(sc32.double() * t2).float().to(dt)
                for t1 in (_fl(gz - _fl(p1)), _fl(gz - p1)) for t2 in (_fl(t1 - _fl(q * ic)), _fl(t1 - q * ic))]
        ok = (dx_t == outs[0]) | (dx_t == outs[1]) | (dx_t == outs[2]) | (dx_t == outs[3])
        assert bool(ok.all()), f"{name}: scalar apply dx: {int((~ok).sum())} elements match none of the four roundings"
        assert_bitwise(f"{name}: dgamma", dg_t, SGX.float())
        assert_bitwise(f"{name}: dbeta", db_t, SG.float())
        assert bool(dx_r.isnan().all()) and bool(dg_r.isnan().all()), f"{name}: apply_renorm must not run on this route"
    assert_bitwise(f"{name}: eval apply dx", dx_e, (sc32.double() * gz).float().to(dt))
    assert_bitwise(f"{name}: activation-only apply dx", dx_a, (g64 * _act_grad(x64, act, SLOPE_INT)).float().to(dt))
    if small:
        assert_bitwise(f"{name}: small dx", dx_s, d.to(dt))
        assert_bitwise(f"{name}: small dx (renorm)", dx_sm, d_r.to(dt))
        for tag, dg, db in (("small", dg_s, db_s), ("small renorm", dg_sm, db_sm)):
            assert_bitwise(f"{name}: {tag} dgamma", dg, SGX.float())
            assert_bitwise(f"{name}: {tag} dbeta", db, SG.float())

    # refusals on the scalar route: nothing launched, nothing written
    if not vec:
        before = _lib.launch_count()
        y0, cf0, nb0 = nan(count, c, dtype=dt), nan(4, c), torch.tensor([5], dtype=torch.int64, device=dev)
        rm1, rv1, s0 = rm0.clone(), rv0.clone(), acc0.clone()
        dx0 = nan(count, c, dtype=dt)
        assert lib.pcb_bn_forward_fused(x.data_ptr(), dcode, count, c, exact_sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                        rm1.data_ptr(), rv1.data_ptr(), nb0.data_ptr(), MOM, EPS, act, SLOPE_INT, None, y0.data_ptr(),
                                        cf0.data_ptr(), st) != 0
        assert lib.pcb_bn_act_backward_reduce_acc(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, s0.data_ptr(), st) != 0
        assert lib.pcb_bn_act_backward_apply_renorm(gy.data_ptr(), x.data_ptr(), dcode, count, c, *bargs, ex[0].data_ptr(),
                                                    ex[1].data_ptr(), 1, msum.data_ptr(), dx0.data_ptr(), None, None, st) != 0
        torch.cuda.synchronize()
        assert _lib.launch_count() == before, f"{name}: a refused call launched a kernel"
        assert bool(y0.isnan().all()) and bool(cf0.isnan().all()) and int(nb0) == 5 and bool(dx0.isnan().all())
        assert bool((rm1 == rm0).all()) and bool((rv1 == rv0).all()) and bool((s0 == acc0).all())
    del x, x64, gy, g64, z, gz, t_gx, y_fused, y_t, y_e, y_a, dx_t, dx_r, dx_e, dx_a, dx_s, dx_sm, d, d_r, inner, res

    # ================= Gaussian regime: fp32 storage, the forward's own coefficients, derived bounds
    xg = torch.randn(count, c, generator=gen, device=dev)
    if sp["illcond"]:
        xg = xg + torch.where(torch.arange(c, device=dev) % 2 == 0, 64.0, 1.0) * (1 + torch.rand(c, generator=gen, device=dev))
    xg64 = xg.double()
    rg = torch.randn(count, c, generator=gen, device=dev) if sp["res"] else None
    L = _chain(count, c, 16)
    ax = xg64.abs()
    Sg, Qg = xg64.sum(0), (xg64 * xg64).sum(0)
    dS, dQ = (L + 1) * U * ax.sum(0), (L + 2) * U * (ax * ax).sum(0)
    sums = nan(2, c, dtype=torch.float64)
    _lib.check(lib.pcb_bn_stats(xg.data_ptr(), F32, count, c, sums[0].data_ptr(), sums[1].data_ptr(), st))
    torch.cuda.synchronize()
    assert_within(f"{name}: Gaussian sum", sums[0], Sg, dS)
    assert_within(f"{name}: Gaussian sum of squares", sums[1], Qg, dQ)
    # the two-pass reference of mean and variance
    m2 = Sg / count
    var2 = ((xg64 - m2) ** 2).sum(0) / count
    Rg = _coef_ref(Sg, var2 * count + m2 * m2 * count, dS, dQ + 2.0 ** -50 * Qg, count, gamma.double(), beta.double())
    Rg["var"] = var2
    if not vec:
        return
    y, cf = nan(count, c), nan(4, c)
    rm_g, rv_g, nb_g = rm0.clone(), rv0.clone(), torch.tensor([0], dtype=torch.int64, device=dev)
    _lib.check(lib.pcb_bn_forward_fused(xg.data_ptr(), F32, count, c, sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(), rm_g.data_ptr(),
                                        rv_g.data_ptr(), nb_g.data_ptr(), MOM, EPS, act, SLOPE, _p(rg), y.data_ptr(), cf.data_ptr(), st))
    torch.cuda.synchronize()
    _check_coef(f"{name}: Gaussian fused forward", Rg, cf[2], cf[3], cf[0], cf[1])
    _check_running(f"{name}: Gaussian fused forward", Rg, rm0, rv0, rm_g, rv_g, count)
    assert int(nb_g) == 1
    sc, sh, mu, iv = (cf[i].double() for i in range(4))
    zg = xg64 * sc + sh
    yref = act_ref(zg, act, SLOPE, f32_slope=True) + (rg.double() if rg is not None else 0)
    assert_within(f"{name}: Gaussian y", y, yref, 2 * U * ((xg64 * sc).abs() + sh.abs()) + U * yref.abs() * 2)
    if sp["illcond"]:                    # for comparison: torch's own (Welford) statistics kernel on the same fp32 input
        ref_inv = 1 / torch.sqrt(var2 + EPS)
        err = float(((cf[3].double() - ref_inv) / ref_inv).abs().max())
        t_err = float(((torch.batch_norm_stats(xg, EPS)[1].double() - ref_inv) / ref_inv).abs().max())
        print(f"{name}: invstd max relative error {err:.3e} (bound {float((Rg['d_inv'] / Rg['inv']).max()):.3e}), "
              f"torch.batch_norm_stats {t_err:.3e}")

    # backward from the forward's coefficients
    gg = torch.randn(count, c, generator=gen, device=dev)
    gg64 = gg.double()
    spread = 2 * U * ((xg64 * sc).abs() + sh.abs())
    lo, hi = _act_grad(zg - spread, act, SLOPE), _act_grad(zg + spread, act, SLOPE)
    kink = (lo - hi).abs()
    gzg = gg64 * _act_grad(zg, act, SLOPE)
    xm = (xg64 - mu)
    SGg, SGXg = gzg.sum(0), (gzg * xm * iv).sum(0)
    Lb = _chain(count, c, 16)
    dSG = (Lb + 1) * U * gzg.abs().sum(0) + (gg64.abs() * kink).sum(0)
    dSGX = (Lb + 4) * U * (gzg * xm * iv).abs().sum(0) + (gg64.abs() * kink * xm.abs() * iv).sum(0)
    rsum = nan(2, c, dtype=torch.float64)
    _lib.check(lib.pcb_bn_act_backward_reduce(gg.data_ptr(), xg.data_ptr(), F32, count, c, cf[0].data_ptr(), cf[1].data_ptr(),
                                              cf[2].data_ptr(), cf[3].data_ptr(), act, SLOPE, rsum[0].data_ptr(), rsum[1].data_ptr(), st))
    dxg, dgg, dbg = nan(count, c), nan(c), nan(c)
    _lib.check(lib.pcb_bn_act_backward_apply_renorm(gg.data_ptr(), xg.data_ptr(), F32, count, c, cf[0].data_ptr(), cf[1].data_ptr(),
                                                    cf[2].data_ptr(), cf[3].data_ptr(), act, SLOPE, rsum[0].data_ptr(), rsum[1].data_ptr(),
                                                    1, msum.data_ptr(), dxg.data_ptr(), dgg.data_ptr(), dbg.data_ptr(), st))
    torch.cuda.synchronize()
    assert_within(f"{name}: Gaussian sum gz", rsum[0], SGg, dSG)
    assert_within(f"{name}: Gaussian sum gz xhat", rsum[1], SGXg, dSGX)
    assert_within(f"{name}: Gaussian dbeta", dbg, SGg, dSG + U * SGg.abs())
    assert_within(f"{name}: Gaussian dgamma", dgg, SGXg, dSGX + U * SGXg.abs())
    Bg, Cg = -sc * iv * SGXg / count, -sc * SGg / count
    dB = (sc * iv / count).abs() * (dSGX + 4 * U * SGXg.abs())
    dC = (sc / count).abs() * (dSG + 3 * U * SGg.abs())
    dref = sc * gzg + Bg * xm + Cg
    bd = xm.abs() * dB + dC + U * (xm.abs() * Bg.abs() + 2 * (Bg * xm + Cg).abs() + 2 * dref.abs()) + (sc * gg64).abs() * kink + 2 * U * (sc * gzg).abs()
    s64 = msum.double()[:, None]
    rsd = torch.where(s64 == 0, torch.zeros_like(s64), 1 / torch.where(s64 == 0, torch.ones_like(s64), s64))
    assert_within(f"{name}: Gaussian apply_renorm dx", dxg, dref * rsd, (bd + 2 * U * dref.abs()) * rsd)
    if small:
        dxs, dgg, dbg = nan(count, c), nan(c), nan(c)
        _lib.check(lib.pcb_bn_act_backward_small(gg.data_ptr(), xg.data_ptr(), F32, count, c, cf.data_ptr(), act, SLOPE, None,
                                                 dxs.data_ptr(), dgg.data_ptr(), dbg.data_ptr(), st))
        torch.cuda.synchronize()
        Ls = math.ceil(count / 1024) + 5 + 32
        dSGs = (Ls + 1) * U * gzg.abs().sum(0) + (gg64.abs() * kink).sum(0)
        dSGXs = (Ls + 4) * U * (gzg * xm * iv).abs().sum(0) + (gg64.abs() * kink * xm.abs() * iv).sum(0)
        assert_within(f"{name}: Gaussian small dbeta", dbg, SGg, dSGs)
        assert_within(f"{name}: Gaussian small dgamma", dgg, SGXg, dSGXs)
        dBs = (sc * iv / count).abs() * (dSGXs + 4 * U * SGXg.abs())
        dCs = (sc / count).abs() * (dSGs + 3 * U * SGg.abs())
        bds = xm.abs() * dBs + dCs + U * (xm.abs() * Bg.abs() + 2 * (Bg * xm + Cg).abs() + 2 * dref.abs()) + (sc * gg64).abs() * kink + 2 * U * (sc * gzg).abs()
        assert_within(f"{name}: Gaussian small dx", dxs, dref, bds)

"""What the fp64 kernel suites (test_gpu_conv_routes.py, test_gpu_dwconv.py, test_gpu_batchnorm.py, test_gpu_glue_ops.py) share:
the route trace, the assertion helpers, the activation reference, prefilled buffers, hole planes, NCHW views and the fixture
loaders.  Each suite keeps its own idea of a route and hands it to `traced` as a check on the kernel records of a trace."""
import collections
import json
import os
import re
import time
import warnings

import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from text_segmentation_image_inpainting_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HOLE_VALUE = 1024.0          # x under the holes: a read that ignores the mask is far outside any bound (exact in bf16)
SENTINEL = -8192.0           # channels past those of a strided view: inputs must not be read there, outputs not written
KERNEL_NAME = re.compile(r"(?<![A-Za-z0-9_])([A-Za-z0-9_]+?_kernel)(?:<([^()]*)>)?")
PROFILER_PAD_S = 0.05        # idle margins: the profiler drops device activity at the edges of its window
PROFILER_TRIES = 20          # traces taken at most per case (see traced)
MARKER, MARKER_CYCLES = "spin_kernel", 1000   # torch.cuda._sleep's kernel brackets every trace


# ------------------------------------------------------------------------------------------------ route traces
def kernel_records(prof):
    """(Counter of (kernel name, template arguments) -> launches, number of marker kernels) of a trace's device activity;
    the template arguments are a tuple of strings without white space, () for a kernel that is not a template"""
    records, markers = collections.Counter(), 0
    for e in prof.events():
        if getattr(e, "device_type", DeviceType.CUDA) != DeviceType.CUDA:
            continue
        if MARKER in e.name:
            markers += 1
            continue
        m = KERNEL_NAME.search(e.name)
        if m:
            args = tuple(re.sub(r"\s+", "", a) for a in m.group(2).split(",")) if m.group(2) else ()
            records[(m.group(1), args)] += 1
    return records, markers


def traced(name, fn, check, state):
    """Run fn inside a torch.profiler trace and hand the kernel records of the trace (kernel_records) to check, which raises
    AssertionError when they are not the route the case covers.  The profiler loses device activity records now and then
    (whole traces come back empty, even of several kernels and after an idle margin), so every trace is bracketed by two
    marker kernels, the second after a synchronisation, and a trace in which either marker is missing is not evidence either
    way.  Such a trace, or one that check rejects, is taken again, up to PROFILER_TRIES times, from the same state: `state`
    lists (tensor, initial value) pairs reset before each attempt (outputs back to NaN, accumulators back to their operands),
    so the last attempt is the one the value checks read.  A route is a host-side decision on the arguments alone: a wrong
    route repeats on every complete trace and still fails.  Losses come in stretches of seconds, so a case may see no
    complete trace at all: it then warns that its route went unchecked (other cases of the same route still check it) and
    keeps every value check.  Returns the records of the last complete trace, or None."""
    last = None
    for _ in range(PROFILER_TRIES):
        for t, v in state:
            t.copy_(v) if isinstance(v, torch.Tensor) else t.fill_(v)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(PROFILER_PAD_S)
            torch.cuda._sleep(MARKER_CYCLES)
            fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(MARKER_CYCLES)
            torch.cuda.synchronize()
            time.sleep(PROFILER_PAD_S)
        records, markers = kernel_records(prof)
        if markers == 2:
            last = records
            try:
                check(records)
                return records
            except AssertionError:
                pass
    if last is None:       # no complete trace: the route cannot be judged, the value checks that follow still run
        warnings.warn(f"{name}: the profiler recorded no complete trace in {PROFILER_TRIES} attempts; route not checked")
        return None
    check(last)
    return last


# ------------------------------------------------------------------------------------------------ assertions
def _equal(got, want, nan_equal):
    return (got == want) | (got.isnan() & want.isnan()) if nan_equal else got == want


def assert_bitwise(name, got, want, alt=None, nan_equal=False):
    """every element of got equals want (or alt, the other accepted rounding); NaN compares unequal unless nan_equal, which
    still fails a NaN prefill left unwritten wherever want is not NaN"""
    ok = _equal(got, want, nan_equal)
    if alt is not None:
        ok = ok | _equal(got, alt, nan_equal)
    if not bool(ok.all()):
        bad = tuple((~ok).nonzero()[0].tolist())
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements differ from the exact result; first at {list(bad)}: "
                             f"got {float(got[bad])}, want {float(want[bad])}" + ("" if alt is None else f" or {float(alt[bad])}"))


def assert_within(name, got, ref, bound):
    """|got - ref| <= bound everywhere, got finite (an unwritten NaN prefill fails); got is compared in fp64"""
    got = got.double()
    assert bool(torch.isfinite(got).all()), f"{name}: output left unwritten or not finite"
    excess = (got - ref).abs() - bound
    worst = int(excess.argmax())
    assert float(excess.max()) <= 0.0, (f"{name}: |err| exceeds the bound at flat index {worst}: err "
                                        f"{float((got - ref).abs().flatten()[worst]):.3e}, bound {float(bound.flatten()[worst]):.3e}")


# ------------------------------------------------------------------------------------------------ references and buffers
def act_ref(z, act, slope, f32_slope=False):
    """the library's activations; LeakyReLU multiplies by slope as given, or with f32_slope by fp32(slope) in z's dtype (the
    value the kernels multiply by)"""
    if act == _lib.ACT_RELU:
        return torch.where(z > 0, z, torch.zeros_like(z))
    if act == _lib.ACT_LEAKY:
        if f32_slope:
            slope = torch.tensor(slope, dtype=torch.float32, device=z.device).to(z.dtype)
        return torch.where(z > 0, z, z * slope)
    if act == _lib.ACT_RELU6:
        return z.clamp(0, 6)
    return z


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def strided(shape, cs, fill, dtype):
    """[..., cs] buffer: channels [0, shape[-1]) = fill (a tensor, or a value), [shape[-1], cs) = SENTINEL"""
    buf = torch.full((*shape[:-1], cs), SENTINEL, dtype=dtype, device="cuda")
    buf[..., :shape[-1]] = fill
    return buf


def sentinel_kept(buf, c):
    return bool((buf[..., c:] == SENTINEL).all())


def holes(n, h, w, gen):
    """uint8 plane, 1 = valid: a rectangle per image plus scattered single pixels"""
    m = (torch.rand(n, h, w, generator=gen) > 0.15).to(torch.uint8)
    for i in range(n):
        y0, x0 = int(torch.randint(0, max(1, h // 2), (1,), generator=gen)), int(torch.randint(0, max(1, w // 2), (1,), generator=gen))
        m[i, y0:y0 + max(1, h // 3), x0:x0 + max(2, w // 3)] = 0
    return m


def nchw(buf, c=None):
    """fp64 NCHW view of the first c channels (all by default) of an NHWC buffer"""
    return buf[..., :c].double().permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------ fixtures
def conv_dispatch_cases():
    """the cases of golden/conv_dispatch.json: {"conv": descriptor, "expect": host queries}"""
    with open(os.path.join(GOLDEN, "conv_dispatch.json")) as f:
        return json.load(f)["cases"]


def elementwise_sites():
    """the call sites of golden/elementwise_sites.json"""
    with open(os.path.join(GOLDEN, "elementwise_sites.json")) as f:
        return json.load(f)

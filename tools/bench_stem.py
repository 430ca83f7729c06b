"""Stem forward and weight-gradient times of the production ImageFillOrigin stem (7x7 / stride 2, 3 -> 64, 512x512, batch 8,
bf16, random holes), through the C ABI (pcb_pconv_forward / pcb_pconv_backward_weight, which reach pcb_stem_forward /
pcb_stem_wgrad).

    python tools/bench_stem.py [--calls 100] [--rounds 5] [--other-lib PATH] [--kernels] [--json OUT]

Every call is bracketed by CUDA events; the result is the median per direction over --calls calls per round.  With
--other-lib (another build of libpconv_b200.so, e.g. the parent commit's) the two libraries alternate round by round in one
process on the same inputs, and the outputs of both are compared.  --kernels adds, from a torch.profiler trace taken after the
timed rounds, each kernel's mean device time per call and direction (the mask pass, the space-to-depth pass, the GEMM).  Prints the card's name, power limit and maximum SM clock."""
import argparse
import collections
import ctypes
import json
import os
import re
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from text_segmentation_image_inpainting_b200 import _lib  # noqa: E402

N, H, W, C, CO = 8, 512, 512, 3, 64


def open_lib(path):
    lib = ctypes.CDLL(path)
    for name, (res, args) in _lib._SIGS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def conv_desc(x, mask):
    cv = _lib.Conv()
    cv.n, cv.h, cv.w, cv.cin, cv.cout, cv.kh, cv.kw = N, H, W, C, CO, 7, 7
    cv.stride, cv.pad_h, cv.pad_w, cv.dil, cv.groups, cv.ho, cv.wo = 2, 3, 3, 1, 1, H // 2, W // 2
    cv.dtype = _lib.PCB_BF16
    cv.nparts = 1
    p = cv.parts[0]
    p.x, p.mask, p.c, p.x_cstride = x.data_ptr(), mask.data_ptr(), C, 8
    return cv


class Stem:
    def __init__(self, lib, x, mask, wm, bias, dc, dev):
        self.lib, self.stream = lib, torch.cuda.current_stream().cuda_stream
        self.cv = conv_desc(x, mask)
        self.ref = ctypes.byref(self.cv)
        fe, de = ctypes.c_size_t(), ctypes.c_size_t()
        lib.pcb_conv_weight_layout(self.ref, ctypes.byref(fe), ctypes.byref(de))
        self.wf = torch.zeros(fe.value, dtype=torch.bfloat16, device=dev)
        self.wd = torch.zeros(max(1, de.value), dtype=torch.bfloat16, device=dev)
        self.ws = torch.zeros(max(16, int(lib.pcb_pconv_workspace(self.ref))), dtype=torch.uint8, device=dev)
        self.check(lib.pcb_conv_weight_prepare(self.ref, wm.data_ptr(), self.wf.data_ptr(), self.wd.data_ptr() if de.value else None, self.stream))
        m = N * (H // 2) * (W // 2)
        self.y = torch.zeros(N, H // 2, W // 2, CO, dtype=torch.bfloat16, device=dev)
        self.msum = torch.zeros(m, device=dev)
        self.newmask = torch.zeros(m, dtype=torch.uint8, device=dev)
        self.dw = torch.zeros(CO, 7, 7, C, device=dev)
        self.bias, self.dc = bias, dc

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.pcb_last_error().decode(errors="replace"))

    def fwd(self):
        self.check(self.lib.pcb_pconv_forward(self.ref, self.wf.data_ptr(), self.bias.data_ptr(), self.y.data_ptr(), CO, self.msum.data_ptr(),
                                              self.newmask.data_ptr(), self.ws.data_ptr(), self.stream))

    def wgrad(self):
        self.check(self.lib.pcb_pconv_backward_weight(self.ref, self.dc.data_ptr(), CO, self.dw.data_ptr(), self.ws.data_ptr(), self.stream))


def timed(fn, calls):
    ts = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def kernel_times(fn, calls):
    """mean device time (ms) per call of each kernel fn launches, from a torch.profiler trace of `calls` calls"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    tot = collections.Counter()
    for e in prof.events():
        if getattr(e, "device_type", None) != DeviceType.CUDA:
            continue
        m = re.search(r"([A-Za-z0-9_]+_kernel)", e.name)
        tot[m.group(1) if m else e.name[:60]] += getattr(e, "device_time", 0.0)
    return {k: round(v / calls / 1000.0, 4) for k, v in tot.most_common()}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--other-lib", default=None)
    ap.add_argument("--kernels", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_stem.py needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.zeros(N, H, W, 8, dtype=torch.bfloat16, device=dev)
    x[..., :C] = torch.randn(N, H, W, C, generator=g, device=dev).to(torch.bfloat16)
    mask = (torch.rand(N, H, W, generator=g, device=dev) > 0.2).to(torch.uint8)
    wm = torch.randn(CO, 7, 7, C, generator=g, device=dev) * 0.1
    bias = torch.randn(CO, generator=g, device=dev) * 0.1
    dc = torch.randn(N, H // 2, W // 2, CO, generator=g, device=dev).to(torch.bfloat16)
    libs = {"this": open_lib(_lib.load()._name)}
    if args.other_lib:
        libs["other"] = open_lib(os.path.abspath(args.other_lib))
    stems = {k: Stem(l, x, mask, wm, bias, dc, dev) for k, l in libs.items()}
    for s in stems.values():                 # warm-up: module load, smem opt-in, first launches
        for _ in range(5):
            s.fwd(); s.wgrad()
    torch.cuda.synchronize()
    res = {k: {"fwd_ms": [], "wgrad_ms": []} for k in stems}
    for _ in range(args.rounds):
        for k, s in stems.items():
            res[k]["fwd_ms"].append(timed(s.fwd, args.calls))
            res[k]["wgrad_ms"].append(timed(s.wgrad, args.calls))
    out = {"card": card(), "calls_per_round": args.calls, "rounds": args.rounds}
    for k, r in res.items():
        out[k] = {d: round(statistics.median(v), 4) for d, v in r.items()}
        out[k]["per_round"] = {d: [round(t, 4) for t in v] for d, v in r.items()}
    if args.kernels:
        for k, s in stems.items():
            out[k]["kernels"] = {"fwd": kernel_times(s.fwd, 20), "wgrad": kernel_times(s.wgrad, 20)}
    if "other" in stems:
        a, b = stems["this"], stems["other"]
        for s in (a, b):
            s.fwd(); s.dw.zero_(); s.wgrad()
        torch.cuda.synchronize()
        out["y_max_abs_diff"] = float((a.y.float() - b.y.float()).abs().max())
        out["dw_rel_l2"] = float((a.dw - b.dw).norm() / b.dw.norm())
        t, o = out["this"], out["other"]
        out["speedup_fwd_plus_wgrad"] = round((o["fwd_ms"] + o["wgrad_ms"]) / (t["fwd_ms"] + t["wgrad_ms"]), 3)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""Per-layer weight-gradient times of one eager ImageFillOrigin training step (512x512, batch 8, bf16).

    python tools/wgrad_layers.py [--reps 5] [--json OUT]

Every conv call of the step is bracketed by CUDA events (ops.set_profile); while that is on, the weight gradients run on
the main stream, not beside the data gradients, so each time belongs to its own launch.  The table gives, per tensor-core
wgrad call, the median over --reps profiled steps with its FLOPs and achieved TFLOP/s, then every family's total.  The
card's name, power limit and maximum SM clock are printed with it: the numbers mean nothing without them.
Development tool; the events add gaps between launches, so the totals are not bench.py values."""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from text_segmentation_image_inpainting_b200 import _lib, ops
from text_segmentation_image_inpainting_b200.engine import TrainStep
from text_segmentation_image_inpainting_b200.models.image_inpainting import ImageFillOrigin
from text_segmentation_image_inpainting_b200.synthetic import random_hole_masks


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        return out.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(0) + " (nvidia-smi unavailable)"


def measure(reps):
    """(family, layer label, call index) -> (median ms over `reps` profiled eager steps, FLOPs), in call order"""
    dev = torch.device("cuda:0")
    lib = _lib.load()
    torch.manual_seed(0)
    ts = TrainStep(ImageFillOrigin().to(dev), compute_dtype=torch.bfloat16, process_group=None, use_graph=False)
    x = torch.randn(8, 3, 512, 512).to(dev)
    m = torch.from_numpy(random_hole_masks(8, 512, 512, seed=0)).to(dev)
    for _ in range(3):
        ts.step(x, m)
    torch.cuda.synchronize()
    times = collections.defaultdict(list)      # (family, layer label, call index) -> [ms per rep]
    work = {}
    for _ in range(reps):
        rec = []
        ops.set_profile(rec)
        ts._fwd_bwd(x, m)
        torch.cuda.synchronize()
        ops.set_profile(None)
        seen = collections.Counter()
        for kind, g, s, e in rec:
            c = g.struct(None)
            tc = bool(lib.pcb_conv_uses_tensor_cores(_lib.ctypes.byref(c)))
            fam = ("tc_" if tc else "other_") + kind
            label = f"{g.cin}->{g.cout} k{g.kh} s{g.stride} d{g.dil} @{g.h}x{g.w}"
            key = (fam, label, seen[(fam, label)])
            seen[(fam, label)] += 1
            times[key].append(s.elapsed_time(e))
            work[key] = 2.0 * g.n * g.ho * g.wo * g.cout * (g.cin // g.groups) * g.kh * g.kw
    return [(k, statistics.median(v), work[k]) for k, v in times.items()]


def report(rows, families, json_path=None):
    """print the per-layer table of `families` and every family's total (optionally also as JSON)"""
    print(f"card: {card()}")
    for want in families:
        print(f"{'layer (' + want + ')':40s} {'GFLOP':>8s} {'ms':>8s} {'TFLOP/s':>8s}")
        for (fam, label, i), ms, fl in rows:
            if fam == want:
                print(f"{label:40s} {fl / 1e9:8.2f} {ms:8.3f} {fl / 1e9 / ms:8.1f}")
    fams = collections.defaultdict(lambda: [0.0, 0.0, 0])
    for (fam, _label, _i), ms, fl in rows:
        f = fams[fam]
        f[0] += fl; f[1] += ms; f[2] += 1
    for fam, (fl, ms, n) in sorted(fams.items(), key=lambda kv: -kv[1][1]):
        print(f"== {fam:12s} launches={n:3d} {fl / 1e9:8.1f} GFLOP {ms:8.3f} ms {fl / 1e9 / max(ms, 1e-9):8.1f} TFLOP/s")
    if json_path:
        with open(json_path, "w") as f:
            json.dump({"card": card(), "rows": [{"family": k[0], "layer": k[1], "call": k[2], "ms": ms, "gflop": fl / 1e9}
                                                for k, ms, fl in rows]}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    report(measure(args.reps), ("tc_wgrad",), args.json)

if __name__ == "__main__":
    main()

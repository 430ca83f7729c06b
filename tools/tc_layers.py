"""Per-layer forward and data-gradient times of one eager ImageFillOrigin training step (512x512, batch 8, bf16).

    python tools/tc_layers.py [--reps 5] [--json OUT]

The same measurement as tools/wgrad_layers.py (every conv call bracketed by CUDA events, median over --reps profiled steps,
weight gradients serialised on the main stream), tabulated for the tensor-core forward and data-gradient calls, then every
family's total, with the card's name, power limit and maximum SM clock.  Development tool; the events add gaps between
launches, so the totals are not bench.py values."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from wgrad_layers import measure, report  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    report(measure(args.reps), ("tc_fwd", "tc_dgrad"), args.json)


if __name__ == "__main__":
    main()

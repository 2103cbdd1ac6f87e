"""Timing of SamplesLoss("energy") and SamplesLoss("laplacian") on the tensor-core kernels (8 < D <= 64), with the
gaussian timed in the same run for comparison.

    python tools/bench_norms_tc.py [--reps 3] [--sizes 1000000:64,400000:16] [--out DIR]

For every (N = M, D): forward, and forward + backward w.r.t. x, of each loss; the losses alternate within every
repetition so that clock and co-tenant drift hit them alike.  Times are CUDA-event times of one call, after one
warm-up call of the same shape.  pairs/s counts the N x M pairs of the three kernel matvecs (K_xx, K_yy, K_xy) of
the forward; the backward adds the row gradients of K_xx and K_xy.  Prints one JSON line per measurement and the
card's name and power limit (nvidia-smi query) first.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import SamplesLoss  # noqa: E402

LOSSES = [("gaussian", 1.0), ("laplacian", 1.0), ("energy", None)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return q


def time_call(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1000000:64,400000:16")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_norms_tc needs a CUDA device")
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for spec in args.sizes.split(","):
        n, d = (int(v) for v in spec.split(":"))
        x = torch.rand(n, d, generator=g, device="cuda")
        y = torch.rand(n, d, generator=g, device="cuda") * 0.9 + 0.15
        calls = {}
        for loss, blur in LOSSES:
            f = SamplesLoss(loss, blur=blur if blur is not None else 0.05)
            xg = x.clone().requires_grad_(True)
            calls[(loss, "fwd")] = lambda f=f: f(x, y).item()
            calls[(loss, "fwd+bwd")] = lambda f=f, xg=xg: torch.autograd.grad(f(xg, y), xg)[0].sum().item()
        for fn in calls.values():  # warm-up: module loads, scratch allocation
            fn()
        times = {k: [] for k in calls}
        for _ in range(args.reps):
            for k, fn in calls.items():
                times[k].append(time_call(fn))
        for (loss, mode), ts in times.items():
            pairs = 3.0 * n * n + (2.0 * n * n if mode == "fwd+bwd" else 0.0)
            print(json.dumps({"loss": loss, "mode": mode, "N": n, "M": n, "D": d, "seconds": ts,
                              "pairs_per_s": [pairs / t for t in ts]}), flush=True)


if __name__ == "__main__":
    main()

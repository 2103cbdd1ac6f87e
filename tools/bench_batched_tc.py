"""Timing of SamplesLoss on batches of mid-dimensional clouds (B > 1, 8 < D <= 64): the batched tensor-core path
(one launch group per reduction for the whole batch) against the per-element loop (B one-problem losses, which call
the unbatched operators).

    python tools/bench_batched_tc.py [--reps 3] [--shapes 64:500:16,64:500:64,8:4096:16,...]

Shapes are B:N:D with M = N.  For every shape and loss (sinkhorn at blur .05, gaussian at blur 1): forward, and
forward + gradient w.r.t. x, of both paths.  The loop shares the batch's diameter, so that both paths run the same
eps-schedule.  The four (path, mode) calls alternate within every repetition so that clock and co-tenant drift hit
them alike; times are CUDA-event times of one call, after one warm-up call of each.  Prints one JSON line per
measurement and the card's name and power limit (nvidia-smi query) first.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import SamplesLoss, samples_loss  # noqa: E402
from geomloss_b200.sinkhorn import max_diameter  # noqa: E402

SHAPES = "64:500:16,64:500:64,8:4096:16,8:4096:64,2:100000:16,2:100000:64"
LOSSES = [("sinkhorn", 0.05), ("gaussian", 1.0)]


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
    ap.add_argument("--shapes", default=SHAPES)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batched_tc needs a CUDA device")
    # the batched path at every size: the size above which SamplesLoss prefers the loop is what this measures
    samples_loss.BATCHED_TC_MAX_PAIRS = float("inf")
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for spec in args.shapes.split(","):
        B, n, d = (int(v) for v in spec.split(":"))
        x = torch.rand(B, n, d, generator=g, device="cuda")
        y = torch.rand(B, n, d, generator=g, device="cuda") * 0.9 + 0.15
        diam = max_diameter(x.view(-1, d), y.view(-1, d))
        for loss, blur in LOSSES:
            f = SamplesLoss(loss, blur=blur, diameter=diam if loss == "sinkhorn" else None)
            xg = x.clone().requires_grad_(True)

            def loop(xs):
                return torch.stack([f(xs[k], y[k]) for k in range(B)])

            calls = {
                ("batched", "fwd"): lambda: f(x, y).sum().item(),
                ("loop", "fwd"): lambda: loop(x).sum().item(),
                ("batched", "fwd+grad"): lambda: torch.autograd.grad(f(xg, y).sum(), xg)[0].sum().item(),
                ("loop", "fwd+grad"): lambda: torch.autograd.grad(loop(xg).sum(), xg)[0].sum().item(),
            }
            with torch.no_grad():
                vb, vl = f(x, y), loop(x)
            rel = ((vb - vl).abs().max() / vl.abs().max()).item()
            for fn in calls.values():  # warm-up: module loads, scratch allocation
                fn()
            times = {k: [] for k in calls}
            for _ in range(args.reps):
                for k, fn in calls.items():
                    times[k].append(time_call(fn))
            for (path, mode), ts in times.items():
                print(json.dumps({"loss": loss, "blur": blur, "path": path, "mode": mode, "B": B, "N": n, "M": n,
                                  "D": d, "seconds": ts, "batched_vs_loop_rel_diff": rel}), flush=True)


if __name__ == "__main__":
    main()

"""Timing of the p = 1 Sinkhorn divergence in the tensor-core dimensions (8 < D <= 64), next to p = 2 at the same shapes.

    python tools/bench_sinkhorn_p1_tc.py [--reps 3] [--ops 1000000:16,1000000:64,400000:16,400000:64]
                                         [--loss 100000:16,100000:64] [--batched 64:500,2:100000]

Three parts, each p = 1 and p = 2 alternated within every repetition so that clock and co-tenant drift hit them alike;
times are CUDA-event times of one call after one warm-up call of each:
  * ops: one softmin (forward) and one softmin + row gradient at N = M, unit-cube clouds, eps = 0.1;
  * loss: SamplesLoss("sinkhorn", blur=0.1, scaling=0.5) forward, and forward + gradient w.r.t. x, at N = M;
  * batched: SamplesLoss on B:N batches at D = 64, the batched launch group against the per-element loop (the route
    samples_loss.BATCHED_TC_MAX_PAIRS chooses between), forward + gradient.
Pairs/s counts the N x M pairs of every reduction a call runs (softmins and row gradients).  Prints the card's name and
power limit (nvidia-smi query) first, then one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import SamplesLoss, ops, samples_loss  # noqa: E402
from geomloss_b200.sinkhorn import epsilon_schedule, max_diameter  # noqa: E402

DEV = "cuda:0"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_call(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e-3


def shapes(spec):
    return [tuple(int(float(v)) for v in s.split(":")) for s in spec.split(",") if s]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def run_ops(n, d, reps):
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.rand(n, d, device=DEV, generator=g)
    y = torch.rand(n, d, device=DEV, generator=g)
    h = torch.zeros(n, device=DEV)
    go = torch.ones(n, device=DEV)
    c = ops.default_center(x, y)
    eps = 0.1

    def fwd(p):
        return lambda: (ops.softmin_l1_raw if p == 1 else ops.softmin_raw)(eps, x, y, h, p=p, center=c)

    def grad(p):
        def f():
            xg = x.clone().requires_grad_(True)
            out = (ops.softmin_l1 if p == 1 else ops.softmin)(eps, xg, y, h, p=p, center=c)
            torch.autograd.grad(out, xg, go)
        return f

    calls = {(p, mode): (fwd(p) if mode == "fwd" else grad(p), 1 if mode == "fwd" else 2)
             for p in (1, 2) for mode in ("fwd", "fwd+grad")}
    for fn, _ in calls.values():
        fn()
    for r in range(reps):
        for (p, mode), (fn, red) in calls.items():
            t = time_call(fn)
            emit(part="ops", rep=r, p=p, mode=mode, N=n, M=n, D=d, seconds=t, pairs_per_s=red * n * n / t)


def run_loss(n, d, reps):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.rand(n, d, device=DEV, generator=g)
    y = torch.rand(n, d, device=DEV, generator=g)
    diam = max_diameter(x, y)
    calls = {}
    for p in (1, 2):
        loss = SamplesLoss("sinkhorn", p=p, blur=0.1, scaling=0.5, diameter=diam)
        n_eps = len(epsilon_schedule(p, diam, 0.1, 0.5))
        softmins = 4 * (n_eps + 2)  # init, one per eps, final extrapolation; four softmins each (debias)

        def fwd(loss=loss):
            loss(x, y)

        def both(loss=loss):
            xg = x.clone().requires_grad_(True)
            torch.autograd.grad(loss(xg, y), xg)

        calls[(p, "fwd")] = (fwd, softmins)
        calls[(p, "fwd+grad")] = (both, softmins + 2)  # + the row gradients of f_ba and f_aa
    for fn, _ in calls.values():
        fn()
    for r in range(reps):
        for (p, mode), (fn, red) in calls.items():
            t = time_call(fn)
            emit(part="loss", rep=r, p=p, mode=mode, N=n, M=n, D=d, seconds=t, pairs_per_s=red * n * n / t)


def run_batched(b, n, reps, d=64):
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.rand(b, n, d, device=DEV, generator=g)
    y = torch.rand(b, n, d, device=DEV, generator=g)
    diam = max_diameter(x.view(-1, d), y.view(-1, d))
    calls = {}
    for p in (1, 2):
        loss = SamplesLoss("sinkhorn", p=p, blur=0.1, scaling=0.5, diameter=diam)

        def batched(loss=loss):
            keep = samples_loss.BATCHED_TC_MAX_PAIRS
            samples_loss.BATCHED_TC_MAX_PAIRS = float("inf")
            try:
                xg = x.clone().requires_grad_(True)
                torch.autograd.grad(loss(xg, y).sum(), xg)
            finally:
                samples_loss.BATCHED_TC_MAX_PAIRS = keep

        def loop(loss=loss):
            xg = x.clone().requires_grad_(True)
            torch.autograd.grad(sum(loss(xg[k], y[k]) for k in range(b)), xg)

        calls[(p, "batched")] = batched
        calls[(p, "loop")] = loop
    for fn in calls.values():
        fn()
    for r in range(reps):
        for (p, path), fn in calls.items():
            emit(part="batched", rep=r, p=p, path=path, B=b, N=n, M=n, D=d, seconds=time_call(fn))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ops", default="1000000:16,1000000:64,400000:16,400000:64")
    ap.add_argument("--loss", default="100000:16,100000:64")
    ap.add_argument("--batched", default="64:500,2:100000")
    a = ap.parse_args()
    emit(card=card())
    for n, d in shapes(a.ops):
        run_ops(n, d, a.reps)
    for n, d in shapes(a.loss):
        run_loss(n, d, a.reps)
    for b, n in shapes(a.batched):
        run_batched(b, n, a.reps)


if __name__ == "__main__":
    main()

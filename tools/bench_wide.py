"""Timing of the operators above D = 64 (csrc/tcwide.cuh), next to the chunked fp32 torch softmin a user would write.

    python tools/bench_wide.py [--reps 3] [--n 200000] [--dims 128,256,512,1024] [--no-loss]

Prints the card's name and power limit first (nvidia-smi, in the same call), then one JSON line per measurement.
Times are CUDA-event times of one call after one warm-up call; the variants of one shape are alternated within every
repetition so that clock and co-tenant drift hit them alike, and the median is reported.
  * ops at N = M = n: softmin forward, softmin forward + row gradient (p = 2, eps = 0.1), gaussian and energy kernel
    convolution forward + row gradient;
  * the same softmin forward as chunked fp32 torch: x @ y.T and logsumexp over column chunks that fit in memory, TF32
    off;
  * end to end: SamplesLoss("sinkhorn", blur=.05) forward + backward at N = M = 1e4, D = 512, and at B = 16 x N = 1000,
    D = 256.
Flop model (tensor-core share of 989 TFLOP/s dense fp16): the exponent costs 3 x 2 dk + 2 x 16 flops per pair (the
hh, hl, lh products and the bf16 rank-one chunk); a row gradient runs it once per 64-dimension slice and adds GEMM 2,
2 x 2 x 128 + 2 x 64 flops per pair and slice (hi.[Y_h | Y_l], lo.Y_h).
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import SamplesLoss, ops  # noqa: E402

DEV = "cuda:0"
PEAK = 989e12


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
    return start.elapsed_time(end) / 1e3


def flops_fwd(D):
    dk = -(-D // 16) * 16
    return 3 * 2 * dk + 2 * 16


def flops_bwd(D):
    slices = -(-D // 64)
    return slices * (flops_fwd(D) + 2 * 2 * 128 + 2 * 64)


def torch_softmin(eps, x, y, h, chunk):
    """-eps logsumexp_j(h_j - |x_i - y_j|^2 / 2 eps) in fp32, column chunks, running logsumexp."""
    xx = (x * x).sum(1, keepdim=True) / 2
    acc = None
    for j in range(0, y.shape[0], chunk):
        yc = y[j:j + chunk]
        s = h[j:j + chunk] - ((y[j:j + chunk] * yc).sum(1) / 2 - x @ yc.T + xx) / eps
        m = torch.logsumexp(s, dim=1)
        acc = m if acc is None else torch.logaddexp(acc, m)
    return -eps * acc


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def bench_ops(n, D, reps):
    g = torch.Generator(device=DEV).manual_seed(D)
    x = torch.rand(n, D, device=DEV, generator=g)
    y = torch.rand(n, D, device=DEV, generator=g)
    h = torch.zeros(n, device=DEV)
    w = torch.rand(n, device=DEV, generator=g)
    go = torch.ones(n, device=DEV)
    c = ops.default_center(x, y)
    eps = 0.1
    lse = ops.softmin_wide_raw(eps, x, y, h, center=c, want_lse2=True)[1]
    free = torch.cuda.mem_get_info()[0]
    chunk = max(1024, min(n, int(free * 0.25 / (n * 4 * 3))))
    calls = {
        "softmin_fwd": lambda: ops.softmin_wide_raw(eps, x, y, h, center=c),
        "softmin_fwd_bwd": lambda: (ops.softmin_wide_raw(eps, x, y, h, center=c, want_lse2=True),
                                    ops.softmin_wide_grad_rows(eps, x, y, h, None, 0.0, lse, go, center=c)),
        "gaussian_fwd_bwd": lambda: (ops.kernel_conv_wide_raw("gaussian", x, y, w, 0.5, center=c),
                                     ops.kernel_conv_wide_grad_rows("gaussian", x, y, w, 0.5, go, center=c)),
        "energy_fwd_bwd": lambda: (ops.kernel_conv_wide_raw("energy", x, y, w, 0.5, center=c),
                                   ops.kernel_conv_wide_grad_rows("energy", x, y, w, 0.5, go, center=c)),
        "torch_fp32_softmin_fwd": lambda: torch_softmin(eps, x, y, h, chunk),
    }
    flops = {"softmin_fwd": flops_fwd(D), "softmin_fwd_bwd": flops_fwd(D) + flops_bwd(D),
             "gaussian_fwd_bwd": flops_fwd(D) + flops_bwd(D), "energy_fwd_bwd": flops_fwd(D) + flops_bwd(D)}
    torch.backends.cuda.matmul.allow_tf32 = False
    for fn in calls.values():
        fn()
    times = {k: [] for k in calls}
    for _ in range(reps):
        for k, fn in calls.items():
            times[k].append(time_call(fn))
    pairs = float(n) * n
    for k, t in times.items():
        s = median(t)
        rec = {"part": "ops", "op": k, "N": n, "M": n, "D": D, "seconds": s, "pairs_per_s": pairs / s}
        if k in flops:
            rec["tc_share"] = pairs * flops[k] / s / PEAK
        else:
            rec["chunk"] = chunk
        print(json.dumps(rec), flush=True)


def bench_loss(reps):
    for B, n, D in ((0, 10000, 512), (16, 1000, 256)):
        g = torch.Generator(device=DEV).manual_seed(n)
        lead = (B,) if B else ()
        x = torch.rand(*lead, n, D, device=DEV, generator=g).requires_grad_(True)
        y = torch.rand(*lead, n, D, device=DEV, generator=g)
        L = SamplesLoss("sinkhorn", blur=0.05)

        def step():
            v = L(x, y).sum()
            v.backward()

        step()
        t = median([time_call(step) for _ in range(reps)])
        print(json.dumps({"part": "loss", "B": B, "N": n, "M": n, "D": D, "seconds": t}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dims", default="128,256,512,1024")
    ap.add_argument("--no-loss", action="store_true")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for D in (int(d) for d in a.dims.split(",")):
        bench_ops(a.n, D, a.reps)
    if not a.no_loss:
        bench_loss(a.reps)


if __name__ == "__main__":
    main()

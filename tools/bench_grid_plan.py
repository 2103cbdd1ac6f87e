"""Timing of the plan applied to K value channels on a grid (ops.grid_plan_apply_raw, one b200ot_grid_plan_apply call)
against the evaluation it replaces, 2K + 1 grid softmins (ops.softmin_grid_axes_raw): one for the denominator and one
per channel and sign of V, P V = exp((f - softmin(log V+)) / eps) - exp((f - softmin(log V-)) / eps); then
``ot.solve_grid`` end to end.

    python tools/bench_grid_plan.py [--reps 5] [--solve 512:100]

Shapes of the operator comparison: a 1024^2 batch of 4 images with K = 2 and a 256^3 volume with K = 3.  The two
evaluations alternate within every repetition so that clock and co-tenant drift hit them alike; times are the median
CUDA-event times of one synchronised call after one warm-up call of each.  ``pairs_per_s`` counts the (output, input)
pairs of every pass (sum over axes of P N_d, times the launches of one slab chain), each one exponential, against the
MUFU.EX2 rate of b200ot_ubench measured in the same run.  Prints the card's name and power limit first (read, never
set), then one JSON line per measurement.  Needs a GPU.
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import _lib, ops, ot  # noqa: E402
from geomloss_b200.sinkhorn import log_weights  # noqa: E402

DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name}, {q}"


def time_call(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e-3, out


def mufu_rate():
    L = _lib.lib()
    sink = torch.zeros(256, dtype=torch.float32, device=DEV)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    ops_per, iters, blocks = ctypes.c_int32(0), 8192, sms * 8
    best = None
    for r in range(4):
        t, _ = time_call(lambda: _lib.check(L.b200ot_ubench(0, iters, blocks, ops._ptr(sink), ctypes.byref(ops_per),
                                                             ops._stream(DEV)), "ubench"))
        if r > 0:
            best = t if best is None else min(best, t)
    return float(blocks) * 256 * iters * ops_per.value / best


def by_softmins(eps, h, v, geo):
    """(sm0, s): the denominator's softmin and the conditional means from 2K + 1 softmins."""
    sm0 = ops.softmin_grid_axes_raw(eps, h, **geo)
    out = []
    for k in range(v.shape[0]):
        acc = torch.zeros_like(h)
        for sign in (1.0, -1.0):
            part = (sign * v[k]).clamp_min(0.0)
            smk = ops.softmin_grid_axes_raw(eps, h, log_weights(part), 1.0, **geo)
            acc = acc + sign * torch.exp((sm0 - smk) / eps)
        out.append(acc)
    return sm0, torch.stack(out)


def apply_compare(shape, K, reps, mufu):
    g = torch.Generator(device=DEV).manual_seed(0)
    h = 0.1 * torch.randn(shape, device=DEV, generator=g)
    v = torch.randn((K,) + shape, device=DEV, generator=g)
    sides = shape[1:]
    geo = dict(pitch=[1.0 / n for n in sides], periodic=[False] * len(sides))
    eps = 2.0 * (2.0 / max(sides)) ** 2  # a kernel a few pixels wide
    fused = lambda: ops.grid_plan_apply_raw(eps, h, None, 0.0, v, **geo)  # noqa: E731
    slow = lambda: by_softmins(eps, h, v, geo)  # noqa: E731
    fused(), slow()
    tf, ts = [], []
    for _ in range(reps):
        t, (ell, s) = time_call(fused)
        tf.append(t)
        t, (sm0, s_ref) = time_call(slow)
        ts.append(t)
    P = h.numel()
    pairs = sum(P * n for n in sides) * -(-K // ops.GRID_APPLY_SLAB)
    err = ((s - s_ref).abs().max() / v.abs().max()).item()
    t_f, t_s = statistics.median(tf), statistics.median(ts)
    return dict(what="grid_plan_apply", shape=list(shape), K=K, fused_s=t_f, softmins_s=t_s, speedup=t_s / t_f,
                pairs_per_s=pairs / t_f, mufu_ex2_per_s=mufu, fraction_of_mufu=pairs / t_f / mufu,
                max_diff_over_max_v=err, ell_vs_softmin=(-eps * math.log(2.0) * ell - sm0).abs().max().item())


def solve(n, max_iter, reps):
    g = torch.Generator(device=DEV).manual_seed(1)
    a = torch.rand(2, n, n, device=DEV, generator=g) + 0.1
    b = torch.rand(2, n, n, device=DEV, generator=g) + 0.1
    a, b = a / a.sum((1, 2), keepdim=True), b / b.sum((1, 2), keepdim=True)
    run = lambda: ot.solve_grid(a, b, reg=1e-3, max_iter=max_iter).potential_a  # noqa: E731
    run()
    times = [time_call(run)[0] for _ in range(reps)]
    return dict(what="solve_grid", shape=[2, n, n], max_iter=max_iter, reg=1e-3, seconds=statistics.median(times),
                softmin_calls=2 * (max_iter + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--solve", default="512:100", help="side:max_iter of the end-to-end solve_grid run (B = 2)")
    args = ap.parse_args()
    print(f"# {card()}", flush=True)
    mufu = mufu_rate()
    with torch.no_grad():
        for shape, K in (((4, 1024, 1024), 2), ((1, 256, 256, 256), 3)):
            print(json.dumps(apply_compare(shape, K, args.reps, mufu)), flush=True)
        n, it = (int(t) for t in args.solve.split(":"))
        print(json.dumps(solve(n, it, max(1, args.reps // 2))), flush=True)


if __name__ == "__main__":
    main()

"""Timing of ``SamplesLoss("sinkhorn", cost=callable)`` and of its grouped row-softmin operator
(ops.dense_softmin_rows_raw, csrc/b200ot_dense.cu dense_rows_kernel):

    python tools/bench_samples_cost.py [--reps 5] [--iters 20] [--parts a,b,c]

(a) the row kernel alone on one 16384^2 and one 32768^2 matrix: kernel device time (torch.profiler, the partials kernel
    only) and the time of the whole call (CUDA events, with its finalize); the kernel's share of the H100 SXM
    data-sheet 3.35 TB/s and of the read rate ``C.sum()`` reaches in the same run; the pair kernel of ot.solve
    (ops.dense_softmin_pair_raw, both directions) on the same matrix.
(b) one Jacobi iteration of the debiased loop (4 softmins) at N = M = 5000 and at B = 64 x 512^2: the grouped call,
    the pair kernel run once per matrix (the alternative without a new kernel), and the reference's
    ``softmin_tensorized`` formula in torch; the host enqueue time of the grouped call (a host clock around the
    calls, no synchronise) against its device time.
(c) ``SamplesLoss("sinkhorn", cost=c)`` forward + backward against the UNMODIFIED reference (oracle/_ref, imported as
    bench.py imports it; skipped when it is not installed) at N = M = 5000, D = 3 and D = 2048: time and peak memory.
The arms of (a) and (b) are alternated within every repetition after a warm-up of each; medians over the repetitions.
Prints the card's name and power limit first (read, never set), then one JSON line per measurement.  Needs a GPU.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from geomloss_b200 import SamplesLoss, ops  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return f"{name}, {q}"


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def alternate(arms, reps, iters):
    """{name: median ms} over ``reps`` windows of ``iters`` calls, the arms alternated within every repetition."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            times[k].append(timed(fn, iters))
    return {k: statistics.median(v) for k, v in times.items()}


def kernel_ms(fn, iters, names):
    """Device time per call of the kernels whose names contain one of ``names`` (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names)) / 1e3 / iters


def inputs(gen, B, N, M):
    C = torch.rand(B, N, M, device=DEV, generator=gen)
    log_w = torch.full((B, M), -math.log(M), device=DEV)
    pot = 0.01 * torch.randn(B, M, device=DEV, generator=gen)
    old = 0.01 * torch.randn(B, N, device=DEV, generator=gen)
    return C, log_w, pot, old


def part_a(args, eps=0.05):
    gen = torch.Generator(device=DEV).manual_seed(0)
    for n in (16384, 32768):
        C, log_w, pot, old = inputs(gen, 1, n, n)
        log_a = torch.full((1, n), -math.log(n), device=DEV)

        def rows():
            ops.dense_softmin_rows_raw(eps, [(C, log_w, pot, old)], alpha_old=0.5, beta=0.5)

        def pair():
            ops.dense_softmin_pair_raw(eps, C, log_a, log_w, old, pot, alpha_old=0.5, beta=0.5)

        def read():
            C.sum()

        t = alternate(dict(rows=rows, pair=pair, read=read), args.reps, args.iters)
        k_rows = kernel_ms(rows, args.iters, ("dense_rows_kernel",))
        k_pair = kernel_ms(pair, args.iters, ("dense_pair_kernel",))
        nbytes = 4.0 * n * n
        read_rate = nbytes / (t["read"] * 1e-3)
        print(json.dumps(dict(part="a", N=n, M=n, rows_kernel_ms=round(k_rows, 4), rows_call_ms=round(t["rows"], 4),
                              pair_kernel_ms=round(k_pair, 4), pair_call_ms=round(t["pair"], 4),
                              c_sum_ms=round(t["read"], 4),
                              rows_kernel_share_of_3_35TBps=round(nbytes / (k_rows * 1e-3) / HBM, 3),
                              rows_kernel_share_of_c_sum=round(nbytes / (k_rows * 1e-3) / read_rate, 3),
                              c_sum_share_of_3_35TBps=round(read_rate / HBM, 3),
                              pair_kernel_share_of_3_35TBps=round(nbytes / (k_pair * 1e-3) / HBM, 3))), flush=True)
        del C


def part_b(args, eps=0.05):
    gen = torch.Generator(device=DEV).manual_seed(1)
    for B, n in ((1, 5000), (64, 512)):
        probs = [inputs(gen, B, n, n) for _ in range(4)]
        log_a = torch.full((B, n), -math.log(n), device=DEV)

        def grouped():
            ops.dense_softmin_rows_raw(eps, probs, alpha_old=0.5, beta=0.5)

        def pair_per_matrix():
            for C, log_w, pot, old in probs:
                ops.dense_softmin_pair_raw(eps, C, log_a, log_w, old, pot, alpha_old=0.5, beta=0.5)

        def torch_formula():  # softmin_tensorized (sinkhorn_samples.py:32-71) and the loop's averaging
            for C, log_w, pot, old in probs:
                0.5 * old + 0.5 * (-eps * ((log_w + pot / eps).view(B, 1, -1) - C / eps).logsumexp(2).view(B, -1))

        t = alternate(dict(grouped=grouped, pair_per_matrix=pair_per_matrix, torch=torch_formula), args.reps,
                      args.iters)
        dev_ms = kernel_ms(grouped, args.iters, ("dense_rows_kernel", "softmin_finalize"))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            grouped()
        enqueue_us = (time.perf_counter() - t0) / args.iters * 1e6
        torch.cuda.synchronize()
        print(json.dumps(dict(part="b", B=B, N=n, M=n, softmins=4, grouped_ms=round(t["grouped"], 4),
                              pair_per_matrix_ms=round(t["pair_per_matrix"], 4), torch_ms=round(t["torch"], 4),
                              grouped_device_ms=round(dev_ms, 4), grouped_enqueue_us=round(enqueue_us, 1))),
              flush=True)
        del probs


def half_sqdist_mm(x, y):
    """|x - y|^2 / 2 through one matmul, at any D."""
    return ((x * x).sum(-1)[:, :, None] + (y * y).sum(-1)[:, None, :] - 2 * x @ y.transpose(1, 2)) / 2


def reference_samples_loss():
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(ref_dir):
        return None
    sys.path.insert(0, ref_dir)
    try:
        from geomloss import SamplesLoss as RefSamplesLoss
    finally:
        sys.path.remove(ref_dir)
    return RefSamplesLoss


def part_c(args):
    Ref = reference_samples_loss()
    gen = torch.Generator(device=DEV).manual_seed(2)
    for D in (3, 2048):
        x = torch.rand(5000, D, device=DEV, generator=gen) / math.sqrt(D)
        y = torch.rand(5000, D, device=DEV, generator=gen) / math.sqrt(D)
        arms = {"engine": SamplesLoss}
        if Ref is not None:
            arms["reference"] = Ref
        res, vals = {}, {}
        for _ in range(2):  # warm-up, then one alternated measurement window per repetition
            for name, cls in arms.items():
                xg = x.clone().requires_grad_(True)
                v = cls("sinkhorn", cost=half_sqdist_mm, backend="tensorized")(xg, y)
                v.backward()
                vals[name] = float(v)
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for name, cls in arms.items():
                xg = x.clone().requires_grad_(True)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                cls("sinkhorn", cost=half_sqdist_mm, backend="tensorized")(xg, y).backward()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3)
                res[name + "_peak_MiB"] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        for name in arms:
            res[name + "_fwd_bwd_ms"] = round(statistics.median(times[name]), 2)
        print(json.dumps(dict(part="c", N=5000, M=5000, D=D, **res, values=vals,
                              reference="oracle/_ref" if Ref is not None else "not installed")), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--parts", default="a,b,c")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_samples_cost.py needs a CUDA device")
    print(card(), flush=True)
    parts = args.parts.split(",")
    for name, fn in (("a", part_a), ("b", part_b), ("c", part_c)):
        if name in parts:
            fn(args)


if __name__ == "__main__":
    main()

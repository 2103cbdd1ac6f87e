"""Timing of one symmetric Sinkhorn update on an explicit cost matrix: the fused pair update
(ops.dense_softmin_pair_raw, one pass over C for both potentials) against the reference's ``softmin_dense`` formula
restated in torch on C and on a contiguous copy of C^T (ot/_implementations/matrix.py:29-94, :646-651), with the
same averaging.

    python tools/bench_ot_matrix.py [--reps 5] [--shapes 1:4096:4096,1:16384:16384,1:32768:32768,64:512:512]

A shape is B:N:M.  The two paths are alternated within every repetition after one warm-up call of each, and timed
with CUDA events over ``--iters`` updates; the median over repetitions is reported.  Effective bandwidth counts the
4 B N M bytes of C one update must read, over the fused time, and its share of the H100 SXM data-sheet 3.35 TB/s.
``fused_kernel_ms`` is the device time of the update's three kernels from torch.profiler (below ``fused_ms`` where
the host enqueue of a small update is the bound), and ``torch_sum_read`` the share a plain ``C.sum()`` reaches: the
read rate the card delivers in the same run.
``solve_ms`` is one ``ot.solve_batch(max_iter=100)``.  Peak memory is what one update of each path allocates above C
(and C^T for torch).  ``max_diff`` is the largest difference between the two paths' potentials.  Prints the card's
name and power limit first (read, never set), then one JSON line per shape.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import ops, ot  # noqa: E402
from geomloss_b200.sinkhorn import log_weights  # noqa: E402

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


def torch_pair(eps, C, CT, log_a, log_b, f, g):
    """softmin_dense on C and C^T (scores materialised, then logsumexp), averaged like the solver's loop."""
    ft = -eps * torch.logsumexp((log_b + g / eps)[:, None, :] - C / eps, dim=2)
    gt = -eps * torch.logsumexp((log_a + f / eps)[:, None, :] - CT / eps, dim=2)
    return 0.5 * (f + ft), 0.5 * (g + gt)


def fused_pair(eps, C, CT, log_a, log_b, f, g):
    return ops.dense_softmin_pair_raw(eps, C, log_a, log_b, f, g, alpha_old=0.5, beta=0.5)[:2]


def timed(fn, iters, *args):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        out = fn(*args)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters, out


def profiled_kernel_ms(iters, *args):
    """Device time per update of the kernels of the fused path (the pass and its two finalizes), from torch.profiler:
    what one update costs once host enqueue is out of the picture."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fused_pair(*args)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "dense_pair" in e.key or "softmin_finalize" in e.key)
    return us / 1e3 / iters


def peak_extra(fn, *args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn(*args)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1:4096:4096,1:16384:16384,1:32768:32768,64:512:512")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ot_matrix.py needs a CUDA device")
    print(card(), flush=True)
    for shape in args.shapes.split(","):
        B, N, M = (int(s) for s in shape.split(":"))
        gen = torch.Generator(device=DEV).manual_seed(0)
        C = torch.rand(B, N, M, device=DEV, generator=gen)
        CT = C.transpose(1, 2).contiguous()
        log_a = log_weights(torch.full((B, N), 1.0 / N, device=DEV))
        log_b = log_weights(torch.full((B, M), 1.0 / M, device=DEV))
        f = 0.01 * torch.randn(B, N, device=DEV, generator=gen)
        g = 0.01 * torch.randn(B, M, device=DEV, generator=gen)
        eps = 0.05
        inputs = (eps, C, CT, log_a, log_b, f, g)
        (fa, ga), (fb, gb) = fused_pair(*inputs), torch_pair(*inputs)  # warm-up
        max_diff = max(float((fa - fb).abs().max()), float((ga - gb).abs().max()))
        t_fused, t_torch = [], []
        for _ in range(args.reps):
            t_fused.append(timed(fused_pair, args.iters, *inputs)[0])
            t_torch.append(timed(torch_pair, args.iters, *inputs)[0])
        mem_fused, mem_torch = peak_extra(fused_pair, *inputs), peak_extra(torch_pair, *inputs)
        kernel_ms = profiled_kernel_ms(args.iters, *inputs)
        read_ms = statistics.median(timed(torch.sum, args.iters, C)[0] for _ in range(args.reps))
        del CT
        ot.solve_batch(C, reg=eps, max_iter=2)
        torch.cuda.synchronize()
        solve_ms = timed(lambda: ot.solve_batch(C, reg=eps, max_iter=100), 1)[0]
        tf, tt = statistics.median(t_fused), statistics.median(t_torch)
        bw = 4.0 * B * N * M / (tf * 1e-3)
        kbw = 4.0 * B * N * M / (kernel_ms * 1e-3)
        print(json.dumps(dict(B=B, N=N, M=M, fused_ms=round(tf, 4), torch_ms=round(tt, 4), speedup=round(tt / tf, 2),
                              fused_kernel_ms=round(kernel_ms, 4), kernel_share_of_3_35TBps=round(kbw / HBM, 3),
                              torch_sum_read_share_of_3_35TBps=round(4.0 * B * N * M / (read_ms * 1e-3) / HBM, 3),
                              fused_spread_ms=[round(min(t_fused), 4), round(max(t_fused), 4)],
                              effective_TBps=round(bw / 1e12, 3), share_of_3_35TBps=round(bw / HBM, 3),
                              solve_100_ms=round(solve_ms, 2), peak_extra_MiB_fused=round(mem_fused / 2**20, 1),
                              peak_extra_MiB_torch=round(mem_torch / 2**20, 1), max_diff=max_diff)), flush=True)
        del C


if __name__ == "__main__":
    main()

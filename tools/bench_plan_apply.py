"""Timing of ``plan @ V`` on the fused operator (ops.plan_apply_raw) against the evaluation it replaces, one softmin
per column and sign of V, restated here from ops.softmin_raw.

    python tools/bench_plan_apply.py [--reps 3] [--shapes 1000000:3:3:signed,1000000:3:10:onehot,200000:64:64:signed]

A shape is N(=M):D:K:kind, kind = signed (gaussian V) or onehot (class indicators).  Old and new are alternated within
every repetition so that clock and co-tenant drift hit them alike; times are CUDA-event times of one synchronised call
after one warm-up call of each.  ``new`` is one application with lse2 cached (what every application after the first
costs), ``new_first`` includes the forward softmin that produces lse2.  The row-gradient kernel of the same shape
(b200ot_softmin_bwd_x: the same exponent and a D-column second reduction) is timed next to them as the yardstick, and
pairs/s counts N x M pairs per pass over the pairs.  Prints the card's name and power limit first (read, never set),
then one JSON line per measurement.  Needs a GPU: there is nothing to time without one.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import ops  # noqa: E402
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


def run(n, d, k, kind, reps):
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.rand(n, d, device=DEV, generator=g)
    y = torch.rand(n, d, device=DEV, generator=g)
    b = torch.full((n,), 1.0 / n, device=DEV)
    pot = 0.01 * torch.randn(n, device=DEV, generator=g)
    f = 0.01 * torch.randn(n, device=DEV, generator=g)
    if kind == "onehot":
        v = torch.nn.functional.one_hot(torch.randint(0, k, (n,), device=DEV, generator=g), k).float()
    else:
        v = torch.randn(n, k, device=DEV, generator=g)
    c = ops.default_center(x, y)
    reg = 2 * 0.05 ** 2 * d / 3  # C = |x - y|^2, temperature reg: the kernel runs at eps = reg / 2
    e2, inv = 0.5 * reg, 1.0 / reg
    log_b = log_weights(b)

    def old():
        # plan-weighted columns b_j V_jk as log-weights, positive and negative parts apart, one softmin each
        out = []
        for col in range(k):
            s = b * v[:, col]
            acc = torch.zeros(n, device=DEV)
            for sign in (1.0, -1.0):
                part = (sign * s).clamp_min(0.0)
                if bool((part > 0).any()):
                    sm = ops.softmin_raw(e2, x, y, log_weights(part), pot, inv, p=2, center=c, beta=2.0)[0]
                    acc = acc + sign * torch.exp((f - sm) * inv)
            out.append(acc)
        return torch.stack(out, 1)

    state = {}

    def first():
        sm, lse2 = ops.softmin_raw(e2, x, y, log_b, pot, inv, p=2, center=c, beta=2.0, want_lse2=True)
        state["lse2"], state["r"] = lse2, torch.exp((f - sm) * inv)
        return new()

    def new():
        return ops.plan_apply_raw(e2, x, y, log_b, pot, inv, state["lse2"], v, row_factor=state["r"], center=c)

    def grad_rows():
        return ops.softmin_grad_rows(e2, x, y, log_b, pot, inv, state["lse2"], b, p=2, center=c)

    calls = {"old": old, "new_first": first, "new": new, "row_gradient": grad_rows}
    outs = {name: fn() for name, fn in calls.items()}  # warm-up of every shape timed below
    scale = outs["old"].abs().max().item()
    diff = (outs["old"] - outs["new"]).abs().max().item() / scale
    times = {name: [] for name in calls}
    for _ in range(reps):
        for name, fn in calls.items():
            times[name].append(time_call(fn)[0])
    slab = 8 if d <= ops.MAX_D else 64
    passes = {"old": sum(1 + int(bool((v[:, col] < 0).any())) for col in range(k)) if kind == "signed" else k,
              "new_first": 1 + -(-k // slab), "new": -(-k // slab), "row_gradient": 1}
    for name in calls:
        t = sorted(times[name])[len(times[name]) // 2]
        print(json.dumps({"N": n, "M": n, "D": d, "K": k, "values": kind, "call": name, "median_s": round(t, 5),
                          "all_s": [round(u, 5) for u in times[name]], "passes": passes[name],
                          "pairs_per_s": round(passes[name] * float(n) * n / t, 0),
                          "speedup_vs_old": round(sorted(times["old"])[len(times["old"]) // 2] / t, 2),
                          "max_diff_old_new_rel": float(f"{diff:.3e}")}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="1000000:3:3:signed,1000000:3:10:onehot,200000:64:64:signed")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_plan_apply needs a CUDA device")
    print("card:", card(), flush=True)
    for spec in args.shapes.split(","):
        n, d, k, kind = spec.split(":")
        run(int(float(n)), int(d), int(k), kind, args.reps)

"""Timing of ``plan @ V`` on the fused operator (ops.plan_apply_raw; ops.plan_apply_wide_raw above D = 64) against
the evaluations it replaces: one softmin per column and sign of V, restated here from ops.softmin_raw (D <= 64 only:
above, K = D would take 2 D softmins), and a dense fp32 torch evaluation in row chunks with TF32 off
(x @ y.T -> softmax weights -> @ V).

    python tools/bench_plan_apply.py [--reps 3] [--shapes 1000000:3:3:signed,1000000:3:10:onehot,200000:64:64:signed]
    python tools/bench_plan_apply.py --shapes 200000:512:10:onehot,200000:512:64:signed,200000:512:512:signed
    python tools/bench_plan_apply.py --solve 100000:512:20     # solve_sample(max_iter=20) + a_to_b, N = M = 1e5

A shape is N(=M):D:K:kind, kind = signed (gaussian V) or onehot (class indicators).  The calls are alternated within
every repetition so that clock and co-tenant drift hit them alike; times are CUDA-event times of one synchronised call
after one warm-up call of each.  ``new`` is one application with lse2 cached (what every application after the first
costs), ``new_first`` includes the forward softmin that produces lse2.  The row-gradient kernel of the same shape
(b200ot_softmin_bwd_x / b200ot_wide_softmin_bwd_x: the same exponent and a D-column second reduction) is timed next
to them as the yardstick, and pairs/s counts N x M pairs per pass over the pairs.  Prints the card's name and power
limit first (read, never set), then one JSON line per measurement.  Needs a GPU: there is nothing to time without one.
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


def torch_fp32(x, y, h, inv, v, r, chunk):
    """r_i sum_j softmax_j(h_j - |x_i - y_j|^2 inv) v_j in fp32 on the CUDA cores (TF32 off), row chunks"""
    yy = (y * y).sum(1)
    out = []
    for i in range(0, x.shape[0], chunk):
        xc = x[i:i + chunk]
        logits = h[None, :] - ((xc * xc).sum(1)[:, None] - 2.0 * (xc @ y.T) + yy[None, :]) * inv
        out.append(torch.softmax(logits, dim=1) @ v)
    return r[:, None] * torch.cat(out)


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
    wide = d > ops.MAX_D_TC
    softmin = ops.softmin_wide_raw if wide else ops.softmin_raw
    apply = ops.plan_apply_wide_raw if wide else ops.plan_apply_raw
    grad = ops.softmin_wide_grad_rows if wide else ops.softmin_grad_rows
    # C = |x - y|^2, temperature reg (the kernel runs at eps = reg / 2): blur 0.05 at D = 3, reg ~ D / 120 above
    reg = 2 * 0.05 ** 2 * d / 3 if d <= ops.MAX_D_TC else d / 120.0
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
                    sm = softmin(e2, x, y, log_weights(part), pot, inv, p=2, center=c, beta=2.0)[0]
                    acc = acc + sign * torch.exp((f - sm) * inv)
            out.append(acc)
        return torch.stack(out, 1)

    state = {}

    def first():
        sm, lse2 = softmin(e2, x, y, log_b, pot, inv, p=2, center=c, beta=2.0, want_lse2=True)
        state["lse2"], state["r"] = lse2, torch.exp((f - sm) * inv)
        return new()

    def new():
        return apply(e2, x, y, log_b, pot, inv, state["lse2"], v, row_factor=state["r"], center=c)

    def grad_rows():
        return grad(e2, x, y, log_b, pot, inv, state["lse2"], b, p=2, center=c)

    def dense():
        return torch_fp32(x, y, log_b + pot * inv, inv, v, state["r"], max(1, (1 << 29) // n))

    calls = {"new_first": first, "new": new, "row_gradient": grad_rows, "torch_fp32": dense}
    if not wide:
        calls = {"old": old, **calls}
    base = "torch_fp32" if wide else "old"
    outs = {name: fn() for name, fn in calls.items()}  # warm-up of every shape timed below
    scale = outs[base].abs().max().item()
    diff = (outs[base] - outs["new"]).abs().max().item() / scale
    times = {name: [] for name in calls}
    for _ in range(reps):
        for name, fn in calls.items():
            times[name].append(time_call(fn)[0])
    slab = 8 if d <= ops.MAX_D else 64
    passes = {"old": sum(1 + int(bool((v[:, col] < 0).any())) for col in range(k)) if kind == "signed" else k,
              "new_first": 1 + -(-k // slab), "new": -(-k // slab), "row_gradient": 1, "torch_fp32": 1}
    if wide:
        passes["row_gradient"] = -(-(-(-d // 16) * 16) // 64)  # one recomputed exponent per 64-dimension slice
    for name in calls:
        t = sorted(times[name])[len(times[name]) // 2]
        print(json.dumps({"N": n, "M": n, "D": d, "K": k, "values": kind, "call": name, "median_s": round(t, 5),
                          "all_s": [round(u, 5) for u in times[name]], "passes": passes[name],
                          "pairs_per_s": round(passes[name] * float(n) * n / t, 0),
                          f"speedup_vs_{base}": round(sorted(times[base])[len(times[base]) // 2] / t, 2),
                          f"max_diff_{base}_new_rel": float(f"{diff:.3e}")}), flush=True)


def solve(n, d, max_iter, reps):
    """solve_sample(..., max_iter) then a_to_b, end to end (synchronised), unit-cube clouds, reg = D / 120"""
    from geomloss_b200 import ot

    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.rand(n, d, device=DEV, generator=g)
    y = torch.rand(n, d, device=DEV, generator=g) * 0.8 + 0.1

    def once():
        res = ot.solve_sample(x, y, reg=d / 120.0, max_iter=max_iter)
        return res.a_to_b

    once()
    for _ in range(reps):
        t, ab = time_call(once)
        assert torch.isfinite(ab).all()
        print(json.dumps({"N": n, "M": n, "D": d, "call": f"solve_sample(max_iter={max_iter}) + a_to_b",
                          "s": round(t, 4)}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="1000000:3:3:signed,1000000:3:10:onehot,200000:64:64:signed")
    ap.add_argument("--solve", default="", help="N:D:max_iter of an end-to-end solve_sample + a_to_b run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_plan_apply needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False  # the torch baseline computes in fp32
    print("card:", card(), flush=True)
    for spec in filter(None, args.shapes.split(",")):
        n, d, k, kind = spec.split(":")
        run(int(float(n)), int(d), int(k), kind, args.reps)
    if args.solve:
        n, d, it = args.solve.split(":")
        solve(int(float(n)), int(d), int(it), args.reps)

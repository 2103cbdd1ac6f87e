"""Where the time of bench.py's step goes: the four Jacobi updates of configs[1] (N = M, D = 3, p = 2, blur = .01)
timed with CUDA events (L2 flushed before every step), then, in a separate profiled run, every softmin_pair_kernel
launch of the step: its time, CTAs, registers, resident CTAs per SM, waves, and exponentials per second as a fraction
of the MUFU.EX2 rate of b200ot_ubench, with the card's name, power limit and sampled SM clock.

    python tools/bench_softmin_step.py [--n 1000000] [--steps 10] [--out DIR]

Exponentials of the step's paired kernels: N M for the xy / yx pair and, for each self update, the off-diagonal blocks
once and the diagonal blocks whole, (N^2 + sum_b |B_b|^2) / 2 over the blocks B_b of pair_blocks
(csrc/b200ot_softmin.cu).  A launch that serves the whole step is charged all of them."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pair_sizes(n):
    """Points per block of pair_blocks(n) at the default tiles per block."""
    tiles = -(-n // 1024)
    nb = -(-tiles // -(-tiles // 64))
    return [min(n, (b + 1) * tiles // nb * 1024) - b * tiles // nb * 1024 for b in range(nb)]


def resident_ctas(regs, threads, smem):
    """CTAs per SM an sm_90 SM holds at this register count (allocated per warp in units of 256), block size and
    dynamic shared memory (228 KB per SM, 1 KB reserved per CTA)."""
    warps = -(-threads // 32)
    by_regs = 65536 // (warps * (-(-regs * 32 // 256) * 256)) if regs else 32
    by_smem = (233472 // (smem + 1024)) if smem else 32
    return max(0, min(by_regs, by_smem, 64 // warps, 32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--blur", type=float, default=0.01)
    ap.add_argument("--out", default=None, help="directory for the JSON result")
    args = ap.parse_args()

    import torch

    import bench
    from geomloss_b200 import _lib, ops
    from geomloss_b200.sinkhorn import softmin_many

    dev = torch.device("cuda", 0)
    L = _lib.lib()
    n = args.n
    eps = args.blur ** 2
    g = torch.Generator().manual_seed(0)
    x, y = torch.rand(n, 3, generator=g).to(dev), torch.rand(n, 3, generator=g).to(dev)
    a_log = torch.full((n,), -math.log(n), device=dev)
    b_log = a_log.clone()
    c = ops.default_center(x, y)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    pots = [ops.softmin_raw(eps, r, col, lw, p=2, center=c)[0] for r, col, lw in
            ((x, y, b_log), (y, x, a_log), (x, x, a_log), (y, y, b_log))]
    kw = dict(p=2, center=c, alpha_old=0.5, beta=0.5)

    def step(pt):
        f, gg, fa, gb = pt
        res = softmin_many(ops.softmin_raw, [((eps, x, y, b_log, gg, 1 / eps), dict(out_old=f, **kw)),
                                             ((eps, y, x, a_log, f, 1 / eps), dict(out_old=gg, **kw)),
                                             ((eps, x, x, a_log, fa, 1 / eps), dict(out_old=fa, **kw)),
                                             ((eps, y, y, b_log, gb, 1 / eps), dict(out_old=gb, **kw))])
        return [o for o, _ in res]

    for _ in range(3):
        pots = step(pots)
    torch.cuda.synchronize(dev)
    ms = []
    sampler = bench.ClockSampler(0)
    with sampler:
        for _ in range(args.steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pots = step(pots)
            e1.record()
            torch.cuda.synchronize(dev)
            ms.append(e0.elapsed_time(e1))

    # per-kernel times from a profiled run of its own
    from torch.profiler import ProfilerActivity, profile

    prof_steps = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(prof_steps):
            flush.zero_()
            pots = step(pots)
        torch.cuda.synchronize(dev)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    kern = [e for e in trace.get("traceEvents", []) if e.get("cat") == "kernel" and "softmin_pair_kernel" in e["name"]]
    kern.sort(key=lambda e: e["ts"])
    per_step = len(kern) // prof_steps
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    mufu = bench.pipe_ceilings(L, ops, torch, dev)["mufu_ex2_per_s"]
    sym = (float(n) * n + sum(float(s) ** 2 for s in pair_sizes(n))) / 2
    exps = [float(n) * n + 2 * sym] if per_step == 1 else [float(n) * n, sym, sym][:per_step]
    kernels = []
    for k in range(per_step):
        evs = [kern[s * per_step + k] for s in range(prof_steps)]
        a = evs[0].get("args", {})
        dur_ms = sorted(e["dur"] for e in evs)[len(evs) // 2] * 1e-3
        grid = a.get("grid", [0, 1, 1])
        block = a.get("block", [0, 1, 1])
        regs = a.get("registers per thread", 0)
        smem = a.get("shared memory", 0)
        ctas = grid[0] * grid[1] * grid[2]
        per_sm = resident_ctas(regs, block[0] * block[1] * block[2], smem)
        kernels.append({"name": evs[0]["name"][:120], "ms": dur_ms, "ctas": ctas, "regs": regs, "ctas_per_sm": per_sm,
                        "waves": ctas / (per_sm * sms) if per_sm else None, "exps": exps[k],
                        "exp_per_s": exps[k] / (dur_ms * 1e-3), "frac_mufu": exps[k] / (dur_ms * 1e-3) / mufu})
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    step_ms = sorted(ms)[len(ms) // 2]
    res = {"n": n, "eps": eps, "card": smi, "clocks": sampler.summary(), "mufu_ex2_per_s": mufu,
           "step_ms_median": step_ms, "step_ms": ms, "pair_kernels_per_step": per_step,
           "pair_kernels_ms": sum(k["ms"] for k in kernels), "step_exps": sum(exps),
           "step_frac_mufu": sum(exps) / (step_ms * 1e-3) / mufu, "kernels": kernels}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_softmin_step.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

"""A/B of the paired softmins in one process: bench.py's step (the four Jacobi updates of configs[1], N = M, D = 3,
p = 2, blur = .01) with $B200OT_PAIR on and off, alternated, L2 flushed before every step; the exponentials per second
of the paired step against the MUFU.EX2 rate of b200ot_ubench; the SM clock (NVML) and the card's name and power limit.

    python tools/bench_softmin_pair.py [--n 1000000] [--steps 5] [--rounds 3] [--out DIR]

Exponentials per step: unpaired 2 N M + N^2 + M^2; paired N M for the xy / yx pair and, for each self update, the
off-diagonal blocks once and the diagonal blocks whole: (N^2 + sum_b |B_b|^2) / 2 over the blocks B_b of the
symmetric kernel (csrc/b200ot_softmin.cu, pair_blocks)."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
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

    def timed(paired, pt):
        os.environ["B200OT_PAIR"] = "1" if paired else "0"
        for _ in range(2):
            pt = step(pt)
        ms = []
        for _ in range(args.steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            pt = step(pt)
            e1.record()
            torch.cuda.synchronize(dev)
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2], pt

    arms = {"paired": [], "unpaired": []}
    sampler = bench.ClockSampler(0)
    with sampler:
        for _ in range(args.rounds):
            for name in ("unpaired", "paired"):
                t, pots = timed(name == "paired", pots)
                arms[name].append(t)
    os.environ.pop("B200OT_PAIR", None)
    mufu = bench.pipe_ceilings(L, ops, torch, dev)["mufu_ex2_per_s"]
    tiles = -(-n // 1024)
    nb = -(-tiles // -(-tiles // 64))
    sizes = [min(n, (b + 1) * tiles // nb * 1024) - b * tiles // nb * 1024 for b in range(nb)]
    exps = {"paired": float(n) * n + float(n) * n + sum(float(s) ** 2 for s in sizes), "unpaired": 4.0 * n * n}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"n": n, "eps": eps, "card": smi, "clocks": sampler.summary(), "mufu_ex2_per_s": mufu, "rounds": {}}
    for name, ts in arms.items():
        best = min(ts)
        res["rounds"][name] = {"ms_per_step": ts, "exp_per_s": exps[name] / (best * 1e-3),
                               "frac_mufu": exps[name] / (best * 1e-3) / mufu}
    res["speedup_median"] = sorted(arms["unpaired"])[len(ts) // 2] / sorted(arms["paired"])[len(ts) // 2]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_softmin_pair.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

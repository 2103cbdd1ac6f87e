"""Labelled two-scale Sinkhorn (backend="multiscale" with user labels, block-sparse tensor-core softmins above D = 8)
against the dense single-scale loss at the same blur, forward and forward + gradient.

    python tools/bench_labels_hd.py [--n 200000] [--dims 16,64] [--blobs 2000] [--runs 3] [--blur 0.05]
                                    [--cluster-scale 0.1] [--truncate 5]

Workload: N = M points in `blobs` Gaussian blobs (labels = blob ids), y a slightly shifted copy of x's blob layout.
The two paths alternate, `runs` times each.  Prints one JSON line per (D, path, pass) with the times of every run, and
per D the kept-pair fraction of the truncation mask and the fraction of pairs the kernels compute once every cluster
is padded to whole 128-point tiles (both averaged over the four fine-phase problems xy, yx, xx, yy).  The card name
and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import SamplesLoss, multiscale  # noqa: E402

DEV = "cuda:0"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def clouds(n, d, blobs, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    centers = torch.rand(blobs, d, generator=g, device=DEV) / (d / 3) ** 0.5
    s = 0.05 / d ** 0.5
    lx = torch.randint(0, blobs, (n,), generator=g, device=DEV)
    ly = torch.randint(0, blobs, (n,), generator=g, device=DEV)
    x = centers[lx] + s * torch.randn(n, d, generator=g, device=DEV)
    y = centers[ly] + 0.02 / d ** 0.5 + s * torch.randn(n, d, generator=g, device=DEV)
    # compact labels (every blob id present with overwhelming probability; relabel to be safe)
    lx = torch.unique(lx, return_inverse=True)[1]
    ly = torch.unique(ly, return_inverse=True)[1]
    a = torch.full((n,), 1.0 / n, device=DEV)
    return lx, a, x, ly, a.clone(), y


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=200000)
    ap.add_argument("--dims", default="16,64")
    ap.add_argument("--blobs", type=int, default=2000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--blur", type=float, default=0.05)
    # the scale of the jump from clusters to points: cluster_scale^2 ~ the eps at which the truncation mask is built
    # (0: the reference's default, diameter / (sqrt(D) 2000^(1/D)))
    ap.add_argument("--cluster-scale", type=float, default=0.1)
    ap.add_argument("--truncate", type=float, default=5.0)
    args = ap.parse_args()
    print(json.dumps({"card": card(), "n": args.n, "blobs": args.blobs, "blur": args.blur,
                      "cluster_scale": args.cluster_scale, "truncate": args.truncate}), flush=True)
    probs = []
    build = multiscale.LocalEngine.build

    def recording_build(self, *a, **kw):
        p = build(self, *a, **kw)
        probs.append(p)
        return p

    multiscale.LocalEngine.build = recording_build
    for d in (int(v) for v in args.dims.split(",")):
        lx, a, x, ly, b, y = clouds(args.n, d, args.blobs)
        two = SamplesLoss("sinkhorn", p=2, blur=args.blur, backend="multiscale",
                          cluster_scale=args.cluster_scale or None,
                          truncate=args.truncate)
        dense = SamplesLoss("sinkhorn", p=2, blur=args.blur, backend="online")
        paths = {"two_scale": lambda xx: two(lx, a, xx, ly, b, y), "dense": lambda xx: dense(a, xx, b, y)}
        times = {(k, ps): [] for k in paths for ps in ("fwd", "fwd_bwd")}
        values = {}
        for k, f in paths.items():  # warm-up: builds, scratch, first-launch attributes
            values[k] = f(x).item()
        probs.clear()
        for _ in range(args.runs):
            for k, f in paths.items():
                times[(k, "fwd")].append(timed(lambda: f(x)))
                xg = x.clone().requires_grad_(True)
                times[(k, "fwd_bwd")].append(timed(lambda: torch.autograd.grad(f(xg), xg)))
        kept = sum(p.density for p in probs) / max(len(probs), 1)
        computed = sum(p.computed for p in probs) / max(len(probs), 1)
        print(json.dumps({"D": d, "values": values, "kept_pairs": kept, "computed_pairs": computed}), flush=True)
        for (k, ps), ts in times.items():
            print(json.dumps({"D": d, "path": k, "pass": ps, "seconds": [round(t, 4) for t in ts]}), flush=True)
    multiscale.LocalEngine.build = build


if __name__ == "__main__":
    main()

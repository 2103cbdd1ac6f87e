"""Golden fixtures for the reference's two-scale Sinkhorn with user cluster labels above D = 3:
``SamplesLoss(backend="multiscale")(l_x, a, x, l_y, b, y)``, which always routes to ``sinkhorn_multiscale``
(_legacy/samples_loss.py:220-230) and clusters by the given labels in any dimension (``clusterize``,
_legacy/sinkhorn_samples.py:453-490; kernel truncation :493-530; the jump of sinkhorn_divergence.py:519-606).

    python tests/golden/make_golden_labels_highdim.py

Same procedure as make_golden_multiscale.py: the UNMODIFIED reference on the dense pykeops shim, fp32 and fp64 runs,
saved as ``labels_hd_*.npz``: fp64 inputs (the fp32 run reads them cast to fp32), labels, hyper-parameters, the fp64
value + autograd gradients or potentials (``*_f64``), and the fp32 run's value or potentials only, which keeps the
high-dimensional files small.  The clouds are labelled Gaussian blobs whose sizes include 1, 127, 128, 129 and a few
hundred points: cluster tiles of the tensor-core kernels that are nearly empty, exactly full and one point over.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_multiscale import npy, run  # noqa: E402  (imports the reference on the shim)

# blob sizes of x and y: up to D = 16, and (smaller files) above
SIZES = {False: ([1, 127, 128, 129, 300, 60, 17, 90], [129, 1, 300, 128, 127, 33, 78, 64]),
         True: ([1, 129, 200, 60, 17], [128, 127, 90, 33, 50])}


def save(name, a, x, b, y, kw, labels, potentials):
    arrays = dict(a_f64=npy(a), x_f64=npy(x), b_f64=npy(b), y_f64=npy(y), labels_x=npy(labels[0]),
                  labels_y=npy(labels[1]), potentials=int(potentials))
    for k, v in kw.items():
        arrays["kw_" + k] = np.array("None" if v is None else v)
    key = ("pot_f", "pot_g") if potentials else ("value",)
    r32 = run(a, x, b, y, torch.float32, labels=labels, potentials=potentials, **kw)
    r64 = run(a, x, b, y, torch.float64, labels=labels, potentials=potentials, **kw)
    arrays.update({k: r32[k] for k in key})
    arrays.update({k + "_f64": v for k, v in r64.items()})
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **arrays)
    print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB  {key[0]} fp32 {np.ravel(r32[key[0]])[:1]} "
          f"fp64 {np.ravel(r64[key[0]])[:1]}")


def blobs(seed, d, weights="random"):
    """Blobs shared by both clouds (y's shifted a little); labels = blob ids, points in random order."""
    g = torch.Generator().manual_seed(seed)
    sizes_x, sizes_y = SIZES[d > 16]
    # neighbouring blobs overlap at the final blur, so that truncation drops blocks that carry mass
    centers = 0.5 * torch.rand(len(sizes_x), d, generator=g, dtype=torch.float64) / np.sqrt(d / 3)
    shift = 0.05 * torch.randn(d, generator=g, dtype=torch.float64) / np.sqrt(d)
    s = 0.15 / np.sqrt(d)  # blob radius ~ 0.15 whatever the dimension

    def cloud(sizes, off):
        lab = torch.cat([torch.full((n,), k, dtype=torch.int32) for k, n in enumerate(sizes)])
        pts = centers[lab.long()] + off + s * torch.randn(len(lab), d, generator=g, dtype=torch.float64)
        perm = torch.randperm(len(lab), generator=g)
        return pts[perm], lab[perm]

    x, lx = cloud(sizes_x, 0.0)
    y, ly = cloud(sizes_y, shift)
    n, m = len(x), len(y)
    if weights == "uniform":
        a, b = torch.ones(n, dtype=torch.float64) / n, torch.ones(m, dtype=torch.float64) / m
    else:
        a = torch.rand(n, generator=g, dtype=torch.float64) + 0.1
        b = torch.rand(m, generator=g, dtype=torch.float64) + 0.1
        a, b = a / a.sum(), b / b.sum()
        if weights == "unbalanced":
            b = b * 1.3
    return (lx, ly), a, x, b, y


CASES = [
    # (name suffix, seed, D, weights, SamplesLoss kwargs, potentials)
    ("d5_trunc2", 1, 5, "random", dict(p=2, blur=0.1, truncate=2, cluster_scale=0.15), False),
    ("d5_p1", 2, 5, "random", dict(p=1, blur=0.1, truncate=2, cluster_scale=0.15), False),
    ("d16_trunc1", 3, 16, "random", dict(p=2, blur=0.1, truncate=1, cluster_scale=0.15), False),
    ("d16_exact", 4, 16, "uniform", dict(p=2, blur=0.1, truncate=None, cluster_scale=0.15), False),
    ("d16_potentials", 5, 16, "random", dict(p=2, blur=0.1, truncate=2, cluster_scale=0.15), True),
    ("d33_trunc3_reach", 6, 33, "unbalanced", dict(p=2, blur=0.1, reach=0.5, truncate=3, cluster_scale=0.15), False),
    ("d33_lastjump", 7, 33, "random", dict(p=2, blur=0.1, truncate=2, cluster_scale=0.05), False),
    ("d64_trunc2", 8, 64, "random", dict(p=2, blur=0.1, truncate=2, cluster_scale=0.15), False),
    ("d33_nodebias", 9, 33, "random", dict(p=2, blur=0.1, truncate=3, cluster_scale=0.15, debias=False), False),
]


def main():
    only = sys.argv[1:]
    for suffix, seed, d, w, kw, pot in CASES:
        if only and suffix not in only:
            continue
        labels, a, x, b, y = blobs(seed, d, w)
        save("labels_hd_" + suffix, a, x, b, y, dict(loss="sinkhorn", backend="multiscale", **kw), labels, pot)


if __name__ == "__main__":
    main()

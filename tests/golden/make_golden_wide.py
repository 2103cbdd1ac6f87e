"""Golden fixtures above D = 64 (the K-slab tensor-core operators) from the REAL reference.

    python tests/golden/make_golden_wide.py

Imports geomloss from /root/reference/src (or $GEOMLOSS_REFERENCE) and runs SamplesLoss(backend="tensorized") in fp32
and fp64 with autograd gradients: the Sinkhorn divergence for p = 1 and 2 and the three kernel norms at D = 96, 128
and 512, and one batched Sinkhorn.  Coordinates are uniform in a cube of side 2 / sqrt(D) (a cloud of radius about 1
whatever D: the regime where the expansion error of the tensor-core exponent stays below the potentials' bar, DESIGN.md
section 3.5d).  The reference's own fp32 run is kept for information; the tests compare with the fp64 run.  Written
as wide_*.npz, each below 1 MB (the D = 512 cases keep fewer than 128 points per cloud).
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get("GEOMLOSS_REFERENCE", "/root/reference/src"))
from geomloss import SamplesLoss  # noqa: E402

torch.set_num_threads(8)


def npy(t):
    return t.detach().cpu().numpy()


# (name, seed, B (0: unbatched), N, M, D, SamplesLoss keywords)
CASES = [
    ("wide_sinkhorn_p2_d96", 71, 0, 400, 380, 96, dict(loss="sinkhorn", p=2, blur=0.1, scaling=0.6)),
    ("wide_sinkhorn_p2_d512", 72, 0, 80, 72, 512, dict(loss="sinkhorn", p=2, blur=0.1, scaling=0.6)),
    ("wide_sinkhorn_p1_d128", 73, 0, 350, 360, 128, dict(loss="sinkhorn", p=1, blur=0.2, scaling=0.6)),
    ("wide_sinkhorn_p1_d512", 74, 0, 72, 80, 512, dict(loss="sinkhorn", p=1, blur=0.2, scaling=0.6)),
    ("wide_gaussian_d96", 75, 0, 400, 350, 96, dict(loss="gaussian", blur=0.5)),
    ("wide_laplacian_d128", 76, 0, 350, 330, 128, dict(loss="laplacian", blur=0.5)),
    ("wide_energy_d512", 77, 0, 80, 76, 512, dict(loss="energy")),
    ("wide_batched_sinkhorn_p2_d128", 78, 3, 150, 130, 128, dict(loss="sinkhorn", p=2, blur=0.1, scaling=0.6)),
]


def main():
    for name, seed, B, n, m, d, kw in CASES:
        g = torch.Generator().manual_seed(seed)
        lead = (B,) if B else ()
        s = 2.0 / math.sqrt(d)
        # fp32-representable inputs: the fp64 run of the reference sees exactly the same numbers (x.double())
        x = torch.rand(*lead, n, d, generator=g) * s
        y = torch.rand(*lead, m, d, generator=g) * (0.9 * s) + 0.1 * s
        a = torch.rand(*lead, n, generator=g) + 0.1
        b = torch.rand(*lead, m, generator=g) + 0.1
        a, b = a / a.sum(-1, keepdim=True), b / b.sum(-1, keepdim=True)
        kw = dict(backend="tensorized", **kw)
        arrays = dict(a=npy(a), x=npy(x), b=npy(b), y=npy(y))
        for k, v in kw.items():
            arrays["kw_" + k] = np.array(v)
        for dtype, suf in ((torch.float32, ""), (torch.float64, "_f64")):
            leaves = [t.to(dtype).requires_grad_(True) for t in (a, x, b, y)]
            out = SamplesLoss(**kw)(*leaves)
            ga, gx, gb, gy = torch.autograd.grad(out.sum(), leaves)
            arrays.update({"value" + suf: npy(out), "grad_a" + suf: npy(ga), "grad_b" + suf: npy(gb)})
            if suf:  # point gradients: the fp64 run only, stored in fp32 (far below the tests' bars)
                arrays.update({"grad_x" + suf: npy(gx).astype(np.float32), "grad_y" + suf: npy(gy).astype(np.float32)})
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **arrays)
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB value fp32 {arrays['value']} fp64 {arrays['value_f64']}")


if __name__ == "__main__":
    main()

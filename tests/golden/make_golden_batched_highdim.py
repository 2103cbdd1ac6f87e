"""Golden fixtures of batched losses in the tensor-core dimensions (B > 1, 8 < D <= 64) from the REAL reference's
tensorized backend on (B, N, D) inputs.

    python tests/golden/make_golden_batched_highdim.py

Imports geomloss from /root/reference/src (commit 00e493f); fp32 and fp64 runs of
SamplesLoss(..., backend="tensorized") on batched clouds, with autograd gradients of a, x, b and y taken on the sum of
the B loss values, in the style of make_golden_highdim_norms.py.  Writes only the batched_hd_* files.  The batch
elements differ in scale and offset, so that one element's weights or extent cannot stand in for another's.
"""
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


CASES = [
    ("batched_hd_sinkhorn_d16", 61, 4, 150, 170, 16, dict(loss="sinkhorn", p=2, blur=0.1)),
    ("batched_hd_sinkhorn_d64_reach", 62, 3, 130, 129, 64, dict(loss="sinkhorn", p=2, blur=0.3, reach=0.5)),
    ("batched_hd_gaussian_d64", 63, 3, 200, 150, 64, dict(loss="gaussian", blur=2.0)),
    ("batched_hd_laplacian_d16", 64, 5, 129, 140, 16, dict(loss="laplacian", blur=0.5)),
    ("batched_hd_energy_d33", 65, 3, 160, 129, 33, dict(loss="energy", blur=0.05)),
]


def main():
    for name, seed, B, n, m, d, kw in CASES:
        g = torch.Generator().manual_seed(seed)
        # fp32-representable inputs: the fp64 run of the reference sees exactly the same numbers (x.double())
        s = (0.5 + torch.arange(B, dtype=torch.float32) / B).view(B, 1, 1)
        x = torch.rand(B, n, d, generator=g) * s
        y = torch.rand(B, m, d, generator=g) * s * 0.9 + 0.15
        a = torch.rand(B, n, generator=g) + 0.1
        b = torch.rand(B, m, generator=g) + 0.1
        a, b = a / a.sum(1, keepdim=True), b / b.sum(1, keepdim=True)
        arrays = dict(a=npy(a), x=npy(x), b=npy(b), y=npy(y))
        for k, v in kw.items():
            arrays["kw_" + k] = np.array(v)
        for dtype, suf in ((torch.float32, ""), (torch.float64, "_f64")):
            leaves = [t.to(dtype).requires_grad_(True) for t in (a, x, b, y)]
            val = SamplesLoss(backend="tensorized", **kw)(*leaves)
            ga, gx, gb, gy = torch.autograd.grad(val.sum(), leaves)
            arrays.update({"value" + suf: npy(val), "grad_a" + suf: npy(ga), "grad_b" + suf: npy(gb)})
            if suf:  # point gradients: the fp64 run only
                arrays.update({"grad_x" + suf: npy(gx).astype(np.float32), "grad_y" + suf: npy(gy).astype(np.float32)})
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **arrays)
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB value fp64 {arrays['value_f64']}")


if __name__ == "__main__":
    main()

"""Golden fixtures of the laplacian and energy kernel norms in dimensions 16, 33 and 64 (the tensor-core kernels)
from the REAL reference's tensorized backend.

    python tests/golden/make_golden_highdim_norms.py

Imports geomloss from /root/reference/src (commit 00e493f); fp32 and fp64 runs of
SamplesLoss("laplacian" | "energy", backend="tensorized") with autograd gradients of a, x, b and y, in the style of
make_golden_highdim.py.  Writes only the hd_laplacian_* / hd_energy_* files.  The "_dup" case repeats rows of x
inside x and inside y: coincident pairs across and within the clouds, where the reference's 1e-8 clamp gives the
value sqrt(1e-8) (energy) or exp(-1e-4) (laplacian) and a zero gradient.  The energy cases store the reference's
default blur (.05), which the energy distance does not use.
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
    ("hd_laplacian_d16_blur05", 51, 600, 550, 16, dict(loss="laplacian", blur=0.5), False),
    ("hd_laplacian_d64_blur2", 52, 500, 520, 64, dict(loss="laplacian", blur=2.0), False),
    ("hd_laplacian_d33_blur02", 53, 450, 470, 33, dict(loss="laplacian", blur=0.2), False),
    ("hd_energy_d16", 54, 600, 550, 16, dict(loss="energy", blur=0.05), False),
    ("hd_energy_d33", 55, 450, 470, 33, dict(loss="energy", blur=0.05), False),
    ("hd_energy_d64", 56, 500, 520, 64, dict(loss="energy", blur=0.05), False),
    ("hd_energy_d64_dup", 57, 400, 300, 64, dict(loss="energy", blur=0.05), True),
    ("hd_laplacian_d64_blur2_dup", 58, 400, 300, 64, dict(loss="laplacian", blur=2.0), True),
]


def main():
    for name, seed, n, m, d, kw, dup in CASES:
        g = torch.Generator().manual_seed(seed)
        # fp32-representable inputs: the fp64 run of the reference sees exactly the same numbers (x.double())
        x = torch.rand(n, d, generator=g)
        y = torch.rand(m, d, generator=g) * 0.9 + 0.15
        if dup:
            x[n // 2:n // 2 + 20] = x[:20]  # duplicates within x
            y[:40] = x[100:140]  # copies of rows of x in y
        a = torch.rand(n, generator=g) + 0.1
        b = torch.rand(m, generator=g) + 0.1
        a, b = a / a.sum(), b / b.sum()
        arrays = dict(a=npy(a), x=npy(x), b=npy(b), y=npy(y))
        for k, v in kw.items():
            arrays["kw_" + k] = np.array(v)
        for dtype, suf in ((torch.float32, ""), (torch.float64, "_f64")):
            leaves = [t.to(dtype).requires_grad_(True) for t in (a, x, b, y)]
            val = SamplesLoss(backend="tensorized", **kw)(*leaves)
            ga, gx, gb, gy = torch.autograd.grad(val, leaves)
            arrays.update({"value" + suf: npy(val), "grad_a" + suf: npy(ga), "grad_b" + suf: npy(gb)})
            if suf:  # point gradients: the fp64 run only
                arrays.update({"grad_x" + suf: npy(gx).astype(np.float32), "grad_y" + suf: npy(gy).astype(np.float32)})
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **arrays)
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB value fp32 {arrays['value']} fp64 {arrays['value_f64']}")


if __name__ == "__main__":
    main()

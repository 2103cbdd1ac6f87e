"""Golden fixtures of the p = 1 Sinkhorn divergence in the tensor-core dimensions (8 < D <= 64) from the REAL reference.

    python tests/golden/make_golden_highdim_p1.py

Imports geomloss from /root/reference/src (commit 00e493f), with tests/golden/pykeops_shim first on ``sys.path`` for
the one "online" case (a dense pure-torch stand-in for pykeops, see make_golden_multiscale.py); the "tensorized" cases
never touch it.  fp32 and fp64 runs of SamplesLoss("sinkhorn", p=1) with autograd gradients, or the potentials.  The
reference's own fp32 run is 1e-4 to 1e-3 relative off its fp64 run on these cases, so the tests compare with the fp64
run only.  Written as p1hd_*.npz (the hd_* prefix belongs to make_golden_highdim.py's fixtures).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ.get("GEOMLOSS_REFERENCE", "/root/reference/src"))
sys.path.insert(0, os.path.join(HERE, "pykeops_shim"))
import pykeops  # noqa: E402

assert pykeops.__version__.startswith("shim"), "the dense pykeops shim must shadow any real pykeops"
from geomloss import SamplesLoss  # noqa: E402

torch.set_num_threads(8)


def npy(t):
    return t.detach().cpu().numpy()


# (name, seed, N, M, D, duplicated points, SamplesLoss keywords)
CASES = [
    ("p1hd_d16", 61, 500, 550, 16, 0, dict(blur=0.3, scaling=0.6)),
    ("p1hd_d33", 62, 480, 520, 33, 0, dict(blur=0.5, scaling=0.6)),
    ("p1hd_d64", 63, 500, 450, 64, 0, dict(blur=1.0, scaling=0.6)),
    ("p1hd_d33_reach", 64, 450, 500, 33, 0, dict(blur=0.5, reach=2.0, scaling=0.7)),
    ("p1hd_d16_nodebias", 65, 500, 470, 16, 0, dict(blur=0.4, scaling=0.6, debias=False)),
    ("p1hd_d64_dup", 66, 500, 500, 64, 120, dict(blur=1.0, scaling=0.6)),
    ("p1hd_d16_potentials", 67, 430, 500, 16, 0, dict(blur=0.3, scaling=0.6, potentials=True)),
    ("p1hd_d33_online", 68, 500, 510, 33, 40, dict(blur=0.5, scaling=0.6, backend="online")),
]


def main():
    for name, seed, n, m, d, dup, kw in CASES:
        g = torch.Generator().manual_seed(seed)
        # fp32-representable inputs: the fp64 run of the reference sees exactly the same numbers (x.double())
        x = torch.rand(n, d, generator=g)
        y = torch.rand(m, d, generator=g) * 0.9 + 0.15
        if dup:
            # copies within each cloud and across the two clouds: coincident pairs in xx, yy, xy and yx
            x[n - dup // 2:] = x[: dup // 2]
            y[: dup // 2] = x[dup // 2: dup]
            y[m - dup // 4:] = y[dup // 2: dup // 2 + dup // 4]
        a = torch.rand(n, generator=g) + 0.1
        b = torch.rand(m, generator=g) + 0.1
        a, b = a / a.sum(), b / b.sum()
        kw = dict(loss="sinkhorn", p=1, **{"backend": "tensorized", **kw})
        arrays = dict(a=npy(a), x=npy(x), b=npy(b), y=npy(y))
        for k, v in kw.items():
            arrays["kw_" + k] = np.array(v)
        for dtype, suf in ((torch.float32, ""), (torch.float64, "_f64")):
            leaves = [t.to(dtype).requires_grad_(True) for t in (a, x, b, y)]
            out = SamplesLoss(**kw)(*leaves)
            if kw.get("potentials"):
                arrays.update({"pot_f" + suf: npy(out[0]).ravel(), "pot_g" + suf: npy(out[1]).ravel()})
                continue
            ga, gx, gb, gy = torch.autograd.grad(out, leaves)
            arrays.update({"value" + suf: npy(out), "grad_a" + suf: npy(ga), "grad_b" + suf: npy(gb)})
            if suf:  # point gradients: the fp64 run only, stored in fp32 (far below the tests' 2e-3 bar)
                arrays.update({"grad_x" + suf: npy(gx).astype(np.float32), "grad_y" + suf: npy(gy).astype(np.float32)})
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **arrays)
        what = "potentials" if kw.get("potentials") else f"value fp32 {arrays['value']} fp64 {arrays['value_f64']}"
        print(f"{name}: {os.path.getsize(path) / 1024:.0f} KiB {what}")


if __name__ == "__main__":
    main()

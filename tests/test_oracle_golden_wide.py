"""The fp64 oracle (oracle/geomloss_oracle.py) against the reference's runs above D = 64 (tests/golden/wide_*.npz,
make_golden_wide.py): the fixtures the GPU tests hold the wide operators to are the reference's, to fp64 rounding.
CPU only."""
import numpy as np
import pytest
import torch

from conftest import golden_kwargs, golden_names, load_golden
from oracle import geomloss_oracle as O

NAMES = golden_names("wide_")
F64 = dict(rtol=1e-10, atol=1e-12)


def test_fixture_set():
    assert len(NAMES) == 8
    gs = [load_golden(n) for n in NAMES]
    assert {g["x"].shape[-1] for g in gs} == {96, 128, 512}
    kws = [golden_kwargs(g) for g in gs]
    assert {(k["loss"], k.get("p")) for k in kws} >= {("sinkhorn", 1), ("sinkhorn", 2), ("gaussian", None),
                                                      ("laplacian", None), ("energy", None)}
    assert any(g["x"].ndim == 3 for g in gs)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fp64(name):
    g = load_golden(name)
    kw = golden_kwargs(g)
    kw.pop("backend")
    leaves = [torch.from_numpy(g[k]).double().requires_grad_(True) for k in "axby"]
    out = O.samples_loss(*leaves, **kw)
    np.testing.assert_allclose(out.detach().numpy(), g["value_f64"], **F64)
    grads = torch.autograd.grad(out.sum(), leaves)
    for got, key in zip(grads, ("grad_a", "grad_x", "grad_b", "grad_y")):
        ref = g[key + "_f64"]
        # point gradients are stored in fp32
        atol = (1e-6 if key in ("grad_x", "grad_y") else 1e-11) * max(1.0, np.abs(ref).max())
        np.testing.assert_allclose(got.numpy().reshape(ref.shape), ref, rtol=0, atol=atol)

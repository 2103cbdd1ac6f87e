"""The fp64 oracle (oracle/geomloss_oracle.py) against the reference's p = 1 Sinkhorn runs above D = 8
(tests/golden/p1hd_*.npz, make_golden_highdim_p1.py): the fixtures the GPU tests hold the engine to are the
reference's, to fp64 rounding, in both cost conventions.  CPU only."""
import numpy as np
import pytest
import torch

from conftest import golden_kwargs, golden_names, load_golden
from oracle import geomloss_oracle as O

NAMES = golden_names("p1hd_")
F64 = dict(rtol=1e-10, atol=1e-12)


def test_fixture_set():
    assert len(NAMES) == 8
    kws = [golden_kwargs(load_golden(n)) for n in NAMES]
    assert {load_golden(n)["x"].shape[1] for n in NAMES} == {16, 33, 64}
    assert any("reach" in k for k in kws) and any(k.get("debias") is False for k in kws)
    assert any(k.get("potentials") for k in kws) and any(k["backend"] == "online" for k in kws)
    assert all(k["p"] == 1 and k["loss"] == "sinkhorn" for k in kws)
    dup = load_golden("p1hd_d64_dup")
    assert len(np.unique(np.concatenate([dup["x"], dup["y"]]), axis=0)) < len(dup["x"]) + len(dup["y"])


def _oracle(g, leaves):
    kw = golden_kwargs(g)
    backend = kw.pop("backend")
    kw.pop("loss")
    a, x, b, y = leaves
    if backend == "online":
        out = O.sinkhorn_online(a[None], x[None], b[None], y[None], **kw)
        return (out[0][0], out[1][0]) if kw.get("potentials") else out[0]
    return O.samples_loss(a, x, b, y, loss="sinkhorn", **kw)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fp64(name):
    g = load_golden(name)
    pot = bool(golden_kwargs(g).get("potentials", False))
    leaves = [torch.from_numpy(g[k]).double().requires_grad_(not pot) for k in "axby"]
    out = _oracle(g, leaves)
    if pot:
        np.testing.assert_allclose(out[0].detach().numpy().ravel(), g["pot_f_f64"], **F64)
        np.testing.assert_allclose(out[1].detach().numpy().ravel(), g["pot_g_f64"], **F64)
        return
    np.testing.assert_allclose(out.detach().numpy(), g["value_f64"], **F64)
    grads = torch.autograd.grad(out, leaves)
    for got, key in zip(grads, ("grad_a", "grad_x", "grad_b", "grad_y")):
        ref = g[key + "_f64"]
        # point gradients are stored in fp32
        atol = (1e-6 if key in ("grad_x", "grad_y") else 1e-11) * max(1.0, np.abs(ref).max())
        np.testing.assert_allclose(got.numpy().reshape(ref.shape), ref, rtol=0, atol=atol)

"""The fp64 oracle's two-scale Sinkhorn (oracle.geomloss_oracle.sinkhorn_multiscale_dense) against the reference's
labelled runs above D = 3 (tests/golden/labels_hd_*.npz, make_golden_labels_highdim.py): the algorithm the GPU tests
hold the engine to is the reference's, to fp64 rounding.  CPU only."""
import numpy as np
import pytest
import torch

from conftest import golden_kwargs, golden_names, load_golden
from oracle import geomloss_oracle as O

NAMES = golden_names("labels_hd_")
F64 = dict(rtol=1e-11, atol=1e-11)


def _run(g, **over):
    kw = golden_kwargs(g)
    kw.pop("loss"), kw.pop("backend")
    kw.update(over)
    a, x, b, y = (torch.from_numpy(g[k + "_f64"]) for k in "axby")
    lab = dict(labels_x=torch.from_numpy(g["labels_x"]), labels_y=torch.from_numpy(g["labels_y"]))
    pot = bool(g["potentials"])
    leaves = [t.clone().requires_grad_(not pot) for t in (a, x, b, y)]
    return O.sinkhorn_multiscale_dense(*leaves, potentials=pot, **lab, **kw), leaves, pot


def test_fixture_set():
    assert len(NAMES) == 9
    dims = {load_golden(n)["x_f64"].shape[1] for n in NAMES}
    assert dims == {5, 16, 33, 64}
    sizes = set()
    for n in NAMES:
        g = load_golden(n)
        sizes |= set(np.bincount(g["labels_x"]).tolist()) | set(np.bincount(g["labels_y"]).tolist())
    assert {1, 127, 128, 129} <= sizes and max(sizes) >= 200


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fp64(name):
    g = load_golden(name)
    out, leaves, pot = _run(g)
    if pot:
        np.testing.assert_allclose(out[0].detach().numpy(), g["pot_f_f64"].ravel(), **F64)
        np.testing.assert_allclose(out[1].detach().numpy(), g["pot_g_f64"].ravel(), **F64)
        return
    np.testing.assert_allclose(out.detach().numpy().ravel(), g["value_f64"].ravel(), **F64)
    grads = torch.autograd.grad(out.sum(), leaves)
    for got, key in zip(grads, ("grad_a", "grad_x", "grad_b", "grad_y")):
        ref = g[key + "_f64"]
        np.testing.assert_allclose(got.numpy().reshape(ref.shape), ref, rtol=0, atol=1e-11 * max(1.0, np.abs(ref).max()))


@pytest.mark.parametrize("name", ["labels_hd_d5_trunc2", "labels_hd_d16_trunc1"])
def test_labels_and_truncation_are_visible_in_the_fixtures(name):
    """The two-scale value is not the single-scale one (the labels matter), and the truncated value is not the exact
    two-scale one (the block mask matters): both far beyond the GPU tests' 1e-4 bar."""
    g = load_golden(name)
    ref = float(g["value_f64"])
    exact, _, _ = _run(g, truncate=None)
    assert abs(exact.item() - ref) > 1e-4 * abs(ref)
    kw = golden_kwargs(g)
    a, x, b, y = (torch.from_numpy(g[k + "_f64"]) for k in "axby")
    single = O.sinkhorn_online(a[None], x[None], b[None], y[None], p=kw["p"], blur=kw["blur"], reach=kw.get("reach"))
    assert abs(float(single.ravel()[0]) - ref) > 1e-3 * abs(ref)

"""The fp64 restatement of ``SamplesLoss("sinkhorn", cost=callable)`` on the reference's "tensorized" backend reproduces
the reference's fixtures (tests/golden/make_golden_samples_cost.py): values or potentials, and the fp64 autograd
gradients w.r.t. x, y, a and b.  The host and GPU tests hold the engine to the same fixtures."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, golden_kwargs, golden_names, load_golden
from oracle import geomloss_oracle as O

CASES = golden_names("samples_cost_case")


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_samples_cost",
                                                  os.path.join(GOLDEN, "make_golden_samples_cost.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _generator()


def sinkhorn_cost_fp64(a, x, b, y, cost, p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, debias=True,
                       potentials=False, duals=False):
    """sinkhorn_tensorized with ``cost`` (sinkhorn_samples.py:74-221) on the oracle's loop, softmin and value formula:
    unbatched (N,) (N,D) inputs are lifted to a batch of one like the reference does.  ``duals``: also return the
    largest of the four dual terms <a, f_ba>, <a, f_aa>, <b, g_ab>, <b, g_bb> (the scale of a value that cancels)."""
    batched = x.dim() == 3
    if not batched:
        a, x, b, y = a[None], x[None], b[None], y[None]
    C_xy, C_yx = cost(x, y.detach()), cost(y, x.detach())
    C_xx, C_yy = (cost(x, x.detach()), cost(y, y.detach())) if debias else (None, None)
    diameter, eps, eps_list, rho = O.scaling_parameters(x, y, p, blur, reach, diameter, scaling)
    f_aa, g_bb, g_ab, f_ba = O.sinkhorn_loop(O.softmin_dense, O.log_weights(a), O.log_weights(b), C_xx, C_yy, C_xy,
                                             C_yx, eps_list, rho, debias=debias)
    out = O.sinkhorn_value(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=debias, potentials=potentials)
    if potentials:
        return out[0].view_as(a), out[1].view_as(b)
    out = out if batched else out[0]
    if duals:
        terms = [O._dot(w, f).abs().max().item() for w, f in ((a, f_ba), (a, f_aa), (b, g_ab), (b, g_bb))
                 if f is not None]
        return out, max(terms)
    return out


def fixture(name):
    g = load_golden(name)
    kw = golden_kwargs(g)
    return g, G.COSTS[str(g["cost"])], kw


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name):
    g, cost, kw = fixture(name)
    a, x, b, y = (torch.from_numpy(g[k]).double().requires_grad_(True) for k in ("a", "x", "b", "y"))
    out = sinkhorn_cost_fp64(a, x, b, y, cost, **kw)
    if kw.get("potentials"):
        np.testing.assert_allclose(out[0].detach().numpy(), g["F_f64"], rtol=0, atol=1e-11)
        np.testing.assert_allclose(out[1].detach().numpy(), g["G_f64"], rtol=0, atol=1e-11)
        return
    np.testing.assert_allclose(out.detach().numpy(), g["value_f64"], rtol=0, atol=1e-11)
    grads = torch.autograd.grad(out.sum(), [x, y, a, b])
    for k, gr in zip(("grad_x", "grad_y", "grad_a", "grad_b"), grads):
        np.testing.assert_allclose(gr.numpy(), g[k + "_f64"], rtol=0, atol=1e-11, err_msg=k)


def test_fixtures_cover_the_cases():
    assert len(CASES) == len(G.CASES) == 10
    for name in CASES:
        assert os.path.getsize(os.path.join(GOLDEN, name + ".npz")) < 400 * 1024

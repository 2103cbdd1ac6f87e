"""The fp64 restatement of ``geomloss.ot.solve`` / ``solve_batch`` on explicit cost matrices reproduces the reference's
fixtures (tests/golden/make_golden_ot_matrix.py): every result attribute in fp64 and fp32, and the fp64 autograd
gradients of the value w.r.t. C, a and b.  The GPU tests hold the CUDA solver to the same fixtures."""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import geomloss_oracle as O

CASES = golden_names("ot_matrix_case")


def ot_solve_matrix(C, a, b, reg, unbalanced=None, max_iter=None, v=None):
    """Dense restatement of ``ot.solve(C, a=a, b=b, reg=reg, ...)`` (C (N, M)) or ``ot.solve_batch`` (C (B, N, M)),
    built on the oracle's softmin and value formula; returns the result attributes (and ``plan_v = plan @ v``).

    matrix.py:620-660 (the batched driver) -> sinkhorn_ot.py:17-29 (eps = +inf start, minus half of <a, f> per
    problem: with (B, N) vectors bk.dot_products reduces each row), :240-288 (symmetric averaged updates on the eps
    ladder of annealing.py:131-170 from max(C) - min(C) over the whole batch), :419-436 (one last update with detached
    log-weights and potentials, so the value depends on C through both softmins of that update), unbalanced_ot.py
    (value), matrix.py:188-330 (density, plan, operators) and _ot_result.py:388-406 (marginals)."""
    batched = C.dim() == 3
    if not batched:
        C, a, b = C[None], a[None], b[None]
        v = None if v is None else v[None]
    rho = unbalanced
    log_a, log_b = O.log_weights(a), O.log_weights(b)
    CT = C.transpose(1, 2)

    def sm(eps, lw, Cm, pot):  # the reference's softmin_dense, element by element of the batch
        return torch.stack([O.ot_softmin(eps, lw[k], Cm[k], pot[k]) for k in range(Cm.shape[0])])

    def damp(eps):
        return 1.0 if rho is None else 1.0 / (1.0 + eps / rho)

    eps_list = O.ot_annealing_eps(float(C.detach().max() - C.detach().min()), reg, max_iter)
    with torch.no_grad():
        lam = damp(eps_list[0])

        def init(lw_self, lw_other, Cm):
            f = sm(float("inf"), lw_other, Cm, 0 * lw_other)
            return lam * (f - 0.5 * (lw_self.exp() * f).sum(-1, keepdim=True))

        f, g = init(log_a, log_b, C), init(log_b, log_a, CT)
        for eps in eps_list:
            lam = damp(eps)
            ft, gt = lam * sm(eps, log_b, C, g), lam * sm(eps, log_a, CT, f)
            f, g = 0.5 * (f + ft), 0.5 * (g + gt)
    la, lb = log_a.detach(), log_b.detach()
    f, g = lam * sm(eps, lb, C, g.detach()), lam * sm(eps, la, CT, f.detach())
    value = torch.stack([O.ot_sinkhorn_cost(a[k], b[k], None, None, g[k], f[k], reg, rho, False)
                         for k in range(C.shape[0])])
    density = torch.exp((f[:, :, None] + g[:, None, :] - C) / reg)
    plan = density * a[:, :, None] * b[:, None, :]
    out = dict(value=value, potential_a=f, potential_b=g, marginal_a=a * (density @ b[..., None])[..., 0],
               marginal_b=b * (density.transpose(1, 2) @ a[..., None])[..., 0], plan=plan)
    if v is not None:
        out["plan_v"] = plan @ v
    return {k: t if batched else t[0] for k, t in out.items()}


def case(name, dtype):
    z = load_golden(name)
    kw = dict(reg=float(z["kw_reg"]), max_iter=int(z["kw_max_iter"]),
              unbalanced=float(z["kw_unbalanced"]) if "kw_unbalanced" in z else None)
    t = {k: torch.from_numpy(z[k]).to(dtype) for k in ("C", "a", "b", "v")}
    return z, t, kw


def test_fixture_set_is_complete():
    assert len(CASES) == 10


@pytest.mark.parametrize("name", CASES)
def test_oracle_ot_solve_matrix_matches_reference(name):
    for dtype, suffix, tol in ((torch.float64, "_f64", 1e-9), (torch.float32, "", 2e-4)):
        z, t, kw = case(name, dtype)
        out = ot_solve_matrix(t["C"], t["a"], t["b"], v=t["v"], **kw)
        for key, val in out.items():
            ref = z[key + suffix]
            assert val.shape == ref.shape, key
            np.testing.assert_allclose(val.detach().numpy(), ref, atol=tol * max(1.0, float(np.abs(ref).max())),
                                       err_msg=f"{key}{suffix} {name}")


@pytest.mark.parametrize("name", CASES)
def test_oracle_ot_solve_matrix_gradients_match_reference(name):
    z, t, kw = case(name, torch.float64)
    leaves = [t[k].clone().requires_grad_(True) for k in ("C", "a", "b")]
    value = ot_solve_matrix(*leaves, **kw)["value"]
    grads = torch.autograd.grad(value.sum(), leaves)
    for got, key in zip(grads, ("grad_C", "grad_a", "grad_b")):
        ref = z[key + "_f64"]
        np.testing.assert_allclose(got.numpy(), ref, atol=1e-9 * max(1.0, float(np.abs(ref).max())), err_msg=key)


def test_doctest_gradient_is_twice_the_plan():
    """At convergence the value's gradient w.r.t. C is ~2 plan: the last update is differentiated through the row
    AND the column softmin, each of which contributes one plan."""
    z = load_golden("ot_matrix_case00")
    np.testing.assert_allclose(z["grad_C_f64"], [[2, 2, 0], [0, 0, 4]], atol=2e-3)
    np.testing.assert_allclose(z["plan_f64"], [[1, 1, 0], [0, 0, 2]], atol=2e-3)

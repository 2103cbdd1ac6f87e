"""Pin the CPU oracle (oracle/geomloss_oracle.py) against outputs of the real reference.

The fixtures in tests/golden/ were produced by tests/golden/make_golden.py, which imports
jeanfeydy/geomloss @ 00e493f from /root/reference/src.  The oracle runs the same dense torch
arithmetic, so fp32 agreement is expected to a few ulps; tolerances are stated per test.
"""
import math

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import geomloss_oracle as O

T = torch.from_numpy


def _kw(g):
    reach = float(g["reach"])
    return dict(loss="sinkhorn", p=int(g["p"]), blur=float(g["blur"]), reach=None if reach < 0 else reach,
                debias=bool(g["debias"]), scaling=float(g["scaling"]))


def test_cfg1_value_potentials_gradients():
    g = load_golden("cfg1_sinkhorn_n1000")
    a, x, b, y = (T(g[k]) for k in "axby")
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = O.samples_loss(ag, xg, bg, yg, loss="sinkhorn", p=2, blur=0.05)
    # SURVEY.md section 8c anchor: 2.2802867e-3 (fp32)
    assert abs(val.item() - 2.2802867e-3) < 2e-9
    np.testing.assert_allclose(val.item(), g["value_f32"], rtol=2e-6)
    np.testing.assert_allclose(val.item(), g["value_f64"], rtol=2e-6)
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    np.testing.assert_allclose(ga.numpy(), g["grad_a_f32"], atol=2e-7)
    np.testing.assert_allclose(gb.numpy(), g["grad_b_f32"], atol=2e-7)
    np.testing.assert_allclose(gx.numpy(), g["grad_x_f32"], atol=2e-9 + 1e-5 * np.abs(g["grad_x_f32"]).max())
    np.testing.assert_allclose(gy.numpy(), g["grad_y_f32"], atol=2e-9 + 1e-5 * np.abs(g["grad_y_f32"]).max())
    F, G = O.samples_loss(a, x, b, y, loss="sinkhorn", p=2, blur=0.05, potentials=True)
    assert F.shape == (1, 1000) and G.shape == (1, 1000)  # the reference's (1,N) quirk, SURVEY A-12
    np.testing.assert_allclose(F.numpy(), g["pot_f_f32"], atol=2e-7)
    np.testing.assert_allclose(G.numpy(), g["pot_g_f32"], atol=2e-7)
    # weights' gradients ARE the potentials (SURVEY.md section 3.2)
    np.testing.assert_allclose(ga.numpy(), F.numpy()[0], atol=2e-7)


@pytest.mark.parametrize("name", golden_names("sinkhorn_case"))
def test_sinkhorn_cases(name):
    g = load_golden(name)
    a, x, b, y = (T(g[k]) for k in "axby")
    kw = _kw(g)
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = O.samples_loss(ag, xg, bg, yg, **kw)
    scale = max(abs(float(g["value"])), 1e-6)
    assert abs(val.item() - float(g["value"])) <= 5e-6 * scale + 1e-8
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    for got, key in ((ga, "grad_a"), (gb, "grad_b"), (gx, "grad_x"), (gy, "grad_y")):
        ref = g[key]
        np.testing.assert_allclose(got.numpy(), ref, atol=1e-5 * max(np.abs(ref).max(), 1e-3))
    F, G = O.samples_loss(a, x, b, y, potentials=True, **kw)
    np.testing.assert_allclose(F.numpy(), g["pot_f"], atol=1e-5 * max(np.abs(g["pot_f"]).max(), 1e-3))
    np.testing.assert_allclose(G.numpy(), g["pot_g"], atol=1e-5 * max(np.abs(g["pot_g"]).max(), 1e-3))


def test_sinkhorn_batched():
    g = load_golden("sinkhorn_batched")
    a, x, b, y = (T(g[k]) for k in "axby")
    val = O.samples_loss(a, x, b, y, loss="sinkhorn", p=2, blur=0.1)
    assert val.shape == (2,)
    np.testing.assert_allclose(val.numpy(), g["value"], rtol=5e-6)
    F, G = O.samples_loss(a, x, b, y, loss="sinkhorn", p=2, blur=0.1, potentials=True)
    np.testing.assert_allclose(F.numpy(), g["pot_f"], atol=2e-7)
    np.testing.assert_allclose(G.numpy(), g["pot_g"], atol=2e-7)


@pytest.mark.parametrize("name", golden_names("kernel_gaussian") + golden_names("kernel_laplacian")
                         + golden_names("kernel_energy"))
def test_kernel_losses(name):
    g = load_golden(name)
    kind = name.split("_")[1]
    a, x, b, y = (T(g[k]) for k in "axby")
    blur = float(g["blur"])
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = O.samples_loss(ag, xg, bg, yg, loss=kind, blur=blur)
    np.testing.assert_allclose(val.item(), g["value"], rtol=1e-5, atol=1e-9)
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    for got, key in ((ga, "grad_a"), (gb, "grad_b"), (gx, "grad_x"), (gy, "grad_y")):
        np.testing.assert_allclose(got.numpy(), g[key], atol=1e-5 * max(np.abs(g[key]).max(), 1e-3))
    F, G = O.samples_loss(a, x, b, y, loss=kind, blur=blur, potentials=True)
    np.testing.assert_allclose(F.numpy(), g["pot_f"], atol=1e-5 * np.abs(g["pot_f"]).max())
    np.testing.assert_allclose(G.numpy(), g["pot_g"], atol=1e-5 * np.abs(g["pot_g"]).max())


def test_softmin_operator():
    g = load_golden("softmin_operator")
    x, y, b, pot = (T(g[k]) for k in ("x", "y", "b", "pot"))
    for p in (1, 2):
        C = O.cost_matrix(x.unsqueeze(0), y.unsqueeze(0), p)
        for e, eps in enumerate(g["eps"]):
            eps = float(eps)
            h = O.log_weights(b) + pot / eps
            ref = g[f"softmin_p{p}_eps{e}"]
            got = O.softmin_dense(eps, C, h.unsqueeze(0))[0].numpy()
            np.testing.assert_allclose(got, ref, atol=1e-6 * max(1.0, np.abs(ref).max()))
            # the blocked point-cloud form is the same operator
            got2 = O.softmin_points(eps, x, y, h, p=p, row_block=16).numpy()
            np.testing.assert_allclose(got2, ref, atol=1e-6 * max(1.0, np.abs(ref).max()))


def test_epsilon_schedule():
    g = load_golden("epsilon_schedule")
    for i in range(4):
        p, diam, blur, scaling = g[f"args{i}"]
        got = np.array(O.epsilon_schedule(int(p), diam, blur, scaling))
        np.testing.assert_array_equal(got, g[f"eps{i}"])  # same numpy expressions -> bit-exact
    # SURVEY.md appendix C: 10 / 51 values for blur .01 at scaling .5 / .9 on the unit cube
    assert len(O.epsilon_schedule(2, 3**0.5, 0.01, 0.5)) == 10
    assert len(O.epsilon_schedule(2, 3**0.5, 0.01, 0.9)) == 51


def test_kernel_operator():
    g = load_golden("kernel_operator")
    x, y = T(g["x"]), T(g["y"])
    for name in ("gaussian", "laplacian", "energy"):
        got = O.kernel_matrix(name, x, y, float(g["blur"])).numpy()
        np.testing.assert_allclose(got, g[name], atol=1e-6)


def test_counting_helpers():
    # SURVEY.md appendix C: 40 softmins (debias) / 20 at 8 eps values; BASELINE.md: 2.12e14 pairs at cfg 2
    assert O.n_softmins(8, True) == 40 and O.n_softmins(8, False) == 20
    assert abs(O.pair_interactions(51, 10**6, 10**6) - 2.12e14) < 1e12


@pytest.mark.parametrize("d,n", [(2, 8), (3, 4)])
def test_grid_softmin_is_the_full_grid_softmin(d, n):
    """The (unpinned) grid restatement must equal the pinned dense softmin on the explicit pixel coordinates:
    p=2: cost |x-y|^2/2; p=1: the per-axis (L1) cost the separable reference formula implies."""
    g = torch.Generator().manual_seed(d)
    h = torch.randn(1, 1, *([n] * d), generator=g, dtype=torch.float64)
    coords = torch.stack(torch.meshgrid(*[torch.arange(n, dtype=torch.float64) / n] * d, indexing="ij"), -1).reshape(-1, d)
    for p in (1, 2):
        C = O.cost_matrix(coords, coords, 2) if p == 2 else (coords[:, None, :] - coords[None, :, :]).abs().sum(-1)
        for eps in (0.5, 0.02):
            ref = O.softmin_dense(eps, C[None], h.reshape(1, -1))[0]
            got = O.softmin_grid_dense(eps, p, h).reshape(-1)
            assert (got - ref).abs().max().item() < 1e-12


def grid64_vs_oracle(device):
    """The largest relative difference between fp64_refs.grid_softmin64 (full and sampled, small line blocks) and
    oracle.softmin_grid_dense, at sides and grids of every dimension where the oracle's dense broadcast is cheap."""
    from fp64_refs import grid_softmin64

    g = torch.Generator().manual_seed(4)
    worst = 0.0
    for dim, n in ((1, 1), (1, 9), (2, 1), (2, 7), (2, 17), (3, 5), (3, 12)):
        h = (torch.randn(2, 3, *([n] * dim), generator=g, dtype=torch.float64) * 3.0).to(device)
        h.view(6, -1)[1, ::3] = -10000.0
        h.view(6, -1)[2, :] = -math.inf
        h.view(6, -1)[3, 1:] = -math.inf
        rows = [torch.randint(0, n, (3,), generator=g) for _ in range(dim)]
        for p in (1, 2):
            for eps in (2.0, 0.1, (0.5 / n) ** p):
                ref = O.softmin_grid_dense(eps, p, h)
                sub = ref
                for axis, r in enumerate(rows):
                    sub = sub.index_select(2 + axis, r.to(device))
                for got, want in ((grid_softmin64(eps, p, h, dim, device=device, budget=64), ref),
                                  (grid_softmin64(eps, p, h, dim, rows=rows, device=device, budget=64), sub)):
                    assert got.device == want.device and got.shape == want.shape
                    fin = torch.isfinite(want)
                    assert torch.equal(got[~fin], want[~fin]) and bool(torch.isfinite(got[fin]).all())
                    err = (got[fin] - want[fin]).abs().max().item() / max(1.0, want[fin].abs().max().item())
                    worst = max(worst, err)
    return worst


def test_fp64_grid_reference_is_the_grid_oracle():
    """CPU half of the cross-check of the grid softmin's fp64 reference (test_gpu_grid.py runs it on the GPU)."""
    assert grid64_vs_oracle("cpu") <= 1e-11


def test_grid_pyramid_and_schedule():
    a = torch.rand(2, 1, 16, 16)
    lv = O.grid_pyramid(a)
    assert [t.shape[-1] for t in lv] == [1, 2, 4, 8, 16]
    for t in lv:  # sum-pooling preserves mass
        np.testing.assert_allclose(t.sum((1, 2, 3)).numpy(), a.sum((1, 2, 3)).numpy(), rtol=1e-5)
    v = O.sinkhorn_images(a.double(), a.double().flip(-1), blur=1 / 16)
    assert v.shape == (2,) and (v > 0).all()
    assert torch.allclose(O.sinkhorn_images(a.double(), a.double()), torch.zeros(2, dtype=torch.float64), atol=1e-12)


# ------------------------------------------------------------------------------------------------
# geomloss.ot.solve_sample (new API) — oracle restatement vs the reference's fp32 / fp64 runs
# ------------------------------------------------------------------------------------------------
def _ot_case(name, dtype):
    z = load_golden(name)
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    if "max_iter" in kw:
        kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    t = lambda k: torch.from_numpy(z[k]).to(dtype)  # noqa: E731
    args = dict(X_a=t("X_a"), X_b=t("X_b"), a=t("a") if "a" in z else None, b=t("b") if "b" in z else None)
    return z, args, kw


@pytest.mark.parametrize("idx", range(8))
def test_oracle_ot_solve_sample_matches_reference(idx):
    for dtype, suffix, tol in ((torch.float64, "_f64", 1e-9), (torch.float32, "", 2e-4)):
        z, args, kw = _ot_case(f"ot_sample_case{idx:02d}", dtype)
        out = O.ot_solve_sample(**args, **kw)
        for name, val in out.items():
            ref = z[name + suffix]
            scale = max(1.0, float(np.abs(ref).max()))
            np.testing.assert_allclose(val.numpy(), ref, atol=tol * scale, err_msg=f"{name}{suffix} case {idx}")
    # autograd contract of the new API (last update differentiated through the cost matrices; direct dependence of
    # the value on a and b): gradients of the reference's fp64 run
    z, args, kw = _ot_case(f"ot_sample_case{idx:02d}", torch.float64)
    n, m = args["X_a"].shape[0], args["X_b"].shape[0]
    if args["a"] is None:
        args["a"], args["b"] = torch.full((n,), 1.0 / n, dtype=torch.float64), torch.full((m,), 1.0 / m, dtype=torch.float64)
    leaves = {k: v.clone().requires_grad_(True) for k, v in args.items()}
    val = O.ot_solve_sample(**leaves, **kw)["value"]
    grads = torch.autograd.grad(val, [leaves[k] for k in ("X_a", "X_b", "a", "b")])
    for g, name in zip(grads, ("grad_X_a", "grad_X_b", "grad_a", "grad_b")):
        ref = z[name + "_f64"]
        np.testing.assert_allclose(g.numpy(), ref, atol=1e-9 * max(1.0, float(np.abs(ref).max())), err_msg=name)

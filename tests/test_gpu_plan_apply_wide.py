"""The plan-times-values operator above D = 64 on the GPU (b200ot_wide_plan_apply, ops.plan_apply_wide_raw: the K-slab
kernel tc_wide_apply_kernel) and ``ot.solve_sample`` with its result object above D = 64, against dense or row-chunked
fp64 evaluations on the device and against the reference's fixtures (tests/golden/make_golden_ot_wide.py).

Bar of the operator: 5e-5 max_j |V_jk| per value column, plus the effect of the exponent's rounding on the weights,
computed from the fp64 data by DESIGN.md section 3.5d's bound: the kernels' d^2 is off by at most
(3 dk/16 + 9) 2^-23 (|X_i|^2 + |Y_j|^2) in their scaled coordinates, so the log2 exponent of row i by at most
delta_i = (3 dk/16 + 9) 2^-24 (|X_i|^2 + max_j |Y_j|^2), and the normalised weights by 2 (2^delta_i - 1) relative."""
import math

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOG2E = 1.4426950408889634
CASES = golden_names("ot_sample_wide_case")


def _cd(d):
    return 3 * (-(-d // 16) * 16) // 16 + 9


def _clouds(n, m, d, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g).to(DEV)
    y = torch.rand(m, d, generator=g).to(DEV)
    h = (0.3 * torch.randn(m, generator=g)).to(DEV)
    return x, y, h, g


def _eps_for(d):
    return 0.01 * d  # unit cubes: |x - y|^2 ~ d / 6 with a spread ~ sqrt(7 d / 180) over a row


def _exponent64(x, y, h, eps):
    return h.double()[None, :] - 0.5 * torch.cdist(x.double(), y.double()) ** 2 / eps


def _ref(x, y, h, eps, v, chunk=1024):
    out = []
    for i in range(0, x.shape[0], chunk):
        out.append(torch.softmax(_exponent64(x[i:i + chunk], y, h, eps), dim=1) @ v.double())
    return torch.cat(out)


def _center(x, y):
    from geomloss_b200 import ops

    return ops.default_center(x, y)


def _run(x, y, h, eps, v, row_factor=None, h_b=None, h_scale_b=0.0):
    from geomloss_b200 import ops

    c = _center(x, y)
    _, lse2 = ops.softmin_wide_raw(eps, x, y, h, h_b, h_scale_b, p=2, center=c, want_lse2=True)
    return ops.plan_apply_wide_raw(eps, x, y, h, h_b, h_scale_b, lse2, v, row_factor=row_factor, center=c)


def _delta(x, y, eps):
    """delta_i of every row (log2 units), from the fp64 data and the centre the operator uses"""
    c = _center(x, y).double()
    s2 = LOG2E / eps
    xx, yy = s2 * ((x.double() - c) ** 2).sum(1), s2 * ((y.double() - c) ** 2).sum(1)
    return _cd(x.shape[1]) * 2.0**-24 * (xx + yy.max())


def _check(out, ref, v, delta, bar=5e-5):
    scale = v.double().abs().reshape(v.shape[0], -1).max(0).values.clamp_min(1e-300)
    err = (out.double() - ref).abs().reshape(out.shape[0], -1) / scale
    bound = bar + 2.0 * (2.0 ** delta - 1.0)[:, None]
    assert (err <= bound).all(), (err.max().item(), bound.max().item())
    return err.max().item()


@pytest.mark.parametrize("d", [65, 96, 128, 200, 512, 1024])
@pytest.mark.parametrize("k", [1, 15, 16, 17, 64, 65, 130])
def test_dimensions_and_value_widths(d, k):
    """partial last K slab at 65 and 200; value slabs of 16 .. 64 columns and several passes"""
    x, y, h, g = _clouds(500, 700, d, 13 * d + k)
    eps = _eps_for(d)
    v = torch.randn(700, k, generator=g).to(DEV)
    out = _run(x, y, h, eps, v)
    assert out.shape == (500, k)
    _check(out, _ref(x, y, h, eps, v), v, _delta(x, y, eps))
    if k == 1:  # a vector of values gives a vector
        out1 = _run(x, y, h, eps, v[:, 0])
        assert out1.shape == (500,) and torch.equal(out1, out[:, 0])


@pytest.mark.parametrize("d", [96, 200])
@pytest.mark.parametrize("n,m", [(1, 1), (1, 129), (127, 128), (128, 127), (129, 129), (1000, 1100), (1031, 3000)])
@pytest.mark.parametrize("splits", [0, 1, 3])
def test_tile_edges_and_splits(d, n, m, splits, monkeypatch):
    """around the 128-row and 128-column tiles; splits > 0 forces the column split count ($B200OT_FORCE_SPLITS)"""
    if splits:
        monkeypatch.setenv("B200OT_FORCE_SPLITS", str(splits))
    x, y, h, g = _clouds(n, m, d, 7 * n + m + d)
    eps = _eps_for(d)
    v = torch.randn(m, 20, generator=g).to(DEV)
    _check(_run(x, y, h, eps, v), _ref(x, y, h, eps, v), v, _delta(x, y, eps))


@pytest.mark.parametrize("d", [96, 512])
def test_values_of_any_sign_and_scale(d):
    n, m = 900, 1500
    x, y, h, g = _clouds(n, m, d, 5 + d)
    eps = _eps_for(d)
    delta = _delta(x, y, eps)
    v = torch.randn(m, 6, generator=g)
    v[:, 1] *= 1e-6
    v[:, 2] *= 1e6  # side by side with the 1e-6 column: every column is judged on its own scale
    v[:, 3] = v[:, 3].abs()
    v[:, 4] = 2.5  # constant
    v[:, 5] = 1.0
    v = v.to(DEV)
    out = _run(x, y, h, eps, v)
    _check(out, _ref(x, y, h, eps, v), v, delta)
    # a constant comes back: the weights are normalised by the kernel's own sum
    assert (out[:, 4] - 2.5).abs().max().item() <= 2.5 * 2e-6
    assert (out[:, 5] - 1.0).abs().max().item() <= 2e-6
    # strided values, and a row factor applied by the finalize
    wide = torch.randn(m, 10, generator=g).to(DEV)
    r = torch.rand(n, generator=g).to(DEV) + 0.5
    out_s = _run(x, y, h, eps, wide[:, ::2], row_factor=r)
    assert not wide[:, ::2].is_contiguous()
    _check(out_s / r[:, None], _ref(x, y, h, eps, wide[:, ::2]), wide[:, ::2], delta)
    # h = h_a + h_scale_b h_b is fused like the softmin's
    hb = torch.randn(m, generator=g).to(DEV)
    _check(_run(x, y, h, eps, v, h_b=hb, h_scale_b=0.7), _ref(x, y, h + 0.7 * hb, eps, v), v, delta)


@pytest.mark.parametrize("d", [128, 1024])
def test_zero_weight_columns_duplicates_and_translation(d):
    n, m = 700, 1200
    x, y, h, g = _clouds(n, m, d, 40 + d)
    eps = _eps_for(d)
    v = torch.randn(m, 4, generator=g).to(DEV)
    dead = torch.zeros(m, dtype=torch.bool, device=DEV)
    dead[::7] = True
    h0 = torch.where(dead, torch.full_like(h, -1.0e5), h)
    v_big = torch.where(dead[:, None], torch.full_like(v, 1.0e6), v)  # must not leak: the weight is exactly 0
    out = _run(x, y, h0, eps, v_big)
    _check(out, _ref(x, y[~dead], h[~dead], eps, v[~dead]), v, _delta(x, y, eps))
    # duplicated points on both sides
    xd, yd = torch.cat([x, x[:50]]), torch.cat([y, y[:300], y[:300]])
    hd, vd = torch.cat([h, h[:300], h[:300]]), torch.cat([v, v[:300], -v[:300]])
    _check(_run(xd, yd, hd, eps, vd), _ref(xd, yd, hd, eps, vd), vd, _delta(xd, yd, eps))
    # clouds far from the origin: the centre of the expansion travels with them
    shift = torch.full((d,), 1.0e3, device=DEV)
    xs, ys = x + shift, y + shift
    _check(_run(xs, ys, h, eps, v), _ref(xs, ys, h, eps, v), v, _delta(xs, ys, eps), bar=2e-4)


# ------------------------------------------------------------------------------------------------
# ot.solve_sample above D = 64
# ------------------------------------------------------------------------------------------------
def _solve(name, grads=False):
    from geomloss_b200 import ot

    z = load_golden(name)
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    n, m = z["X_a"].shape[0], z["X_b"].shape[0]
    a0 = torch.from_numpy(z["a"]) if "a" in z else torch.full((n,), 1.0 / n)
    b0 = torch.from_numpy(z["b"]) if "b" in z else torch.full((m,), 1.0 / m)
    leaves = [t.to(DEV) for t in (torch.from_numpy(z["X_a"]), torch.from_numpy(z["X_b"]), a0, b0)]
    if grads:
        leaves = [t.requires_grad_(True) for t in leaves]
    else:
        leaves[2] = leaves[2] if "a" in z else None
        leaves[3] = leaves[3] if "b" in z else None
    res = ot.solve_sample(leaves[0], leaves[1], a=leaves[2], b=leaves[3], **kw)
    return z, kw, res, leaves


def _slack_potential(z, res):
    """the expansion error of one softmin in potential units (C = |x - y|^2, no 1/2): 2 (3 dk/16 + 9) 2^-24
    (max |x - c|^2 + max |y - c|^2), with the facade's centre"""
    xa, xb = torch.from_numpy(z["X_a"]).double(), torch.from_numpy(z["X_b"]).double()
    c = res._sm.center.double().cpu()
    n2 = float(((xa - c) ** 2).sum(1).max() + ((xb - c) ** 2).sum(1).max())
    return 2.0 * _cd(xa.shape[1]) * 2.0**-24 * n2


@pytest.mark.parametrize("name", CASES)
def test_ot_solve_sample_wide_vs_reference_goldens(name):
    """value 1e-4 relative, potentials 2e-5 of their scale, marginals / plan 3e-4 of their largest entry (the bars of
    the D <= 64 fixtures), each plus the expansion error of section 3.5d carried to it"""
    z, kw, res, _ = _solve(name)
    reg = kw["reg"]
    sp = _slack_potential(z, res)
    rel = math.expm1(3.0 * sp / reg)  # a plan entry: f, g and the cost each off by up to sp
    ref = float(z["value_f64"])
    mass = float(z["a"].sum() + z["b"].sum()) if "a" in z else 2.0
    assert abs(res.value.item() - ref) <= 1e-4 * abs(ref) + 4.0 * mass * sp, (res.value.item(), ref)
    names = ["potential_a", "potential_b", "marginal_a", "marginal_b", "plan"]
    if kw.get("debias"):
        names += ["potential_aa", "potential_bb"]
    for attr in names:
        r = z[attr + "_f64"]
        out = getattr(res, attr).cpu().numpy()
        assert out.shape == r.shape, attr
        rmax = float(np.abs(r).max())
        tol = 2e-5 * max(1.0, rmax) + 2.0 * sp if "potential" in attr else (3e-4 + rel) * rmax
        np.testing.assert_allclose(out, r, atol=tol, err_msg=attr)


@pytest.mark.parametrize("name", CASES)
def test_ot_solve_sample_wide_gradients_vs_reference(name):
    z, kw, res, leaves = _solve(name, grads=True)
    rel = math.expm1(3.0 * _slack_potential(z, res) / kw["reg"])
    grads = torch.autograd.grad(res.value, leaves)
    for g, gname in zip(grads, ("grad_X_a", "grad_X_b", "grad_a", "grad_b")):
        assert torch.isfinite(g).all(), gname
        if gname + "_f64" not in z:  # cloud gradients are stored up to D = 200 (make_golden_ot_wide.py)
            continue
        r = z[gname + "_f64"]
        np.testing.assert_allclose(g.cpu().numpy(), r, atol=(2e-3 + 4.0 * rel) * float(np.abs(r).max()), err_msg=gname)


@pytest.mark.parametrize("name", CASES)
def test_ot_wide_operators_vs_dense_fp64_plan(name):
    """plan @ V, .T @ W, density @ V, a_to_b, b_to_a and the gradient w.r.t. V against the dense fp64 plan built from
    the returned potentials: 3e-4 of the result's scale plus the exponent term of the operator (and of the row factor,
    from the softmin that produced it)"""
    z, kw, res, _ = _solve(name)
    reg = kw["reg"]
    Xa, Xb = torch.from_numpy(z["X_a"]).to(DEV).double(), torch.from_numpy(z["X_b"]).to(DEV).double()
    n, m = Xa.shape[0], Xb.shape[0]
    a = torch.from_numpy(z["a"]).to(DEV).double() if "a" in z else torch.full((n,), 1.0 / n, device=DEV).double()
    b = torch.from_numpy(z["b"]).to(DEV).double() if "b" in z else torch.full((m,), 1.0 / m, device=DEV).double()
    C = torch.cdist(Xa, Xb) ** 2
    dens = torch.exp((res.potential_a.double()[:, None] + res.potential_b.double()[None, :] - C) / reg)
    P = a[:, None] * b[None, :] * dens
    # the operator runs at eps = reg / 2: its exponent bound in both directions
    dab = float(_delta(Xa.float(), Xb.float(), reg / 2).max())
    dba = float(_delta(Xb.float(), Xa.float(), reg / 2).max())
    ea, eb = 3.0 * (2.0**dab - 1.0), 3.0 * (2.0**dba - 1.0)
    g = torch.Generator().manual_seed(len(name))
    V = torch.randn(m, 70, generator=g).to(DEV)
    W = torch.randn(n, 3, generator=g).to(DEV)
    out = (res.plan_operator @ V).double()
    assert (out - P @ V.double()).abs().max() <= (3e-4 + ea) * (P @ V.double().abs()).max()
    outT = (res.plan_operator.T @ W).double()
    assert (outT - P.t() @ W.double()).abs().max() <= (3e-4 + eb) * (P.t() @ W.double().abs()).max()
    outD = (res.density_operator @ V[:, :5]).double()
    assert (outD - dens @ V[:, :5].double()).abs().max() <= (3e-4 + ea) * (dens @ V[:, :5].double().abs()).max()
    span = max(Xa.abs().max().item(), Xb.abs().max().item())
    ab = (P @ Xb) / P.sum(1, keepdim=True) - Xa
    ba = (P.t() @ Xa) / P.sum(0)[:, None] - Xb
    assert (res.a_to_b.double() - ab).abs().max() <= (3e-4 + ea) * span
    assert (res.b_to_a.double() - ba).abs().max() <= (3e-4 + eb) * span
    Vg = V[:, :3].clone().requires_grad_(True)
    (gv,) = torch.autograd.grad(((res.plan_operator @ Vg) * W).sum(), Vg)
    assert (gv.double() - P.t() @ W.double()).abs().max() <= (3e-4 + eb) * (P.t() @ W.double().abs()).max()


def test_ot_wide_large_problem_sampled_rows():
    """N = M = 5e4, D = 256, K = 256 (four value slabs): the barycentric map against fp64 rows, and plan @ 1 against
    the marginal"""
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(11)
    n = m = 50_000
    d = 256
    X_a, X_b = torch.rand(n, d, generator=g).to(DEV), (torch.rand(m, d, generator=g) * 0.8 + 0.1).to(DEV)
    reg = d / 120.0
    res = ot.solve_sample(X_a, X_b, reg=reg, max_iter=10)
    ab = res.a_to_b
    assert ab.shape == (n, d)
    rows = torch.randint(0, n, (64,), generator=g).to(DEV)
    C = torch.cdist(X_a[rows].double(), X_b.double()) ** 2
    P = torch.exp((res.potential_a.double()[rows, None] + res.potential_b.double()[None, :] - C) / reg) / (n * m)
    ref = (P @ X_b.double()) / P.sum(1, keepdim=True) - X_a[rows].double()
    delta = float(_delta(X_a, X_b, reg / 2)[rows].max())
    assert (ab[rows].double() - ref).abs().max() <= 3e-4 + 2.0 * (2.0**delta - 1.0)
    # plan @ 1 is the row factor times sum_j P_ij / sum_j P_ij, the numerator accumulated by GEMM 2 on the tensor
    # cores and the denominator by fp32 FADDs: over 5e4 columns the two drift apart by up to 7.2e-5 (measured on an
    # H100 80GB HBM3, 700 W; DESIGN.md section 3.5e)
    ones = res.plan_operator @ torch.ones(m, device=DEV)
    assert ((ones - res.marginal_a).abs() / res.marginal_a).max().item() <= 2e-4

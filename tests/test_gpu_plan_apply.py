"""The plan-times-values operator on the GPU (b200ot_plan_apply, ops.plan_apply_raw) and the result-object accessors
built on it (plan_operator / density_operator, a_to_b / b_to_a, the gradient w.r.t. the values), against dense or
row-chunked fp64 evaluations on the device.  Bar of the operator: 5e-5 max_j |V_jk| per value column.  D <= 8 runs the
CUDA-core kernels (planapply.cuh), D > 8 the tensor-core ones (tcapply.cuh); both tile shapes of the CUDA-core plan
and several column splits are visited."""
import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOG2E = 1.4426950408889634


def _clouds(n, m, d, seed, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    x = (spread * torch.rand(n, d, generator=g)).to(DEV)
    y = (spread * torch.rand(m, d, generator=g)).to(DEV)
    h = (0.3 * torch.randn(m, generator=g)).to(DEV)
    return x, y, h, g


def _exponent64(x, y, h, eps):
    """h_j - |x_i - y_j|^2 / (2 eps) in fp64 (N, M)"""
    return h.double()[None, :] - 0.5 * torch.cdist(x.double(), y.double()) ** 2 / eps


def _ref(x, y, h, eps, v, chunk=2048):
    out = []
    for i in range(0, x.shape[0], chunk):
        out.append(torch.softmax(_exponent64(x[i:i + chunk], y, h, eps), dim=1) @ v.double())
    return torch.cat(out)


def _run(x, y, h, eps, v, center="mid", row_factor=None, h_b=None, h_scale_b=0.0):
    from geomloss_b200 import ops

    c = ops.default_center(x, y) if isinstance(center, str) else center
    _, lse2 = ops.softmin_raw(eps, x, y, h, h_b, h_scale_b, p=2, center=c, want_lse2=True)
    return ops.plan_apply_raw(eps, x, y, h, h_b, h_scale_b, lse2, v, row_factor=row_factor, center=c)


def _check(out, ref, v, bar=5e-5):
    scale = v.double().abs().reshape(v.shape[0], -1).max(0).values.clamp_min(1e-300)
    err = ((out.double() - ref).abs().reshape(out.shape[0], -1) / scale).max().item()
    assert err <= bar, err
    return err


def _eps_for(d):
    return 0.02 * d  # unit cubes: |x - y|^2 ~ d / 6, a softmax over many columns at every dimension


@pytest.mark.parametrize("d", [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 33, 64])
def test_every_dimension(d):
    x, y, h, g = _clouds(700, 1100, d, d)
    v = torch.randn(1100, 5, generator=g).to(DEV)
    _check(_run(x, y, h, _eps_for(d), v), _ref(x, y, h, _eps_for(d), v), v)


@pytest.mark.parametrize("d", [3, 8, 16])
@pytest.mark.parametrize("n,m", [(128, 128), (512, 1024), (1023, 1025), (1025, 1023), (4100, 4097), (4609, 5121),
                                 (300, 200_000)])
def test_tile_edges_and_splits(d, n, m):
    """around the 128 / 512-row and 128 / 256 / 1024-column tiles; N, M >= 4096 takes the 512 x 1024 CUDA-core shape;
    M = 2e5 against few rows is cut into many column splits"""
    x, y, h, g = _clouds(n, m, d, 100 * d + n % 97)
    v = torch.randn(m, 4 if d == 3 else 6, generator=g).to(DEV)
    _check(_run(x, y, h, _eps_for(d), v), _ref(x, y, h, _eps_for(d), v), v)


@pytest.mark.parametrize("d", [3, 16])
@pytest.mark.parametrize("k", [1, 3, 4, 8, 9, 64, 65, 130])
def test_value_widths(d, k):
    x, y, h, g = _clouds(600, 900, d, 7 * k + d)
    v = torch.randn(900, k, generator=g).to(DEV)
    out = _run(x, y, h, _eps_for(d), v)
    assert out.shape == (600, k)
    _check(out, _ref(x, y, h, _eps_for(d), v), v)
    if k == 1:  # a vector of values gives a vector
        out1 = _run(x, y, h, _eps_for(d), v[:, 0])
        assert out1.shape == (600,) and torch.equal(out1, out[:, 0])


@pytest.mark.parametrize("d", [2, 3, 16, 64])
@pytest.mark.parametrize("eps", [0.5, 0.05, 1e-3, 1e-5])
def test_temperatures(d, eps):
    """From a flat softmax down to one column taking all the weight.  Where the fp64 exponents of a row put its best
    column 40 (log2 units) ahead of the second, out is that column's row of V whatever the kernels' exponent error;
    elsewhere the bar is widened by the effect on the weights of the exponent's own rounding, computed from the fp64
    data: 2^-18 (|X_i|^2 + |Y_j|^2) at worst for the tensor cores' expansion (csrc/tcconv.cuh), 2^-20 of the same
    for the fp32 FMA chain of the CUDA cores (it vanishes next to the bar from eps ~ 1e-2 up)."""
    n, m = 500, 800
    x, y, h, g = _clouds(n, m, d, 11 * d)
    v = torch.randn(m, 3, generator=g).to(DEV)
    out = _run(x, y, h, eps, v).double()
    t = _exponent64(x, y, h, eps) * LOG2E
    top = t.topk(2, dim=1)
    sure = (top.values[:, 0] - top.values[:, 1]) > 40.0
    ref = _ref(x, y, h, eps, v)
    vmax = v.double().abs().max(0).values
    if sure.any():
        assert ((out[sure] - v.double()[top.indices[sure, 0]]).abs() / vmax).max().item() <= 5e-5
    if eps <= 1e-4:
        assert sure.float().mean().item() > 0.1
    rest = ~sure
    if rest.any():
        c = 0.5 * (torch.minimum(x.min(0).values, y.min(0).values) + torch.maximum(x.max(0).values, y.max(0).values))
        s2 = LOG2E / eps
        xx, yy = s2 * ((x - c).double() ** 2).sum(1), s2 * ((y - c).double() ** 2).sum(1)
        delta = (2.0 ** -18 if d > 8 else 2.0 ** -20) * (xx + yy.max())
        bound = 5e-5 + 2.0 * (2.0 ** delta - 1.0)[:, None]
        assert (((out - ref).abs() / vmax) <= bound)[rest].all(), ((out - ref).abs() / vmax)[rest].max().item()


@pytest.mark.parametrize("d", [3, 16])
def test_values_of_any_sign_and_scale(d):
    n, m = 900, 1500
    x, y, h, g = _clouds(n, m, d, 5 + d)
    eps = _eps_for(d)
    v = torch.randn(m, 6, generator=g)
    v[:, 1] *= 1e-6
    v[:, 2] *= 1e6  # side by side with the 1e-6 column: every column is judged on its own scale
    v[:, 3] = v[:, 3].abs()
    v[:, 4] = 2.5  # constant
    v[:, 5] = 1.0
    v = v.to(DEV)
    out = _run(x, y, h, eps, v)
    _check(out, _ref(x, y, h, eps, v), v)
    # a constant comes back: the weights are normalised by the kernel's own sum
    assert (out[:, 4] - 2.5).abs().max().item() <= 2.5 * 2e-6
    if d <= 8:
        assert torch.equal(out[:, 5], torch.ones_like(out[:, 5]))  # FFMA(e, 1, T) is the FADD of the weight sum
    else:
        assert (out[:, 5] - 1.0).abs().max().item() <= 2e-6
    # strided values, and a row factor applied by the finalize
    wide = torch.randn(m, 10, generator=g).to(DEV)
    r = torch.rand(n, generator=g).to(DEV) + 0.5
    out_s = _run(x, y, h, eps, wide[:, ::2], row_factor=r)
    assert not wide[:, ::2].is_contiguous()
    _check(out_s / r[:, None], _ref(x, y, h, eps, wide[:, ::2]), wide[:, ::2])
    # h = h_a + h_scale_b h_b is fused like the softmin's
    hb = torch.randn(m, generator=g).to(DEV)
    _check(_run(x, y, h, eps, v, h_b=hb, h_scale_b=0.7), _ref(x, y, h + 0.7 * hb, eps, v), v)


@pytest.mark.parametrize("d", [3, 16])
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
    _check(out, _ref(x, y[~dead], h[~dead], eps, v[~dead]), v)
    # duplicated points on both sides
    xd, yd = torch.cat([x, x[:50]]), torch.cat([y, y[:300], y[:300]])
    hd, vd = torch.cat([h, h[:300], h[:300]]), torch.cat([v, v[:300], -v[:300]])
    _check(_run(xd, yd, hd, eps, vd), _ref(xd, yd, hd, eps, vd), vd)
    # clouds far from the origin: the centre of the expansion travels with them
    shift = torch.full((d,), 1.0e3, device=DEV)
    _check(_run(x + shift, y + shift, h, eps, v), _ref(x + shift, y + shift, h, eps, v), v, bar=2e-4)


# ------------------------------------------------------------------------------------------------
# the result object of ot.solve_sample
# ------------------------------------------------------------------------------------------------
def _solve_golden(idx):
    from geomloss_b200 import ot

    z = load_golden(f"ot_sample_case{idx:02d}")
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    t = lambda k: torch.from_numpy(z[k]).to(DEV)  # noqa: E731
    res = ot.solve_sample(t("X_a"), t("X_b"), a=t("a") if "a" in z else None, b=t("b") if "b" in z else None, **kw)
    return z, res


@pytest.mark.parametrize("idx", range(8))
def test_ot_operators_maps_and_gradient_vs_reference_plan(idx):
    z, res = _solve_golden(idx)
    P = torch.from_numpy(z["plan_f64"]).to(DEV)
    n, m = P.shape
    g = torch.Generator().manual_seed(100 + idx)
    V = torch.randn(m, 7, generator=g).to(DEV)
    W = torch.randn(n, 7, generator=g).to(DEV)
    out = (res.plan_operator @ V).double()
    assert out.shape == (n, 7)
    assert (out - P @ V.double()).abs().max() <= 3e-4 * (P @ V.double().abs()).max()
    outT = (res.plan_operator.T @ W).double()
    assert (outT - P.t() @ W.double()).abs().max() <= 3e-4 * (P.t() @ W.double().abs()).max()
    # barycentric maps against the same dense plan
    Xa, Xb = torch.from_numpy(z["X_a"]).to(DEV).double(), torch.from_numpy(z["X_b"]).to(DEV).double()
    span = max(Xa.abs().max().item(), Xb.abs().max().item())
    ab = (P @ Xb) / P.sum(1, keepdim=True) - Xa
    ba = (P.t() @ Xa) / P.sum(0)[:, None] - Xb
    assert res.a_to_b.shape == Xa.shape and res.b_to_a.shape == Xb.shape
    ok_a, ok_b = P.sum(1) > 1e-12, P.sum(0) > 1e-12
    assert (res.a_to_b.double() - ab)[ok_a].abs().max() <= 3e-4 * span
    assert (res.b_to_a.double() - ba)[ok_b].abs().max() <= 3e-4 * span
    # gradient w.r.t. the values: the transposed operator, against the dense plan's autograd
    Vg = V.clone().requires_grad_(True)
    (gv,) = torch.autograd.grad(((res.plan_operator @ Vg) * W).sum(), Vg)
    Vd = V.double().requires_grad_(True)
    (gd,) = torch.autograd.grad(((P @ Vd) * W.double()).sum(), Vd)
    assert (gv.double() - gd).abs().max() <= 3e-4 * (P.t() @ W.double().abs()).max()
    res.cache_clear()
    assert "_apply_cache" not in res.__dict__


@pytest.mark.parametrize("d,reg", [(16, 0.5), (64, 2.0)])
def test_ot_high_dimension_vs_dense_fp64_plan(d, reg):
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(d)
    n, m = 900, 1100
    X_a, X_b = torch.rand(n, d, generator=g).to(DEV), (torch.rand(m, d, generator=g) * 0.9 + 0.1).to(DEV)
    a = torch.rand(n, generator=g).to(DEV) + 0.1
    b = torch.rand(m, generator=g).to(DEV) + 0.1
    a, b = a / a.sum(), b / b.sum()
    res = ot.solve_sample(X_a, X_b, a=a, b=b, reg=reg, max_iter=20)
    C = torch.cdist(X_a.double(), X_b.double()) ** 2
    P = a.double()[:, None] * b.double()[None, :] * torch.exp(
        (res.potential_a.double()[:, None] + res.potential_b.double()[None, :] - C) / reg)
    V = torch.randn(m, d, generator=g).to(DEV)
    out = (res.plan_operator @ V).double()
    assert (out - P @ V.double()).abs().max() <= 3e-4 * (P @ V.double().abs()).max()
    W = torch.randn(n, 3, generator=g).to(DEV)
    outT = (res.plan_operator.T @ W).double()
    assert (outT - P.t() @ W.double()).abs().max() <= 3e-4 * (P.t() @ W.double().abs()).max()
    ab = (P @ X_b.double()) / P.sum(1, keepdim=True) - X_a.double()
    assert (res.a_to_b.double() - ab).abs().max() <= 3e-4


def test_ot_large_problem_sampled_rows():
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(9)
    n = m = 200_000
    X_a, X_b = torch.rand(n, 3, generator=g).to(DEV), (torch.rand(m, 3, generator=g) * 0.8 + 0.2).to(DEV)
    reg = 2 * 0.05 ** 2
    res = ot.solve_sample(X_a, X_b, reg=reg, max_iter=10)
    out = res.plan_operator @ X_b
    rows = torch.randint(0, n, (64,), generator=g).to(DEV)
    C = torch.cdist(X_a[rows].double(), X_b.double()) ** 2
    P = (1.0 / n) * (1.0 / m) * torch.exp(
        (res.potential_a.double()[rows, None] + res.potential_b.double()[None, :] - C) / reg)
    ref = P @ X_b.double()
    assert (out[rows].double() - ref).abs().max() <= 3e-4 * ref.abs().max()
    ones = res.plan_operator @ torch.ones(m, device=DEV)
    assert ((ones - res.marginal_a).abs() / res.marginal_a).max().item() <= 1e-5

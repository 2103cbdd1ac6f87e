"""The p = 1 softmin on the tensor cores for 8 < D <= 64 (csrc/tcconv.cuh tc_reduce_kernel<6>, csrc/tcbwd.cuh
tc_bwd_kernel<7>; ops.softmin_l1_raw / softmin_l1), in both cost conventions: the reference's tensorized
sqrt(max(d^2, 1e-8)) and the pykeops one (no clamp, zero gradient at 0), selected by P_UNCLAMPED.

Every comparison is against float64.  Operator values: 3e-6 max(1, |f|) plus the error of the norm expansion carried
to each row: d^2 is off by at most 2^-18 (|x_i - c|^2 + |y_j - c|^2) (tcconv.cuh), so d_ij by that over 2 d_ij (at most
its square root), and f_i by the softmax-weighted sum of those.  Row gradients: 2e-4 of the largest entry against
autograd of the fp64 operator, 5e-5 at M = 65536 (the bar of test_gpu_tc_streaming.py).  Batches: the bars of
test_gpu_tc_batched.py::test_batched_equals_per_element_loop.  SamplesLoss: the bars of the hd_* fixtures
(test_gpu_reference_goldens.py) against the reference's fp64 runs (tests/golden/p1hd_*.npz)."""
import math

import numpy as np
import pytest
import torch

from conftest import golden_kwargs, golden_names, load_golden
from test_gpu_tc_variants import env

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
UNCLAMPED = 0x100
LN2 = math.log(2.0)


def _clouds(n, m, d, seed, b=None, dup=0):
    g = torch.Generator().manual_seed(seed)
    lead = () if b is None else (b,)
    x = torch.rand(*lead, n, d, generator=g, dtype=torch.float64)
    y = torch.rand(*lead, m, d, generator=g, dtype=torch.float64) * 0.9 + 0.15
    if dup:
        y[..., :dup, :] = x[..., torch.arange(dup) % n, :]  # columns that coincide with rows
    h = torch.randn(*lead, m, generator=g, dtype=torch.float64) * 0.5
    go = torch.randn(*lead, n, generator=g, dtype=torch.float64)
    return tuple(t.float().double().to(DEV) for t in (x, y, h, go))  # fp32-representable


def _dist(x, y, keops):
    if keops:  # pykeops' Norm2: exact differences, sqrt(0) = 0 with a zero gradient
        sq = ((x.unsqueeze(-2) - y.unsqueeze(-3)) ** 2).sum(-1)
        pos = sq > 0
        return torch.where(pos, sq, torch.ones_like(sq)).sqrt() * pos.to(sq.dtype)
    sq = (x * x).sum(-1, keepdim=True) - 2 * x @ y.transpose(-1, -2) + (y * y).sum(-1).unsqueeze(-2)
    return sq.clamp_min(1e-8).sqrt()  # the reference's `distances` (utils.py:56-61)


def _ref(eps, x, y, h, keops, go=None):
    """fp64 softmin (and its row gradient for `go`): -eps logsumexp_j(h_j - d_ij / eps)."""
    xr = x.detach().clone().requires_grad_(go is not None)
    f = -eps * torch.logsumexp(h.unsqueeze(-2) - _dist(xr, y, keops) / eps, dim=-1)
    if go is None:
        return f.detach(), None
    (gx,) = torch.autograd.grad((f * go).sum(), xr)
    return f.detach(), gx


def _slack(eps, x, y, h, center, keops):
    """sum_j w_ij dd_ij, dd = min(dq / (2 d), sqrt(dq)), dq = 2^-18 (|x_i - c|^2 + |y_j - c|^2)."""
    xc, yc = x - center, y - center
    dq = 2.0**-18 * ((xc * xc).sum(-1).unsqueeze(-1) + (yc * yc).sum(-1).unsqueeze(-2))
    d = _dist(x, y, keops)
    dd = torch.minimum(dq / (2 * d.clamp_min(1e-30)), dq.sqrt())
    w = torch.softmax(h.unsqueeze(-2) - d / eps, dim=-1)
    return (w * dd).sum(-1)


def _close(got, ref, bar, what):
    got, ref = got.detach().double(), ref.detach().double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs()
    bar = torch.as_tensor(bar, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > bar
    i = int(torch.argmax(err - bar))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {err.numel()} off, worst {err.flatten()[i]:.3e} " \
                          f"(bar {bar.flatten()[i]:.3e})"


def _center(x, y):
    xf, yf = x.reshape(-1, x.shape[-1]), y.reshape(-1, y.shape[-1])
    lo = torch.minimum(xf.min(0).values, yf.min(0).values)
    hi = torch.maximum(xf.max(0).values, yf.max(0).values)
    return (0.5 * (lo + hi)).float().double()


def _f32(*ts):
    return [None if t is None else t.float().contiguous() for t in ts]


def _check_values(eps, x, y, h, keops, what, center=None, **kw):
    from geomloss_b200 import ops

    p = 1 | (UNCLAMPED if keops else 0)
    center = _center(x, y) if center is None else center
    out, lse2 = ops.softmin_l1_raw(eps, *_f32(x, y, h), p=p, center=center.float(), want_lse2=True, **kw)
    ref, _ = _ref(eps, x, y, h, keops)
    bar = 3e-6 * ref.abs().clamp_min(1.0) + _slack(eps, x, y, h, center, keops)
    _close(out, ref, bar, what)
    # the saved lse2 is the value in log2 units: out = -eps ln2 lse2 to fp32 rounding
    _close(out, -eps * LN2 * lse2.double(), 2e-6 * out.double().abs().clamp_min(1e-3), f"{what} lse2")
    return out, lse2


# ------------------------------------------------------------------------------------------------
# 1. operator values: every padded-dimension boundary, small and large eps, both conventions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("eps", [0.5, 0.01, 5e-4])
@pytest.mark.parametrize("d", [9, 16, 17, 33, 48, 63, 64])
def test_operator_values(d, eps, keops):
    x, y, h, _ = _clouds(300, 700, d, seed=d)
    _check_values(eps, x, y, h, keops, f"D={d} eps={eps} keops={keops}")


@pytest.mark.parametrize("n,m", [(1, 1), (127, 129), (128, 128), (129, 127), (255, 1025), (1000, 257)])
@pytest.mark.parametrize("splits", [1, 3, 7])
def test_ragged_shapes_and_splits(n, m, splits):
    x, y, h, _ = _clouds(n, m, 33, seed=n + m)
    with env(B200OT_FORCE_SPLITS=splits):
        _check_values(0.05, x, y, h, False, f"{n}x{m} splits={splits}")


def test_uncentred_and_translated_clouds():
    x, y, h, _ = _clouds(200, 300, 24, seed=5)
    _check_values(0.1, x + 3.0, y + 3.0, h, False, "translated, centred", center=_center(x + 3.0, y + 3.0))
    _check_values(0.1, x, y, h, True, "no centre", center=torch.zeros(24, dtype=torch.float64, device=DEV))


def test_fused_epilogue_and_zero_weights():
    from geomloss_b200 import ops

    eps = 0.2
    x, y, h, _ = _clouds(300, 400, 40, seed=11)
    hb = torch.randn_like(h)
    h = h.clone()
    h[::3] = -1e5  # zero weights: log_weights pins them at -1e5
    old = torch.randn(300, dtype=torch.float64, device=DEV).float().double()
    c = _center(x, y)
    out, _ = ops.softmin_l1_raw(eps, *_f32(x, y, h, hb), 0.7, center=c.float(), out_old=old.float(), alpha_old=0.5,
                                beta=0.25)
    hh = h + 0.7 * hb
    ref, _ = _ref(eps, x, y, hh, False)
    ref = 0.5 * old + 0.25 * ref
    _close(out, ref, 3e-6 * ref.abs().clamp_min(1.0) + 0.25 * _slack(eps, x, y, hh, c, False), "fused epilogue")


# ------------------------------------------------------------------------------------------------
# 2. row gradients
# ------------------------------------------------------------------------------------------------
def _check_grad(eps, x, y, h, go, keops, what, tol=2e-4, floor=0.0):
    from geomloss_b200 import ops

    p = 1 | (UNCLAMPED if keops else 0)
    c = _center(x, y)
    xg = x.float().requires_grad_(True)
    f = ops.softmin_l1(eps, xg, y.float(), h.float(), p=p, center=c.float())
    (gx,) = torch.autograd.grad(f, xg, go.float())
    _, gref = _ref(eps, x, y, h, keops, go)
    _close(gx, gref, tol * max(floor, gref.abs().max().item()), what)
    return gx, gref


@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("eps", [0.5, 0.05, 2e-3])
@pytest.mark.parametrize("d", [9, 16, 33, 48, 64])
def test_row_gradient(d, eps, keops):
    x, y, h, go = _clouds(300, 520, d, seed=100 + d)
    _check_grad(eps, x, y, h, go, keops, f"D={d} eps={eps} keops={keops}")


@pytest.mark.parametrize("pattern", ["distinct", "copies"])
@pytest.mark.parametrize("eps", [2.0, 0.3])
def test_row_gradient_large_m(pattern, eps):
    """M = 65536 columns at D = 64: near-uniform softmax weights ~2^-16 (eps = 2), where Q = P / d must stay out of
    fp16's subnormal range, and 128 atoms x 512 copies, where a bias of the fp16 image would add up."""
    g = torch.Generator().manual_seed(7)
    n, m, d = 256, 65536, 64
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    if pattern == "distinct":
        y = torch.rand(m, d, generator=g, dtype=torch.float64)
    else:
        y = torch.rand(128, d, generator=g, dtype=torch.float64).repeat(512, 1)
    h = torch.zeros(m, dtype=torch.float64)
    go = torch.randn(n, generator=g, dtype=torch.float64)
    x, y, h, go = (t.float().double().to(DEV) for t in (x, y, h, go))
    _check_grad(eps, x, y, h, go, False, f"M=65536 {pattern} eps={eps}", tol=5e-5)


@pytest.mark.parametrize("keops", [False, True])
def test_coincident_points(keops):
    """Rows that coincide with columns, and the xx term itself: such a pair keeps its weight at d = sqrt(clamp) and has
    no gradient, in each convention.  In the xx term the diagonal takes nearly all the weight, the gradient is a sum
    of weights ~e^-20 (below Q's normal fp16 range, tcconv.cuh kTcL1QLog2) and nearly zero: its bar is taken on the
    scale of a sum of unit vectors, as in test_gpu_tc_streaming.py."""
    from geomloss_b200 import ops

    eps = 0.1
    x, y, h, go = _clouds(200, 300, 33, seed=3, dup=150)
    _check_values(eps, x, y, h, keops, f"cross copies keops={keops}")
    _check_grad(eps, x, y, h, go, keops, f"cross copies keops={keops}")
    # the self term (x is y): the diagonal is exact
    hx = h[:200]
    _check_values(eps, x, x, hx, keops, f"xx keops={keops}")
    _check_grad(eps, x, x, hx, go, keops, f"xx keops={keops}", floor=1.0)
    # a row all of whose columns coincide with it has a zero gradient
    p = 1 | (UNCLAMPED if keops else 0)
    xr = x[:1].repeat(5, 1).float().requires_grad_(True)
    f = ops.softmin_l1(eps, xr, x[:1].repeat(7, 1).float(), torch.zeros(7, device=DEV), p=p)
    (gx,) = torch.autograd.grad(f.sum(), xr)
    assert (gx == 0).all()


# ------------------------------------------------------------------------------------------------
# 3. batches
# ------------------------------------------------------------------------------------------------
def test_batch_of_one_is_the_single_problem():
    from geomloss_b200 import ops

    x, y, h, go = _clouds(300, 400, 33, seed=21)
    c = _center(x, y).float()
    one, l1 = ops.softmin_l1_raw(0.1, *_f32(x, y, h), center=c, want_lse2=True)
    bat, lb = ops.softmin_l1_raw(0.1, *_f32(x[None], y[None], h[None]), center=c, want_lse2=True)
    assert bat.shape == (1, 300) and torch.equal(bat[0], one) and torch.equal(lb[0], l1)
    xg = x.float().requires_grad_(True)
    (g1,) = torch.autograd.grad(ops.softmin_l1(0.1, xg, y.float(), h.float(), center=c), xg, go.float())
    xb = x[None].float().requires_grad_(True)
    (gb,) = torch.autograd.grad(ops.softmin_l1(0.1, xb, y[None].float(), h[None].float(), center=c), xb,
                                go[None].float())
    assert torch.equal(gb[0], g1)


@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("d", [16, 64])
def test_batched_equals_per_element_loop(d, keops):
    from geomloss_b200 import ops

    B, n, m, eps = 5, 200, 333, 0.2
    p = 1 | (UNCLAMPED if keops else 0)
    x, y, h, go = _clouds(n, m, d, seed=31 + d, b=B)
    x, y, h, go = _f32(x, y, h, go)
    c = _center(x, y).float()
    xb = x.clone().requires_grad_(True)
    out = ops.softmin_l1(eps, xb, y, h, p=p, center=c)
    (gb,) = torch.autograd.grad(out, xb, go)
    for k in range(B):
        xk = x[k].clone().requires_grad_(True)
        ok = ops.softmin_l1(eps, xk, y[k], h[k], p=p, center=c)
        (gk,) = torch.autograd.grad(ok, xk, go[k])
        _close(out[k], ok, 5e-6 * ok.detach().abs().double().clamp_min(1e-30), f"element {k} values")
        _close(gb[k], gk, 1e-4 * gk.abs().max().item(), f"element {k} gradients")


# ------------------------------------------------------------------------------------------------
# 4. SamplesLoss against the reference's fp64 runs
# ------------------------------------------------------------------------------------------------
NAMES = golden_names("p1hd_")


def test_fixture_set():
    assert len(NAMES) == 8


@pytest.mark.parametrize("name", NAMES)
def test_samples_loss_matches_reference(name):
    from geomloss_b200 import SamplesLoss

    g = load_golden(name)
    kw = golden_kwargs(g)
    pot = bool(kw.get("potentials", False))
    leaves = [torch.from_numpy(g[k]).to(DEV).requires_grad_(not pot) for k in "axby"]
    out = SamplesLoss(**kw)(*leaves)
    if pot:
        for got, key in zip(out, ("pot_f_f64", "pot_g_f64")):
            ref = torch.from_numpy(g[key]).to(DEV)
            _close(got.view(-1), ref, 1e-4 * max(1.0, ref.abs().max().item()), f"{name} {key}")
        return
    ref = float(g["value_f64"])
    assert abs(out.item() - ref) <= 1e-4 * abs(ref), (name, out.item(), ref)
    grads = torch.autograd.grad(out, leaves)
    for got, key in zip(grads, ("grad_a", "grad_x", "grad_b", "grad_y")):
        r = torch.from_numpy(g[key + "_f64"]).to(DEV).double()
        _close(got.view_as(r), r, 2e-3 * r.abs().max().item(), f"{name} {key}")


def test_samples_loss_batched_equals_loop():
    from geomloss_b200 import SamplesLoss

    g = torch.Generator().manual_seed(5)
    x = torch.rand(3, 300, 40, generator=g).to(DEV)
    y = torch.rand(3, 350, 40, generator=g).to(DEV)
    loss = SamplesLoss("sinkhorn", p=1, blur=0.3, scaling=0.7, diameter=3.0)
    xb = x.clone().requires_grad_(True)
    vals = loss(xb, y)
    (gb,) = torch.autograd.grad(vals.sum(), xb)
    for k in range(3):
        xk = x[k].clone().requires_grad_(True)
        vk = loss(xk, y[k])
        (gk,) = torch.autograd.grad(vk, xk)
        assert abs(vals[k].item() - vk.item()) <= 5e-6 * abs(vk.item()) + 1e-7, (k, vals[k].item(), vk.item())
        _close(gb[k], gk, 1e-4 * gk.abs().max().item(), f"element {k}")


def test_low_dimensions_keep_the_cuda_core_kernels(monkeypatch):
    """D <= 8 never reaches the tensor-core p = 1 operators and still matches the fp64 oracle."""
    from geomloss_b200 import SamplesLoss, ops, sinkhorn_small
    from oracle import geomloss_oracle as O

    def refuse(*a, **k):
        raise AssertionError("the p = 1 tensor-core softmin was called at D <= 8")

    monkeypatch.setattr(ops, "softmin_l1_raw", refuse)
    monkeypatch.setattr(ops, "softmin_l1", refuse)
    monkeypatch.setattr(sinkhorn_small, "SMALL_MAX", 0)  # the tiled kernels, not the one-launch ones
    g = torch.Generator().manual_seed(9)
    for d in (3, 8):
        x, y = torch.rand(700, d, generator=g), torch.rand(650, d, generator=g)
        ref = float(O.samples_loss(x.double(), y.double(), loss="sinkhorn", p=1, blur=0.1, scaling=0.7))
        val = SamplesLoss("sinkhorn", p=1, blur=0.1, scaling=0.7)(x.to(DEV), y.to(DEV)).item()
        assert abs(val - ref) <= 1e-4 * abs(ref), (d, val, ref)

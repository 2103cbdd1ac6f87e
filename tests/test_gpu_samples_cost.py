"""``SamplesLoss("sinkhorn", cost=callable)`` and its grouped row-softmin operator on the GPU: the reference's fixtures,
agreement with the built-in cost, asymmetric costs, the operator against fp64 over shapes, groups, batches, layouts
and planted jumps, equal bits from both load paths, the backward, a 46341^2 matrix, D = 2048, launches and memory."""
import math

import numpy as np
import pytest
import torch

from geomloss_b200 import SamplesLoss, ops, sinkhorn
from test_oracle_samples_cost import CASES, G, fixture, sinkhorn_cost_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _loss(cost, **kw):
    return SamplesLoss("sinkhorn", cost=cost, backend="tensorized", **kw)


@pytest.mark.parametrize("name", CASES)
def test_fixture_parity(name):
    g, cost, kw = fixture(name)
    host = [torch.from_numpy(g[k]) for k in ("a", "x", "b", "y")]
    a, x, b, y = (t.to(DEV).requires_grad_(True) for t in host)
    out = _loss(cost, **kw)(a, x, b, y)
    if kw.get("potentials"):
        xb, yb = (t.double()[None] if t.dim() == 2 else t.double() for t in (host[1], host[3]))
        cmax = max(float(cost(u, v).abs().max()) for u, v in ((xb, yb), (yb, xb), (xb, xb), (yb, yb)))
        for got, ref in zip(out, (g["F_f64"], g["G_f64"])):
            assert got.shape == ref.shape
            assert float(np.abs(got.detach().cpu().double().numpy() - ref).max()) <= 1e-5 * max(1.0, cmax)
        return
    _, duals = sinkhorn_cost_fp64(*(t.double() for t in host), cost, duals=True, **kw)
    ref = g["value_f64"]
    assert out.shape == ref.shape
    scale = max(float(np.abs(ref).max()), duals)
    assert float(np.abs(out.detach().cpu().double().numpy() - ref).max()) <= 1e-4 * scale
    grads = torch.autograd.grad(out.sum(), [x, y, a, b])
    for k, got in zip(("grad_x", "grad_y", "grad_a", "grad_b"), grads):
        ref = g[k + "_f64"]
        assert float(np.abs(got.cpu().double().numpy() - ref).max()) <= 5e-4 * float(np.abs(ref).max()), k


def test_matches_the_builtin_cost():
    gen = torch.Generator().manual_seed(5)
    for shape_x, shape_y in (((700, 3), (500, 3)), ((4, 300, 3), (4, 200, 3))):
        x, y = torch.rand(*shape_x, generator=gen).to(DEV), torch.rand(*shape_y, generator=gen).to(DEV)
        got = _loss(G.half_sqdist)(x, y)
        ref = SamplesLoss("sinkhorn", backend="tensorized")(x, y)
        assert got.shape == ref.shape
        assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


def test_asymmetric_cost_is_not_transposed():
    """C_yx of an asymmetric cost is not C_xy^T: reading C_xy^T in its place gives the value of another cost."""
    gen = torch.Generator().manual_seed(6)
    x, y = torch.rand(300, 3, generator=gen), torch.rand(400, 3, generator=gen)

    def transposing(u, v):  # C_yx := C_xy^T, C_xx, C_yy as the asymmetric cost gives them
        return G.asymmetric(v, u).transpose(1, 2) if u.shape[1] == 400 and v.shape[1] == 300 else G.asymmetric(u, v)

    F = _loss(G.asymmetric, blur=0.1, potentials=True)(x.to(DEV), y.to(DEV))[0].cpu().double()
    F_ref = sinkhorn_cost_fp64(torch.full((300,), 1 / 300, dtype=torch.float64), x.double(),
                               torch.full((400,), 1 / 400, dtype=torch.float64), y.double(), G.asymmetric, blur=0.1,
                               potentials=True)[0]
    F_wrong = sinkhorn_cost_fp64(torch.full((300,), 1 / 300, dtype=torch.float64), x.double(),
                                 torch.full((400,), 1 / 400, dtype=torch.float64), y.double(), transposing, blur=0.1,
                                 potentials=True)[0]
    assert float((F - F_ref).abs().max()) <= 1e-5
    assert float((F_ref - F_wrong).abs().max()) > 1e-2


# ---- the grouped operator against fp64 ---------------------------------------------------------------------------------
def _ref_rows(eps, C, log_w, pot, out_old, alpha, beta):
    h = log_w.double() + (0 if pot is None else pot.double() / eps)
    lse = torch.logsumexp(h.unsqueeze(-2) - C.double() / eps, dim=-1)
    out = beta * (-eps * lse) + (0 if out_old is None else alpha * out_old.double())
    return out, lse / math.log(2)


def _problem(gen, B, N, M, eps, zero=False, jumps=False, pot=True, old=True):
    lead = (B,) if B else ()
    C = torch.rand(*lead, N, M, generator=gen, device=DEV) * 2
    w = torch.rand(*lead, M, generator=gen, device=DEV) + 0.1
    if zero:
        w[..., ::3] = 0.0
    log_w = sinkhorn.log_weights(w / w.sum(-1, keepdim=True))
    if jumps:  # entries far below the rest, met after the running max has settled: > 64 log2 units
        C[..., M // 2:] -= 150 * eps
    p = torch.randn(*lead, M, generator=gen, device=DEV) * 0.3 if pot else None
    o = torch.randn(*lead, N, generator=gen, device=DEV) if old else None
    return C, log_w, p, o


def _check_group(eps, problems, alpha=0.5, beta=0.7, tol=2e-5):
    res = ops.dense_softmin_rows_raw(eps, problems, alpha_old=alpha, beta=beta, want_lse2=True)
    assert len(res) == len(problems)
    for (C, log_w, pot, old), (out, lse2) in zip(problems, res):
        ref, ref2 = _ref_rows(eps, C, log_w, pot, old, alpha if old is not None else 0.0, beta)
        assert out.shape == ref.shape
        scale = max(1.0, float(ref.abs().max()))
        assert float((out.double() - ref).abs().max()) <= tol * scale, tuple(C.shape)
        assert float((lse2.double() - ref2).abs().max()) <= tol * max(1.0, float(ref2.abs().max()))
    return res


SIZES = (1, 31, 32, 33, 127, 128, 129, 1000, 4097)


@pytest.mark.parametrize("N", SIZES)
def test_rows_over_shapes(N):
    gen = torch.Generator(device=DEV).manual_seed(N)
    for M in SIZES:
        _check_group(0.1, [_problem(gen, 0, N, M, 0.1)])


def test_groups_batches_and_layouts():
    gen = torch.Generator(device=DEV).manual_seed(21)
    shapes = [(0, 33, 129), (3, 128, 31), (2, 1000, 257), (0, 1, 4097)]
    for k in range(1, 5):
        _check_group(0.05, [_problem(gen, *s, 0.05) for s in shapes[:k]])
    # no potential and no previous output (the first update of the loop), zero weights, planted jumps
    _check_group(0.05, [_problem(gen, 2, 100, 300, 0.05, pot=False, old=False), _problem(gen, 0, 77, 513, 0.05, True),
                        _problem(gen, 0, 200, 1024, 0.05, jumps=True), _problem(gen, 3, 64, 9, 0.01, True, True)])
    # a batch view off the 16-byte grid, odd n_cols, a non-contiguous C
    buf = torch.rand(3 * 64 * 128 + 1, generator=gen, device=DEV)
    C, log_w, pot, old = _problem(gen, 3, 64, 128, 0.1)
    mis = buf[1:].view(3, 64, 128)
    odd = _problem(gen, 2, 70, 131, 0.1)
    t = torch.rand(2, 131, 70, generator=gen, device=DEV).transpose(1, 2)
    _check_group(0.1, [(mis, log_w, pot, old), odd, (t, *odd[1:])])


@pytest.mark.parametrize("B, N, M", [(1, 300, 1024), (3, 129, 4096), (2, 1000, 128)])
def test_aligned_and_scalar_paths_give_equal_bits(B, N, M):
    gen = torch.Generator(device=DEV).manual_seed(B + N + M)
    C, log_w, pot, old = _problem(gen, B, N, M, 0.05, zero=True, jumps=True)
    buf = torch.empty(C.numel() + 1, device=DEV)
    mis = buf[1:].view_as(C)
    mis.copy_(C)
    outs = [ops.dense_softmin_rows_raw(0.05, [(X, log_w, pot, old)], alpha_old=0.5, beta=0.5, want_lse2=True)[0]
            for X in (C, mis)]
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("B, N, M", [(0, 33, 129), (2, 300, 257), (1, 4097, 31)])
def test_rows_gradient(B, N, M):
    gen = torch.Generator(device=DEV).manual_seed(7 * N + M)
    eps = 0.05
    C, log_w, pot, _ = _problem(gen, B, N, M, eps, zero=True)
    (_, lse2), = ops.dense_softmin_rows_raw(eps, [(C, log_w, pot, None)], want_lse2=True)
    go = torch.randn(lse2.shape, generator=gen, device=DEV)
    grad = ops.dense_softmin_rows_grad(eps, C, log_w, pot, lse2, go)
    Cr = C.double().requires_grad_(True)
    out, _ = _ref_rows(eps, Cr, log_w, pot, None, 0.0, 1.0)
    (ref,) = torch.autograd.grad((out * go.double()).sum(), Cr)
    assert float((grad.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    (_, l2), = ops.dense_softmin_rows_raw(eps, [(C, log_w, None, None)], want_lse2=True)
    grad0 = ops.dense_softmin_rows_grad(eps, C, log_w, None, l2, go)
    out0, _ = _ref_rows(eps, Cr, log_w, None, None, 0.0, 1.0)
    (ref0,) = torch.autograd.grad((out0 * go.double()).sum(), Cr)
    assert float((grad0.double() - ref0).abs().max()) <= 1e-5 * float(ref0.abs().max())


def test_large_matrix_in_a_group():
    N = 46341  # N * N > 2^31
    gen = torch.Generator(device=DEV).manual_seed(11)
    C = torch.rand(1, N, N, device=DEV, generator=gen)
    log_w = torch.full((1, N), -float(np.log(N)), device=DEV)
    pot = torch.randn(1, N, device=DEV, generator=gen) * 0.1
    small = _problem(gen, 0, 100, 77, 0.05)
    (f, _), (fs, _) = ops.dense_softmin_rows_raw(0.05, [(C, log_w, pot, None), small])
    idx = torch.cat([torch.arange(8), torch.randint(0, N, (24,), generator=torch.Generator().manual_seed(3)),
                     torch.arange(N - 8, N)]).to(DEV)
    ref, _ = _ref_rows(0.05, C[0, idx], log_w[0], pot[0], None, 0.0, 1.0)
    assert float((f[0, idx].double() - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))
    ref_s, _ = _ref_rows(0.05, small[0], small[1], small[2], small[3], 0.0, 1.0)
    assert float((fs.double() - ref_s).abs().max()) <= 2e-5 * max(1.0, float(ref_s.abs().max()))


def cosine(u, v):
    un, vn = u / u.norm(dim=-1, keepdim=True), v / v.norm(dim=-1, keepdim=True)
    return 1 - un @ vn.transpose(1, 2)


def test_any_dimension():
    gen = torch.Generator().manual_seed(12)
    x, y = torch.randn(2, 300, 2048, generator=gen), torch.randn(2, 250, 2048, generator=gen)
    a, b = torch.full((2, 300), 1 / 300), torch.full((2, 250), 1 / 250)
    xg = x.to(DEV).requires_grad_(True)
    val = _loss(cosine, blur=0.1)(a.to(DEV), xg, b.to(DEV), y.to(DEV))
    (gx,) = torch.autograd.grad(val.sum(), xg)
    xr = x.double().requires_grad_(True)
    ref, duals = sinkhorn_cost_fp64(a.double(), xr, b.double(), y.double(), cosine, blur=0.1, duals=True)
    (gref,) = torch.autograd.grad(ref.sum(), xr)
    assert float((val.detach().cpu().double() - ref.detach()).abs().max()) <= 1e-4 * max(duals, 1e-3)
    assert float((gx.cpu().double() - gref).abs().max()) <= 5e-4 * float(gref.abs().max())


def test_launches_per_iteration():
    gen = torch.Generator().manual_seed(13)
    x, y = torch.rand(500, 16, generator=gen).to(DEV), torch.rand(400, 16, generator=gen).to(DEV)
    n_eps = len(sinkhorn.scaling_parameters(x, y, 2, 0.05, None, None, 0.5)[2])
    for debias, k in ((True, 4), (False, 2)):
        n0 = ops.launches()
        _loss(G.half_sqdist, debias=debias)(x, y)
        assert ops.launches() - n0 == (n_eps + 2) * (1 + k), debias  # D = 16: the diameter takes torch reductions


def test_memory_beyond_the_four_matrices():
    N = 8192
    gen = torch.Generator(device=DEV).manual_seed(14)
    x, y = torch.rand(N, 3, device=DEV, generator=gen), torch.rand(N, 3, device=DEV, generator=gen)
    _loss(G.half_sqdist)(x[:256], y[:256])  # library and scratch warmed up
    mats = [torch.rand(1, N, N, device=DEV, generator=gen) for _ in range(4)]
    calls = iter(mats)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    _loss(lambda u, v: next(calls))(x, y).item()
    extra = torch.cuda.max_memory_allocated() - base
    total = sum(m.numel() * 4 for m in mats)
    assert extra < 0.02 * total, f"{extra / 2**20:.1f} MiB over the matrices' {total / 2**20:.0f} MiB"

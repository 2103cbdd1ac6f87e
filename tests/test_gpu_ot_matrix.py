"""``ot.solve`` / ``ot.solve_batch`` and the one-pass pair update on an H100: parity with the reference's fp64 fixtures
(tests/golden/make_golden_ot_matrix.py), the reference's doctest values, the properties of OT restated (transpose,
scaling, permutations), every pair update against a fp64 restatement over shapes, alignments and batches, a C with
more than 2^31 entries, the launch count and the memory the solver adds to C."""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from geomloss_b200 import ops, ot

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = golden_names("ot_matrix_case")
LOG2E = 1.4426950408889634


def _case(name):
    z = load_golden(name)
    kw = dict(reg=float(z["kw_reg"]), max_iter=int(z["kw_max_iter"]),
              unbalanced=float(z["kw_unbalanced"]) if "kw_unbalanced" in z else None)
    t = {k: torch.from_numpy(z[k]).to(DEV) for k in ("C", "a", "b", "v")}
    return z, t, kw


def _solve(C, **kw):
    return (ot.solve if C.dim() == 2 else ot.solve_batch)(C, **kw)


def _close(got, ref, atol, what):
    got = got.detach().double().cpu().numpy()
    assert got.shape == ref.shape, what
    err = np.abs(got - ref).max()
    assert err <= atol, f"{what}: max error {err:.3e} > {atol:.3e}"


@pytest.mark.parametrize("name", CASES)
def test_fixture_parity(name):
    z, t, kw = _case(name)
    C, a, b = (t[k].clone().requires_grad_(True) for k in ("C", "a", "b"))
    res = _solve(C, a=a, b=b, **kw)
    ref = z["value_f64"]
    _close(res.value, ref, 1e-4 * np.abs(ref).max(), "value")
    scale = max(1.0, float(np.abs(z["C"]).max()))
    for key in ("potential_a", "potential_b"):
        _close(getattr(res, key), z[key + "_f64"], 1e-5 * scale, key)
    # a marginal is w exp((f - softmin) / eps): one fp32 ulp of f is ulp / eps relative in it (2.4e-4 at the doctests'
    # eps = 1e-3, f ~ 2), and f - softmin carries the rounding of both: the bar is the larger of 1e-5 |C|max and four
    # such ulps
    f_max = max(np.abs(z["potential_a_f64"]).max(), np.abs(z["potential_b_f64"]).max())
    ulp_rel = 4.0 * float(np.spacing(np.float32(f_max))) / kw["reg"]
    for key in ("marginal_a", "marginal_b"):
        ref = z[key + "_f64"]
        _close(getattr(res, key), ref, max(1e-5 * scale, ulp_rel * np.abs(ref).max()), key)
    for key, got in (("plan", res.plan), ("plan_v", res.plan_operator @ t["v"])):
        _close(got, z[key + "_f64"], 1e-4 * np.abs(z[key + "_f64"]).max(), key)
    grads = torch.autograd.grad(res.value.sum(), [C, a, b])
    for got, key in zip(grads, ("grad_C", "grad_a", "grad_b")):
        ref = z[key + "_f64"]
        _close(got, ref, 5e-4 * max(np.abs(ref).max(), 1e-30), key)
    for key in ("potential_a", "potential_b", "marginal_a", "marginal_b", "plan", "density"):
        assert not getattr(res, key).requires_grad, key
    assert res.lazy_plan is None and res.lazy_density is None


def test_doctests():
    C = torch.tensor([[0.0, 1.0, 4.0], [2.0, 1.0, 0.0]], device=DEV)
    res = ot.solve(C, a=torch.tensor([2.0, 2.0], device=DEV), b=torch.tensor([1.0, 1.0, 2.0], device=DEV), reg=1e-3,
                   max_iter=100)
    assert f"{res.value:.3f}" == "0.997"
    np.testing.assert_allclose(res.plan.cpu().numpy(), [[1, 1, 0], [0, 0, 2]], atol=1e-3)
    np.testing.assert_allclose((res.plan_operator @ torch.tensor([-2.0, 1.0, 1.0], device=DEV)).cpu().numpy(), [-1, 2],
                               atol=1e-3)
    Cb = torch.tensor([[[0.0, 1.0, 4.0], [2.0, 1.0, 0.0]], [[0.0, 2.0, 3.0], [1.0, 0.0, 1.0]]], device=DEV)
    res = ot.solve_batch(Cb, a=torch.tensor([[2.0, 2.0], [1.0, 3.0]], device=DEV),
                         b=torch.tensor([[1.0, 1.0, 2.0], [2.0, 1.0, 1.0]], device=DEV), reg=1e-3, max_iter=1000)
    np.testing.assert_allclose(res.value.cpu().numpy(), [0.997, 1.995], atol=5e-4)
    assert res.plan.shape == (2, 2, 3) and res.potential_a.shape == (2, 2) and res.marginal_b.shape == (2, 3)
    assert (res.density_operator @ torch.ones(2, 3, 4, device=DEV)).shape == (2, 2, 4)
    assert (res.plan_operator.T @ torch.ones(2, 2, device=DEV)).shape == (2, 3)
    res.cache_clear()
    np.testing.assert_allclose(res.value.cpu().numpy(), [0.997, 1.995], atol=5e-4)


def _random_problem(g, B, N, M, unbalanced=False):
    C = torch.rand(B, N, M, generator=g, dtype=torch.float64)
    a = torch.rand(B, N, generator=g, dtype=torch.float64) + 0.1
    b = torch.rand(B, M, generator=g, dtype=torch.float64) + 0.1
    a, b = a / a.sum(-1, keepdim=True), b / b.sum(-1, keepdim=True)
    if unbalanced:
        b = 1.3 * b
    return C.float().to(DEV), a.float().to(DEV), b.float().to(DEV)


@pytest.mark.parametrize("rho", [None, 0.5])
def test_transpose_swaps_everything(rho):
    g = torch.Generator().manual_seed(5)
    C, a, b = _random_problem(g, 3, 40, 57, unbalanced=rho is not None)
    kw = dict(reg=0.05, max_iter=30, unbalanced=rho)
    ab = ot.solve_batch(C, a=a, b=b, **kw)
    ba = ot.solve_batch(C.transpose(1, 2), a=b, b=a, **kw)  # a non-contiguous C
    torch.testing.assert_close(ba.value, ab.value, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ba.plan, ab.plan.transpose(1, 2), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(ba.potential_a, ab.potential_b, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(ba.potential_b, ab.potential_a, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("s", [0.01, 1.0, 100.0])
@pytest.mark.parametrize("rho", [None, 0.3])
def test_cost_scaling(s, rho):
    """solve(s C, reg = s reg, unbalanced = s rho): same plan, s times the value (no additive offset: the eps = +inf
    start is not translation-invariant)."""
    g = torch.Generator().manual_seed(6)
    C, a, b = _random_problem(g, 1, 33, 48, unbalanced=rho is not None)
    C, a, b = C[0], a[0], b[0]
    ref = ot.solve(C, a=a, b=b, reg=0.05, max_iter=25, unbalanced=rho)
    res = ot.solve(s * C, a=a, b=b, reg=s * 0.05, max_iter=25, unbalanced=None if rho is None else s * rho)
    torch.testing.assert_close(res.plan, ref.plan, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(res.value, s * ref.value, rtol=1e-4, atol=1e-7 * s)


def test_permutation_cost():
    """A cost with a unique optimal permutation: at small reg the plan is the permutation matrix over N."""
    N = 50
    g = torch.Generator().manual_seed(7)
    perm = torch.randperm(N, generator=g)
    C = torch.rand(N, N, generator=g) + 1.0
    C[torch.arange(N), perm] = 0.0
    res = ot.solve(C.to(DEV), reg=1e-3, max_iter=100)
    P = torch.zeros(N, N)
    P[torch.arange(N), perm] = 1.0 / N
    torch.testing.assert_close(res.plan.cpu(), P, rtol=0, atol=1e-5)


def _pair_ref(eps, C, log_a, log_b, f, g, alpha, beta):
    """fp64 restatement of one fused pair update, in the kernel's log2 units."""
    C, log_a, log_b, f, g = (t.double() for t in (C, log_a, log_b, f, g))
    t = (log_b + g / eps)[..., None, :] - C / eps
    u = (log_a + f / eps)[..., :, None] - C / eps
    lse_r, lse_c = torch.logsumexp(t, -1), torch.logsumexp(u, -2)
    return alpha * f - beta * eps * lse_r, alpha * g - beta * eps * lse_c, LOG2E * lse_r, LOG2E * lse_c


def _pair_inputs(gen, B, N, M, eps, offset=0):
    buf = torch.rand(B * N * M + offset, generator=gen)
    C = buf[offset:].view(B, N, M).to(DEV) if offset == 0 else buf.to(DEV)[offset:].view(B, N, M)
    vec = lambda n, s: (s * torch.randn(B, n, generator=gen)).to(DEV)  # noqa: E731
    log_a = torch.log_softmax(vec(N, 1.0), -1)
    log_b = torch.log_softmax(vec(M, 1.0), -1)
    return C, log_a, log_b, vec(N, 20 * eps), vec(M, 20 * eps)


@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("N", [1, 5, 129])
@pytest.mark.parametrize("M", [1, 3, 127, 128, 1001])
def test_pair_update_shapes(B, N, M):
    gen = torch.Generator().manual_seed(B * 10007 + N * 101 + M)
    eps = 0.1
    offset = 1 if (B, N, M) in ((3, 5, 128), (64, 129, 128)) else 0  # element offsets off the 16-byte grid
    C, log_a, log_b, f, g = _pair_inputs(gen, B, N, M, eps, offset)
    if offset:
        assert C.data_ptr() % 16 != 0
    n0 = ops.launches()
    fo, go, l2r, l2c = ops.dense_softmin_pair_raw(eps, C, log_a, log_b, f, g, alpha_old=0.5, beta=0.7, want_lse2=True)
    assert ops.launches() - n0 == 3
    refs = _pair_ref(eps, C, log_a, log_b, f, g, 0.5, 0.7)
    for got, ref, what in zip((fo, go, l2r, l2c), refs, ("f", "g", "lse2_row", "lse2_col")):
        assert got.shape == ref.shape
        tol = 1e-5 * max(1.0, float(ref.abs().max()))
        assert float((got.double() - ref).abs().max()) <= tol, what
    # the 2-D form of one problem, and a non-contiguous C
    if B == 1:
        fo2, go2, _, _ = ops.dense_softmin_pair_raw(eps, C[0].t().contiguous().t(), log_a[0], log_b[0], f[0], g[0],
                                                    alpha_old=0.5, beta=0.7)
        assert fo2.shape == (N,) and go2.shape == (M,)
        torch.testing.assert_close(fo2, fo[0], rtol=0, atol=0)
        torch.testing.assert_close(go2, go[0], rtol=0, atol=0)
        Ct = C[0].t().contiguous().t()  # same values, transposed strides
        assert not Ct.is_contiguous() or M == 1 or N == 1
        fo3, _, _, _ = ops.dense_softmin_pair_raw(eps, Ct, log_a[0], log_b[0], f[0], g[0], alpha_old=0.5, beta=0.7)
        torch.testing.assert_close(fo3, fo[0], rtol=0, atol=0)


@pytest.mark.parametrize("B, N, M", [(1, 129, 128), (3, 5, 1000), (2, 300, 4096), (64, 17, 36)])
def test_aligned_and_general_paths_agree(B, N, M):
    """C 16-byte aligned with M % 4 == 0 takes the cp.async ring, the same values one float off that grid take the
    scalar loads: the same sums in the same order, so the same bits."""
    gen = torch.Generator().manual_seed(B + N + M)
    eps = 0.05
    C, log_a, log_b, f, g = _pair_inputs(gen, B, N, M, eps)
    assert C.data_ptr() % 16 == 0 and M % 4 == 0
    buf = torch.empty(C.numel() + 1, device=DEV)
    buf[1:] = C.reshape(-1)
    C_off = buf[1:].view(B, N, M)
    outs = [ops.dense_softmin_pair_raw(eps, X, log_a, log_b, f, g, alpha_old=0.5, beta=0.5, want_lse2=True)
            for X in (C, C_off)]
    for got, ref in zip(*outs):
        assert torch.equal(got, ref)
    refs = _pair_ref(eps, C, log_a, log_b, f, g, 0.5, 0.5)
    for got, ref in zip(outs[0], refs):
        assert float((got.double() - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("B, N, M", [(1, 1, 1), (1, 5, 1001), (3, 129, 127), (64, 5, 3), (2, 300, 513)])
def test_pair_gradient(B, N, M):
    gen = torch.Generator().manual_seed(N * M + B)
    eps = 0.07
    C, log_a, log_b, f, g = _pair_inputs(gen, B, N, M, eps)
    _, _, l2r, l2c = ops.dense_softmin_pair_raw(eps, C, log_a, log_b, f, g, want_lse2=True)
    go_f, go_g = torch.randn(B, N, generator=gen).to(DEV), torch.randn(B, M, generator=gen).to(DEV)
    grad = ops.dense_softmin_pair_grad(eps, C, log_a, log_b, f, g, l2r, l2c, go_f, go_g)
    Cd = C.double().requires_grad_(True)
    fr, gr, _, _ = _pair_ref(eps, Cd, log_a, log_b, f, g, 0.0, 1.0)
    (ref,) = torch.autograd.grad((fr * go_f.double()).sum() + (gr * go_g.double()).sum(), [Cd])
    assert float((grad.double() - ref).abs().max()) <= 1e-5 * max(1.0, float(ref.abs().max()))


def test_solve_launches():
    """Each annealing step is one pass plus two finalizes (3 launches), whatever the shape."""
    for B, N, M in ((1, 7, 9), (4, 300, 129), (1, 2000, 3000)):
        C = torch.rand(B, N, M, device=DEV)
        for K in (1, 6):
            n0 = ops.launches()
            ot.solve_batch(C, reg=0.05, max_iter=K)
            assert ops.launches() - n0 == 3 * (K + 1), (B, N, M, K)


def test_large_problem_over_2_31_entries():
    N = 46341  # N * N > 2^31
    gen = torch.Generator(device=DEV).manual_seed(11)
    C = torch.rand(1, N, N, device=DEV, generator=gen)
    assert C.numel() > 2**31
    log_a = torch.full((1, N), -float(np.log(N)), device=DEV)
    f, g = torch.zeros(1, N, device=DEV), torch.zeros(1, N, device=DEV)
    eps = 0.05
    for _ in range(5):
        f_prev, g_prev = f, g
        f, g, l2r, l2c = ops.dense_softmin_pair_raw(eps, C, log_a, log_a, f, g, alpha_old=0.5, beta=0.5,
                                                    want_lse2=True)
    assert bool(torch.isfinite(f).all()) and bool(torch.isfinite(g).all())
    idx = torch.cat([torch.arange(8), torch.randint(0, N, (24,), generator=torch.Generator().manual_seed(3)),
                     torch.arange(N - 8, N)]).to(DEV)
    la, fp, gp = log_a[0].double(), f_prev[0].double(), g_prev[0].double()
    rows = C[0, idx].double()  # (k, N): sampled rows
    ref_f = 0.5 * fp[idx] - 0.5 * eps * torch.logsumexp((la + gp / eps)[None, :] - rows / eps, 1)
    cols = C[0][:, idx].double()  # (N, k): sampled columns
    ref_g = 0.5 * gp[idx] - 0.5 * eps * torch.logsumexp((la + fp / eps)[:, None] - cols / eps, 0)
    assert float((f[0, idx].double() - ref_f).abs().max()) <= 1e-5
    assert float((g[0, idx].double() - ref_g).abs().max()) <= 1e-5
    # the last entries of the last row: int64 offsets past 2^31
    assert float(C[0, N - 1, N - 1]) == float(C.view(-1)[-1])


def test_memory_is_c_plus_vectors():
    """No transposed copy, no scores matrix: a solve adds at most 5 % of C's bytes to what C takes."""
    N = 16384
    ot.solve(torch.rand(64, 64, device=DEV), reg=0.1, max_iter=3)  # library, scratch and cuBLAS workspace warmed up
    C = torch.rand(N, N, device=DEV)
    ot.solve(C[:256, :256].contiguous(), reg=0.1, max_iter=2)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    res = ot.solve(C, reg=0.01, max_iter=10)
    res.potential_a.sum().item()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra <= 0.05 * C.numel() * 4, f"{extra / 2**20:.1f} MiB over C's {C.numel() * 4 / 2**20:.0f} MiB"

"""Entropic OT on regular grids: the per-axis grid softmin (b200ot_softmin_grid_axes), the plan applied to K value
channels (b200ot_grid_plan_apply, grid_apply_kernel) and ``ot.solve_grid`` with its result object.

  A. the softmin against a separable fp64 evaluation: 1-, 2- and 3-D grids with mixed sides from
     {1, 7, 8, 9, 33, 880, 881, 1024}, unequal pitches, every periodic mask; on square grids of pitch 1/N it also
     agrees with b200ot_softmin_grid;
  B. the apply kernel against a dense fp64 plan: K in {1, 4 (one slab), 5, 7}, signed values, zero-weight and -inf
     pixels (s = 0, never NaN), lazy-max spikes along each axis, periodic axes, the 32-, 16- and 8-line tiles, and the
     launch count D ceil(K / 4);
  C. ``solve_grid`` against ``solve_sample`` on the pixel-centre cloud: balanced and unbalanced, with and without
     debias, 1-, 2- and 3-D non-square grids, custom axes; value, potentials, marginals, a_to_b, b_to_a, plan @ V;
  D. periodic grids against an fp64 dense restatement of the solver loop, the value gradient in a and b against fp64
     autograd, the gradient of plan_operator @ V in V against the dense plan;
  E. identities: plan @ 1 = marginal_a, plan.T @ 1 = marginal_b, swapping a and b swaps the potentials, one element
     solved alone equals the same element inside a batch bit for bit;
  F. a 1024^2 batch of two images and a 256^3 volume, with peak memory O(B P K) (a P^2 buffer would not fit).

Bars.  A: 3e-6 max(1, |ref|), that of the square-grid softmin (test_gpu_grid.py), which runs the same pass kernel.
B: l as the softmin it encodes (-eps ln2 l) under the same bar; s under 5e-5 max|V| per channel, the bar of the
point-cloud plan-times-values kernel (test_gpu_plan_apply.py): the conditional means are convex combinations computed
with one fp32 exponential per pair, so their error is a few ulp of the exponent times max|V|.  C: the two solvers run
different fp32 reductions of the same sums (separable passes against direct pair sums) through the same eps ladder;
the Sinkhorn map contracts, so the gap stays at the one-update level: potentials and displacements within 2e-4 of the
problem's cost scale (diameter^2 or the grid pitch), value and marginals within 2e-4 relative.  D: the fp64
restatement follows the same ladder, so the same 2e-4, for the gradients as well.  E: 1e-4 relative
(plan @ 1 runs the apply kernel, the marginal the softmin kernel), bitwise for the batch check.
"""
import math

import pytest
import torch

from fp64_refs import check

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LN2 = math.log(2.0)
VALUE_BAR = 3e-6
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    torch.cuda.init()
    yield
    for sec in sorted(RATIOS):
        what, r = RATIOS[sec]
        print(f"\n[ot_grid] section {sec}: largest error / bar = {r:.3g} ({what})")


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _axis_cost(n, h, periodic):
    k = torch.arange(n, dtype=torch.float64, device=DEV)
    d = (k[:, None] - k[None, :]).abs()
    if periodic:
        d = torch.minimum(d, n - d)
    return (d * h) ** 2


def _softmin64(eps, h, pitch, periodic, budget=2**26):
    """-eps log sum_j exp(h_j - |x_i - x_j|^2 / (2 eps)) on the grid, one exact fp64 log-sum-exp per axis."""
    t = h.double()
    for d in range(t.dim() - 1):
        ax = 1 + d
        n = t.shape[ax]
        K = _axis_cost(n, pitch[d], periodic[d]) / (2 * eps)
        tt = t.movedim(ax, -1)
        flat = tt.reshape(-1, n)
        out = torch.empty_like(flat)
        step = max(1, budget // (n * n))
        for r in range(0, flat.shape[0], step):
            out[r:r + step] = torch.logsumexp(flat[r:r + step, None, :] - K[None], -1)
        t = out.reshape(tt.shape).movedim(-1, ax)
    return -eps * t


def _dense_cost(sides, pitch, periodic):
    idx = torch.meshgrid(*[torch.arange(n, device=DEV) for n in sides], indexing="ij")
    return sum(_axis_cost(n, h, per)[k.reshape(-1)][:, k.reshape(-1)]
               for n, h, per, k in zip(sides, pitch, periodic, idx))


def _apply64(eps, h, v, pitch, periodic):
    """(softmin, s) of the dense fp64 plan: v (K, B, *grid)."""
    B, sides = h.shape[0], tuple(h.shape[1:])
    C = _dense_cost(sides, pitch, periodic)
    E = h.double().reshape(B, 1, -1) - C[None] / (2 * eps)  # (B, P, P)
    sm = -eps * torch.logsumexp(E, -1)
    W = torch.softmax(E, -1)
    W = torch.nan_to_num(W, nan=0.0)
    s = torch.einsum("bij,kbj->kbi", W, v.double().reshape(v.shape[0], B, -1))
    return sm.reshape(h.shape), s.reshape(v.shape)


# ---------------------------------------------------------------------------------------------------------------------
# A. the softmin
# ---------------------------------------------------------------------------------------------------------------------
SHAPES_A = ([(n,) for n in (1, 7, 8, 9, 33, 880, 881, 1024)]
            + [(7, 1024), (1024, 9), (881, 33), (1, 880), (33, 881), (8, 8)]
            + [(9, 33, 8), (1, 7, 881), (33, 8, 9)])


def _masks(dim):
    return [tuple(bool(m >> d & 1) for d in range(dim)) for m in range(1 << dim)]


@pytest.mark.parametrize("shape", SHAPES_A, ids=lambda s: "x".join(map(str, s)))
def test_softmin_axes_vs_fp64(shape):
    from geomloss_b200 import ops

    g = torch.Generator().manual_seed(sum(shape))
    dim = len(shape)
    pitch = [(0.7 + 0.6 * d) / n for d, n in enumerate(shape)]
    h = torch.randn((2,) + shape, generator=g).to(DEV)
    old = torch.randn((2,) + shape, generator=g).to(DEV)
    hb = torch.randn((2,) + shape, generator=g).to(DEV)
    for per in _masks(dim):
        for eps in (0.3 * max(pitch) ** 2, 0.02):
            out = ops.softmin_grid_axes_raw(eps, h, hb, 0.25, pitch=pitch, periodic=per, out_old=old, alpha_old=0.5,
                                            beta=1.5)
            ref = 0.5 * old.double() + 1.5 * _softmin64(eps, h.double() + 0.25 * hb.double(), pitch, per)
            bar = VALUE_BAR * 1.5 * ref.abs().reshape(2, -1).amax(1).clamp_min(1.0)
            check(RATIOS, "A", f"{shape} periodic={per} eps={eps:.3g}", out.reshape(2, -1), ref.reshape(2, -1), bar)


@pytest.mark.parametrize("n,dim", [(8, 2), (33, 2), (880, 2), (881, 2), (1024, 1), (16, 3), (33, 3)])
def test_softmin_axes_matches_square_entry(n, dim):
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn_images import softmin_grid

    g = torch.Generator().manual_seed(n + dim)
    h = torch.randn((2,) + (n,) * dim, generator=g).to(DEV)
    for eps in (1e-3, 0.05):
        out = ops.softmin_grid_axes_raw(eps, h, pitch=[1.0 / n] * dim, periodic=[False] * dim)
        if dim == 1:
            ref = torch.empty_like(h)
            ops._call(h.device, "b200ot_softmin_grid", h, None, 0.0, None, 0.0, 1.0, ref, 2, n, 1, 2, float(eps),
                      launches=1)
        else:
            ref = softmin_grid(eps, 2, h[:, None])[:, 0]
        bar = VALUE_BAR * ref.abs().reshape(2, -1).amax(1).clamp_min(1.0)
        check(RATIOS, "A", f"square {n}^{dim} eps={eps}", out.reshape(2, -1), ref.reshape(2, -1), bar)


# ---------------------------------------------------------------------------------------------------------------------
# B. the apply kernel
# ---------------------------------------------------------------------------------------------------------------------
def _check_apply(sec, what, eps, h, v, pitch, periodic):
    from geomloss_b200 import ops

    K = v.shape[0]
    n0 = ops.launches()
    ell, s = ops.grid_plan_apply_raw(eps, h, None, 0.0, v, pitch=pitch, periodic=periodic)
    assert ops.launches() - n0 == (h.dim() - 1) * -(-K // ops.GRID_APPLY_SLAB)
    assert not torch.isnan(s).any() and not torch.isnan(ell).any()
    sm_ref, s_ref = _apply64(eps, h, v, pitch, periodic)
    live = torch.isfinite(sm_ref)
    assert torch.equal(torch.isfinite(ell), live), what
    assert (s[:, ~live] == 0).all(), what
    sm = torch.where(live, -eps * LN2 * ell.double(), torch.zeros_like(sm_ref))
    sm_ref = torch.where(live, sm_ref, torch.zeros_like(sm_ref))
    B = h.shape[0]
    check(RATIOS, sec, what + " l", sm.reshape(B, -1), sm_ref.reshape(B, -1),
          VALUE_BAR * sm_ref.abs().reshape(B, -1).amax(1).clamp_min(1.0))
    vmax = v.abs().reshape(K, -1).amax(1).double()
    check(RATIOS, sec, what + " s", s.reshape(K, -1), s_ref.reshape(K, -1), 5e-5 * vmax)


@pytest.mark.parametrize("K", [1, 4, 5, 7])
@pytest.mark.parametrize("shape", [(1024,), (300,), (33, 31), (3, 1024), (9, 8, 7)],
                         ids=lambda s: "x".join(map(str, s)))
def test_apply_vs_dense(shape, K):
    g = torch.Generator().manual_seed(K * 1000 + sum(shape))
    dim = len(shape)
    pitch = [(0.5 + 0.5 * d) / n for d, n in enumerate(shape)]
    h = torch.randn((2,) + shape, generator=g).to(DEV)
    h[0].view(-1)[:: 5] = -1e5  # zero-weight pixels (log_weights' floor)
    h[1].view(-1)[1:: 7] = -math.inf
    v = (4 * torch.randn((K, 2) + shape, generator=g) - 1).to(DEV)  # signed values
    for per in (_masks(dim) if dim < 3 else [(False,) * 3, (True, False, True), (True,) * 3]):
        for eps in (0.5 * max(pitch) ** 2, 2e-3):
            _check_apply("B", f"{shape} K={K} periodic={per} eps={eps:.3g}", eps, h, v, pitch, per)


def test_apply_all_inputs_infinite():
    """Outputs none of whose inputs carry weight: l = -inf and s = 0 (a wholly -inf batch element, and, along the
    first axis of a 2-D grid, rows whose every pixel is -inf)."""
    from geomloss_b200 import ops

    h = torch.randn(3, 16, 9, device=DEV)
    h[1] = -math.inf
    v = torch.randn(5, 3, 16, 9, device=DEV)
    ell, s = ops.grid_plan_apply_raw(0.01, h, None, 0.0, v, pitch=[0.1, 0.1], periodic=[False, False])
    assert torch.isneginf(ell[1]).all() and (s[:, 1] == 0).all()
    assert torch.isfinite(ell[0]).all() and torch.isfinite(s).all()


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("spike", [66.0, 140.0, 300.0])
def test_apply_lazy_max_spikes(axis, spike):
    """A plateau 60 log2 units up and a spike far above it at every position of a chunk, along each axis; the rebase
    must rescale the denominator and every numerator alike."""
    g = torch.Generator().manual_seed(int(spike) + axis)
    shape = (40, 24)
    h = torch.randn((1,) + shape, generator=g)
    sl = [slice(None)] * 3
    sl[1 + axis] = slice(10, 30)
    h[tuple(sl)] += 60 * LN2
    for pos in range(8):
        hh = h.clone()
        idx = [0, 5, 5]
        idx[1 + axis] = 16 + pos
        hh[tuple(idx)] += spike * LN2
        v = torch.randn((5, 1) + shape, generator=g)
        _check_apply("B", f"spike {spike} axis {axis} pos {pos}", 2e-3, hh.to(DEV), v.to(DEV), [0.02, 0.03],
                     (axis == 1, False))


@pytest.mark.parametrize("n,K", [(300, 4), (1024, 1), (1024, 4), (600, 2)])
def test_apply_tile_widths(n, K):
    """1-D lines that select the 32-line (n = 300, 4 channels), 16-line (n = 1024 with one, n = 600 with two) and
    8-line (n = 1024 with four) tiles, with more lines than one tile holds."""
    g = torch.Generator().manual_seed(n * K)
    h = torch.randn(37, n, generator=g).to(DEV)
    v = torch.randn(K, 37, n, generator=g).to(DEV)
    for per in (False, True):
        _check_apply("B", f"tiles n={n} K={K} periodic={per}", 3.0 / n**2, h, v, [1.0 / n], [per])


# ---------------------------------------------------------------------------------------------------------------------
# C. solve_grid against solve_sample
# ---------------------------------------------------------------------------------------------------------------------
def _weights(shape, seed, holes=False):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(shape, generator=g) + 0.1
    b = torch.rand(shape, generator=g) + 0.1
    if holes:
        a.view(-1)[::7] = 0.0
    dims = tuple(range(1, len(shape)))
    return (a / a.sum(dims, keepdim=True)).to(DEV), (b / b.sum(dims, keepdim=True)).to(DEV)


def _close(sec, what, got, ref, scale, rel=2e-4):
    check(RATIOS, sec, what, got.reshape(1, -1), ref.reshape(1, -1), rel * scale)


CASES_C = [
    dict(shape=(2, 37), axes=None),
    dict(shape=(2, 12, 9), axes=((-1.0, 2.0), (0.0, 0.5))),
    dict(shape=(1, 16, 16), axes=(0.0, 1.0)),
    dict(shape=(2, 5, 7, 6), axes=((0.0, 1.0), (0.0, 2.0), (1.0, 1.5))),
]


@pytest.mark.parametrize("case", range(len(CASES_C)))
@pytest.mark.parametrize("unbalanced,debias", [(None, False), (None, True), (0.5, False), (0.5, True)])
def test_solve_grid_matches_solve_sample(case, unbalanced, debias):
    from geomloss_b200 import ot

    shape, axes = CASES_C[case]["shape"], CASES_C[case]["axes"]
    a, b = _weights(shape, case, holes=(case == 1))
    reg = 0.01
    kw = dict(reg=reg, unbalanced=unbalanced, debias=debias, max_iter=30)
    res = ot.solve_grid(a, b, axes=axes, **kw)
    geo = res._grid
    X = geo.points(DEV)
    D = len(shape) - 1
    scale = geo.diameter ** 2
    V = torch.randn(shape + (3,), device=DEV)
    pv = res.plan_operator @ V
    ptv = res.plan_operator.T @ V
    for k in range(shape[0]):
        ref = ot.solve_sample(X, X, a[k].reshape(-1), b[k].reshape(-1), **kw)
        w = f"case {case} rho={unbalanced} debias={debias} k={k}"
        _close("C", w + " value", res.value[k], ref.value, abs(ref.value.item()) + 1e-3 * scale)
        _close("C", w + " f", res.potential_a[k], ref.potential_a, scale)
        _close("C", w + " g", res.potential_b[k], ref.potential_b, scale)
        if debias:
            _close("C", w + " f_aa", res.potential_aa[k], ref.potential_aa, scale)
            _close("C", w + " g_bb", res.potential_bb[k], ref.potential_bb, scale)
        _close("C", w + " marginal_a", res.marginal_a[k], ref.marginal_a, ref.marginal_a.abs().max().item())
        _close("C", w + " marginal_b", res.marginal_b[k], ref.marginal_b, ref.marginal_b.abs().max().item())
        pitch = max(geo.pitch)
        _close("C", w + " a_to_b", res.a_to_b[k].reshape(-1, D), ref.a_to_b, pitch, rel=2e-3)
        _close("C", w + " b_to_a", res.b_to_a[k].reshape(-1, D), ref.b_to_a, pitch, rel=2e-3)
        Vk = V[k].reshape(-1, 3)
        r1 = ref.plan_operator @ Vk
        _close("C", w + " plan @ V", pv[k].reshape(-1, 3), r1, r1.abs().max().item())
        r2 = ref.plan_operator.T @ Vk
        _close("C", w + " plan.T @ V", ptv[k].reshape(-1, 3), r2, r2.abs().max().item())


# ---------------------------------------------------------------------------------------------------------------------
# D. periodic grids against an fp64 dense restatement of the loop, and gradients
# ---------------------------------------------------------------------------------------------------------------------
def _solve64(a, b, C, reg, rho, debias, max_iter, diameter):
    from geomloss_b200.ot import annealing_eps
    from geomloss_b200.sinkhorn import log_weights

    B = a.shape[0]
    a, b = a.reshape(B, -1).double(), b.reshape(B, -1).double()
    la, lb = log_weights(a), log_weights(b)

    def damp(e):
        return 1.0 if rho is None else 1.0 / (1.0 + e / rho)

    def sm(e, lw, pot):
        return -e * torch.logsumexp(lw[:, None, :] + (pot[:, None, :] - C[None]) / e, -1)

    def inf(wr, wc, lam):
        f = (C[None] * wc[:, None, :]).sum(-1) / wc.sum(-1, keepdim=True)
        return lam * (f - 0.5 * wr * f)

    eps_list = annealing_eps(diameter**2, reg, max_iter)
    lam = damp(eps_list[0])
    f, g = inf(a, b, lam), inf(b, a, lam)
    faa, gbb = inf(a, a, lam), inf(b, b, lam)
    for e in eps_list:
        lam = damp(e)
        f, g, faa, gbb = (0.5 * f + 0.5 * lam * sm(e, lb, g), 0.5 * g + 0.5 * lam * sm(e, la, f),
                          0.5 * faa + 0.5 * lam * sm(e, la, faa), 0.5 * gbb + 0.5 * lam * sm(e, lb, gbb))
    f, g, faa, gbb = lam * sm(e, lb, g), lam * sm(e, la, f), lam * sm(e, la, faa), lam * sm(e, lb, gbb)
    return (f, g, faa, gbb) if debias else (f, g, None, None)


@pytest.mark.parametrize("shape,periodic", [((2, 24), True), ((2, 10, 12), (True, False)), ((1, 9, 8), True),
                                            ((2, 5, 6, 4), (False, True, True))])
@pytest.mark.parametrize("unbalanced,debias", [(None, True), (0.3, False)])
def test_periodic_vs_dense_loop_and_gradients(shape, periodic, unbalanced, debias):
    from geomloss_b200 import ot

    a, b = _weights(shape, 7 + len(shape))
    reg = 0.02
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    res = ot.solve_grid(ag, bg, periodic=periodic, reg=reg, unbalanced=unbalanced, debias=debias, max_iter=25)
    geo = res._grid
    C = _dense_cost(geo.sides, geo.pitch, geo.periodic)
    f, g, faa, gbb = _solve64(a, b, C, reg, unbalanced, debias, 25, geo.diameter)
    scale, B = geo.diameter**2, shape[0]
    w = f"{shape} periodic={periodic} rho={unbalanced}"
    _close("D", w + " f", res.potential_a.reshape(B, -1), f, scale)
    _close("D", w + " g", res.potential_b.reshape(B, -1), g, scale)
    if debias:
        _close("D", w + " f_aa", res.potential_aa.reshape(B, -1), faa, scale)
    # value and its gradient in a and b (potentials are constants of the value, as in solve_sample)
    a64, b64 = a.reshape(B, -1).double().requires_grad_(True), b.reshape(B, -1).double().requires_grad_(True)
    val64 = _value64(a64, b64, f, g, reg, unbalanced, faa, gbb)
    _close("D", w + " value", res.value, val64, val64.abs().max().item())
    ga, gb = torch.autograd.grad(res.value.sum(), (ag, bg))
    ra, rb = torch.autograd.grad(val64.sum(), (a64, b64))
    _close("D", w + " d/da", ga.reshape(B, -1), ra, ra.abs().max().item(), rel=2e-4)
    _close("D", w + " d/db", gb.reshape(B, -1), rb, rb.abs().max().item(), rel=2e-4)
    # the gradient of plan @ V in V: the transposed dense plan applied to the upstream gradient
    V = torch.randn(shape + (2,), device=DEV, requires_grad=True)
    out = res.plan_operator @ V
    go = torch.randn_like(out)
    (gv,) = torch.autograd.grad(out, V, go)
    plan = (torch.exp((f[:, :, None] + g[:, None, :] - C[None]) / reg) * a.reshape(B, -1, 1).double()
            * b.reshape(B, 1, -1).double())
    ref_out = plan @ V.detach().reshape(B, -1, 2).double()
    _close("D", w + " plan @ V", out.reshape(B, -1, 2), ref_out, ref_out.abs().max().item())
    ref_gv = plan.transpose(1, 2) @ go.reshape(B, -1, 2).double()
    _close("D", w + " d(plan @ V)/dV", gv.reshape(B, -1, 2), ref_gv, ref_gv.abs().max().item())


def _value64(a, b, f, g, eps, rho, faa, gbb):
    if rho is None:
        F, G = (f - faa, g - gbb) if faa is not None else (f, g)
    elif faa is None:
        F = (rho + eps / 2 * b.sum(-1, keepdim=True)) - (rho + eps / 2) * torch.exp(-f / rho)
        G = (rho + eps / 2 * a.sum(-1, keepdim=True)) - (rho + eps / 2) * torch.exp(-g / rho)
    else:
        F = (rho + eps / 2) * (torch.exp(-faa / rho) - torch.exp(-f / rho))
        G = (rho + eps / 2) * (torch.exp(-gbb / rho) - torch.exp(-g / rho))
    return (a * F).sum(-1) + (b * G).sum(-1)


# ---------------------------------------------------------------------------------------------------------------------
# E. identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,periodic,unbalanced", [((3, 20, 30), False, None), ((2, 64), True, 0.2),
                                                       ((2, 6, 5, 7), (True, False, False), None)])
def test_identities(shape, periodic, unbalanced):
    from geomloss_b200 import ot

    a, b = _weights(shape, 11)
    kw = dict(periodic=periodic, reg=0.01, unbalanced=unbalanced, debias=True, max_iter=20)
    res = ot.solve_grid(a, b, **kw)
    ones = torch.ones_like(a)
    w = f"{shape} periodic={periodic}"
    _close("E", w + " plan @ 1", res.plan_operator @ ones, res.marginal_a, res.marginal_a.max().item(), rel=1e-4)
    _close("E", w + " plan.T @ 1", res.plan_operator.T @ ones, res.marginal_b, res.marginal_b.max().item(), rel=1e-4)
    swapped = ot.solve_grid(b, a, **kw)
    assert torch.equal(swapped.potential_a, res.potential_b) and torch.equal(swapped.potential_b, res.potential_a)
    assert torch.equal(swapped.potential_aa, res.potential_bb)
    for k in range(shape[0]):
        alone = ot.solve_grid(a[k:k + 1], b[k:k + 1], **kw)
        assert torch.equal(alone.potential_a[0], res.potential_a[k]), k
        assert torch.equal(alone.potential_b[0], res.potential_b[k]), k
        assert torch.equal(alone.value[0], res.value[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# F. scale
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,K", [((2, 1024, 1024), 2), ((1, 256, 256, 256), 3)])
def test_scale_memory_is_linear(shape, K):
    from geomloss_b200 import ot

    g = torch.Generator(device=DEV).manual_seed(5)
    a = torch.rand(shape, device=DEV, generator=g) + 0.5
    b = torch.rand(shape, device=DEV, generator=g) + 0.5
    dims = tuple(range(1, len(shape)))
    a, b = a / a.sum(dims, keepdim=True), b / b.sum(dims, keepdim=True)
    V = torch.randn(shape + (K,), device=DEV, generator=g)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    res = ot.solve_grid(a, b, reg=1e-3, max_iter=4)
    out = res.plan_operator @ V
    disp = res.a_to_b
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    unit = a.numel() * 4 * max(K, len(shape) - 1)  # bytes of one (B, *grid, K) fp32 tensor
    print(f"\n[ot_grid] {shape} K={K}: peak {peak / 2**20:.0f} MiB = {peak / unit:.1f} x B P K fp32")
    assert peak < 16 * unit
    assert torch.isfinite(res.value).all() and torch.isfinite(out).all() and torch.isfinite(disp).all()
    _close("F", f"{shape} plan @ 1", (res.plan_operator @ torch.ones_like(a)), res.marginal_a,
           res.marginal_a.max().item(), rel=1e-4)

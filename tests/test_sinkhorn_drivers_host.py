"""The Sinkhorn drivers' schedules on CPU: every operator replaced by an fp64 dense stand-in that records its calls.

Each driver must make exactly the calls the eps-scaling schedule defines (the initialisation at eps_0, one averaged
Jacobi step per temperature, the extrapolations and the last, gradient-carrying step: eps, alpha_old, beta or
scale_out, the slot's rows, columns and log-weights, whether it reads and averages potentials, whether its rows carry
a gradient), and reproduce the fp64 oracle's values, potentials and gradients."""
import os
import tempfile

import pytest
import torch

from geomloss_b200 import multiscale, ops, ranges, sinkhorn, sinkhorn_images
from oracle import geomloss_oracle as O
from test_host_logic import _dense_grid_softmin, _pair_mask
from test_samples_cost_host import rows_grad, rows_raw

RTOL = 1e-9
# the two-scale port clusters and extrapolates with its own fp64 arithmetic: its gradients agree to ~2e-7 here
MS_RTOL = 1e-6


def _close(got, ref, rtol=RTOL):
    assert got.shape == ref.shape
    assert (got.detach() - ref.detach()).abs().max() <= rtol * ref.detach().abs().max() + 1e-15


class Recorder:
    """fp64 dense softmins with the signatures of ops.softmin_raw / ops.softmin (an optional ranges problem after
    h_scale_b masks the pairs it does not list); each call logs (op, eps, alpha_old, beta | scale_out, rows, columns,
    log-weights, reads a potential, averages a potential, rows carry a gradient)."""

    def __init__(self, clouds, weights):
        self.clouds, self.weights, self.log = clouds, weights, []

    @staticmethod
    def _name(t, table):
        names = [k for k, v in table.items() if v.numel() == t.numel() and torch.equal(v.reshape(-1), t.reshape(-1))]
        assert len(names) == 1, names
        return names[0]

    def _softmin(self, op, eps, x, y, h_a, h_b, h_scale_b, prob, p, coef, alpha_old, out_old):
        self.log.append((op, eps, alpha_old, coef, self._name(x.detach(), self.clouds),
                         self._name(y, self.clouds), self._name(h_a, self.weights), h_b is not None,
                         out_old is not None, x.requires_grad))
        C = ((x[..., :, None, :] - y[..., None, :, :]) ** 2).sum(-1)
        C = C / 2 if p & 0xFF == 2 else C.sqrt()
        h = (h_a if h_b is None else h_a + h_scale_b * h_b).reshape(y.shape[:-1])
        t = h[..., None, :] - C / eps
        if prob is not None:
            t = t.masked_fill(_pair_mask(prob, x.shape[0], y.shape[0]) == 0, -float("inf"))
        out = -eps * coef * torch.logsumexp(t, -1)
        return out if out_old is None else out + alpha_old * out_old.reshape(out.shape)

    def raw(self, eps, x, y, h_a, h_b=None, h_scale_b=0.0, prob=None, *, p=2, center=None, out_old=None,
            alpha_old=0.0, beta=1.0, out=None, want_lse2=False):
        return self._softmin("raw", eps, x, y, h_a, h_b, h_scale_b, prob, p, beta, alpha_old, out_old), None

    def grad(self, eps, x, y, h_a, h_b=None, h_scale_b=0.0, prob=None, *, p=2, center=None, scale_out=1.0):
        h_b = None if h_b is None else h_b.detach()
        return self._softmin("grad", eps, x, y.detach(), h_a.detach(), h_b, h_scale_b, prob, p, scale_out, 0.0, None)


# the (f_ba, g_ab, f_aa, g_bb) slots: rows, columns, log-weights of the columns
SLOTS = [("x", "y", "b"), ("y", "x", "a"), ("x", "x", "a"), ("y", "y", "b")]


def _schedule(eps_list, rho, slots, init=True, last=True, last_slots=None):
    """The calls of descend(eps_list) (with or without its initialisation) and of a last gradient-carrying step."""
    steps = []
    if init:
        lam = sinkhorn.damping(eps_list[0], rho)
        steps.append([("raw", eps_list[0], 0.0, lam, *s, False, False, False) for s in slots])
    for eps in eps_list:
        steps.append([("raw", eps, 0.5, 0.5 * sinkhorn.damping(eps, rho), *s, True, True, False) for s in slots])
    if last:
        lam = sinkhorn.damping(eps_list[-1], rho)
        steps.append([("grad", eps_list[-1], 0.0, lam, *s, True, False, True) for s in last_slots or slots])
    return steps


def _steps(log, n):
    """The call log cut into steps of n independent calls, each in a canonical order (the order within is free)."""
    assert len(log) % n == 0
    return [sorted(log[i:i + n], key=repr) for i in range(0, len(log), n)]


def _clouds(B, N, M, D, seed):
    g = torch.Generator().manual_seed(seed)
    shape = (B,) if B else ()
    x = torch.rand(*shape, N, D, generator=g, dtype=torch.float64)
    y = torch.rand(*shape, M, D, generator=g, dtype=torch.float64) * 0.8 + 0.15
    a = torch.rand(*shape, N, generator=g, dtype=torch.float64) + 0.2
    b = torch.rand(*shape, M, generator=g, dtype=torch.float64) + 0.2
    return a / a.sum(-1, keepdim=True), x, b / b.sum(-1, keepdim=True), y


# ---- point clouds: one problem (D = 3, 16), a batch (D <= 8: ranges problems, D > 8: batched operators) ------------
@pytest.mark.parametrize("B, D", [(0, 3), (0, 16), (3, 3), (3, 16)])
@pytest.mark.parametrize("kw", [dict(), dict(reach=0.3, debias=False)])
def test_points(monkeypatch, B, D, kw):
    a, x, b, y = _clouds(B, 11, 7, D, D + B)
    rec = Recorder(dict(x=x, y=y), dict(a=sinkhorn.log_weights(a), b=sinkhorn.log_weights(b)))
    for raw, grad in (("softmin_raw", "softmin"), ("softmin_batched_raw", "softmin_batched")):
        monkeypatch.setattr(ops, raw, rec.raw)
        monkeypatch.setattr(ops, grad, rec.grad)
    monkeypatch.setattr(ranges, "softmin_ranges_raw", rec.raw)
    monkeypatch.setattr(ranges, "softmin_ranges", rec.grad)
    drive = sinkhorn.sinkhorn_points_batched if B else sinkhorn.sinkhorn_points
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    val = drive(a, xg, b, yg, blur=0.1, **kw)

    debias = kw.get("debias", True)
    slots = SLOTS[:4 if debias else 2]
    eps_list = sinkhorn.scaling_parameters(x, y, 2, 0.1, kw.get("reach"), None, 0.5)[2]
    rho = None if "reach" not in kw else kw["reach"] ** 2
    assert _steps(rec.log, len(slots)) == [sorted(s, key=repr) for s in _schedule(eps_list, rho, slots)]

    ob = (lambda t: t) if B else (lambda t: t[None])
    xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ref = O.sinkhorn_dense(ob(a), ob(xr), ob(b), ob(yr), blur=0.1, **kw)
    _close(val, ref if B else ref[0])
    for g, r in zip(torch.autograd.grad(val.sum(), [xg, yg]), torch.autograd.grad(ref.sum(), [xr, yr])):
        _close(g, r)
    F, G = drive(a, x, b, y, blur=0.1, potentials=True, **kw)
    Fr, Gr = O.sinkhorn_dense(ob(a), ob(x), ob(b), ob(y), blur=0.1, potentials=True, **kw)
    _close(F, Fr if B else Fr[0])
    _close(G, Gr if B else Gr[0])


# ---- user cost matrices ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("debias", [True, False])
def test_cost_matrices(monkeypatch, debias):
    a, x, b, y = _clouds(2, 9, 6, 3, 7)
    log = []

    def raw(eps, problems, *, alpha_old=0.0, beta=1.0, want_lse2=False):
        log.append((eps, alpha_old, beta, tuple((pot is not None, old is not None) for _, _, pot, old in problems)))
        return rows_raw(eps, problems, alpha_old=alpha_old, beta=beta, want_lse2=want_lse2)

    monkeypatch.setattr(ops, "dense_softmin_rows_raw", raw)
    monkeypatch.setattr(ops, "dense_softmin_rows_grad", rows_grad)
    cost = lambda u, v: O.cost_matrix(u, v, 2)  # noqa: E731
    xg = x.clone().requires_grad_(True)
    val = sinkhorn.sinkhorn_cost_matrices(a, xg, b, y, cost, blur=0.1, debias=debias)
    n = 4 if debias else 2
    eps_list = sinkhorn.scaling_parameters(x, y, 2, 0.1, None, None, 0.5)[2]
    assert log == [(eps_list[0], 0.0, 1.0, ((False, False),) * n)] + [
        (eps, 0.5, 0.5, ((True, True),) * n) for eps in eps_list] + [(eps_list[-1], 0.0, 1.0, ((True, False),) * n)]
    xr = x.clone().requires_grad_(True)
    ref = O.sinkhorn_dense(a, xr, b, y, blur=0.1, debias=debias)
    _close(val, ref)
    _close(torch.autograd.grad(val.sum(), xg)[0], torch.autograd.grad(ref.sum(), xr)[0])


# ---- two scales ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("truncate", [None, 5])
@pytest.mark.parametrize("blur, cluster_scale, last_is_jump", [(0.05, 0.2, False), (0.2, 0.15, True)])
def test_multiscale(monkeypatch, truncate, blur, cluster_scale, last_is_jump):
    a, x, b, y = _clouds(0, 40, 30, 2, 11)
    (a_c, x_c), (a_s, x_s), *_ = multiscale.clusterize(a, x, scale=cluster_scale)
    (b_c, y_c), (b_s, y_s), *_ = multiscale.clusterize(b, y, scale=cluster_scale)
    lw = sinkhorn.log_weights
    rec = Recorder(dict(x=x_s, y=y_s, xc=x_c, yc=y_c), dict(a=lw(a_s), b=lw(b_s), ac=lw(a_c), bc=lw(b_c)))
    for name, op in (("dense_raw", rec.raw), ("dense", rec.grad), ("sparse_raw", rec.raw), ("sparse", rec.grad)):
        monkeypatch.setattr(multiscale.LocalEngine, name, staticmethod(op))
    kw = dict(blur=blur, reach=0.5, truncate=truncate, cluster_scale=cluster_scale)
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    val = multiscale.sinkhorn_multiscale(a, xg, b, yg, **kw)

    eps_list = sinkhorn.scaling_parameters(x, y, 2, blur, None, None, 0.5)[2]
    jump = next((i + 1 for i, e in enumerate(eps_list[2:]) if cluster_scale ** 2 > e), len(eps_list) - 1)
    assert (jump == len(eps_list) - 1) == last_is_jump
    rho = 0.25
    coarse = [(r + "c", c + "c", w + "c") for r, c, w in SLOTS]
    extrapolation = [(r, c + "c", w + "c") for r, c, w in SLOTS]
    want = _schedule(eps_list[:jump + 1], rho, coarse, last=False)
    lam = sinkhorn.damping(eps_list[jump], rho)
    if last_is_jump:
        want.append([("grad", eps_list[jump], 0.0, lam, *s, True, False, True) for s in extrapolation])
    else:
        want.append([("raw", eps_list[jump], 0.0, lam, *s, True, False, False) for s in extrapolation])
        want += _schedule(eps_list[jump + 1:], rho, SLOTS, init=False)
    assert _steps(rec.log, 4) == [sorted(s, key=repr) for s in want]

    xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ref = O.sinkhorn_multiscale_dense(a, xr, b, yr, **kw)
    _close(val, ref, MS_RTOL)
    for g, r in zip(torch.autograd.grad(val, [xg, yg]), torch.autograd.grad(ref, [xr, yr])):
        _close(g, r, MS_RTOL)
    for got, r in zip(multiscale.sinkhorn_multiscale(a, x, b, y, potentials=True, **kw),
                      O.sinkhorn_multiscale_dense(a, x, b, y, potentials=True, **kw)):
        _close(got, r, MS_RTOL)


# ---- images ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 1, 16, 16), (1, 2, 8, 8, 8)])
@pytest.mark.parametrize("scaling, last_jump_is_last", [(0.5, True), (0.7, False)])
def test_images(monkeypatch, shape, scaling, last_jump_is_last):
    log = []

    def grid(eps, p, h_a, h_b=None, h_scale_b=0.0, *, out_old=None, alpha_old=0.0, beta=1.0):
        log.append(("raw", eps, alpha_old, beta, tuple(h_a.shape[2:]), h_b is not None, out_old is not None))
        return _dense_grid_softmin(eps, p, h_a, h_b, h_scale_b, out_old=out_old, alpha_old=alpha_old, beta=beta)

    monkeypatch.setattr(sinkhorn_images, "softmin_grid", grid)
    g = torch.Generator().manual_seed(len(shape))
    dims = tuple(range(2, len(shape)))
    a = torch.rand(*shape, generator=g, dtype=torch.float64) + 0.01
    b = torch.rand(*shape, generator=g, dtype=torch.float64) + 0.01
    a, b = a / a.sum(dims, keepdim=True), b / b.sum(dims, keepdim=True)
    blur = 1 / shape[-1]
    kw = dict(blur=blur, reach=0.3, scaling=scaling)
    ag = a.clone().requires_grad_(True)
    val = sinkhorn_images.sinkhorn_divergence(ag, b, **kw)

    eps_list = sinkhorn.epsilon_schedule(2, 1, blur, scaling)
    sides = [2 ** k for k in range(1, shape[-1].bit_length())]
    jumps, level = [], 0
    for i, eps in enumerate(eps_list[1:]):
        if (1 / sides[level]) ** 2 > eps:
            jumps.append(i + 1)
            level += 1
    assert (jumps[-1] == len(eps_list) - 1) == last_jump_is_last
    rho, level, want = 0.09, 0, []
    lam = sinkhorn.damping(eps_list[0], rho)
    want.append([("raw", eps_list[0], 0.0, lam, (sides[0],) * len(dims), False, False)] * 4)
    for i, eps in enumerate(eps_list):
        want.append([("raw", eps, 0.5, 0.5 * sinkhorn.damping(eps, rho), (sides[level],) * len(dims), True, True)] * 4)
        level += i in jumps
    if not last_jump_is_last:
        lam = sinkhorn.damping(eps_list[-1], rho)
        want.append([("raw", eps_list[-1], 0.0, lam, (sides[-1],) * len(dims), True, False)] * 4)
    assert _steps(log, 4) == want

    ar = a.clone().requires_grad_(True)
    ref = O.sinkhorn_images(ar, b, **kw)
    _close(val, ref)
    _close(torch.autograd.grad(val.sum(), ag)[0], torch.autograd.grad(ref.sum(), ar)[0])
    for got, r in zip(sinkhorn_images.sinkhorn_divergence(a, b, potentials=True, **kw),
                      O.sinkhorn_images(a, b, potentials=True, **kw)):
        _close(got, r)


# ---- column-sharded engine (world 1, gloo): what reaches softmin_raw_many --------------------------------------------
def test_sharded_engine_groups_the_points_steps_only():
    import torch.distributed as dist

    from geomloss_b200.distributed import ColumnShardedEngine
    from test_distributed_gloo import OracleStages

    with tempfile.TemporaryDirectory() as tmp:
        dist.init_process_group("gloo", init_method="file://" + os.path.join(tmp, "store"), rank=0, world_size=1)
        try:
            eng = ColumnShardedEngine(stages=OracleStages())
            groups = []
            many = eng.softmin_raw_many
            eng.softmin_raw_many = lambda calls: groups.append([kw.get("alpha_old", 0.0) for _, kw in calls]) or \
                many(calls)
            a, x, b, y = (t.float() for t in _clouds(0, 40, 30, 2, 3))
            sinkhorn.sinkhorn_points(a, x, b, y, blur=0.1, softmin_raw=eng.softmin_raw, softmin_grad=eng.softmin)
            eps_list = sinkhorn.scaling_parameters(x, y, 2, 0.1, None, None, 0.5)[2]
            assert [g for g in groups if g[0] == 0.5] == [[0.5] * 4] * len(eps_list)
            assert all(len(g) == 4 for g in groups)
            groups.clear()
            multiscale.sinkhorn_multiscale(a, x, b, y, blur=0.05, cluster_scale=0.2, engine=eng)
            assert groups == []
        finally:
            dist.destroy_process_group()

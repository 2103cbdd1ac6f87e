"""The operators above D = 64 on the K-slab tensor-core kernels (csrc/tcwide.cuh; ops.softmin_wide*,
ops.kernel_conv_wide*), against float64.

Bars: the project's (values 3e-6 max(1, |f|) of the operator, potentials 1e-5, gradients 5e-4 of the largest entry,
loss 1e-4 relative) plus the expansion error of d^2 carried to each output, computed here from the fp64 data
(DESIGN.md section 3.5d): |computed d^2 - d^2| <= e_ij = (3 dk/16 + 9) 2^-23 (|X_i|^2 + |Y_j|^2) in the kernels'
scaled coordinates, i.e. (3 dk/16 + 9) 2^-24 (|x_i - c|^2 + |y_j - c|^2) in potential units for the p = 2 softmin,
whatever eps.  Distances are then off by min(e / 2d, sqrt(e)), and pairs closer than the row's coincidence bound T_i
count as coincident (d = sqrt(clamp), no gradient)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
UNCLAMPED = 0x100
LOG2E = 1.0 / math.log(2.0)


def _dk(d):
    return -(-d // 16) * 16


def _cd(d):
    return 3 * _dk(d) // 16 + 9


def _clouds(n, m, d, seed, b=None, dup=0, spread=2.0):
    """Coordinates of norm ~ spread / sqrt(3) about the centre whatever D (a cube of side spread / sqrt(D))."""
    g = torch.Generator().manual_seed(seed)
    lead = () if b is None else (b,)
    s = spread / math.sqrt(d)
    x = torch.rand(*lead, n, d, generator=g, dtype=torch.float64) * s
    y = torch.rand(*lead, m, d, generator=g, dtype=torch.float64) * s * 0.9 + 0.1 * s
    if dup:
        y[..., :dup, :] = x[..., torch.arange(dup) % n, :]
    h = torch.randn(*lead, m, generator=g, dtype=torch.float64) * 0.3
    w = torch.rand(*lead, m, generator=g, dtype=torch.float64) + 0.1
    go = torch.randn(*lead, n, generator=g, dtype=torch.float64)
    return tuple(t.float().double().to(DEV) for t in (x, y, h, w, go))


def _center(x, y):
    xf, yf = x.reshape(-1, x.shape[-1]), y.reshape(-1, y.shape[-1])
    lo = torch.minimum(xf.min(0).values, yf.min(0).values)
    hi = torch.maximum(xf.max(0).values, yf.max(0).values)
    return (0.5 * (lo + hi)).float().double()


def _sq(x, y):
    return ((x * x).sum(-1).unsqueeze(-1) - 2 * x @ y.transpose(-1, -2) + (y * y).sum(-1).unsqueeze(-2)).clamp_min(0)


def _n2(x, c):
    return ((x - c) ** 2).sum(-1)


def _dist(x, y, keops):
    sq = _sq(x, y)
    if keops:
        pos = sq > 1e-24
        return torch.where(pos, sq, torch.ones_like(sq)).sqrt() * pos.to(sq.dtype)
    return sq.clamp_min(1e-8).sqrt()


def _energy_scale(x, y, c):
    amax = max(float((x - c).abs().max()), float((y - c).abs().max()))
    _, e = math.frexp(amax)
    return 2.0 ** max(-40, min(40, 10 - e))


def _dist_slack(x, y, c, d, scale):
    """Error bound of the kernels' d_ij in real units (expansion error and coincidence bound)."""
    D = x.shape[-1]
    nx, ny = _n2(x, c), _n2(y, c)
    e = _cd(D) * 2.0**-23 * (nx.unsqueeze(-1) + ny.unsqueeze(-2))
    rel = max(2.0**-17, _cd(D) * 2.0**-22)
    T = (rel * nx + 2.0**-14 / scale**2).unsqueeze(-1)
    dd = torch.minimum(e / (2 * d.clamp_min(1e-30)), e.sqrt())
    near = d * d < 2 * (T + e)
    return torch.where(near, (T + e).sqrt() * 2, dd), near


def _close(got, ref, bar, what):
    got, ref = got.detach().double(), ref.detach().double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs()
    bar = torch.as_tensor(bar, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > bar
    i = int(torch.argmax(err - bar))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {err.numel()} off, worst {err.flatten()[i]:.3e} " \
                          f"(bar {bar.flatten()[i]:.3e})"


def _f32(*ts):
    return [None if t is None else t.float().contiguous() for t in ts]


# ------------------------------------------------------------------------------------------------
# softmin, p = 1 and 2
# ------------------------------------------------------------------------------------------------
def _softmin_ref(eps, x, y, h, p, keops, go):
    xr = x.detach().clone().requires_grad_(True)
    C = _sq(xr, y) / 2 if p == 2 else _dist(xr, y, keops)
    f = -eps * torch.logsumexp(h.unsqueeze(-2) - C / eps, dim=-1)
    (gx,) = torch.autograd.grad((f * go).sum(), xr)
    w = torch.softmax(h.unsqueeze(-2) - C.detach() / eps, dim=-1)
    return f.detach(), gx, w


def _check_softmin(eps, x, y, h, go, p, keops, what, grad=True):
    from geomloss_b200 import ops

    c = _center(x, y)
    pk = p | (UNCLAMPED if keops else 0)
    xf, yf, hf = _f32(x, y, h)
    f_ref, g_ref, w = _softmin_ref(eps, x, y, h, p, keops, go)
    D = x.shape[-1]
    if p == 2:
        slack_f = _cd(D) * 2.0**-24 * (_n2(x, c).unsqueeze(-1) + _n2(y, c).unsqueeze(-2))
        near = torch.zeros_like(slack_f, dtype=torch.bool)
    else:
        slack_f, near = _dist_slack(x, y, c, _dist(x, y, keops), _energy_scale(x, y, c))
    out, lse2 = ops.softmin_wide_raw(eps, xf, yf, hf, p=pk, center=c.float(), want_lse2=True)
    _close(out, f_ref, 3e-6 * f_ref.abs().clamp_min(1.0) + (w * slack_f).sum(-1), f"{what} value")
    if not grad:
        return
    xg = xf.clone().requires_grad_(True)
    val = ops.softmin_wide(eps, xg, yf, hf, p=pk, center=c.float())
    (gx,) = torch.autograd.grad((val * go.float()).sum(), xg)
    # a relative error delta_ij = slack / eps of the softmax weights moves row i's gradient by at most
    # 2 |go_i| sum_j w_ij delta_ij |x_i - y_j| per coordinate (p = 1: the unit vectors, and coincident pairs fully)
    diff = (x.unsqueeze(-2) - y.unsqueeze(-3)).abs()
    if p == 2:
        move = 2 * (w * slack_f / eps).unsqueeze(-1) * diff
    else:
        d = _dist(x, y, keops).unsqueeze(-1)
        move = (w * slack_f / eps).unsqueeze(-1) * 2 + (w * near).unsqueeze(-1) * 2 + \
            (w.unsqueeze(-1) * 2 * slack_f.unsqueeze(-1) / d.clamp_min(1e-30)).clamp_max(2 * w.unsqueeze(-1))
    slack_g = go.abs().unsqueeze(-1) * move.sum(-2)
    _close(gx, g_ref, 5e-4 * g_ref.abs().max() + slack_g, f"{what} gradient")


@pytest.mark.parametrize("d", [65, 72, 96, 127, 128, 200, 256, 512, 1000, 1024])
@pytest.mark.parametrize("p,keops", [(2, False), (1, False), (1, True)])
def test_softmin_dimensions(d, p, keops):
    x, y, h, _, go = _clouds(300, 257, d, seed=d + p)
    for eps in (0.5, 0.02):
        _check_softmin(eps, x, y, h, go, p, keops, f"D={d} p={p} keops={keops} eps={eps}")


@pytest.mark.parametrize("n,m", [(1, 1), (1, 129), (127, 1), (128, 128), (129, 127), (257, 4000), (4000, 257)])
@pytest.mark.parametrize("d", [65, 128, 200])
@pytest.mark.parametrize("p", [1, 2])
def test_softmin_tile_edges(n, m, d, p):
    x, y, h, _, go = _clouds(n, m, d, seed=n + m + d)
    _check_softmin(0.1, x, y, h, go, p, False, f"N={n} M={m} D={d} p={p}")


@pytest.mark.parametrize("p", [1, 2])
def test_softmin_many_columns(p):
    """M = 65536: P (p = 2) and Q (p = 1) stay inside fp16's range over 512 column tiles."""
    x, y, h, _, go = _clouds(128, 65536, 128, seed=7)
    _check_softmin(0.05, x, y, h, go, p, False, f"M=65536 p={p}")
    # 128 atoms repeated 512 times: every row sees the same weights many times over
    atoms = y[:128]
    _check_softmin(0.05, x, atoms.repeat(512, 1), h, go, p, False, f"M=65536 repeated p={p}")


@pytest.mark.parametrize("p,keops", [(2, False), (1, False), (1, True)])
def test_softmin_duplicates_and_self(p, keops):
    x, y, h, _, go = _clouds(200, 300, 96, seed=3, dup=150)
    _check_softmin(0.05, x, y, h, go, p, keops, "duplicated points")
    xs, _, hs, _, _ = _clouds(257, 257, 160, seed=4)
    _check_softmin(0.05, xs, xs, hs, go[:257] if go.shape[0] >= 257 else torch.ones(257, dtype=torch.float64,
                                                                                       device=DEV), p, keops, "x == y")


@pytest.mark.parametrize("b", [1, 3, 17])
@pytest.mark.parametrize("p", [1, 2])
def test_softmin_batches(b, p):
    x, y, h, _, go = _clouds(129, 200, 96 if b == 17 else 300, seed=b, b=b)
    _check_softmin(0.1, x, y, h, go, p, False, f"B={b} p={p}")


# ------------------------------------------------------------------------------------------------
# kernel convolutions
# ------------------------------------------------------------------------------------------------
def _kernel_ref(kind, x, y, w, blur, keops):
    if kind == 0:
        return torch.exp(-_sq(x, y) / (2 * blur * blur))
    d = _dist(x, y, keops)
    return torch.exp(-d / blur) if kind == 1 else -d


def _check_conv(kind, x, y, w, go, blur, keops, what, grads=True):
    from geomloss_b200 import ops

    c = _center(x, y)
    kid = kind | (UNCLAMPED if keops else 0)
    D = x.shape[-1]
    xf, yf, wf = _f32(x, y, w)
    K = _kernel_ref(kind, x, y, w, blur, keops)
    ref = (K * w.unsqueeze(-2)).sum(-1)
    if kind == 0:
        eS = _cd(D) * 2.0**-24 * LOG2E * (_n2(x, c).unsqueeze(-1) + _n2(y, c).unsqueeze(-2)) / blur**2
        pair = K.abs() * math.log(2) * eS
        near = torch.zeros_like(K, dtype=torch.bool)
        dd = None
    else:
        scale = _energy_scale(x, y, c) if kind == 2 else LOG2E / blur
        d = _dist(x, y, keops)
        dd, near = _dist_slack(x, y, c, d, scale)
        pair = K.abs() * dd / blur if kind == 1 else dd
    out = ops.kernel_conv_wide_raw(kid, xf, yf, wf, blur, center=c.float())
    bar = 3e-6 * (K.abs() * w.abs().unsqueeze(-2)).sum(-1) + (pair * w.abs().unsqueeze(-2)).sum(-1) + 1e-7
    _close(out, ref, bar, f"{what} value")
    if not grads:
        return
    # x, y and w gradients through autograd of both
    leaves = [t.clone().requires_grad_(True) for t in (xf, yf, wf)]
    val = ops.kernel_conv_wide(kid, *leaves, blur, center=c.float())
    got = torch.autograd.grad((val * go.float()).sum(), leaves)
    rl = [t.detach().clone().requires_grad_(True) for t in (x, y, w)]
    Kr = _kernel_ref(kind, rl[0], rl[1], rl[2], blur, keops)
    want = torch.autograd.grad(((Kr * rl[2].unsqueeze(-2)).sum(-1) * go).sum(), rl)
    # every pair's gradient term is off by at most |w_j| |go_i| times the relative error of its kernel value and of
    # its direction (laplacian / energy), and fully for the pairs counted as coincident
    if kind == 0:
        rel = math.log(2) * eS
        term = K.abs() * (rel * (x.unsqueeze(-2) - y.unsqueeze(-3)).abs().amax(-1) / blur**2)
    else:
        dg = _dist(x, y, keops)
        kp = K.abs() / blur if kind == 1 else torch.ones_like(K)
        term = kp * (2 * dd / dg.clamp_min(1e-30) + (dd / blur if kind == 1 else 0)).clamp_max(2.0) + 2 * near * kp
    gw = (go.abs().unsqueeze(-1) * w.abs().unsqueeze(-2) * term)
    slack = {"x": gw.sum(-1).unsqueeze(-1), "y": gw.sum(-2).unsqueeze(-1), "w": (go.abs().unsqueeze(-1) * pair).sum(-2)}
    for name, g, r in zip("xyw", got, want):
        _close(g, r, 5e-4 * r.abs().max() + slack[name] + 3e-6 * r.abs().max(), f"{what} grad {name}")


@pytest.mark.parametrize("d", [65, 72, 96, 127, 128, 200, 256, 512, 1000, 1024])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_conv_dimensions(d, kind):
    x, y, _, w, go = _clouds(300, 257, d, seed=d + kind)
    for blur in (2.0, 0.3):
        _check_conv(kind, x, y, w, go, blur, False, f"kind={kind} D={d} blur={blur}")


@pytest.mark.parametrize("n,m", [(1, 1), (127, 129), (129, 4000), (4000, 128)])
@pytest.mark.parametrize("kind,keops", [(0, False), (1, False), (1, True), (2, False), (2, True)])
def test_conv_tile_edges(n, m, kind, keops):
    x, y, _, w, go = _clouds(n, m, 200, seed=n * 7 + m)
    _check_conv(kind, x, y, w, go, 0.5, keops, f"kind={kind} keops={keops} N={n} M={m}")


@pytest.mark.parametrize("kind,keops", [(0, False), (1, False), (1, True), (2, False), (2, True)])
def test_conv_self_and_duplicates(kind, keops):
    """x == y (the K_xx diagonal is exact) and repeated points."""
    x, y, _, w, go = _clouds(257, 300, 130, seed=11, dup=200)
    _check_conv(kind, x, y, w, go, 0.5, keops, "duplicates")
    _check_conv(kind, x, x, w[:257], go, 0.5, keops, "x == y")


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_conv_many_columns(kind):
    x, y, _, w, go = _clouds(128, 65536, 128, seed=5)
    _check_conv(kind, x, y, w, go, 0.5, False, "M=65536")


@pytest.mark.parametrize("b", [1, 3, 17])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_conv_batches(b, kind):
    x, y, _, w, go = _clouds(129, 200, 96 if b == 17 else 256, seed=b + kind, b=b)
    _check_conv(kind, x, y, w, go, 0.5, False, f"B={b}")


# ------------------------------------------------------------------------------------------------
# SamplesLoss end to end against the fp64 oracle, batched and not
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss,p", [("sinkhorn", 2), ("sinkhorn", 1), ("gaussian", 2), ("laplacian", 2),
                                    ("energy", 2)])
@pytest.mark.parametrize("d", [96, 512])
@pytest.mark.parametrize("batch", [0, 3])
def test_samples_loss(loss, p, d, batch):
    from oracle import geomloss_oracle as O

    from geomloss_b200 import SamplesLoss

    n, m = 300, 200
    x, y, _, _, _ = _clouds(n, m, d, seed=d + batch, b=batch or None)
    g = torch.Generator().manual_seed(d)
    lead = (batch,) if batch else ()
    a = (torch.rand(*lead, n, generator=g, dtype=torch.float64) + 0.5).to(DEV)
    b = (torch.rand(*lead, m, generator=g, dtype=torch.float64) + 0.5).to(DEV)
    a, b = a / a.sum(-1, keepdim=True), b / b.sum(-1, keepdim=True)
    blur = 0.1 if loss == "sinkhorn" else 0.5
    leaves = [t.float().clone().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(loss, p=p, blur=blur)(*leaves)
    got = torch.autograd.grad(val.sum(), leaves)
    refs, rgrads = [], []
    for k in range(batch or 1):
        sel = (lambda t: t[k]) if batch else (lambda t: t)
        rl = [sel(t).detach().clone().requires_grad_(True) for t in (a, x, b, y)]
        r = O.samples_loss(*rl, loss=loss, p=p, blur=blur)
        refs.append(r.detach())
        rgrads.append(torch.autograd.grad(r, rl))
    ref = torch.stack(refs) if batch else refs[0]
    c = _center(x, y)
    spread = float(torch.cat([_n2(x, c).flatten(), _n2(y, c).flatten()]).max())
    # the loss: 1e-4 relative, plus the expansion error on the potentials (sinkhorn: the weights sum to one on each
    # side, four potentials) or the kernel values
    exp_bar = 4 * _cd(d) * 2.0**-24 * 2 * spread * (1.0 if loss == "sinkhorn" else 0.0)
    _close(val, ref, 1e-4 * ref.abs() + exp_bar + 1e-6, f"{loss} p={p} D={d} B={batch} value")
    for i, name in enumerate(["a", "x", "b", "y"]):
        r = torch.stack([gr[i] for gr in rgrads]) if batch else rgrads[0][i]
        # end to end (a whole fp32 Sinkhorn loop against fp64): the bar of the SamplesLoss fixture checks,
        # test_gpu_tc_softmin_l1.py; the operators' own row gradients hold 5e-4 above
        _close(got[i], r, 2e-3 * r.abs().max() + exp_bar / 0.1 * r.abs().max(), f"{loss} p={p} D={d} grad {name}")


def test_wide_route_leaves_low_dims_alone(monkeypatch):
    """D <= 64 still takes the existing operators."""
    from geomloss_b200 import SamplesLoss, ops

    def refuse(*a, **k):
        raise AssertionError("wide operator called at D <= 64")

    for name in ("softmin_wide_raw", "softmin_wide", "kernel_conv_wide_raw", "kernel_conv_wide"):
        monkeypatch.setattr(ops, name, refuse)
    x, y, _, _, _ = _clouds(300, 200, 64, seed=1)
    for loss in ("sinkhorn", "gaussian", "energy"):
        assert torch.isfinite(SamplesLoss(loss, blur=0.5)(x.float(), y.float()))


# ------------------------------------------------------------------------------------------------
# the reference's own runs (tests/golden/wide_*.npz, make_golden_wide.py)
# ------------------------------------------------------------------------------------------------
def _wide_goldens():
    from conftest import golden_names

    return golden_names("wide_")


@pytest.mark.parametrize("name", _wide_goldens())
def test_reference_fixtures(name):
    """SamplesLoss against the reference's fp64 run: the loss to 1e-4 relative, the gradients to the end-to-end bar of
    the other SamplesLoss fixture checks (2e-3 of the largest entry, test_gpu_tc_softmin_l1.py)."""
    from conftest import golden_kwargs, load_golden

    from geomloss_b200 import SamplesLoss

    g = load_golden(name)
    kw = golden_kwargs(g)
    kw.pop("backend")
    loss = kw.pop("loss")
    leaves = [torch.from_numpy(g[k]).float().to(DEV).requires_grad_(True) for k in "axby"]
    val = SamplesLoss(loss, **kw)(*leaves)
    got = torch.autograd.grad(val.sum(), leaves)
    ref = torch.from_numpy(g["value_f64"]).to(DEV)
    _close(val, ref, 1e-4 * ref.abs() + 1e-7, f"{name} value")
    for t, key in zip(got, ("grad_a", "grad_x", "grad_b", "grad_y")):
        r = torch.from_numpy(g[key + "_f64"]).double().to(DEV).view_as(t)
        _close(t, r, 2e-3 * r.abs().max(), f"{name} {key}")

"""Batched problems in the tensor-core dimensions (8 < D <= 64): tc_reduce_kernel / tc_bwd_kernel with BATCH, the
b200ot_*_batched entry points, ops.softmin_batched / kernel_conv_batched and SamplesLoss on (B, N, D) inputs.

Checked: B = 1 equals the one-problem operators bit for bit; no element reads another's columns or weights; every
operator agrees per element with the fp64 oracle (oracle/geomloss_oracle.py, on the device), with per-element weight
normalisation keeping light elements' P in fp16's normal range; whole losses agree with the oracle and with stored
outputs of the reference (tests/golden/batched_hd_*.npz, make_golden_batched_highdim.py); one SamplesLoss call takes the
same number of launches whatever B.  Bars are those of the other tensor-core tests (test_gpu_tc_streaming.py,
test_gpu_tc_norms.py)."""
import os

import numpy as np
import pytest
import torch

from test_gpu_tc_norms import _close, _expansion_slack, _kmat, _loss_bar
from test_gpu_tc_variants import _exponent_slack, env

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LN2 = np.log(2.0)
UNCLAMPED = 0x100
KINDS = {"gaussian": 0, "laplacian": 1, "energy": 2}


def _clouds(B, n, m, d, seed, dup=0):
    """fp64 batched clouds (fp32-representable) whose elements differ in scale and offset."""
    g = torch.Generator().manual_seed(seed)
    s = (0.5 + torch.arange(B, dtype=torch.float64) / B).view(B, 1, 1)
    x = torch.rand(B, n, d, generator=g, dtype=torch.float64) * s
    y = torch.rand(B, m, d, generator=g, dtype=torch.float64) * s * 0.9 + 0.15
    if dup:
        y[:, :dup] = x[:, torch.arange(dup) % n]  # copies of rows of x, element by element
        x[:, n // 2:n // 2 + min(dup, n // 4)] = x[:, :min(dup, n // 4)]  # and repeats within x
    h = torch.randn(B, m, generator=g, dtype=torch.float64) - np.log(m)
    w = torch.randn(B, m, generator=g, dtype=torch.float64) / m
    go = torch.randn(B, n, generator=g, dtype=torch.float64)
    return tuple(t.float().double().to(DEV) for t in (x, y, h, w, go))


def _f32(*ts):
    return tuple(t.float().contiguous() for t in ts)


def _center(x, y):
    from geomloss_b200 import ops

    d = x.shape[-1]
    return ops.default_center(x.reshape(-1, d).float(), y.reshape(-1, d).float())


def _softmin_bar(ref):
    return 1e-5 * max(1.0, ref.abs().max().item())


def _grad_bar(ref):
    return 5e-4 * ref.abs().max().item() + 1e-30


def _gauss_value_bar(x, y, w, blur):
    slack = LN2 * _exponent_slack(x.shape[-1], np.sqrt(np.log2(np.e)) / blur)
    return (2e-5 + slack) * (_kmat("gaussian", x, y, blur, False) @ w.abs()) + 1e-30


def _kernel_loss_bar(ref, a, x, b, y, loss, blur, keops):
    """1e-4 of the value and 2^-22 of the positive summands of 1/2 a K_xx a + 1/2 b K_yy b - a K_xy b, plus the
    kernels' own rounding: the norm expansion of the laplacian and energy (test_gpu_tc_norms._loss_bar), the exponent's
    slack of the gaussian relative to each summand."""
    if loss != "gaussian":
        return _loss_bar(ref, a, x, b, y, loss, blur, keops)
    k = lambda u, v: _kmat(loss, u, v, blur, keops).abs()  # noqa: E731
    pos = (0.5 * a @ k(x, x) @ a + 0.5 * b @ k(y, y) @ b + a @ k(x, y) @ b).item()
    slack = LN2 * _exponent_slack(x.shape[-1], np.sqrt(np.log2(np.e)) / blur)
    return 1e-4 * abs(ref) + (2.0**-22 + slack) * pos


def _check_softmin(eps, x, y, h, go, what, self_term=False):
    """Forward softmin with the h_b fold and the out_old / alpha / beta epilogue, and its row gradient, per element."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    B = x.shape[0]
    g = torch.Generator().manual_seed(x.shape[1] * 31 + y.shape[1])
    old = torch.randn(B, x.shape[1], generator=g, dtype=torch.float64).float().double().to(DEV)
    hb = 0.3 * h.flip(-1)
    xd, yd, hd, hbd, god, oldd = _f32(x, y, h, hb, go, old)
    if self_term:
        yd = xd
    center = _center(x, y)
    out, lse2 = ops.softmin_batched_raw(eps, xd, yd, hd, hbd, 0.5, p=2, center=center, out_old=oldd, alpha_old=0.5,
                                        beta=0.4, want_lse2=True)
    gx = ops.softmin_batched_grad_rows(eps, xd, yd, hd, hbd, 0.5, lse2, god, p=2, center=center)
    assert out.shape == (B, x.shape[1]) and gx.shape == x.shape
    for b in range(B):
        hh = h[b] + 0.5 * hb[b]
        cols = x[b] if self_term else y[b]
        ref = O.softmin_points(eps, x[b], cols, hh, p=2).to(DEV)
        _close(out[b], 0.5 * old[b] + 0.4 * ref, _softmin_bar(ref), f"{what} softmin element {b}")
        gref = O.softmin_grad_rows(eps, x[b], cols, hh, go[b], p=2)
        # x_i - sum_j p_ij y_j cancels when x_i dominates its own softmax (self terms): the bar of
        # test_gpu_tc_streaming, relative to max(1, largest entry)
        _close(gx[b], gref, 5e-5 * max(1.0, gref.abs().max().item()), f"{what} softmin gradient element {b}")


def _check_conv(name, keops, blur, x, y, w, go, what, self_term=False):
    """Kernel convolution, its row gradient and (gaussian) the one-pass value + unit gradient, per element."""
    from geomloss_b200 import ops

    kind = KINDS[name] | (UNCLAMPED if keops else 0)
    B = x.shape[0]
    xd, yd, wd, god = _f32(x, y, w, go)
    if self_term:
        yd = xd
    center = _center(x, y)
    out = ops.kernel_conv_batched_raw(kind, xd, yd, wd, blur, center=center)
    gx = ops.kernel_conv_batched_grad_rows(kind, xd, yd, wd, blur, god, center=center)
    if name == "gaussian":
        val, gunit = ops.kernel_conv_batched_value_and_grad_rows(kind, xd, yd, wd, blur, center=center)
    for b in range(B):
        cols = x[b] if self_term else y[b]
        xr = x[b].clone().requires_grad_(True)
        k = _kmat(name, xr, xr.detach() if self_term else cols, blur, keops)
        ref = k @ w[b]
        (gref,) = torch.autograd.grad(ref, xr, go[b], retain_graph=True)
        ref = ref.detach()
        if name == "gaussian":
            bar = _gauss_value_bar(x[b], cols, w[b], blur)
        else:
            pos = k.detach().abs() @ w[b].abs()
            bar = 1e-4 * pos + 2.0**-22 * pos + _expansion_slack(name, x[b], cols, w[b], blur, center.double())
        tag = f"{what} {name} keops={keops} element {b}"
        _close(out[b], ref, bar, tag)
        # gaussian weights of both signs cancel in the gradient: add 1e-5 of its natural scale
        # max_i |go_i| sum_j |w_j| k_ij |y_j - x_i| / blur^2, as test_gpu_tc_streaming does
        natural = 0.0
        if name == "gaussian":
            natural = (k.detach().abs() @ w[b].abs()).max().item() * np.sqrt(x.shape[-1]) / blur**2
        _close(gx[b], gref, _grad_bar(gref) + 1e-5 * natural * go[b].abs().max().item(), tag + " gradient")
        if name == "gaussian":
            (gu,) = torch.autograd.grad(k @ w[b], xr, torch.ones_like(go[b]))
            _close(val[b], ref, bar, tag + " one-pass value")
            _close(gunit[b], gu, _grad_bar(gu) + 1e-5 * natural, tag + " one-pass gradient")


# ------------------------------------------------------------------------------------------------
# 1. B = 1 is the one-problem operator, bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [0, 1, 3])
@pytest.mark.parametrize("d", [16, 64])
def test_single_element_is_bit_identical(d, splits):
    from geomloss_b200 import ops

    x, y, h, w, go = (t.float() for t in _clouds(1, 300, 128 * 9 - 37, d, seed=d + splits))
    hb = 0.3 * h.flip(-1)
    old = go * 0.7
    center = _center(x, y)
    with env(B200OT_FORCE_SPLITS=splits):
        o1, l1 = ops.softmin_raw(0.3, x[0], y[0], h[0], hb[0], 0.5, p=2, center=center, out_old=old[0], alpha_old=0.5,
                                 beta=0.4, want_lse2=True)
        ob, lb = ops.softmin_batched_raw(0.3, x, y, h, hb, 0.5, p=2, center=center, out_old=old, alpha_old=0.5,
                                         beta=0.4, want_lse2=True)
        pairs = [(o1, ob[0]), (l1, lb[0])]
        g1 = ops.softmin_grad_rows(0.3, x[0], y[0], h[0], hb[0], 0.5, l1, go[0], p=2, center=center)
        gb = ops.softmin_batched_grad_rows(0.3, x, y, h, hb, 0.5, lb, go, p=2, center=center)
        pairs.append((g1, gb[0]))
        for kind in (0, 1, 2, 1 | UNCLAMPED, 2 | UNCLAMPED):
            for yy, ww in ((y, w), (x, old)):  # (x, x): the self term, same buffer
                pairs.append((ops.kernel_conv_raw(kind, x[0], yy[0], ww[0], 0.7, center=center),
                              ops.kernel_conv_batched_raw(kind, x, yy, ww, 0.7, center=center)[0]))
                pairs.append((ops.kernel_conv_grad_rows(kind, x[0], yy[0], ww[0], 0.7, go[0], center=center),
                              ops.kernel_conv_batched_grad_rows(kind, x, yy, ww, 0.7, go, center=center)[0]))
        for yy, ww in ((y, w), (x, old)):
            v1, u1 = ops.kernel_conv_value_and_grad_rows(0, x[0], yy[0], ww[0], 0.7, center=center)
            vb, ub = ops.kernel_conv_batched_value_and_grad_rows(0, x, yy, ww, 0.7, center=center)
            pairs += [(v1, vb[0]), (u1, ub[0])]
    for k, (u, v) in enumerate(pairs):
        assert torch.equal(u, v), f"pair {k}: max difference {(u - v).abs().max().item():.3e}"


# ------------------------------------------------------------------------------------------------
# 2. no cross-talk between elements
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [16, 64])
def test_elements_do_not_interact(d):
    """Element 1's clouds, potentials and weights change (its weights by 1e6); element 0's softmin and gaussian
    outputs and gradients stay bit-identical (explicit centre)."""
    from geomloss_b200 import ops

    x, y, h, w, go = (t.float() for t in _clouds(3, 129, 300, d, seed=5 * d))
    center = _center(x, y)

    def run(y, h, w):
        out, lse2 = ops.softmin_batched_raw(0.3, x, y, h, p=2, center=center, want_lse2=True)
        gx = ops.softmin_batched_grad_rows(0.3, x, y, h, None, 0.0, lse2, go, p=2, center=center)
        conv = ops.kernel_conv_batched_raw(0, x, y, w, 0.7, center=center)
        gc = ops.kernel_conv_batched_grad_rows(0, x, y, w, 0.7, go, center=center)
        val, gu = ops.kernel_conv_batched_value_and_grad_rows(0, x, y, w, 0.7, center=center)
        return [t[0] for t in (out, lse2, gx, conv, gc, val, gu)]

    base = run(y, h, w)
    y2, h2, w2 = y.clone(), h.clone(), w.clone()
    y2[1] = torch.rand_like(y2[1]) * 3 - 1
    h2[1] = h2[1] + 50.0
    w2[1] = w2[1] * 1e6
    for k, (u, v) in enumerate(zip(base, run(y2, h2, w2))):
        assert torch.equal(u, v), f"output {k}: element 0 moved by {(u - v).abs().max().item():.3e}"


# ------------------------------------------------------------------------------------------------
# 3. every operator against fp64, element by element
# ------------------------------------------------------------------------------------------------
SHAPES = [(2, 129, 300), (5, 200, 129), (17, 129, 77)]


@pytest.mark.parametrize("d", [9, 16, 24, 33, 64])
def test_operators_vs_fp64(d):
    for B, n, m in SHAPES:
        x, y, h, w, go = _clouds(B, n, m, d, seed=100 * d + B)
        what = f"D={d} B={B} N={n} M={m}"
        _check_softmin(0.3, x, y, h, go, what)
        for name, blur in (("gaussian", 0.7), ("laplacian", 0.5), ("energy", 1.0)):
            for keops in ((False,) if name == "gaussian" else (False, True)):
                _check_conv(name, keops, blur, x, y, w, go, what)


@pytest.mark.parametrize("d", [16, 64])
def test_self_terms_and_duplicated_points(d):
    """x is y (the K_xx / softmin_xx terms: the exact diagonal, the coincidence rule of the laplacian and energy), and
    y holding copies of rows of x while x repeats rows, within each element."""
    x, y, h, w, go = _clouds(3, 300, 300, d, seed=7 * d, dup=60)
    what = f"D={d}"
    _check_softmin(0.3, x, y, h, go, what + " self", self_term=True)
    _check_softmin(0.3, x, y, h, go, what + " duplicates")
    for name, blur in (("gaussian", 0.7), ("laplacian", 0.5), ("energy", 1.0)):
        for keops in ((False,) if name == "gaussian" else (False, True)):
            _check_conv(name, keops, blur, x, x, go, go, what + " self", self_term=True)
            _check_conv(name, keops, blur, x, y, w, go, what + " duplicates")


@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("d", [16, 64])
def test_forced_splits_over_many_column_tiles(d, splits):
    """M = 128 * 9 - 37 columns per element (9 tiles): one CTA streams all of an element's tiles (1 split) or three
    ragged splits; the splits never leave the element."""
    x, y, h, w, go = _clouds(3, 129, 128 * 9 - 37, d, seed=11 * d + splits)
    with env(B200OT_FORCE_SPLITS=splits):
        what = f"D={d} splits={splits}"
        _check_softmin(0.3, x, y, h, go, what)
        _check_conv("gaussian", False, 0.7, x, y, w, go, what)
        _check_conv("energy", False, 1.0, x, y, w, go, what)


# ------------------------------------------------------------------------------------------------
# 4. per-element weight normalisation: P stays in fp16's normal range
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,blur", [("gaussian", 0.7), ("laplacian", 0.5), ("energy", 1.0)])
def test_light_element_gradient(name, blur):
    """Element 1's weights are 2^-20 times element 0's: normalised by one maximum for the batch, its P would fall on
    fp16's subnormal grid (a bias with repeated points).  Each element must meet the gradient bar on its own."""
    x, y, _, w, go = _clouds(2, 256, 4096, 64, seed=3)
    w = w.abs()
    w[1] = w[1] * 2.0**-20
    rep = torch.arange(4096, device=DEV) % 128  # 128 atoms x 32 copies per element
    y, w = y[:, rep], w[:, rep]
    _check_conv(name, False, blur, x, y, w, go, "light element")


# ------------------------------------------------------------------------------------------------
# 5. whole losses
# ------------------------------------------------------------------------------------------------
SINKHORN = {
    "balanced": dict(blur=0.1),
    "reach": dict(blur=0.3, reach=0.5),
    "nodebias": dict(blur=0.1, debias=False),
}


@pytest.mark.parametrize("backend", ["tensorized", "online"])
@pytest.mark.parametrize("case", sorted(SINKHORN))
@pytest.mark.parametrize("d", [16, 64])
def test_sinkhorn_losses_vs_oracle(d, case, backend):
    """Values, gradients of a, x, b, y and (separately) the potentials, against per-element fp64 oracle runs that
    share the batch's diameter (one eps-schedule for the whole batch, as in the reference)."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    B, n, m = 3, 200, 150
    x, y, _, _, _ = _clouds(B, n, m, d, seed=d + len(case))
    g = torch.Generator().manual_seed(d)
    a = torch.rand(B, n, generator=g, dtype=torch.float64) + 0.1
    b = torch.rand(B, m, generator=g, dtype=torch.float64) + 0.1
    a, b = ((a / a.sum(1, keepdim=True)).float().double().to(DEV), (b / b.sum(1, keepdim=True)).float().double().to(DEV))
    kw = dict(SINKHORN[case])
    diam = O.max_diameter(x.reshape(-1, d), y.reshape(-1, d))
    fl = [t.float().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss("sinkhorn", backend=backend, **kw)(*fl)
    grads = torch.autograd.grad(val.sum(), fl)
    F, G = SamplesLoss("sinkhorn", backend=backend, potentials=True, **kw)(*(t.float() for t in (a, x, b, y)))
    assert val.shape == (B,) and F.shape == (B, n) and G.shape == (B, m)
    for k in range(B):
        leaves = [t[k:k + 1].clone().requires_grad_(True) for t in (a, x, b, y)]
        ref = O.samples_loss(*leaves, loss="sinkhorn", diameter=diam, **kw)
        rgrads = torch.autograd.grad(ref.sum(), leaves)
        what = f"D={d} {case} {backend} element {k}"
        Fr, Gr = O.samples_loss(*(t[k:k + 1] for t in (a, x, b, y)), loss="sinkhorn", diameter=diam, potentials=True,
                                **kw)
        # potentials: 1e-5 of their scale plus the exponent's rounding slack at the last temperature, eps ln2 times
        # _exponent_slack in log2 units; the value: 1e-4 of it and that bar through the four unit-mass dual terms
        eps = kw["blur"] ** 2
        pbar = 1e-5 * max(1.0, Fr.abs().max().item(), Gr.abs().max().item()) + \
            eps * LN2 * _exponent_slack(d, np.sqrt(np.log2(np.e) / eps))
        bar = 1e-4 * abs(ref.item()) + 4 * pbar
        assert abs(val[k].item() - ref.item()) <= bar, (what, val[k].item(), ref.item(), bar)
        for got, r, nm in zip(grads, rgrads, "axby"):
            _close(got[k], r[0], _grad_bar(r), f"{what} grad {nm}")
        _close(F[k], Fr[0], pbar, f"{what} F")
        _close(G[k], Gr[0], pbar, f"{what} G")


@pytest.mark.parametrize("backend", ["tensorized", "online"])
@pytest.mark.parametrize("loss,blur", [("gaussian", 2.0), ("laplacian", 0.5), ("energy", 0.05)])
@pytest.mark.parametrize("d", [16, 64])
def test_kernel_losses_vs_oracle(d, loss, blur, backend):
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    B, n, m = 4, 300, 129
    x, y, _, _, _ = _clouds(B, n, m, d, seed=3 * d + len(loss))
    g = torch.Generator().manual_seed(d + 1)
    a = torch.rand(B, n, generator=g, dtype=torch.float64) + 0.1
    b = torch.rand(B, m, generator=g, dtype=torch.float64) + 0.1
    a, b = ((a / a.sum(1, keepdim=True)).float().double().to(DEV), (b / b.sum(1, keepdim=True)).float().double().to(DEV))
    keops = backend == "online"
    fl = [t.float().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(loss, blur=blur, backend=backend)(*fl)
    grads = torch.autograd.grad(val.sum(), fl)
    F, G = SamplesLoss(loss, blur=blur, backend=backend, potentials=True)(*(t.float() for t in (a, x, b, y)))
    for k in range(B):
        leaves = [t[k:k + 1].clone().requires_grad_(True) for t in (a, x, b, y)]
        ref = (O.mmd_online if keops else O.mmd_dense)(*leaves, loss, blur=blur)
        rgrads = torch.autograd.grad(ref.sum(), leaves)
        what = f"D={d} {loss} {backend} element {k}"
        bar = _kernel_loss_bar(ref.item(), *(t[k] for t in (a, x, b, y)), loss, blur, keops)
        assert abs(val[k].item() - ref.item()) <= bar, (what, val[k].item(), ref.item(), bar)
        for got, r, nm in zip(grads, rgrads, "axby"):
            _close(got[k], r[0], _grad_bar(r), f"{what} grad {nm}")
        Fr, Gr = (O.mmd_online if keops else O.mmd_dense)(*(t[k:k + 1] for t in (a, x, b, y)), loss, blur=blur,
                                                          potentials=True)
        _close(F[k], Fr[0], 2e-4 * Fr.abs().max().item(), f"{what} F")
        _close(G[k], Gr[0], 2e-4 * Gr.abs().max().item(), f"{what} G")


GOLDEN = ["batched_hd_sinkhorn_d16", "batched_hd_sinkhorn_d64_reach", "batched_hd_gaussian_d64",
          "batched_hd_laplacian_d16", "batched_hd_energy_d33"]


@pytest.mark.parametrize("case", GOLDEN)
def test_losses_vs_reference_goldens(case):
    from geomloss_b200 import SamplesLoss

    z = np.load(os.path.join(os.path.dirname(__file__), "golden", case + ".npz"))
    kw = {k[3:]: z[k].item() for k in z.files if k.startswith("kw_")}
    loss = kw.pop("loss")
    a, x, b, y = (torch.tensor(z[k], device=DEV) for k in ("a", "x", "b", "y"))
    leaves = [t.clone().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(loss, backend="tensorized", **kw)(*leaves)
    grads = torch.autograd.grad(val.sum(), leaves)
    ref = torch.tensor(z["value_f64"], device=DEV)
    for k in range(ref.shape[0]):
        if loss == "sinkhorn":
            # 1e-4 of the value, and the potentials' 1e-5 bar at the clouds' cost scale (|x - y|^2 / 2 <= 5 here)
            # through the four unit-mass dual terms
            bar = 1e-4 * abs(ref[k].item()) + 2e-4
        else:
            bar = _kernel_loss_bar(ref[k].item(), *(t[k].double() for t in (a, x, b, y)), loss, kw["blur"], False)
        assert abs(val[k].item() - ref[k].item()) <= bar, (case, k, val[k].item(), ref[k].item(), bar)
    for got, key in zip(grads, ("grad_a_f64", "grad_x_f64", "grad_b_f64", "grad_y_f64")):
        r = torch.tensor(z[key], device=DEV).double()
        _close(got, r, _grad_bar(r), f"{case} {key}")


# ------------------------------------------------------------------------------------------------
# 6. launches do not grow with B
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss", ["sinkhorn", "gaussian", "energy"])
def test_launch_count_does_not_grow_with_batch(loss):
    from geomloss_b200 import SamplesLoss, ops

    def count(B, batched=True):
        x, y, _, _, _ = _clouds(B, 300, 200, 24, seed=B)
        xg = x.float().requires_grad_(True)
        fn = SamplesLoss(loss, blur=0.5, diameter=2.0)
        before = ops.launches()
        if batched:
            val = fn(xg, y.float())
        else:  # the same problems one element at a time
            val = torch.stack([fn(xg[k], y[k].float()) for k in range(B)])
        torch.autograd.grad(val.sum(), xg)
        return ops.launches() - before

    assert count(2) == count(16) > 0
    assert count(16, batched=False) > count(16)
    assert count(16, batched=False) == 8 * count(2, batched=False)

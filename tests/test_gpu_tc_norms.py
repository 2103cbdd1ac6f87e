"""The laplacian and energy kernel norms on the tensor cores (8 < D <= 64; csrc/tcconv.cuh tc_reduce_kernel<4/5>,
csrc/tcbwd.cuh tc_bwd_kernel<4/5>), in both norm conventions: the reference's tensorized sqrt(max(d^2, 1e-8)) and the
pykeops one (no clamp, zero gradient at 0), selected by KERNEL_UNCLAMPED.

Every result is checked against float64 on the device: the oracle's kernels (oracle/geomloss_oracle.py), the stored
outputs of the reference (tests/golden/hd_{laplacian,energy}_*.npz, make_golden_highdim_norms.py) and the oracle's
keops-convention path.  Bars are those of the tensor-core tests: values 1e-4 relative plus 2^-22 of the positive
summands, gradients 2e-4 of the largest entry.  The values also get the distance error of the norm expansion
(_expansion_slack): an error on d^2 of up to 2^-18 (|x_i - c|^2 + |y_j - c|^2) in the kernel's units, the worst case
derived in tcconv.cuh, propagated through d -> k(d) pair by pair."""
import numpy as np
import pytest
import torch

from test_gpu_tc_variants import env

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
UNCLAMPED = 0x100
KINDS = {"laplacian": 1, "energy": 2}


def _clouds(n, m, d, seed, dup=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    y = torch.rand(m, d, generator=g, dtype=torch.float64) * 0.9 + 0.15
    if dup:
        y[:dup] = x[torch.arange(dup) % n]  # copies of rows of x
    w = torch.randn(m, generator=g, dtype=torch.float64) / m  # weights of both signs
    go = torch.randn(n, generator=g, dtype=torch.float64)
    x, y, w, go = (t.float().double().to(DEV) for t in (x, y, w, go))  # fp32-representable
    return x, y, w, go


def _kmat(name, x, y, blur, keops):
    from oracle import geomloss_oracle as O

    return (O.keops_kernel_matrix if keops else O.kernel_matrix)(name, x, y, blur)


def _expansion_slack(name, x, y, w, blur, center):
    """sum_j |w_j| |dk_ij| for an error 2^-18 (|x_i - c|^2 + |y_j - c|^2) on d_ij^2 (in units of blur for the
    laplacian): dd = min(dq / (2 d), sqrt(dq)), dk = k dd (laplacian) or dd (energy)."""
    s = 1.0 / blur if name == "laplacian" else 1.0
    xc, yc = (x - center) * s, (y - center) * s
    dq = 2.0**-18 * ((xc * xc).sum(1)[:, None] + (yc * yc).sum(1)[None, :])
    d = torch.cdist(xc, yc)
    dd = torch.minimum(dq / (2 * d.clamp_min(1e-30)), dq.sqrt())
    dk = torch.exp(-d) * dd if name == "laplacian" else dd
    return dk @ w.abs()


def _value_bar(name, x, y, w, blur, center, keops):
    pos = _kmat(name, x, y, blur, keops).abs() @ w.abs()
    return 1e-4 * pos + 2.0**-22 * pos + _expansion_slack(name, x, y, w, blur, center)


def _close(got, ref, bar, what):
    got, ref = got.detach().double(), ref.detach().double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - ref).abs()
    bar = torch.as_tensor(bar, dtype=torch.float64, device=err.device).expand_as(err)
    bad = err > bar
    i = int(torch.argmax(err - bar))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {err.numel()} off, worst {err.flatten()[i]:.3e} " \
                          f"(bar {bar.flatten()[i]:.3e})"


def _grad_close(got, ref, what):
    _close(got, ref, 2e-4 * ref.abs().max().item() + 1e-30, what)


# ------------------------------------------------------------------------------------------------
# 1. operator values, every padded-dimension boundary, both conventions, many column tiles per CTA
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("name", ["laplacian", "energy"])
@pytest.mark.parametrize("d", [9, 16, 17, 24, 33, 48, 63, 64])
def test_operator_values(d, name, keops):
    from geomloss_b200 import ops

    blur = 0.7
    kind = KINDS[name] | (UNCLAMPED if keops else 0)
    for n, m in ((1, 1), (127, 129), (129, 128 * 13 - 37), (300, 129), (300, 1)):
        x, y, w, _ = _clouds(n, m, d, seed=1000 * d + n + m)
        center = ops.default_center(x.float(), y.float())
        ref = _kmat(name, x, y, blur, keops) @ w
        bar = _value_bar(name, x, y, w, blur, center.double(), keops)
        for splits in (1, 3):
            with env(B200OT_FORCE_SPLITS=splits):
                out = ops.kernel_conv_raw(kind, x.float(), y.float(), w.float(), blur, center=center)
            _close(out, ref, bar, f"{name} keops={keops} D={d} N={n} M={m} splits={splits}")


# ------------------------------------------------------------------------------------------------
# 2. row, column and weight gradients against dense fp64 autograd
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("name,blur", [("laplacian", 0.3), ("laplacian", 2.0), ("energy", 1.0)])
@pytest.mark.parametrize("d", [16, 33, 64])
def test_gradients_vs_autograd(d, name, blur, keops):
    from geomloss_b200 import ops

    x, y, w, go = _clouds(300, 1000, d, seed=7 * d)
    xr, yr, wr = (t.clone().requires_grad_(True) for t in (x, y, w))
    ref = _kmat(name, xr, yr, blur, keops) @ wr
    gx_ref, gy_ref, gw_ref = torch.autograd.grad(ref, (xr, yr, wr), go)
    kind = KINDS[name] | (UNCLAMPED if keops else 0)
    xf, yf, wf = (t.float().requires_grad_(True) for t in (x, y, w))
    out = ops.kernel_conv(kind, xf, yf, wf, blur)
    gx, gy, gw = torch.autograd.grad(out, (xf, yf, wf), go.float())
    what = f"{name} blur={blur} keops={keops} D={d}"
    _grad_close(gx, gx_ref, what + " grad x")
    _grad_close(gy, gy_ref, what + " grad y")
    _grad_close(gw, gw_ref, what + " grad w")


# ------------------------------------------------------------------------------------------------
# 3. full losses: the reference's stored tensorized outputs, the oracle's keops path, potentials
# ------------------------------------------------------------------------------------------------
GOLDEN = ["hd_laplacian_d16_blur05", "hd_laplacian_d64_blur2", "hd_laplacian_d33_blur02", "hd_energy_d16",
          "hd_energy_d33", "hd_energy_d64", "hd_energy_d64_dup", "hd_laplacian_d64_blur2_dup"]


def _load(name):
    import os

    z = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
    kw = {k[3:]: z[k].item() for k in z.files if k.startswith("kw_")}
    return z, kw


def _loss_bar(ref, a, x, b, y, loss, blur, keops):
    """1e-4 of the value, 2^-22 of the positive summands of 1/2 a K_xx a + 1/2 b K_yy b - a K_xy b, and the
    expansion error of every pair (_expansion_slack) weighted like its term."""
    k = lambda u, v: _kmat(loss, u, v, blur, keops).abs()  # noqa: E731
    pos = (0.5 * a @ k(x, x) @ a + 0.5 * b @ k(y, y) @ b + a @ k(x, y) @ b).item()
    c = 0.5 * (torch.minimum(x.min(0).values, y.min(0).values) + torch.maximum(x.max(0).values, y.max(0).values))
    sl = lambda u, v, w: _expansion_slack(loss, u, v, w, blur, c)  # noqa: E731
    slack = (0.5 * a @ sl(x, x, a) + 0.5 * b @ sl(y, y, b) + a @ sl(x, y, b)).item()
    return 1e-4 * abs(ref) + 2.0**-22 * pos + slack


@pytest.mark.parametrize("case", GOLDEN)
def test_samples_loss_vs_reference_goldens(case):
    from geomloss_b200 import SamplesLoss

    z, kw = _load(case)
    loss, blur = kw["loss"], kw.get("blur", 0.05)
    a, x, b, y = (torch.tensor(z[k], device=DEV) for k in ("a", "x", "b", "y"))
    leaves = [t.clone().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(loss, blur=blur, backend="tensorized")(*leaves)
    ga, gx, gb, gy = torch.autograd.grad(val, leaves)
    ref = float(z["value_f64"])
    bar = _loss_bar(ref, a.double(), x.double(), b.double(), y.double(), loss, blur, False)
    assert abs(val.item() - ref) <= bar, (case, val.item(), ref, bar)
    for got, key in ((ga, "grad_a_f64"), (gb, "grad_b_f64"), (gx, "grad_x_f64"), (gy, "grad_y_f64")):
        _grad_close(got, torch.tensor(z[key], device=DEV).double(), f"{case} {key}")


@pytest.mark.parametrize("loss,blur", [("laplacian", 0.5), ("energy", 0.05)])
@pytest.mark.parametrize("d", [16, 64])
def test_samples_loss_online_and_potentials(d, loss, blur):
    """backend="online" against the oracle's keops path (no clamp); potentials=True against the tensorized oracle."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    x, y, _, _ = _clouds(700, 650, d, seed=d)
    g = torch.Generator().manual_seed(d + 1)
    a = (torch.rand(700, generator=g, dtype=torch.float64) + 0.1).to(DEV)
    b = (torch.rand(650, generator=g, dtype=torch.float64) + 0.1).to(DEV)
    a, b = (a / a.sum()).float().double(), (b / b.sum()).float().double()
    leaves = [t.clone().requires_grad_(True) for t in (a, x, b, y)]
    ref = O.mmd_online(*leaves, loss, blur=blur)
    rgrads = torch.autograd.grad(ref, leaves)
    fl = [t.float().requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(loss, blur=blur, backend="online")(*fl)
    grads = torch.autograd.grad(val, fl)
    bar = _loss_bar(ref.item(), a, x, b, y, loss, blur, True)
    assert abs(val.item() - ref.item()) <= bar, (loss, d, val.item(), ref.item(), bar)
    for got, r, nm in zip(grads, rgrads, "axby"):
        _grad_close(got, r, f"online {loss} D={d} grad {nm}")
    F, G = SamplesLoss(loss, blur=blur, backend="tensorized", potentials=True)(*(t.float() for t in (a, x, b, y)))
    Fr, Gr = O.samples_loss(a, x, b, y, loss=loss, blur=blur, potentials=True)
    for got, r, nm in ((F, Fr, "F"), (G, Gr, "G")):
        r = r.reshape(-1)
        _close(got.reshape(-1), r, 2e-4 * r.abs().max().item(), f"potentials {loss} D={d} {nm}")


def test_batched_inputs_take_the_per_batch_loop():
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(3)
    x = torch.rand(2, 300, 24, generator=g, dtype=torch.float64).to(DEV)
    y = torch.rand(2, 280, 24, generator=g, dtype=torch.float64).to(DEV)
    for loss in ("laplacian", "energy"):
        xr = x.clone().requires_grad_(True)
        ref = O.samples_loss(xr, y, loss=loss, blur=0.5)
        (gref,) = torch.autograd.grad(ref.sum(), xr)
        xf = x.float().requires_grad_(True)
        val = SamplesLoss(loss, blur=0.5)(xf, y.float())
        (gx,) = torch.autograd.grad(val.sum(), xf)
        _close(val, ref, 2e-4 * ref.abs().max().item(), f"batched {loss}")
        _grad_close(gx, gref, f"batched {loss} grad x")


# ------------------------------------------------------------------------------------------------
# 4. coincident points, large M
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keops", [False, True])
@pytest.mark.parametrize("name", ["laplacian", "energy"])
def test_self_term_and_duplicated_points(name, keops):
    """S(x, x): the diagonal gets the value of a coincident pair (sqrt(1e-8) / exp(-1e-4), or 0 / 1 without the
    clamp) and no gradient; y holding copies of rows of x (and x repeating rows) must agree the same way."""
    from geomloss_b200 import ops

    blur = 0.5
    kind = KINDS[name] | (UNCLAMPED if keops else 0)
    x, y, w, go = _clouds(300, 700, 40, seed=11, dup=200)
    x[150:170] = x[:20]
    for cols, wc in ((x, go), (y, w)):
        xf, yf, wf = x.float(), cols.float(), wc.float()
        if cols is x:
            yf = xf  # the same buffer: the K_xx term
        center = ops.default_center(xf, yf)
        out = ops.kernel_conv_raw(kind, xf, yf, wf, blur, center=center)
        ref = _kmat(name, x, cols, blur, keops) @ wc
        _close(out, ref, _value_bar(name, x, cols, wc, blur, center.double(), keops),
               f"{name} keops={keops} self={cols is x}")
        gx = ops.kernel_conv_grad_rows(kind, xf, yf, wf, blur, go.float(), center=center)
        xr = x.clone().requires_grad_(True)
        cr = xr.detach() if cols is x else cols
        (gref,) = torch.autograd.grad(_kmat(name, xr, cr, blur, keops) @ wc, xr, go)
        _grad_close(gx, gref, f"{name} keops={keops} self={cols is x} grad")


def test_energy_row_gradients_at_large_m():
    """M = 65536: P = w_j / d_ij of the energy row gradient stays inside fp16's normal range (tcbwd.cuh)."""
    from geomloss_b200 import ops

    x, y, _, go = _clouds(300, 65536, 64, seed=5)
    w = torch.full((65536,), 1.0 / 65536, dtype=torch.float64, device=DEV)
    for kind in (2, 2 | UNCLAMPED):
        gx = ops.kernel_conv_grad_rows(kind, x.float(), y.float(), w.float(), 1.0, go.float())
        xr = x.clone().requires_grad_(True)
        (gref,) = torch.autograd.grad(_kmat("energy", xr, y, 1.0, kind & UNCLAMPED) @ w, xr, go)
        _grad_close(gx, gref, f"energy M=65536 kind={kind:#x}")


# ------------------------------------------------------------------------------------------------
# 5. low dimensions stay on the CUDA cores whatever the routing variables say
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["laplacian", "energy"])
def test_low_dimension_is_unchanged(name):
    from geomloss_b200 import ops

    x, y, w, go = (t.float() for t in _clouds(3000, 2900, 6, seed=6))
    kind = KINDS[name]

    def run():
        out = ops.kernel_conv_raw(kind, x, y, w, 0.3)
        gx = ops.kernel_conv_grad_rows(kind, x, y, w, 0.3, go)
        return out, gx

    base = run()
    with env(B200OT_TC_MIN_D=1, B200OT_TC_MIN_PAIRS=0):
        forced = run()
    for u, v in zip(base, forced):
        assert torch.equal(u, v)

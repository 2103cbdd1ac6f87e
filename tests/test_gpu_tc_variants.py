"""GPU parity of the tensor-core kernels' routing knobs (csrc/b200ot_tc.cu: tc_routed), of the row-gradient
kernel at every padded dimension (csrc/tcbwd.cuh) and of the one-pass value + row-gradient entry
(b200ot_kernel_conv_fwd_bwd_x).  Every route — not only the shipped default — is held to the same bars against the
fp64 oracle as the default kernels in test_gpu_parity.py, so that a default can be flipped from a measurement
(tools/ab_tc_route.py) without changing what is tested."""
import os
from contextlib import contextmanager

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update({k: str(v) for k, v in kv.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


ROUTES = {"cuda-core": dict(B200OT_TC_MIN_D="9", B200OT_TC_MIN_PAIRS="0"),
          "tensor-core": dict(B200OT_TC_MIN_D="1", B200OT_TC_MIN_PAIRS="0")}


def _exponent_slack(d, scale):
    """Absolute error allowed on a log2-domain exponent X.Y - |X|^2/2 - |Y|^2/2 of unit-cube clouds centred on the
    bounding box and scaled by `scale`: a few roundings at the magnitude of |X|^2 <= d (scale/2)^2 — fp32 for the
    CUDA-core expansion (2^-24 each), two-term fp16 operands for the tensor-core one (2^-22)."""
    return 4 * 2.0**-22 * d * (0.5 * scale) ** 2


@pytest.mark.parametrize("route", sorted(ROUTES))
@pytest.mark.parametrize("d", [2, 5, 8])
def test_both_routes_below_nine_dimensions(route, d):
    """D <= 8: the CUDA-core kernels and the (zero-padded, dk = 16) tensor-core kernels serve the same operators; both
    meet the fp64 oracle to the bars of test_softmin_tensor_core_path / test_kernel_conv_vs_oracle, plus the rounding
    of the norm expansion at the magnitude of the scaled coordinates (_exponent_slack, computed, not fitted)."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n, m = 1300, 2100
    g = torch.Generator().manual_seed(100 + d)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    h = torch.randn(m, generator=g) - np.log(m)
    w = torch.rand(m, generator=g) / m
    go = torch.randn(n, generator=g)
    xd, yd, hd, wd, god = (t.to(DEV) for t in (x, y, h, w, go))
    center = ops.default_center(xd, yd)
    ln2, diam = np.log(2.0), float(np.sqrt(d))
    with env(**ROUTES[route]):
        for eps in (0.5, 0.05, 0.01):
            slack = ln2 * _exponent_slack(d, np.sqrt(np.log2(np.e) / eps))  # relative error of a softmax weight
            ref = O.softmin_points(eps, x.double(), y.double(), h.double(), p=2).numpy()
            out, lse2 = ops.softmin_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
            np.testing.assert_allclose(out.cpu().numpy(), ref, atol=5e-6 * max(1.0, np.abs(ref).max()) + eps * slack,
                                       err_msg=f"softmin eps={eps}")
            gref = O.softmin_grad_rows(eps, x.double(), y.double(), h.double(), go.double(), p=2).numpy()
            gx = ops.softmin_grad_rows(eps, xd, yd, hd, None, 0.0, lse2, god, p=2, center=center)
            np.testing.assert_allclose(gx.cpu().numpy(), gref,
                                       atol=5e-5 * max(1.0, np.abs(gref).max()) + slack * diam * go.abs().max().item(),
                                       err_msg=f"softmin gradient eps={eps}")
        for blur in (0.3 * np.sqrt(d / 3.0), 0.15 * np.sqrt(d / 3.0)):
            slack = ln2 * _exponent_slack(d, np.sqrt(np.log2(np.e)) / blur)  # relative error of a kernel value
            ref = O.kernel_conv_points("gaussian", x.double(), y.double(), w.double(), blur).numpy()
            out = ops.kernel_conv_raw("gaussian", xd, yd, wd, blur, center=center)
            np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=2e-5 + slack, atol=1e-30, err_msg=f"conv blur={blur}")
            xr = x.double().requires_grad_(True)
            km = O.kernel_matrix("gaussian", xr, y.double(), blur)
            (gref,) = torch.autograd.grad(km @ w.double(), xr, go.double())
            # the gradient's natural scale: sum_j w_j k_ij |y_j - x_i| / blur^2 (its terms cancel in the sum itself)
            gscale = ((km.detach() @ w.double()) * go.double().abs()).max().item() * diam / blur**2
            gx = ops.kernel_conv_grad_rows("gaussian", xd, yd, wd, blur, god, center=center)
            np.testing.assert_allclose(gx.cpu().numpy(), gref.numpy(),
                                       atol=5e-5 * gref.abs().max().item() + (2e-5 + slack) * gscale,
                                       err_msg=f"conv gradient blur={blur}")


def test_whole_losses_on_the_tensor_core_route_d5():
    """SamplesLoss through the tiled kernels with every p = 2 softmin / gaussian matvec of a D = 5 problem forced onto
    the tensor-core path: value and gradients against the fp64 oracle (bars of test_softmin_tensor_core_path)."""
    from geomloss_b200 import SamplesLoss, sinkhorn_small
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(5)
    x, y = torch.rand(900, 5, generator=g), torch.rand(1100, 5, generator=g)
    keep = sinkhorn_small.SMALL_MAX
    sinkhorn_small.SMALL_MAX = 0
    try:
        with env(**ROUTES["tensor-core"]):
            for kw in (dict(loss="sinkhorn", p=2, blur=0.1, scaling=0.6), dict(loss="gaussian", blur=0.4)):
                xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
                val = SamplesLoss(**kw)(xg, yg)
                gx, gy = torch.autograd.grad(val, [xg, yg])
                xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
                ref = O.samples_loss(xr, yr, **kw)
                rx, ry = torch.autograd.grad(ref, [xr, yr])
                assert abs(val.item() - ref.item()) <= 1e-4 * abs(ref.item()), (kw, val.item(), ref.item())
                assert (gx.cpu().double() - rx).abs().max() <= 2e-4 * rx.abs().max(), kw
                assert (gy.cpu().double() - ry).abs().max() <= 2e-4 * ry.abs().max(), kw
    finally:
        sinkhorn_small.SMALL_MAX = keep


@pytest.mark.parametrize("shape", [(300, 500, 16), (131, 67, 40), (1500, 2300, 64), (257, 300, 24)])
def test_row_gradient_kernel_at_padded_dimensions(shape):
    """tc_bwd_kernel<MODE, DK> at D = 16, 40, 64, 24 (padded dimensions 16, 48, 64, 32): gaussian and softmin row
    gradients against fp64, at the bar of the default kernels."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(n + 7 * d)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    h = torch.randn(m, generator=g) - np.log(m)
    w = torch.rand(m, generator=g) / m
    go = torch.randn(n, generator=g)
    xd, yd, hd, wd, god = (t.to(DEV) for t in (x, y, h, w, go))
    center = ops.default_center(xd, yd)
    for eps in (2.0, 0.3):
        _, lse2 = ops.softmin_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
        ref = O.softmin_grad_rows(eps, x.double(), y.double(), h.double(), go.double(), p=2).numpy()
        gx = ops.softmin_grad_rows(eps, xd, yd, hd, None, 0.0, lse2, god, p=2, center=center)
        np.testing.assert_allclose(gx.cpu().numpy(), ref, atol=5e-5 * max(1.0, np.abs(ref).max()),
                                   err_msg=f"softmin eps={eps}")
    for blur in (2.0, 0.7):
        xr = x.double().requires_grad_(True)
        km = O.kernel_matrix("gaussian", xr, y.double(), blur)
        (ref,) = torch.autograd.grad(km @ w.double(), xr, go.double())
        # natural scale of the gradient (its terms cancel in the sum): sum_j w_j k_ij |y_j - x_i| / blur^2
        gscale = ((km.detach() @ w.double()) * go.double().abs()).max().item() * np.sqrt(d) / blur**2
        gx = ops.kernel_conv_grad_rows("gaussian", xd, yd, wd, blur, god, center=center)
        np.testing.assert_allclose(gx.cpu().numpy(), ref.numpy(),
                                   atol=5e-5 * ref.abs().max().item() + 1e-5 * gscale, err_msg=f"gaussian blur={blur}")


@pytest.mark.parametrize("shape", [(700, 900, 3), (1300, 800, 8), (300, 500, 16), (1000, 2100, 64)])
def test_value_and_unit_gradient_in_one_pass(shape):
    """b200ot_kernel_conv_fwd_bwd_x: out = K(x, y) w and the unit row gradient from one reduction, CUDA-core and
    tensor-core dimensions, cross and self terms (the exact zero exponent of the diagonal included)."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(3 * n + d)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    w, a = torch.rand(m, generator=g) / m, torch.rand(n, generator=g) / n
    xd, yd, wd, ad = (t.to(DEV) for t in (x, y, w, a))
    blurs = (2.0, 0.7) if d > 8 else (0.5, 0.1)
    for blur in blurs:
        for cols, wts, cd, wdv in ((y, w, yd, wd), (x, a, xd, ad)):  # cross term, self term (same buffer)
            center = ops.default_center(xd, cd)
            xr = x.double().requires_grad_(True)
            ref = O.kernel_matrix("gaussian", xr, cols.double(), blur) @ wts.double()
            (gref,) = torch.autograd.grad(ref.sum(), xr)
            out, gunit = ops.kernel_conv_value_and_grad_rows("gaussian", xd, cd, wdv, blur, center=center)
            slack = np.log(2.0) * _exponent_slack(d, np.sqrt(np.log2(np.e)) / blur)
            np.testing.assert_allclose(out.cpu().numpy(), ref.detach().numpy(), rtol=2e-5 + slack, atol=1e-30)
            gscale = ref.detach().max().item() * np.sqrt(d) / blur**2  # natural scale, as above
            np.testing.assert_allclose(gunit.cpu().numpy(), gref.numpy(),
                                       atol=5e-5 * gref.abs().max().item() + (2e-5 + slack) * gscale)
    if d == 64:
        # BASELINE configs[2] regime: the value of the self term is its diagonal, which the kernel takes exactly
        out, _ = ops.kernel_conv_value_and_grad_rows("gaussian", xd, xd, torch.ones(n, device=DEV), 0.05,
                                                     center=ops.default_center(xd, xd))
        ref = O.kernel_conv_points("gaussian", x.double(), x.double(), torch.ones(n).double(), 0.05).numpy()
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-3)


@pytest.mark.parametrize("d", [3, 16, 64])
def test_gaussian_mmd_with_one_pass_gradients(d, monkeypatch):
    """SamplesLoss("gaussian") with ops.FUSED_CONV_GRAD: same value and gradients as the two-pass evaluation and as the
    fp64 oracle (x alone, then x and y requiring gradients; no-grad forward takes the plain path)."""
    from geomloss_b200 import SamplesLoss, ops, sinkhorn_small
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(40 + d)
    x, y = torch.rand(1200, d, generator=g), torch.rand(900, d, generator=g)
    blur = 2.0 if d > 8 else 0.3
    monkeypatch.setattr(sinkhorn_small, "SMALL_MAX", 0)  # the tiled reductions, not the small-cloud kernels
    xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
    ref = O.samples_loss(xr, yr, loss="gaussian", blur=blur)
    rx, ry = torch.autograd.grad(ref, [xr, yr])
    # the value is the small difference of three positive sums; its absolute error bound is 2^-22 of their total (two-term
    # fp16 operands / fp32 sums), computed from the fp64 oracle as in test_gaussian_conv_tensor_core_path
    ua, ub = torch.full((x.shape[0],), 1.0 / x.shape[0]).double(), torch.full((y.shape[0],), 1.0 / y.shape[0]).double()
    xd64, yd64 = x.double(), y.double()
    summands = (0.5 * ua @ O.kernel_matrix("gaussian", xd64, xd64, blur) @ ua
                + 0.5 * ub @ O.kernel_matrix("gaussian", yd64, yd64, blur) @ ub
                + ua @ O.kernel_matrix("gaussian", xd64, yd64, blur) @ ub).item()
    vtol = 1e-4 * abs(ref.item()) + 2.0**-22 * summands
    results = {}
    for fused in (False, True):
        monkeypatch.setattr(ops, "FUSED_CONV_GRAD", fused)
        xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
        before = ops.launches()
        val = SamplesLoss("gaussian", blur=blur)(xg, yg)
        gx, gy = torch.autograd.grad(val, [xg, yg])
        results[fused] = (val.item(), gx.cpu().double(), gy.cpu().double(), ops.launches() - before)
        assert abs(val.item() - ref.item()) <= vtol, (val.item(), ref.item(), vtol)
        assert (gx.cpu().double() - rx).abs().max() <= 2e-4 * rx.abs().max()
        assert (gy.cpu().double() - ry).abs().max() <= 2e-4 * ry.abs().max()
        with torch.no_grad():
            v0 = SamplesLoss("gaussian", blur=blur)(xg, yg).item()
        assert abs(v0 - ref.item()) <= vtol, (v0, ref.item(), vtol)
    # fewer reductions: 3 forward + 4 backward (x and y) two-pass, 1 + 2 one-pass forward and 2 swapped-role backward
    assert results[True][3] < results[False][3]

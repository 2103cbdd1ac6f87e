"""GPU parity tests: the CUDA engine (through the C ABI, via geomloss_b200.ops / SamplesLoss) against
  (a) golden outputs of the real reference (tests/golden/*.npz, made by tests/golden/make_golden.py),
  (b) the CPU oracle (oracle/geomloss_oracle.py, itself pinned to the goldens) on seeded inputs,
  (c) size-independent properties at BASELINE.json's full size (N = M = 1e6).

Tolerances (BASELINE.md section 3 item 7): loss within 1e-4 relative, potentials within 1e-5 absolute on
unit-cube data.  Every golden file holds the reference's output twice: its fp32 run and its fp64 run on
the same inputs.  The fp64 run is the primary target (it is the reference algorithm without rounding
noise); the fp32 run is checked at the level of the reference's own fp32-vs-fp64 gap, which is ~4e-7
for p=2 but ~1e-4..1e-2 for p=1 / laplacian / energy, where its sqrt(clamp(|x|^2-2x.y+|y|^2)) is noisy
for near-zero distances (SURVEY.md section 7.3 and appendix C).
"""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def cu(a):
    return torch.from_numpy(np.asarray(a)).to(DEV)


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()  # fails loudly if libb200ot.so is missing: there is no fallback to test
    yield


def _kw(g):
    reach = float(g["reach"])
    return dict(loss="sinkhorn", p=int(g["p"]), blur=float(g["blur"]), reach=None if reach < 0 else reach,
                debias=bool(g["debias"]), scaling=float(g["scaling"]))


# ------------------------------------------------------------------------------------------------
# operator level
# ------------------------------------------------------------------------------------------------
def test_softmin_operator_vs_reference_golden():
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn import log_weights

    g = load_golden("softmin_operator")
    x, y, b, pot = cu(g["x"]), cu(g["y"]), cu(g["b"]), cu(g["pot"])
    for p in (1, 2):
        for e, eps in enumerate(g["eps"]):
            eps = float(eps)
            ref32, ref64 = g[f"softmin_p{p}_eps{e}"], g[f"softmin_p{p}_eps{e}_f64"]
            out, _ = ops.softmin_raw(eps, x, y, log_weights(b), pot, 1.0 / eps, p=p,
                                     center=ops.default_center(x, y))
            tol = 1e-6 * max(1.0, np.abs(ref64).max())
            np.testing.assert_allclose(out.cpu().numpy(), ref64, atol=tol)
            # the fp32 reference is itself only this close to its fp64 run
            gap = np.abs(ref32 - ref64).max()
            np.testing.assert_allclose(out.cpu().numpy(), ref32, atol=tol + 1.5 * gap)
            # without the centring vector the result must be the same operator
            out2, _ = ops.softmin_raw(eps, x, y, log_weights(b) + pot / eps, p=p)
            np.testing.assert_allclose(out2.cpu().numpy(), ref64, atol=4 * tol)


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("shape", [(1, 1, 3), (3, 1, 2), (1, 5, 1), (257, 131, 3), (130, 1025, 2), (2100, 4099, 3),
                                   (4611, 5003, 3), (700, 300, 5), (300, 4200, 8),
                                   # last tile of the big shape cut to 1 / 1 / 2 / 32 chunks of 32 columns, and whole
                                   (4100, 4097, 3), (4100, 4128, 3), (4100, 4129, 3), (4100, 5120, 3), (4100, 6144, 2)])
def test_softmin_vs_oracle_shapes(p, shape):
    """Ragged sizes around the tile boundaries (2-column packets, 256/1024-column tiles, 128/512-row CTAs),
    both kernel variants (small / big), against the fp64 oracle."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(n * 7 + m)
    x = torch.rand(n, d, generator=g)
    y = torch.rand(m, d, generator=g) * 1.1 - 0.05
    h = torch.randn(m, generator=g) * 2.0 - np.log(m)
    for eps in (0.5, 0.01, 5e-4):
        ref = O.softmin_points(eps, x.double(), y.double(), h.double(), p=p, row_block=512).numpy()
        out, lse2 = ops.softmin_raw(eps, x.to(DEV), y.to(DEV), h.to(DEV), p=p,
                                    center=ops.default_center(x.to(DEV), y.to(DEV)), want_lse2=True)
        got = out.cpu().numpy()
        np.testing.assert_allclose(got, ref, atol=3e-6 * max(1.0, np.abs(ref).max()), err_msg=f"eps={eps}")
        np.testing.assert_allclose(-eps * np.log(2.0) * lse2.cpu().numpy(), got, rtol=1e-6, atol=1e-7)


def test_softmin_fused_epilogue_and_zero_weights():
    """out = alpha*old + beta*softmin(...), and log-weights of -1e5 (zero mass) contribute exactly nothing."""
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn import log_weights
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(5)
    x, y = torch.rand(300, 3, generator=g), torch.rand(411, 3, generator=g)
    b = torch.rand(411, generator=g)
    b[::7] = 0.0
    b = b / b.sum()
    pot = torch.rand(411, generator=g) * 0.1
    old = torch.rand(300, generator=g)
    eps = 0.02
    ref = O.softmin_points(eps, x.double(), y.double(), (O.log_weights(b.double()) + pot.double() / eps)).float()
    out, _ = ops.softmin_raw(eps, x.to(DEV), y.to(DEV), log_weights(b.to(DEV)), pot.to(DEV), 1 / eps,
                             out_old=old.to(DEV), alpha_old=0.5, beta=0.5 * 0.8)
    np.testing.assert_allclose(out.cpu().numpy(), (0.5 * old + 0.4 * ref).numpy(), atol=2e-6)
    keep = b > 0
    ref2 = O.softmin_points(eps, x.double(), y[keep].double(),
                            (b[keep].double().log() + pot[keep].double() / eps)).float()
    np.testing.assert_allclose(ref.numpy(), ref2.numpy(), atol=1e-7)


@pytest.mark.parametrize("p", [1, 2])
def test_softmin_gradient_vs_oracle(p):
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(11)
    n, m = 700, 1300
    x, y = torch.rand(n, 3, generator=g), torch.rand(m, 3, generator=g)
    h = torch.randn(m, generator=g) - np.log(m)
    go = torch.randn(n, generator=g)
    for eps in (0.3, 0.004):
        ref = O.softmin_grad_rows(eps, x.double(), y.double(), h.double(), go.double(), p=p).numpy()
        xg = x.to(DEV).requires_grad_(True)
        out = ops.softmin(eps, xg, y.to(DEV), h.to(DEV), p=p, center=ops.default_center(x.to(DEV), y.to(DEV)))
        (gx,) = torch.autograd.grad(out, xg, go.to(DEV))
        np.testing.assert_allclose(gx.cpu().numpy(), ref, atol=2e-5 * max(1.0, np.abs(ref).max()))


@pytest.mark.parametrize("kind", ["gaussian", "laplacian", "energy"])
def test_kernel_conv_vs_oracle(kind):
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(13)
    for (n, m, d) in [(1, 1, 3), (333, 777, 3), (4200, 4500, 2), (100, 9000, 1), (500, 600, 6)]:
        x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
        w = torch.randn(m, generator=g)
        for blur in (0.05, 0.5):
            ref = O.kernel_conv_points(kind, x.double(), y.double(), w.double(), blur).numpy()
            out = ops.kernel_conv_raw(kind, x.to(DEV), y.to(DEV), w.to(DEV), blur,
                                      center=ops.default_center(x.to(DEV), y.to(DEV)))
            scale = max(1e-3, np.abs(ref).max())
            np.testing.assert_allclose(out.cpu().numpy(), ref, atol=5e-6 * scale + 2e-7 * w.abs().sum().item())


@pytest.mark.parametrize("shape", [(300, 500, 16), (129, 65, 33), (1000, 2100, 64), (4000, 3000, 64), (257, 300, 24)])
def test_gaussian_conv_tensor_core_path(shape):
    """8 < D <= 64: the exponent comes from wgmma (fp16x2 split operands, fp32 accumulate in registers)."""
    from geomloss_b200 import SamplesLoss, ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(n + d)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    w = torch.rand(m, generator=g) / m
    for blur in (2.0, 0.7):  # at D=64, ~unit-cube data, smaller blurs underflow every off-diagonal term
        ref = O.kernel_conv_points("gaussian", x.double(), y.double(), w.double(), blur).numpy()
        out = ops.kernel_conv_raw("gaussian", x.to(DEV), y.to(DEV), w.to(DEV), blur,
                                  center=ops.default_center(x.to(DEV), y.to(DEV))).cpu().numpy()
        np.testing.assert_allclose(out, ref, rtol=2e-5, atol=1e-30, err_msg=f"blur={blur}")
    # gradients of the gaussian MMD at D > 8 (rows, columns, weights) against fp64 autograd of the oracle
    xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
    val = SamplesLoss("gaussian", blur=2.0)(xg, yg)
    gx, gy = torch.autograd.grad(val, [xg, yg])
    xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
    ref = O.samples_loss(xr, yr, loss="gaussian", blur=2.0)
    rx, ry = torch.autograd.grad(ref, [xr, yr])
    # The MMD value is the small difference of three positive sums 1/2 a'K_xx a + 1/2 b'K_yy b - a'K_xy b.  The
    # tensor-core operands are two-term fp16 splits (22 significant bits) and the sums are fp32: the absolute error
    # bound is 2^-22 of the summands' total, computed here from the fp64 oracle — not a fitted constant
    ua, ub = torch.full((n,), 1.0 / n).double(), torch.full((m,), 1.0 / m).double()
    summands = (0.5 * ua @ O.kernel_matrix("gaussian", x.double(), x.double(), 2.0) @ ua
                + 0.5 * ub @ O.kernel_matrix("gaussian", y.double(), y.double(), 2.0) @ ub
                + ua @ O.kernel_matrix("gaussian", x.double(), y.double(), 2.0) @ ub).item()
    assert abs(val.item() - ref.item()) <= 1e-4 * abs(ref.item()) + 2.0**-22 * summands
    assert (gx.cpu().double() - rx).abs().max() <= 2e-4 * rx.abs().max()
    assert (gy.cpu().double() - ry).abs().max() <= 2e-4 * ry.abs().max()
    # BASELINE configs[2] regime (blur = .05 at D = 64): |x/blur|^2 ~ 1e4, every off-diagonal term underflows and
    # the loss is carried by the diagonal of the self terms, whose exponent the kernel sets to its exact value 0
    # (tcconv.cuh, self_mode: rows and columns are the same buffer, as in kernel_loss's K_xx / K_yy).  Bar: 1e-3,
    # the reference's own fp32 error in this regime being ~4e-5 (tests/golden/hd_gaussian_d64_blur005.npz)
    xd, yd = x.to(DEV), y.to(DEV)
    out = ops.kernel_conv_raw("gaussian", xd, xd, torch.ones(n, device=DEV), 0.05,
                              center=ops.default_center(xd, xd)).cpu().numpy()
    ref = O.kernel_conv_points("gaussian", x.double(), x.double(), torch.ones(n).double(), 0.05).numpy()
    np.testing.assert_allclose(out, ref, rtol=1e-3)
    cross = ops.kernel_conv_raw("gaussian", xd, yd, torch.ones(m, device=DEV), 0.05,
                                center=ops.default_center(xd, yd)).cpu().numpy()
    refc = O.kernel_conv_points("gaussian", x.double(), y.double(), torch.ones(m).double(), 0.05).numpy()
    np.testing.assert_allclose(cross, refc, rtol=1e-3, atol=1e-30)
    val = SamplesLoss("gaussian", blur=0.05)(xd, yd).item()
    ref = O.samples_loss(x.double(), y.double(), loss="gaussian", blur=0.05).item()
    assert abs(val - ref) <= 1e-3 * abs(ref), (val, ref)


@pytest.mark.parametrize("shape", [(200, 300, 16), (131, 67, 40), (1500, 2300, 64), (257, 300, 24)])
def test_softmin_tensor_core_path(shape):
    """Forward softmin, p = 2, 8 < D <= 64: exponent from wgmma, lazy-max log-sum-exp epilogue."""
    from geomloss_b200 import SamplesLoss, ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(n * 3 + d)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    h = torch.randn(m, generator=g) - np.log(m)
    for eps in (2.0, 0.3, 0.05):
        ref = O.softmin_points(eps, x.double(), y.double(), h.double(), p=2).numpy()
        out, lse2 = ops.softmin_raw(eps, x.to(DEV), y.to(DEV), h.to(DEV), p=2,
                                    center=ops.default_center(x.to(DEV), y.to(DEV)), want_lse2=True)
        np.testing.assert_allclose(out.cpu().numpy(), ref, atol=5e-6 * max(1.0, np.abs(ref).max()), err_msg=f"eps={eps}")
    # whole Sinkhorn loop (forward / potentials) in dimension d
    F, G = SamplesLoss("sinkhorn", p=2, blur=0.5, scaling=0.6, potentials=True)(x.to(DEV), y.to(DEV))
    Fr, Gr = O.samples_loss(x.double(), y.double(), loss="sinkhorn", p=2, blur=0.5, scaling=0.6, potentials=True)
    assert (F.cpu().double() - Fr).abs().max() < 2e-5 * max(1.0, Fr.abs().max().item())
    assert (G.cpu().double() - Gr).abs().max() < 2e-5 * max(1.0, Gr.abs().max().item())
    # row gradients: two chained wgmma GEMMs (S = X.Y^T -> P = 2^S in registers -> G = P.Y), csrc/tcbwd.cuh
    go = torch.randn(n, generator=g)
    for eps in (2.0, 0.3):
        ref = O.softmin_grad_rows(eps, x.double(), y.double(), h.double(), go.double(), p=2).numpy()
        xg = x.to(DEV).requires_grad_(True)
        out = ops.softmin(eps, xg, y.to(DEV), h.to(DEV), p=2, center=ops.default_center(x.to(DEV), y.to(DEV)))
        (gx,) = torch.autograd.grad(out, xg, go.to(DEV))
        np.testing.assert_allclose(gx.cpu().numpy(), ref, atol=5e-5 * max(1.0, np.abs(ref).max()))
    xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
    val = SamplesLoss("sinkhorn", p=2, blur=0.5, scaling=0.6)(xg, yg)
    gx, gy = torch.autograd.grad(val, [xg, yg])
    xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
    rx, ry = torch.autograd.grad(O.samples_loss(xr, yr, loss="sinkhorn", p=2, blur=0.5, scaling=0.6), [xr, yr])
    assert (gx.cpu().double() - rx).abs().max() <= 1e-4 * rx.abs().max()
    assert (gy.cpu().double() - ry).abs().max() <= 1e-4 * ry.abs().max()


@pytest.mark.parametrize("kind", ["gaussian", "laplacian", "energy"])
def test_kernel_conv_gradients_vs_autograd(kind):
    """Row, column and weight gradients of out = K(x,y) @ w against dense fp64 autograd of the oracle."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(17)
    n, m = 400, 650
    x, y = torch.rand(n, 3, generator=g), torch.rand(m, 3, generator=g)
    w, go = torch.rand(m, generator=g), torch.randn(n, generator=g)
    blur = 0.3
    xr, yr, wr = (t.double().requires_grad_(True) for t in (x, y, w))
    ref_out = O.kernel_matrix(kind, xr, yr, blur) @ wr
    rx, ry, rw = torch.autograd.grad(ref_out, [xr, yr, wr], go.double())
    xg, yg, wg = (t.to(DEV).requires_grad_(True) for t in (x, y, w))
    out = ops.kernel_conv(kind, xg, yg, wg, blur, center=ops.default_center(x.to(DEV), y.to(DEV)))
    gx, gy, gw = torch.autograd.grad(out, [xg, yg, wg], go.to(DEV))
    for got, ref in ((gx, rx), (gy, ry), (gw, rw)):
        ref = ref.numpy()
        np.testing.assert_allclose(got.cpu().numpy(), ref, atol=3e-5 * max(1.0, np.abs(ref).max()))


@pytest.mark.parametrize("m", [257, 288, 289, 4097, 4128, 4129, 5120])
def test_row_reductions_last_tile_lengths(m):
    """The consumers stop at the 32-column chunk holding the last column (plan.cuh: last_pairs) instead of visiting the
    neutral padding of the last tile: softmin row gradients and the three kernel products, small and big tile shape,
    at column counts just before / on / after a chunk and a tile boundary."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n = 4100 if m > 4000 else 300
    g = torch.Generator().manual_seed(m)
    x, y = torch.rand(n, 3, generator=g), torch.rand(m, 3, generator=g)
    h = torch.randn(m, generator=g) - np.log(m)
    w, go = torch.randn(m, generator=g), torch.randn(n, generator=g)
    c = ops.default_center(x.to(DEV), y.to(DEV))
    for p in (1, 2):
        ref = O.softmin_grad_rows(0.02, x.double(), y.double(), h.double(), go.double(), p=p).numpy()
        xg = x.to(DEV).requires_grad_(True)
        (gx,) = torch.autograd.grad(ops.softmin(0.02, xg, y.to(DEV), h.to(DEV), p=p, center=c), xg, go.to(DEV))
        np.testing.assert_allclose(gx.cpu().numpy(), ref, atol=2e-5 * max(1.0, np.abs(ref).max()))
    for kind in ("gaussian", "laplacian", "energy"):
        ref = O.kernel_conv_points(kind, x.double(), y.double(), w.double(), 0.1).numpy()
        out = ops.kernel_conv_raw(kind, x.to(DEV), y.to(DEV), w.to(DEV), 0.1, center=c)
        np.testing.assert_allclose(out.cpu().numpy(), ref,
                                   atol=5e-6 * max(1e-3, np.abs(ref).max()) + 2e-7 * w.abs().sum().item())


@pytest.mark.parametrize("shape", [(1, 0, 3), (5, 7, 1), (1000, 1300, 3), (70000, 5, 2), (300000, 200000, 8)])
def test_cloud_extent_vs_torch(shape):
    """b200ot_cloud_extent (one launch, last-block fold) == torch min / max; repeated calls re-use the ticket scratch."""
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn import max_diameter

    n, m, d = shape
    g = torch.Generator().manual_seed(n + m)
    x = (torch.randn(n, d, generator=g) * 3).to(DEV)
    y = (torch.randn(m, d, generator=g) - 1).to(DEV)
    for _ in range(3):
        lh = ops.cloud_extent(x, y if m else None)
        both = torch.cat([x, y]) if m else x
        assert torch.equal(lh[0], both.min(0).values) and torch.equal(lh[1], both.max(0).values)
    if m:
        ref = (both.max(0).values - both.min(0).values).norm().item()
        assert abs(max_diameter(x, y) - ref) <= 2e-7 * ref
        assert torch.equal(ops.default_center(x, y), 0.5 * (both.min(0).values + both.max(0).values))


@pytest.mark.parametrize("rho", [None, 0.7])
@pytest.mark.parametrize("debias", [True, False])
def test_sinkhorn_cost_small_kernel_vs_host_formula(rho, debias):
    """b200ot_sinkhorn_cost_small: values, d value / d potential and d value / d weight against autograd of the host
    formula (sinkhorn.sinkhorn_cost = sinkhorn_divergence.py:165-255)."""
    import ctypes

    from geomloss_b200 import _lib, ops
    from geomloss_b200.sinkhorn import sinkhorn_cost

    B, N, M, eps = 3, 257, 301, 0.01
    g = torch.Generator().manual_seed(3)
    a = torch.rand(B, N, generator=g).to(DEV).requires_grad_(True)
    b = torch.rand(B, M, generator=g).to(DEV).requires_grad_(True)
    pots = [(torch.randn(B, n, generator=g) * 0.3).to(DEV).requires_grad_(True) for n in (N, M, N, M)]
    f_ba, g_ab, f_aa, g_bb = pots
    ref = sinkhorn_cost(eps, rho, a, b, f_aa if debias else None, g_bb if debias else None, g_ab, f_ba, debias=debias)
    go = torch.tensor([1.0, -2.0, 0.5], device=DEV)
    used = [a, b, f_ba, g_ab] + ([f_aa, g_bb] if debias else [])
    grads = torch.autograd.grad(ref, used, go)
    val = torch.empty(B, device=DEV)
    outs = [torch.zeros(B, n, device=DEV) for n in (N, M, N, M, N, M)]
    P = ops._ptr
    rc = _lib.lib().b200ot_sinkhorn_cost_small(P(a.detach()), P(b.detach()), P(f_ba.detach()), P(g_ab.detach()),
                                               P(f_aa.detach()) if debias else None,
                                               P(g_bb.detach()) if debias else None, B, N, M,
                                               -1.0 if rho is None else rho, eps, P(val), P(outs[0]), P(outs[1]),
                                               P(outs[2]) if debias else None, P(outs[3]) if debias else None,
                                               P(outs[4]), P(outs[5]), ctypes.c_void_p(0))
    assert rc == 0
    torch.cuda.synchronize()
    np.testing.assert_allclose(val.cpu().numpy(), ref.detach().cpu().numpy(), rtol=2e-6, atol=1e-6)
    got = [outs[4], outs[5], outs[0], outs[1]] + ([outs[2], outs[3]] if debias else [])
    for k, (gt, rf) in enumerate(zip(got, grads)):
        np.testing.assert_allclose((gt * go[:, None]).cpu().numpy(), rf.cpu().numpy(), rtol=3e-6, atol=1e-6,
                                   err_msg=f"output {k}")


# ------------------------------------------------------------------------------------------------
# SamplesLoss vs the reference's golden outputs
# ------------------------------------------------------------------------------------------------
def test_cfg1_sinkhorn_n1000(sinkhorn_path):
    """BASELINE.json configs[0]: N=M=1000, D=3, blur=.05 — value, potentials, all four gradients."""
    from geomloss_b200 import SamplesLoss

    g = load_golden("cfg1_sinkhorn_n1000")
    a, x, b, y = (cu(g[k]) for k in "axby")
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = SamplesLoss("sinkhorn", p=2, blur=0.05)(ag, xg, bg, yg)
    assert val.dim() == 0
    ref64 = float(g["value_f64"])
    assert abs(val.item() - ref64) <= 1e-4 * abs(ref64)  # the stated bar
    assert abs(val.item() - ref64) <= 5e-6 * abs(ref64)  # what the engine actually achieves
    assert abs(val.item() - float(g["value_f32"])) <= 5e-6 * abs(ref64)
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    np.testing.assert_allclose(ga.cpu().numpy(), g["grad_a_f64"], atol=1e-6)
    np.testing.assert_allclose(gb.cpu().numpy(), g["grad_b_f64"], atol=1e-6)
    gscale = np.abs(g["grad_x_f64"]).max()
    np.testing.assert_allclose(gx.cpu().numpy(), g["grad_x_f64"], atol=2e-5 * gscale)
    np.testing.assert_allclose(gy.cpu().numpy(), g["grad_y_f64"], atol=2e-5 * gscale)
    F, G = SamplesLoss("sinkhorn", p=2, blur=0.05, potentials=True)(a, x, b, y)
    assert F.shape == (1, 1000) and G.shape == (1, 1000)
    np.testing.assert_allclose(F.cpu().numpy(), g["pot_f_f64"], atol=1e-6)  # bar: 1e-5
    np.testing.assert_allclose(G.cpu().numpy(), g["pot_g_f64"], atol=1e-6)
    # 2-argument form = uniform weights; "auto" / "tensorized" / "online" are one exact engine
    for backend in ("auto", "tensorized", "online"):
        v2 = SamplesLoss("sinkhorn", p=2, blur=0.05, backend=backend)(x, y)
        assert abs(v2.item() - ref64) <= 5e-6 * abs(ref64)
    # "multiscale" is a different (two-scale) iteration scheme: same ballpark, not the same number
    v3 = SamplesLoss("sinkhorn", p=2, blur=0.05, backend="multiscale")(x, y)
    assert abs(v3.item() - ref64) <= 0.15 * abs(ref64)


@pytest.mark.parametrize("name", golden_names("sinkhorn_case"))
def test_sinkhorn_cases(name, sinkhorn_path):
    from geomloss_b200 import SamplesLoss, ops

    g = load_golden(name)
    if not dim_supported(g["x"].shape[-1]):
        pytest.skip("D > 3 kernels not instantiated in this build")
    a, x, b, y = (cu(g[k]) for k in "axby")
    kw = _kw(g)
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = SamplesLoss(**kw)(ag, xg, bg, yg)
    ref = float(g["value_f64"])
    assert abs(val.item() - ref) <= 1e-4 * abs(ref) + 1e-7, (val.item(), ref)
    # fp32 reference: within its own distance to the fp64 run (+ the stated bar)
    gap = abs(float(g["value"]) - ref)
    assert abs(val.item() - float(g["value"])) <= 1e-4 * abs(ref) + 1.5 * gap + 1e-7
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    for got, key in ((ga, "grad_a"), (gb, "grad_b"), (gx, "grad_x"), (gy, "grad_y")):
        r = g[key + "_f64"]
        np.testing.assert_allclose(got.cpu().numpy(), r, atol=1e-4 * max(np.abs(r).max(), 1e-3), err_msg=key)
    F, G = SamplesLoss(potentials=True, **kw)(a, x, b, y)
    np.testing.assert_allclose(F.cpu().numpy(), g["pot_f_f64"], atol=1e-5 * max(1.0, np.abs(g["pot_f_f64"]).max()))
    np.testing.assert_allclose(G.cpu().numpy(), g["pot_g_f64"], atol=1e-5 * max(1.0, np.abs(g["pot_g_f64"]).max()))


def dim_supported(d):
    return d <= 8


def test_sinkhorn_batched(sinkhorn_path):
    from geomloss_b200 import SamplesLoss

    g = load_golden("sinkhorn_batched")
    a, x, b, y = (cu(g[k]) for k in "axby")
    val = SamplesLoss("sinkhorn", p=2, blur=0.1)(a, x, b, y)
    assert val.shape == (2,)
    np.testing.assert_allclose(val.cpu().numpy(), g["value_f64"], rtol=1e-4)
    np.testing.assert_allclose(val.cpu().numpy(), g["value"], rtol=1e-4)
    F, G = SamplesLoss("sinkhorn", p=2, blur=0.1, potentials=True)(a, x, b, y)
    assert F.shape == (2, 40) and G.shape == (2, 30)
    np.testing.assert_allclose(F.cpu().numpy(), g["pot_f_f64"], atol=1e-5)
    np.testing.assert_allclose(G.cpu().numpy(), g["pot_g_f64"], atol=1e-5)
    # weights given as (B,N,1)
    v2 = SamplesLoss("sinkhorn", p=2, blur=0.1)(a.unsqueeze(-1), x, b.unsqueeze(-1), y)
    np.testing.assert_allclose(v2.cpu().numpy(), val.cpu().numpy(), rtol=1e-6)


@pytest.mark.parametrize("name", golden_names("kernel_gaussian") + golden_names("kernel_laplacian")
                         + golden_names("kernel_energy"))
def test_kernel_losses(name, sinkhorn_path):
    from geomloss_b200 import SamplesLoss

    g = load_golden(name)
    if not dim_supported(g["x"].shape[-1]):
        pytest.skip("D > 3 kernels not instantiated in this build")
    kind = name.split("_")[1]
    a, x, b, y = (cu(g[k]) for k in "axby")
    blur = float(g["blur"])
    xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ag, bg = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    val = SamplesLoss(kind, blur=blur)(ag, xg, bg, yg)
    ref = float(g["value_f64"])
    # the reference's own fp32 result is only self-consistent to ~1e-4..1e-3 for laplacian/energy
    # (SURVEY.md appendix C); compare with its fp64 value
    assert abs(val.item() - ref) <= 1e-4 * abs(ref) + 2e-7, (val.item(), ref)
    ga, gx, gb, gy = torch.autograd.grad(val, [ag, xg, bg, yg])
    for got, key in ((ga, "grad_a"), (gb, "grad_b"), (gx, "grad_x"), (gy, "grad_y")):
        r = g[key + "_f64"]
        np.testing.assert_allclose(got.cpu().numpy(), r, atol=1e-4 * max(np.abs(r).max(), 1e-3), err_msg=key)
    F, G = SamplesLoss(kind, blur=blur, potentials=True)(a, x, b, y)
    np.testing.assert_allclose(F.cpu().numpy(), g["pot_f_f64"], atol=2e-5 * np.abs(g["pot_f_f64"]).max())
    np.testing.assert_allclose(G.cpu().numpy(), g["pot_g_f64"], atol=2e-5 * np.abs(g["pot_g_f64"]).max())
    # dL/da is the potential (SURVEY.md appendix A-16)
    np.testing.assert_allclose(ga.cpu().numpy(), F.cpu().numpy().reshape(-1), atol=1e-6)


def test_mid_size_loss_vs_oracle():
    """N=4300, M=4100 (big-kernel variant, ragged): loss and potentials against the dense CPU oracle."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(23)
    x, y = torch.rand(4300, 3, generator=g), torch.rand(4100, 3, generator=g)
    for kw in (dict(blur=0.05, scaling=0.5), dict(blur=0.01, scaling=0.6), dict(blur=0.05, p=1, scaling=0.5),
               dict(blur=0.05, reach=0.5, scaling=0.5)):
        # one dense fp64 oracle run gives both the potentials and (through the value formula) the loss
        a = torch.full((1, 4300), 1 / 4300, dtype=torch.float64)
        b = torch.full((1, 4100), 1 / 4100, dtype=torch.float64)
        Fr, Gr = O.samples_loss(x.double(), y.double(), loss="sinkhorn", potentials=True, **kw)
        F, G = SamplesLoss("sinkhorn", potentials=True, **kw)(x.to(DEV), y.to(DEV))
        assert (F.cpu().double() - Fr).abs().max() < 1e-5 and (G.cpu().double() - Gr).abs().max() < 1e-5
        val = SamplesLoss("sinkhorn", **kw)(x.to(DEV), y.to(DEV)).item()
        if kw.get("reach") is None:  # balanced + debiased: value = <a, F> + <b, G>
            ref = ((a * Fr).sum() + (b * Gr).sum()).item()
        else:
            ref = O.samples_loss(x.double(), y.double(), loss="sinkhorn", **kw).item()
        assert abs(val - ref) <= 1e-4 * abs(ref), (kw, val, ref)


# ------------------------------------------------------------------------------------------------
# full size (BASELINE.json configs[1]): size-independent properties
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def million():
    g = torch.Generator().manual_seed(0)
    x = torch.rand(10**6, 3, generator=g)
    y = torch.rand(10**6, 3, generator=g)
    return x, y


def test_full_size_softmin_properties(million):
    from geomloss_b200 import ops

    x, y = million
    n = m = 10**6
    eps = 1e-4  # blur = .01
    g = torch.Generator().manual_seed(1)
    pot = (torch.rand(m, generator=g) - 0.5) * 0.02
    h_a = torch.full((m,), -np.log(m))
    xd, yd, pd, hd = x.to(DEV), y.to(DEV), pot.to(DEV), h_a.to(DEV)
    c = ops.default_center(xd, yd)
    out, _ = ops.softmin_raw(eps, xd, yd, hd, pd, 1 / eps, center=c)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    # (1) sampled rows against an fp64 brute force
    idx = torch.linspace(0, n - 1, 12).long()
    h64 = h_a.double() + pot.double() / eps
    for i in idx.tolist():
        t = h64 - ((x[i].double() - y.double()) ** 2).sum(1) / (2 * eps)
        ref = -eps * torch.logsumexp(t, 0).item()
        assert abs(out[i].item() - ref) < 2e-7 + 2e-6 * abs(ref)
    # (2) shift equivariance: softmin(h + s) = softmin(h) - eps*s
    out_s, _ = ops.softmin_raw(eps, xd, yd, hd + 3.0, pd, 1 / eps, center=c)
    assert (out_s - (out - 3.0 * eps)).abs().max().item() < 5e-7
    # (3) column permutation invariance (different tiles, splits and summation order)
    perm = torch.randperm(m, generator=g).to(DEV)
    out_p, _ = ops.softmin_raw(eps, xd, yd[perm], hd[perm], pd[perm], 1 / eps, center=c)
    assert (out_p - out).abs().max().item() < 5e-7
    # (4) column-shard consistency: LSE-merging two half problems reproduces the full one
    half = m // 2
    o1, _ = ops.softmin_raw(eps, xd, yd[:half], hd[:half], pd[:half], 1 / eps, center=c)
    o2, _ = ops.softmin_raw(eps, xd, yd[half:], hd[half:], pd[half:], 1 / eps, center=c)
    merged = -eps * torch.logaddexp(-o1 / eps, -o2 / eps)
    assert (merged - out).abs().max().item() < 5e-7
    # (5) soft-min bounds: min_j (C_ij - eps h_j) - eps log M... <= out <= min_j (C_ij - eps h_j)
    i = 12345
    cmin = (((x[i].double() - y.double()) ** 2).sum(1) / 2 - eps * h64).min().item()
    assert cmin - eps * np.log(m) - 1e-6 <= out[i].item() <= cmin + 1e-6


def test_full_size_sinkhorn_iteration_identities(million):
    """One symmetric Sinkhorn iteration at N=M=1e6: OT(a,a) potentials are symmetric by construction
    (f_aa from (x,x) equals itself under a relabelling) and S(a,a) = 0."""
    from geomloss_b200 import SamplesLoss

    x, _ = million
    xd = x.to(DEV)[:200000].contiguous()
    v = SamplesLoss("sinkhorn", p=2, blur=0.05, scaling=0.5)(xd, xd.clone())
    assert abs(v.item()) < 1e-7


# ------------------------------------------------------------------------------------------------
# multiscale (two-scale, block-sparse) vs the dense engine
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(p=2, blur=0.02), dict(p=2, blur=0.03, reach=0.4, debias=False), dict(p=1, blur=0.02),
                                dict(p=2, blur=0.4)])
def test_multiscale_vs_two_scale_oracle(kw):
    """The two-scale scheme (coarse centroids -> jump with kernel truncation -> block-sparse fine phase) against a
    dense CPU restatement of the same algorithm.  NB it is not comparable to the single-scale backends at
    tight tolerance: its iterates differ by design (see multiscale.py).  blur=.4 exercises the 'jump on the last
    iteration' branch.  Our tile-level mask keeps a superset of the reference's cluster-level blocks, so the
    truncated results agree to the (tiny) weight of the pruned terms."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(31)
    n, m = 5200, 4700
    x = torch.rand(n, 3, generator=g)
    y = torch.rand(m, 3, generator=g) * 0.8 + 0.15
    a = torch.rand(n, generator=g) + 0.5
    b = torch.rand(m, generator=g) + 0.5
    a, b = a / a.sum(), b / b.sum()
    cs = 0.12  # ~600 clusters per cloud: several clusters per 512 x 1024 tile, real sparsity at blur = .02
    xd, yd, ad, bd = x.to(DEV), y.to(DEV), a.to(DEV), b.to(DEV)
    for truncate in (None, 5):
        ref = O.sinkhorn_multiscale_dense(a.double(), x.double(), b.double(), y.double(), truncate=truncate,
                                          cluster_scale=cs, **kw).item()
        L = SamplesLoss("sinkhorn", backend="multiscale", truncate=truncate, cluster_scale=cs, **kw)
        val = L(ad, xd, bd, yd).item()
        assert abs(val - ref) <= 5e-5 * abs(ref), (truncate, val, ref)
    Fr, Gr = O.sinkhorn_multiscale_dense(a.double(), x.double(), b.double(), y.double(), truncate=None, cluster_scale=cs,
                                         potentials=True, **kw)
    F, G = SamplesLoss("sinkhorn", backend="multiscale", truncate=None, cluster_scale=cs, potentials=True, **kw)(ad, xd,
                                                                                                              bd, yd)
    assert F.shape == (n,) and G.shape == (m,)  # multiscale returns un-batched potentials (SURVEY A-12), de-permuted
    assert (F.cpu().double() - Fr).abs().max().item() < 2e-5 and (G.cpu().double() - Gr).abs().max().item() < 2e-5
    # autograd contract: d/da = potential (balanced, debiased); d/dx close to the dense engine's gradient
    if kw.get("reach") is None:
        ag, xg = ad.clone().requires_grad_(True), xd.clone().requires_grad_(True)
        val = SamplesLoss("sinkhorn", backend="multiscale", truncate=None, cluster_scale=cs, **kw)(ag, xg, bd, yd)
        ga, gx = torch.autograd.grad(val, [ag, xg])
        assert (ga - F).abs().max().item() < 1e-6
        xg2 = xd.clone().requires_grad_(True)
        (gd,) = torch.autograd.grad(SamplesLoss("sinkhorn", backend="online", **kw)(ad, xg2, bd, yd), xg2)
        cos = torch.nn.functional.cosine_similarity(gx.flatten(), gd.flatten(), dim=0).item()
        assert cos > 0.98, cos
    # user-supplied cluster labels (6-argument form) route to the multiscale backend
    from geomloss_b200.multiscale import grid_labels

    lab = SamplesLoss("sinkhorn", truncate=None, cluster_scale=cs, **kw)(grid_labels(xd, cs), ad, xd, grid_labels(yd, cs),
                                                                            bd, yd)
    plain = SamplesLoss("sinkhorn", backend="multiscale", truncate=None, cluster_scale=cs, **kw)(ad, xd, bd, yd)
    # (centroids are accumulated with float atomics: run-to-run differences of a few ulps are expected)
    assert abs(lab.item() - plain.item()) <= 2e-5 * abs(plain.item())


# ------------------------------------------------------------------------------------------------
# grids (images / volumes): parity against the (unpinned, cross-checked) dense grid oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 1, 8, 8), (1, 2, 32, 32), (1, 1, 64, 64), (1, 1, 16, 16, 16), (2, 1, 32, 32, 32)])
@pytest.mark.parametrize("p", [1, 2])
def test_grid_softmin_vs_oracle(shape, p):
    from geomloss_b200.sinkhorn_images import softmin_grid
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(sum(shape) + p)
    h = torch.randn(*shape, generator=g) * 3.0
    h[..., 0] = -10000.0  # empty pixels (log_dens floor)
    pot = torch.randn(*shape, generator=g) * 0.01
    old = torch.randn(*shape, generator=g)
    n = shape[-1]
    for eps in (1.0, (2.0 / n) ** p, (1.0 / n) ** p):
        ref = O.softmin_grid_dense(eps, p, (h + pot / eps).double())
        out = softmin_grid(eps, p, h.to(DEV), pot.to(DEV), 1.0 / eps)
        scale = max(1.0, ref.abs().max().item())
        assert (out.cpu().double() - ref).abs().max().item() < 3e-6 * scale, eps
        out2 = softmin_grid(eps, p, h.to(DEV), pot.to(DEV), 1.0 / eps, out_old=old.to(DEV), alpha_old=0.5, beta=0.4)
        assert (out2.cpu().double() - (0.5 * old.double() + 0.4 * ref)).abs().max().item() < 3e-6 * scale


@pytest.mark.parametrize("shape", [(2, 1, 32, 32), (1, 1, 16, 16, 16)])
def test_image_sinkhorn_vs_oracle(shape):
    from geomloss_b200 import sinkhorn_divergence
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(len(shape))
    a = torch.rand(*shape, generator=g) ** 3
    b = torch.rand(*shape, generator=g) ** 3
    a[..., :3] = 0.0  # empty pixels
    a, b = a / a.sum(), b / b.sum() * 1.0
    # (blur must resolve the finest pixels, else the reference's own "bug in the multiscale pre-processing"
    #  assertion fires — kept verbatim in both restatements)
    for kw in (dict(p=2), dict(p=2, reach=0.3, scaling=0.7), dict(p=1)):
        ref = O.sinkhorn_images(a.double(), b.double(), **kw)
        ag = a.to(DEV).requires_grad_(True)
        val = sinkhorn_divergence(ag, b.to(DEV), **kw)
        assert val.shape == (shape[0],)
        np.testing.assert_allclose(val.detach().cpu().numpy(), ref.numpy(), rtol=2e-4, atol=1e-9)
        Fr, Gr = O.sinkhorn_images(a.double(), b.double(), potentials=True, **kw)
        F, G = sinkhorn_divergence(a.to(DEV), b.to(DEV), potentials=True, **kw)
        assert (F.cpu().double() - Fr).abs().max() < 1e-5 * max(1.0, Fr.abs().max().item())
        assert (G.cpu().double() - Gr).abs().max() < 1e-5 * max(1.0, Gr.abs().max().item())
        if kw.get("reach") is None:  # balanced: d loss / d a = potential
            (ga,) = torch.autograd.grad(val.sum(), ag)
            assert (ga.cpu().double() - Fr).abs().max() < 1e-5 * max(1.0, Fr.abs().max().item())
    with pytest.raises(ValueError):
        sinkhorn_divergence(a.to(DEV), b.to(DEV), scaling=0.3)


# ------------------------------------------------------------------------------------------------
# error behaviour on the GPU
# ------------------------------------------------------------------------------------------------
def test_errors_on_gpu():
    from geomloss_b200 import SamplesLoss, _lib, ops

    x, y = torch.rand(10, 3, device=DEV), torch.rand(12, 3, device=DEV)
    with pytest.raises(TypeError):
        SamplesLoss("sinkhorn")(x.double(), y.double())
    with pytest.raises(NotImplementedError):
        ops.softmin_raw(0.1, torch.rand(4, 100, device=DEV), torch.rand(5, 100, device=DEV), torch.zeros(5, device=DEV))
    with pytest.raises(NotImplementedError):  # p = 1 has no tensor-core path
        ops.softmin_raw(0.1, torch.rand(4, 40, device=DEV), torch.rand(5, 40, device=DEV), torch.zeros(5, device=DEV), p=1)
    with pytest.raises(ValueError):
        ops.softmin_raw(0.1, x, y, torch.zeros(11, device=DEV))
    with pytest.raises(_lib.B200OTError):
        ops.softmin_raw(-1.0, x, y, torch.zeros(12, device=DEV))


# ------------------------------------------------------------------------------------------------
# geomloss.ot.solve_sample facade (SURVEY.md section 8, row f-3)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("idx", range(8))
def test_ot_solve_sample_vs_reference_goldens(idx):
    """The new-API solver on the CUDA softmin against fp64 / fp32 runs of the real reference (tests/golden/
    make_golden_ot.py): value 1e-4 relative, potentials / marginals 2e-5 of their scale, dense plan."""
    from geomloss_b200 import ot

    z = load_golden(f"ot_sample_case{idx:02d}")
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    t = lambda k: torch.from_numpy(z[k]).to(DEV)  # noqa: E731
    res = ot.solve_sample(t("X_a"), t("X_b"), a=t("a") if "a" in z else None, b=t("b") if "b" in z else None, **kw)
    ref = float(z["value_f64"])
    assert abs(res.value.item() - ref) <= 1e-4 * abs(ref), (res.value.item(), ref)
    # against the fp32 reference run: within the reference's own fp32-vs-fp64 gap (+ our 1e-4 bar)
    assert abs(res.value.item() - float(z["value"])) <= 1e-4 * abs(ref) + 2 * abs(float(z["value"]) - ref)
    names = ["potential_a", "potential_b", "marginal_a", "marginal_b", "plan"]
    if kw.get("debias"):
        names += ["potential_aa", "potential_bb"]
    else:
        with pytest.raises(ValueError):
            res.potential_aa
    for name in names:
        r = z[name + "_f64"]
        out = getattr(res, name).cpu().numpy()
        assert out.shape == r.shape, name
        np.testing.assert_allclose(out, r, atol=2e-5 * max(1.0, float(np.abs(r).max())) if "potential" in name
                                   else 3e-4 * float(np.abs(r).max()), err_msg=name)
    # operators: plan @ 1 = marginal_a, plan.T @ 1 = marginal_b, signed right-hand sides, trailing dimensions
    n, m = z["X_a"].shape[0], z["X_b"].shape[0]
    P = torch.from_numpy(z["plan_f64"])
    g = torch.Generator().manual_seed(idx)
    s = torch.randn(m, 2, generator=g, dtype=torch.float64)
    out = (res.plan_operator @ s.float().to(DEV)).cpu().double()
    assert out.shape == (n, 2)
    assert (out - P @ s).abs().max() <= 3e-4 * (P @ s.abs()).max()
    s = torch.rand(n, generator=g, dtype=torch.float64)
    out = (res.plan_operator.T @ s.float().to(DEV)).cpu().double()
    assert (out - P.t() @ s).abs().max() <= 3e-4 * (P.t() @ s).max()
    assert res.plan_operator.shape == (n, m) and res.lazy_plan is None


@pytest.mark.parametrize("idx", range(8))
def test_ot_solve_sample_gradients_vs_reference(idx):
    """d value / d (X_a, X_b, a, b): the last update differentiated w.r.t. BOTH clouds (row-gradient kernel + the same
    kernel on the swapped problem) against the real reference's fp64 autograd (tests/golden/make_golden_ot.py)."""
    from geomloss_b200 import ot

    z = load_golden(f"ot_sample_case{idx:02d}")
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    n, m = z["X_a"].shape[0], z["X_b"].shape[0]
    a0 = torch.from_numpy(z["a"]) if "a" in z else torch.full((n,), 1.0 / n)
    b0 = torch.from_numpy(z["b"]) if "b" in z else torch.full((m,), 1.0 / m)
    leaves = [t.to(DEV).requires_grad_(True) for t in (torch.from_numpy(z["X_a"]), torch.from_numpy(z["X_b"]), a0, b0)]
    res = ot.solve_sample(leaves[0], leaves[1], a=leaves[2], b=leaves[3], **kw)
    ref = float(z["value_f64"])
    assert abs(res.value.item() - ref) <= 1e-4 * abs(ref)
    grads = torch.autograd.grad(res.value, leaves)
    for g, name in zip(grads, ("grad_X_a", "grad_X_b", "grad_a", "grad_b")):
        r = z[name + "_f64"]
        np.testing.assert_allclose(g.cpu().numpy(), r, atol=2e-3 * float(np.abs(r).max()), err_msg=name)
    assert not res.potential_a.requires_grad and not res.marginal_b.requires_grad


def test_ot_solve_sample_diracs_and_doc_example():
    """The reference's own checks for this solver: tests/test_ot_solve_sample.py::test_correct_values_diracs
    (one point per side: value = C, potentials = C/2, plan = 1, any reg / max_iter) and the doctest of
    solve_sample (sample.py:256-279)."""
    from geomloss_b200 import ot

    rng = np.random.default_rng(0)
    for _ in range(12):
        D = int(rng.integers(1, 6))
        xa, xb = rng.uniform(-10, 10, (1, D)), rng.uniform(-10, 10, (1, D))
        reg, max_iter = float(rng.uniform(1e-2, 10.0)), int(rng.integers(1, 51))
        C = float(((xa - xb) ** 2).sum())
        use_w = bool(rng.integers(0, 2))
        res = ot.solve_sample(torch.tensor(xa, dtype=torch.float32, device=DEV),
                              torch.tensor(xb, dtype=torch.float32, device=DEV),
                              a=torch.ones(1, device=DEV) if use_w else None,
                              b=torch.ones(1, device=DEV) if use_w else None, reg=reg, max_iter=max_iter)
        atol = 1e-2  # the reference's tolerance for this generator (tests/generators/diracs.py)
        assert abs(res.value.item() - C) <= atol + 1e-5 * C
        assert abs(res.potential_a.item() - C / 2) <= atol + 1e-5 * C
        assert abs(res.potential_b.item() - C / 2) <= atol + 1e-5 * C
        assert abs(res.plan.item() - 1.0) <= atol
    sol = ot.solve_sample(torch.tensor([[0.0, 0.0], [0.0, 2.0]], device=DEV), torch.tensor([[2.0, 1.0], [2.0, 2.0]], device=DEV),
                          reg=0.001, max_iter=100)
    np.testing.assert_allclose(sol.plan.cpu().numpy(), [[0.5, 0.0], [0.0, 0.5]], atol=1e-3)
    assert f"{sol.value.item():.3f}" == "4.501"


def test_ot_solve_sample_large_never_dense():
    """N = M = 2e5 (a dense plan would be 160 GB): marginals through the operator, balanced constraints met."""
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(0)
    x = torch.rand(200_000, 3, generator=g).to(DEV)
    y = torch.rand(200_000, 3, generator=g).to(DEV)
    res = ot.solve_sample(x, y, blur=0.05, max_iter=12)
    ma, mb = res.marginal_a, res.marginal_b
    # the last update is simultaneous (Jacobi): both marginals are met to the convergence of a 12-step ladder
    assert abs(ma.sum().item() - 1.0) < 5e-2 and abs(mb.sum().item() - 1.0) < 5e-2
    assert (ma * 200_000 - 1).abs().max().item() < 0.5
    with pytest.raises(MemoryError):
        res.plan
    # the value is the legacy API's OT_eps up to the cost convention: C = |x-y|^2 = 2 * (|x-y|^2 / 2)
    from geomloss_b200 import SamplesLoss

    legacy = SamplesLoss("sinkhorn", p=2, blur=0.05, debias=False, scaling=0.5)(x, y).item()
    assert abs(res.value.item() - 2 * legacy) <= 2e-2 * abs(2 * legacy)


# ------------------------------------------------------------------------------------------------
# ImagesBarycenter on the grid softmin (SURVEY.md section 8, row f-4)
# ------------------------------------------------------------------------------------------------
def _bary_inputs(n, K, B, seed):
    g = torch.Generator().manual_seed(seed)
    ax = torch.linspace(0, 1, n)
    X, Y = torch.meshgrid(ax, ax, indexing="ij")
    imgs = torch.zeros(B, K, n, n)
    for bi in range(B):
        for k in range(K):
            c = 0.2 + 0.6 * torch.rand(2, generator=g)
            s = 0.06 + 0.08 * float(torch.rand(1, generator=g))
            imgs[bi, k] = torch.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2) / (2 * s * s)) + 1e-4
            if k == 0:
                imgs[bi, k][: n // 4] = 0.0  # empty pixels: log_dens floor
    imgs = imgs / imgs.sum((2, 3), keepdim=True)
    w = torch.rand(B, K, generator=g) + 0.2
    return imgs, w / w.sum(1, keepdim=True)


@pytest.mark.parametrize("shape", [(16, 2, 1), (32, 3, 2)])
@pytest.mark.parametrize("p", [1, 2])
def test_images_barycenter_vs_dense_oracle(shape, p):
    from geomloss_b200 import ImagesBarycenter
    from oracle import geomloss_oracle as O

    n, K, B = shape
    imgs, w = _bary_inputs(n, K, B, seed=n + p)
    ref = O.images_barycenter(imgs.double(), w.double(), p=p, scaling_N=4)
    out = ImagesBarycenter(imgs.to(DEV), w.to(DEV), p=p, scaling_N=4).cpu().double()
    assert out.shape == (B, 1, n, n)
    assert (out - ref).abs().max() <= 2e-4 * ref.max(), ((out - ref).abs().max().item(), ref.max().item())
    # (with few steps per scale the scheme's output is not yet a probability image — mass 0.16 at scaling_N = 4,
    #  0.79 at the default 10 in the dense oracle as well; only agreement with the restatement is asserted)


@pytest.mark.parametrize("backward_iterations", [0, 3])
def test_images_barycenter_gradients(backward_iterations):
    """d/d(weights) and d/d(measures) of <barycenter, test image>: closed-form softmin_grid backward (two grid
    softmins) against plain autograd through the dense oracle."""
    from geomloss_b200 import ImagesBarycenter
    from oracle import geomloss_oracle as O

    n, K, B = 16, 3, 1
    imgs, w = _bary_inputs(n, K, B, seed=5)
    imgs = imgs + 1e-3  # strictly positive: log_dens is differentiable everywhere
    imgs = imgs / imgs.sum((2, 3), keepdim=True)
    g = torch.Generator().manual_seed(1)
    probe = torch.rand(B, 1, n, n, generator=g)
    ir, wr = imgs.double().requires_grad_(True), w.double().requires_grad_(True)
    ref = (O.images_barycenter(ir, wr, scaling_N=3, backward_iterations=backward_iterations) * probe.double()).sum()
    ig, wg = imgs.to(DEV).requires_grad_(True), w.to(DEV).requires_grad_(True)
    val = (ImagesBarycenter(ig, wg, scaling_N=3, backward_iterations=backward_iterations) * probe.to(DEV)).sum()
    assert abs(val.item() - ref.item()) <= 2e-4 * abs(ref.item())
    r_w, r_i = torch.autograd.grad(ref, [wr, ir], allow_unused=True)
    g_w, g_i = torch.autograd.grad(val, [wg, ig], allow_unused=True)
    assert (g_w.cpu().double() - r_w).abs().max() <= 2e-3 * r_w.abs().max()
    if backward_iterations == 0:
        assert (g_i.cpu().double() - r_i).abs().max() <= 5e-3 * r_i.abs().max()
    else:
        # measures enter the extra iterations only through constants computed without autograd (as in the reference)
        assert (r_i is None or float(r_i.abs().max()) == 0.0) and (g_i is None or float(g_i.abs().max()) == 0.0)


# ------------------------------------------------------------------------------------------------
# mid / full size against an INDEPENDENT fp64 evaluation on the device (plain torch ops, row-chunked)
# ------------------------------------------------------------------------------------------------
def _chunked_fp64_softmin(p, rows=4096):
    """softmin(eps, (x, y), h) for the oracle's sinkhorn_loop: plain torch fp64 on the device, row-chunked so that it
    reaches N = M = 1e5 (8 GB of temporaries would be needed otherwise).  Independent of libb200ot.so."""

    from torch.utils.checkpoint import checkpoint

    def softmin(eps, C, h):
        x, y = C  # (1, N, D), (1, M, D)
        yy = (y[0] * y[0]).sum(-1)

        def block(xs):
            d2 = ((xs * xs).sum(-1)[:, None] - 2.0 * xs @ y[0].t() + yy[None, :]).clamp_min(0.0)
            cost = d2 / 2 if p == 2 else d2.clamp_min(1e-8).sqrt()
            return -eps * torch.logsumexp(h.reshape(1, -1) - cost / eps, dim=1)

        out = []
        for s in range(0, x.shape[1], rows):
            xs = x[0, s:s + rows]
            # (the gradient-carrying final step: recompute each block in backward instead of keeping its
            #  rows x M fp64 temporaries — 25 blocks of 3 GB each at N = M = 1e5)
            out.append(checkpoint(block, xs, use_reentrant=False) if xs.requires_grad else block(xs))
        return torch.cat(out)[None]

    return softmin


def test_full_sinkhorn_loop_n1e5_vs_chunked_fp64():
    """SURVEY.md 7.1 step 3: the WHOLE eps-scaling loop (10 temperatures, 48 softmins, tiled TMA kernels) at
    N = M = 1e5 against the oracle's sinkhorn_loop driven by a chunked fp64 softmin — value, potentials and the
    gradient w.r.t. x."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(7)
    n = m = 100_000
    x = torch.rand(n, 3, generator=g)
    y = torch.rand(m, 3, generator=g) * 0.9 + 0.1
    kw = dict(p=2, blur=0.02, scaling=0.5)
    xd, yd = x.to(DEV), y.to(DEV)
    xg = xd.clone().requires_grad_(True)
    val = SamplesLoss("sinkhorn", backend="online", **kw)(xg, yd)
    (gx,) = torch.autograd.grad(val, xg)
    F, G = SamplesLoss("sinkhorn", backend="online", potentials=True, **kw)(xd, yd)

    x64, y64 = xd.double()[None], yd.double()[None]
    x64r = x64.clone().requires_grad_(True)
    a = torch.full((1, n), 1.0 / n, dtype=torch.float64, device=DEV)
    b = torch.full((1, m), 1.0 / m, dtype=torch.float64, device=DEV)
    diameter, eps, eps_list, rho = O.scaling_parameters(x64, y64, 2, kw["blur"], None, None, kw["scaling"])
    sm = _chunked_fp64_softmin(2)
    f_aa, g_bb, g_ab, f_ba = O.sinkhorn_loop(sm, O.log_weights(a), O.log_weights(b), (x64r, x64.detach()),
                                             (y64, y64.detach()), (x64r, y64.detach()), (y64, x64.detach()), eps_list,
                                             rho, debias=True)
    ref = O.sinkhorn_value(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba)[0]
    (rgx,) = torch.autograd.grad(ref, x64r)
    assert abs(val.item() - ref.item()) <= 1e-4 * abs(ref.item()), (val.item(), ref.item())
    assert (F[0].double() - (f_ba - f_aa)[0].detach()).abs().max().item() < 1e-5
    assert (G[0].double() - (g_ab - g_bb)[0].detach()).abs().max().item() < 1e-5
    assert (gx.double() - rgx[0]).abs().max().item() <= 5e-4 * rgx.abs().max().item()


def test_grid_softmin_256_cubed_sampled_lines():
    """The 3-D separable grid kernel at BASELINE configs[4]'s side (256: the transposed last-axis path and the
    8-outputs-per-thread tiling at full width) on 8 x 8 sampled output lines vs a separable fp64 evaluation."""
    from geomloss_b200.sinkhorn_images import softmin_grid

    n = 256
    g = torch.Generator().manual_seed(11)
    h = (torch.randn(1, 1, n, n, n, generator=g) * 2.0).to(DEV)
    h[0, 0, :5] = -10000.0  # an empty slab (log_dens floor)
    for p, eps in ((2, (1.0 / n) ** 2), (2, 0.01), (1, 2.0 / n)):
        out = softmin_grid(eps, p, h)
        hh = h[0, 0].double()
        xs = torch.arange(n, device=DEV, dtype=torch.float64) / n
        xs = xs / np.sqrt(2 * eps) if p == 2 else xs / eps
        d = xs[:, None] - xs[None, :]
        k = -(d**2) if p == 2 else -d.abs()
        i0 = torch.randint(0, n, (8,), generator=g).to(DEV)
        i1 = torch.randint(0, n, (8,), generator=g).to(DEV)
        # one first-axis slice at a time: the whole (n, n, n, n) fp64 broadcast is 32 GiB, and logsumexp needs two
        t2 = torch.stack([torch.logsumexp(hh[a][:, None, :] + k[None, :, :], dim=-1) for a in range(n)])
        t1 = torch.logsumexp(t2[:, None, :, :] + k[i1][None, :, :, None], dim=2)
        t0 = torch.logsumexp(t1[None, :, :, :] + k[i0][:, :, None, None], dim=1)
        want = -eps * t0
        got = out[0, 0][i0][:, i1].double()
        assert (got - want).abs().max().item() < 3e-6 * max(1.0, want.abs().max().item()), (p, eps)

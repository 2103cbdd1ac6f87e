"""The tensor-core kernels (8 < D <= 64; csrc/tcconv.cuh tc_reduce_kernel<0/1>, csrc/tcbwd.cuh tc_bwd_kernel<2/3>) in
the regimes they are built for and the other tensor-core tests do not reach: many column tiles streamed through one CTA
(the ring of kTcMaxStage = 4 slots wraps, the row sums and the lazy max carry across tiles), the default plan of a large
row count, the tile and padding edges, and M = 65536 columns, where the softmax weights P ~ 1/M of the row gradients
fall below fp16's normal range unless they are scaled (kTcPScale, csrc/common.cuh).

Every result is checked against the fp64 oracle (oracle/geomloss_oracle.py, evaluated in float64 on the device) with
the bars of test_gpu_parity.py / test_gpu_tc_variants.py for the same operators.  $B200OT_FORCE_SPLITS (csrc/plan.cuh)
forces the number of column splits; test_cabi_symbols.py shows that it reaches the tensor-core plan."""
import numpy as np
import pytest
import torch

from test_gpu_tc_variants import _exponent_slack, env

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LN2 = np.log(2.0)


def _clouds(n, m, d, seed, atoms=None):
    """Unit-cube clouds on the device; `atoms`: y (and h) repeat `atoms` distinct points, M / atoms copies each."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    k = m if atoms is None else atoms
    y = torch.rand(k, d, generator=g, dtype=torch.float64)
    h = torch.randn(k, generator=g, dtype=torch.float64) - np.log(m)
    w = torch.rand(k, generator=g, dtype=torch.float64) / m
    go = torch.randn(n, generator=g, dtype=torch.float64)
    if atoms is not None:
        rep = torch.arange(m) % atoms
        y, h, w = y[rep], h[rep], w[rep]
    return tuple(t.to(DEV) for t in (x, y, h, w, go))


def _f32(*ts):
    return tuple(t.float().contiguous() for t in ts)


def _gauss_ref(x, y, w, blur, go):
    """fp64 oracle of out = K w and of the row gradient of <go, K w>, with the natural scales of both (their terms
    cancel when weights have mixed signs): sum_j |w_j| k_ij and max_i |go_i| sum_j |w_j| k_ij |y_j - x_i| / blur^2."""
    from oracle import geomloss_oracle as O

    xr = x.detach().clone().requires_grad_(True)
    km = O.kernel_matrix("gaussian", xr, y, blur)
    val = km @ w
    (g,) = torch.autograd.grad(val, xr, go)
    absval = km.detach() @ w.abs()
    gscale = (absval * go.abs()).max().item() * np.sqrt(x.shape[1]) / blur**2
    return val.detach(), g, absval, gscale


def _assert_close(got, ref, atol, what):
    got, ref = got.detach().double().cpu().numpy(), ref.detach().double().cpu().numpy()
    atol = np.asarray(atol.detach().cpu().numpy() if torch.is_tensor(atol) else atol)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    err = np.abs(got - ref)
    bad = err > atol
    assert not bad.any(), (f"{what}: {bad.sum()} of {bad.size} entries off, worst {err.max():.3e} "
                           f"(bar {np.broadcast_to(atol, err.shape).flat[np.argmax(err)]:.3e})")


def _softmin_checks(eps, x, y, h, go, what, rows=None):
    """Forward softmin (bar of test_softmin_tensor_core_path) and its row gradient from the forward's lse2 (bar of
    test_row_gradient_kernel_at_padded_dimensions); rows: the sampled row indices checked against the oracle (default:
    all)."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    xd, yd, hd, god = _f32(x, y, h, go)
    center = ops.default_center(xd, yd)
    out, lse2 = ops.softmin_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
    gx = ops.softmin_grad_rows(eps, xd, yd, hd, None, 0.0, lse2, god, p=2, center=center)
    rows = slice(None) if rows is None else rows
    ref = O.softmin_points(eps, x[rows], y, h, p=2)
    _assert_close(out[rows], ref, 5e-6 * max(1.0, ref.abs().max().item()), f"{what} softmin eps={eps}")
    gref = O.softmin_grad_rows(eps, x[rows], y, h, go[rows], p=2)
    _assert_close(gx[rows], gref, 5e-5 * max(1.0, gref.abs().max().item()), f"{what} softmin gradient eps={eps}")


def _gauss_checks(blur, x, y, w, go, what, rows=None, tol_grad=5e-5):
    """Gaussian convolution (rtol 2e-5 + the exponent's rounding slack, of sum |w| k as weights may have mixed signs:
    test_value_and_unit_gradient_in_one_pass) and its row gradient (5e-5 of the largest entry + 1e-5 of the natural
    scale, test_row_gradient_kernel_at_padded_dimensions)."""
    from geomloss_b200 import ops

    xd, yd, wd, god = _f32(x, y, w, go)
    center = ops.default_center(xd, yd)
    out = ops.kernel_conv_raw("gaussian", xd, yd, wd, blur, center=center)
    gx = ops.kernel_conv_grad_rows("gaussian", xd, yd, wd, blur, god, center=center)
    rows = slice(None) if rows is None else rows
    ref, gref, absval, gscale = _gauss_ref(x[rows], y, w, blur, go[rows])
    slack = LN2 * _exponent_slack(x.shape[1], np.sqrt(np.log2(np.e)) / blur)
    _assert_close(out[rows], ref, (2e-5 + slack) * absval + 1e-30, f"{what} gaussian blur={blur}")
    _assert_close(gx[rows], gref, tol_grad * gref.abs().max().item() + 1e-5 * gscale, f"{what} gaussian gradient")


def _one_pass_checks(blur, x, y, w, what, self_term=False):
    """b200ot_kernel_conv_fwd_bwd_x: value and unit row gradient from one pass, bars of
    test_value_and_unit_gradient_in_one_pass (self_term: rows and columns are the same buffer)."""
    from geomloss_b200 import ops

    xd, yd, wd = _f32(x, y, w)
    if self_term:
        yd = xd
    center = ops.default_center(xd, yd)
    out, gunit = ops.kernel_conv_value_and_grad_rows("gaussian", xd, yd, wd, blur, center=center)
    ref, gref, absval, gscale = _gauss_ref(x, x if self_term else y, w, blur, torch.ones_like(x[:, 0]))
    slack = LN2 * _exponent_slack(x.shape[1], np.sqrt(np.log2(np.e)) / blur)
    _assert_close(out, ref, (2e-5 + slack) * absval + 1e-30, f"{what} one-pass value")
    _assert_close(gunit, gref, 5e-5 * gref.abs().max().item() + (2e-5 + slack) * gscale, f"{what} one-pass gradient")


# ------------------------------------------------------------------------------------------------
# 1. many column tiles per CTA
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("d", [9, 17, 48, 64])
def test_many_column_tiles_per_cta(d, splits):
    """M = 128 t - 37 columns with t = 5, 9, 13 tiles, forced into 1 split (one CTA streams all t tiles: the 4-slot
    ring wraps 1-3 times, the producer waits on empty_b and the mbarrier phases flip on reuse) or 3 splits (the last
    one ragged: 2+2+1, 3+3+3, 5+5+3 tiles).  All four tensor-core operators, for row counts that leave one warpgroup
    idle (1), fill one row tile but one row (127), spill one row into a second tile (129) or fill three (300); plus
    the one-pass value + gradient of the self term (rows = columns, same buffer), whose diagonal is met in one tile of
    each row tile."""
    with env(B200OT_FORCE_SPLITS=splits):
        for t in (5, 9, 13):
            m = 128 * t - 37
            for n in (1, 127, 129, 300):
                x, y, h, w, go = _clouds(n, m, d, seed=1000 * d + 10 * t + n)
                what = f"D={d} splits={splits} N={n} M={m}"
                _softmin_checks(0.3, x, y, h, go, what)
                _gauss_checks(0.7, x, y, w, go, what)
            _one_pass_checks(0.7, y, y, w, f"D={d} splits={splits} self term N=M={m}", self_term=True)


# ------------------------------------------------------------------------------------------------
# 2. the lazy max of the softmin across tiles
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("pattern", ["rising", "falling", "late-overflow"])
def test_lazy_max_across_column_tiles(pattern, d, splits):
    """tc_reduce_kernel<1> keeps a running (m, s) per row and rebases only when a tile's sum against the stale max
    leaves 2^64 (or overflows).  The potential is built tile by tile (eps = 4: the cost varies by < 12 in log2 within a
    tile of these clouds, so the offsets set the order):
      rising        each tile's best term beats the previous tile's by 76..97 in log2 (> 64: the guard, not an
                    overflow, triggers the rebase); the first tile has zero mass only;
      falling       the first tile dominates and every later tile underflows completely (< -64 in log2);
      late-overflow tile 6 of 9 exceeds the running max by more than 128 in log2: ex2 overflows to inf.
    Scattered zero-mass columns (log_weights gives -1e5), the h_b / h_scale_b fold and the fused epilogue
    out = alpha_old * out_old + beta * softmin are exercised in the same launches; the row gradient is taken from the
    lse2 of that forward pass."""
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn import log_weights
    from oracle import geomloss_oracle as O

    n, eps = 300, 4.0
    m = 128 * 9 - 37
    g = torch.Generator().manual_seed({"rising": 1, "falling": 2, "late-overflow": 3}[pattern] + 10 * d)
    x = torch.rand(n, d, generator=g, dtype=torch.float64)
    y = torch.rand(m, d, generator=g, dtype=torch.float64)
    tile = torch.arange(m) // 128
    if pattern == "rising":
        off = 60.0 * tile
    elif pattern == "falling":
        off = -60.0 * tile
    else:
        off = torch.where(tile == 6, 150.0, 0.0).double()
    b = torch.rand(m, generator=g, dtype=torch.float64) + 0.1
    b[::7] = 0.0
    if pattern == "rising":
        b[tile == 0] = 0.0
    b = b / b.sum()
    pot = eps * (off + 0.5 * torch.randn(m, generator=g, dtype=torch.float64))
    old = torch.randn(n, generator=g, dtype=torch.float64)
    go = torch.randn(n, generator=g, dtype=torch.float64)
    x, y, b, pot, old, go = (t.to(DEV) for t in (x, y, b, pot, old, go))
    h = O.log_weights(b) + pot / eps
    xd, yd, bd, potd, oldd, god = _f32(x, y, b, pot, old, go)
    center = ops.default_center(xd, yd)
    with env(B200OT_FORCE_SPLITS=splits):
        ha = log_weights(bd)
        out, lse2 = ops.softmin_raw(eps, xd, yd, ha, potd, 1.0 / eps, p=2, center=center, out_old=oldd,
                                    alpha_old=0.5, beta=0.4, want_lse2=True)
        gx = ops.softmin_grad_rows(eps, xd, yd, ha, potd, 1.0 / eps, lse2, god, p=2, center=center)
    ref = O.softmin_points(eps, x, y, h, p=2).to(DEV)
    _assert_close(out, 0.5 * old + 0.4 * ref, 5e-6 * max(1.0, ref.abs().max().item()), f"{pattern} softmin")
    gref = O.softmin_grad_rows(eps, x, y, h, go, p=2)
    _assert_close(gx, gref, 5e-5 * max(1.0, gref.abs().max().item()), f"{pattern} softmin gradient")


# ------------------------------------------------------------------------------------------------
# 3. the default plan of a large row count
# ------------------------------------------------------------------------------------------------
def test_default_plan_with_one_column_split(monkeypatch):
    """N = 4 * SMs * 128 + 37 rows: make_tc_plan asks for ceil(4 SMs / (4 SMs + 1)) = 1 split, so without any hook
    every CTA streams all 10 column tiles of M = 1189 (D = 64).  ~2k sampled rows are checked, among them the first
    and last row of 200 row tiles and the last row of the ragged last tile."""
    from geomloss_b200 import _lib

    monkeypatch.delenv("B200OT_FORCE_SPLITS", raising=False)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, m, d = 4 * sms * 128 + 37, 1189, 64
    L = _lib.lib()
    default = L.b200ot_softmin_scratch_bytes(n, m, d)
    with env(B200OT_FORCE_SPLITS=1):
        assert L.b200ot_softmin_scratch_bytes(n, m, d) == default  # the default plan IS one split
    x, y, h, w, go = _clouds(n, m, d, seed=77)
    g = torch.Generator().manual_seed(78)
    tiles = torch.randperm(-(-n // 128), generator=g)[:200]
    rows = torch.cat([tiles * 128, tiles * 128 + 127, torch.tensor([0, n - 1]),
                      torch.randint(0, n, (1600,), generator=g)])
    rows = torch.unique(rows[rows < n]).to(DEV)
    _softmin_checks(0.3, x, y, h, go, "default plan", rows=rows)
    _gauss_checks(0.7, x, y, w, go, "default plan", rows=rows)


# ------------------------------------------------------------------------------------------------
# 4. tile and padding edges
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [9, 15, 16, 17, 31, 32, 47, 49, 63])
def test_tile_and_padding_edges(d):
    """Dimensions on both sides of every padded dk (16, 32, 48, 64); shapes where only one warpgroup of the 128-row
    tile has live rows (N <= 64), or one row of a second tile, or a single column; gaussian weights of both signs
    with zeros among them, and all-zero weights (max|w| = 0: the outputs must be exact zeros, not NaN)."""
    from geomloss_b200 import ops

    for n, m in ((1, 1), (1, 129), (129, 1), (64, 200), (65, 128)):
        x, y, h, _, go = _clouds(n, m, d, seed=31 * d + n + 7 * m)
        g = torch.Generator().manual_seed(d + n + m)
        w = (torch.randn(m, generator=g, dtype=torch.float64) / m).to(DEV)
        w[::3] = 0.0
        what = f"D={d} N={n} M={m}"
        _softmin_checks(0.3, x, y, h, go, what)
        _gauss_checks(0.7, x, y, w, go, what + " signed weights")
        _one_pass_checks(0.7, x, y, w, what + " signed weights")
        xd, yd, god = _f32(x, y, go)
        zero = torch.zeros(m, device=DEV)
        center = ops.default_center(xd, yd)
        out = ops.kernel_conv_raw("gaussian", xd, yd, zero, 0.7, center=center)
        gx = ops.kernel_conv_grad_rows("gaussian", xd, yd, zero, 0.7, god, center=center)
        val, gunit = ops.kernel_conv_value_and_grad_rows("gaussian", xd, yd, zero, 0.7, center=center)
        for name, t in (("conv", out), ("gradient", gx), ("value", val), ("unit gradient", gunit)):
            assert bool((t == 0).all()), f"{what} zero weights: {name} {t.flatten()[:4].tolist()}"


# ------------------------------------------------------------------------------------------------
# 5. large M: P below fp16's normal range
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [16, 64])
@pytest.mark.parametrize("cloud", ["distinct", "atoms"])
def test_softmin_row_gradient_at_large_m(cloud, d):
    """N = 256 rows against M = 65536 columns: the softmax weights are ~1/M = 1.5e-5, below fp16's smallest normal
    number (6.1e-5), where they would sit on the fixed 6e-8 subnormal grid if tc_bwd_kernel fed them to GEMM 2
    unscaled.  With 128 atoms x 512 copies the rounding repeats identically for every copy: a bias, not noise."""
    n, m = 256, 65536
    x, y, h, _, go = _clouds(n, m, d, seed=5 * d + (1 if cloud == "atoms" else 0),
                             atoms=128 if cloud == "atoms" else None)
    for eps in (2.0, 0.3):
        _softmin_checks(eps, x, y, h, go, f"{cloud} D={d}")


@pytest.mark.parametrize("cloud", ["distinct", "atoms"])
def test_gaussian_row_gradient_and_value_at_large_m(cloud):
    """D = 64, blur = .7, M = 65536: kernel values exp(-|x - y|^2 / (2 blur^2)) ~ 1e-7..1e-3 times weights
    normalised to max|w| put P far into fp16's subnormal range unless scaled.  Two-pass gradient and one-pass
    value + unit gradient."""
    n, m, d = 256, 65536, 64
    x, y, _, w, go = _clouds(n, m, d, seed=11 + (1 if cloud == "atoms" else 0), atoms=128 if cloud == "atoms" else None)
    _gauss_checks(0.7, x, y, w, go, f"{cloud} D=64")
    _one_pass_checks(0.7, x, y, w, f"{cloud} D=64")


@pytest.mark.parametrize("d", [16, 64])
def test_softmin_bwd_sums_at_large_m(d):
    """b200ot_softmin_bwd_sums, the only entry that returns the raw row sums (the multi-GPU engine adds them over the
    column shards), through the single-rank stage of distributed.py: sums[:, 0] = sum_j P_ij ~ 1 and
    sums[:, 1 + k] = sum_j P_ij Y_jk with Y = sqrt(log2(e) / eps) (y - center), against fp64 sums of
    P_ij = 2^(S_ij - lse2_i) over the lse2 the kernel was given.  Any scale the kernel applies to P must be undone."""
    from geomloss_b200 import ops
    from geomloss_b200.distributed import CudaStages

    n, m, eps = 256, 65536, 2.0
    for cloud, atoms in (("distinct", None), ("atoms", 128)):
        x, y, h, _, _ = _clouds(n, m, d, seed=50 + d + (atoms or 0), atoms=atoms)
        xd, yd, hd = _f32(x, y, h)
        center = ops.default_center(xd, yd)
        _, lse2 = ops.softmin_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
        sums = CudaStages().softmin_bwd_shard(eps, xd, yd, hd, None, 0.0, 2, center, lse2)
        scale = np.sqrt(np.log2(np.e) / eps)
        X, Y = scale * (x - center.double()), scale * (y - center.double())
        S = np.log2(np.e) * h[None, :] - 0.5 * ((X * X).sum(1)[:, None] - 2 * X @ Y.T + (Y * Y).sum(1)[None, :])
        P = torch.exp2(S - lse2.double()[:, None])
        ref = torch.cat([P.sum(1, keepdim=True), P @ Y], dim=1)
        what = f"{cloud} D={d}"
        _assert_close(sums[:, 0], torch.ones(n, device=DEV, dtype=torch.float64), 1e-4, f"{what} sum of P")
        _assert_close(sums, ref, 5e-5 * max(1.0, ref.abs().max().item()), f"{what} raw sums")

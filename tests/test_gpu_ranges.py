"""The CUDA-core block-sparse and batched reductions (D <= 8, ranges.BIG / ranges.SMALL) and the column-shard stages of
distributed.CudaStages, against fp64 references of the same operators.

The references are built from the cluster keep matrix and the cluster sizes, never from the descriptors of
ranges.build_problem, so that a wrong segment or piece fails as well as a wrong kernel:

  A. softmin values (b200ot_softmin_pack_gather + b200ot_softmin_partial_ranges + b200ot_softmin_finalize), p = 2, 1
     and 1 | P_UNCLAMPED, three temperatures, a cloud translated by +50, zero-weight columns, the fused epilogue;
  B. softmin row gradients (b200ot_softmin_bwd_partial_ranges + b200ot_softmin_bwd_finalize), also on a self problem
     whose coincident pairs meet the p = 1 clamp;
  C. kernel products and their x, y and w gradients (b200ot_kernel_conv_pack_gather, _partial_ranges forward and
     backward, _finalize, _bwd_finalize), three kernels in both conventions, cross and self problems;
  D. batched (block-diagonal) problems element by element, element independence, and batched SamplesLoss values and
     gradients on the ranges path;
  E. column shards merged on one GPU: dense shards (b200ot_softmin_pack / _partial / _merge, b200ot_softmin_finalize
     with n_part > 1, b200ot_softmin_bwd_sums), ranges shards built with rank / world, kernel product shards;
  F. negative controls: a reference with one kept block flipped, or a merge without one rank, misses the bar by 10x.

Row clusters of 1 ... 513 points and column clusters of 1 ... 1025 points reach idle warps, slivers and multi-segment
clusters (128 / 512 rows per segment), padding slots and pieces at and just past each cap (256 / 1024 columns).  One
row cluster keeps nothing, one keeps everything (a long run cut into several pieces), the rest is random.  Each row
cluster sits on its LAST kept column cluster, so at small eps the max pre-pass (the first 256 column pairs) picks a
stale max and the rebase path runs.

Bars are those the dense CUDA-core operators meet in test_gpu_parity.py (the ranges kernels do the same arithmetic);
the p = 1, laplacian and energy row gradients add, row by row, the fp32 rounding bound of their pair directions
(fp64_refs.direction_slack), which pairs a few ulps apart reach at D = 1 in the unclamped convention.  Every check records its error-to-bar ratio; the largest per section is printed when the module ends.
"""
import functools
import math

import pytest
import torch

from fp64_refs import check, conv64, mid, softmin64
from oracle import geomloss_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

ROW_SIZES = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 511, 512, 513]
COL_SIZES = [1, 15, 16, 17, 255, 256, 257, 1023, 1024, 1025]
EMPTY_ROW, FULL_ROW = 9, 12  # the 129-row cluster keeps nothing, the 513-row cluster keeps every column cluster
CONVS = ("p2", "p1", "p1u")  # p = 2; p = 1 with the clamp of the tensorized cost; p = 1 | P_UNCLAMPED (pykeops)
KINDS = ("gaussian", "laplacian", "energy")
GRID = [(d, v) for d in range(1, 9) for v in ("BIG", "SMALL")]
GRID_IDS = [f"D{d}-{v}" for d, v in GRID]

# bars of the dense CUDA-core operators (test_gpu_parity.py)
SOFTMIN_BAR = 3e-6  # test_softmin_vs_oracle_shapes
GRAD_BAR = 2e-5  # test_softmin_gradient_vs_oracle, test_row_reductions_last_tile_lengths
CONV_REL, CONV_W = 5e-6, 2e-7  # test_kernel_conv_vs_oracle
CONV_GRAD_BAR = 3e-5  # test_kernel_conv_gradients_vs_autograd

RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    yield
    for sec in sorted(RATIOS):
        what, r = RATIOS[sec]
        print(f"\n[ranges] section {sec}: largest error / bar = {r:.3g} ({what})")


def _pv(conv):
    from geomloss_b200 import ops

    return {"p2": 2, "p1": 1, "p1u": 1 | ops.P_UNCLAMPED}[conv]


def _check(sec, what, got, ref, bar):
    check(RATIOS, sec, what, got, ref, bar)


def _softmin_bar(ref):
    return SOFTMIN_BAR * max(1.0, ref.abs().max().item())


def _conv_bar(ref, w):
    return CONV_REL * max(1e-3, ref.abs().max().item()) + CONV_W * w.abs().sum().item()


def _grad_bar(ref, c):
    return c * max(1.0, ref.abs().max().item())


# ------------------------------------------------------------------------------------------------------
# problems
# ------------------------------------------------------------------------------------------------------
def _expand(keep, rc, cc):
    """Point-level mask of a cluster keep matrix (the blocks of rows x columns it keeps)."""
    return keep[torch.repeat_interleave(torch.arange(len(rc)), rc)][:, torch.repeat_interleave(torch.arange(len(cc)), cc)]


@functools.lru_cache(maxsize=None)
def _clusters(D):
    """Clouds of label-sorted clusters on the unit cube, the keep matrix and the per-column / per-row vectors."""
    g = torch.Generator().manual_seed(1000 + D)
    rc, cc = torch.tensor(ROW_SIZES), torch.tensor(COL_SIZES)
    R, C = len(rc), len(cc)
    keep = torch.rand(R, C, generator=g) < 0.4
    for r in range(R):
        if not keep[r].any():
            keep[r, int(torch.randint(C, (1,), generator=g))] = True
    keep[EMPTY_ROW] = False
    keep[FULL_ROW] = True
    ccen = torch.rand(C, D, generator=g) * 0.8
    # every row cluster on its last kept column cluster: the nearest columns come late in column order
    last = [int(keep[r].nonzero().max()) if keep[r].any() else 0 for r in range(R)]
    rcen = ccen[torch.tensor(last)]
    x = rcen[torch.repeat_interleave(torch.arange(R), rc)] + 0.2 * torch.rand(int(rc.sum()), D, generator=g)
    y = ccen[torch.repeat_interleave(torch.arange(C), cc)] + 0.2 * torch.rand(int(cc.sum()), D, generator=g)
    M, N = y.shape[0], x.shape[0]
    b = torch.rand(M, generator=g) + 0.5
    h_a = (b / b.sum()).log()
    h_a[3::7] = -1e5  # zero-weight columns (log_weights of a zero mass)
    pot = 0.2 * torch.rand(M, generator=g)
    old, go = torch.rand(N, generator=g), torch.randn(N, generator=g)
    w = torch.randn(M, generator=g)
    pairs = _expand(keep, rc, cc)
    return dict(x=x, y=y, rc=rc, cc=cc, keep=keep, pairs=pairs, live=pairs.any(1), h_a=h_a, pot=pot, old=old, go=go, w=w)


@functools.lru_cache(maxsize=None)
def _self_problem(D):
    """x against a copy of itself, diagonal blocks kept: coincident pairs in every kept diagonal block."""
    P = _clusters(D)
    g = torch.Generator().manual_seed(2000 + D)
    R = len(ROW_SIZES)
    keep = (torch.rand(R, R, generator=g) < 0.3) | torch.eye(R, dtype=torch.bool)
    keep[EMPTY_ROW] = False
    N = P["x"].shape[0]
    h_a = torch.randn(N, generator=g) * 0.5 - math.log(N)
    pairs = _expand(keep, P["rc"], P["rc"])
    return dict(x=P["x"], y=P["x"].clone(), rc=P["rc"], cc=P["rc"], keep=keep, pairs=pairs, live=pairs.any(1), h_a=h_a,
                pot=0.2 * torch.rand(N, generator=g), go=torch.randn(N, generator=g), w=torch.randn(N, generator=g))


def _problem(P, variant, transposed=False):
    from geomloss_b200 import ranges

    keep = P["keep"]
    rc, cc = (P["cc"], P["rc"]) if transposed else (P["rc"], P["cc"])
    k = keep.t().contiguous() if transposed else keep
    return ranges.build_problem(k.to(DEV), rc.to(DEV), ranges.ColumnLayout(cc.to(DEV)),
                                variant=getattr(ranges, variant))


# ------------------------------------------------------------------------------------------------------
# fp64 references (fp64_refs.py)
# ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _ref_softmin(D, conv, eps, shifted=False, self_problem=False, grad=False):
    P = _self_problem(D) if self_problem else _clusters(D)
    x, y = P["x"], P["y"]
    if shifted:  # the fp32 translated clouds, translated back exactly in fp64
        x, y = (x + 50.0).double() - 50.0, (y + 50.0).double() - 50.0
    h = P["h_a"].double() + P["pot"].double() / eps
    return softmin64(eps, x, y, h, P["pairs"], conv, go=P["go"] if grad else None)


@functools.lru_cache(maxsize=None)
def _ref_conv(D, kind, unclamped, blur, self_problem=False):
    P = _self_problem(D) if self_problem else _clusters(D)
    return conv64(kind, unclamped, P["x"], P["y"], P["w"], blur, P["pairs"], P["go"], mid(P["x"], P["y"]))


# ------------------------------------------------------------------------------------------------------
# A. softmin values
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,variant", GRID, ids=GRID_IDS)
def test_softmin_values(D, variant):
    from geomloss_b200 import ops, ranges

    P = _clusters(D)
    prob = _problem(P, variant)
    live = P["live"]
    assert not bool(live.all()) and bool(live.any())
    ha, pot, old = (P[k].to(DEV) for k in ("h_a", "pot", "old"))
    for conv in CONVS:
        for eps in (0.5, 0.02, 5e-4):
            for shifted in ((False, True) if eps == 0.02 else (False,)):
                what = f"D={D} {variant} {conv} eps={eps}{' +50' if shifted else ''}"
                if shifted:
                    xd, yd = (P["x"] + 50.0).to(DEV), (P["y"] + 50.0).to(DEV)
                    center = ops.default_center(xd, yd)
                else:
                    xd, yd, center = P["x"].to(DEV), P["y"].to(DEV), None
                ref = _ref_softmin(D, conv, eps, shifted)[0]
                out, lse2 = ranges.softmin_ranges_raw(eps, xd, yd, ha, pot, 1.0 / eps, prob, p=_pv(conv), center=center,
                                                      want_lse2=True)
                _check("A", what, out[live.to(DEV)], ref[live], _softmin_bar(ref[live]))
                # rows whose cluster keeps no column: -eps log 0 = +inf, as the tensor-core block path gives
                dead = out[~live.to(DEV)]
                assert bool(torch.isinf(dead).all() and (dead > 0).all()), what
                o, l2 = out[live.to(DEV)].double(), lse2[live.to(DEV)].double()
                assert (-eps * math.log(2.0) * l2 - o).abs().max().item() <= 1e-6 * o.abs().max().item() + 1e-7, what
                fused, _ = ranges.softmin_ranges_raw(eps, xd, yd, ha, pot, 1.0 / eps, prob, p=_pv(conv),
                                                     center=center, out_old=old, alpha_old=0.5, beta=0.7)
                want = 0.5 * P["old"].double() + 0.7 * ref
                _check("A", what + " fused epilogue", fused[live.to(DEV)], want[live], _softmin_bar(want[live]))
                assert bool(torch.isinf(fused[~live.to(DEV)]).all()), what


# ------------------------------------------------------------------------------------------------------
# B. softmin row gradients
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,variant", GRID, ids=GRID_IDS)
def test_softmin_row_gradients(D, variant):
    from geomloss_b200 import ranges

    for self_problem in (False, True):
        P = _self_problem(D) if self_problem else _clusters(D)
        prob = _problem(P, variant)
        live = P["live"]
        xd, yd, ha, pot, go = (P[k].to(DEV) for k in ("x", "y", "h_a", "pot", "go"))
        for conv in CONVS:
            for eps in (0.5, 0.02):
                what = f"D={D} {variant} {conv} eps={eps}{' self' if self_problem else ''}"
                _, gref, allow = _ref_softmin(D, conv, eps, self_problem=self_problem, grad=True)
                xg = xd.clone().requires_grad_(True)
                val = ranges.softmin_ranges(eps, xg, yd, ha, pot, 1.0 / eps, prob, p=_pv(conv), scale_out=0.7)
                (gx,) = torch.autograd.grad(val, xg, go)
                want = 0.7 * gref[live]
                _check("B", what, gx[live.to(DEV)], want, _grad_bar(want, GRAD_BAR) + 0.7 * allow[live])


# ------------------------------------------------------------------------------------------------------
# C. kernel products and their gradients
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,variant", GRID, ids=GRID_IDS)
def test_kernel_products_and_gradients(D, variant):
    from geomloss_b200 import ops, ranges

    for self_problem in (False, True):
        P = _self_problem(D) if self_problem else _clusters(D)
        prob, prob_t = _problem(P, variant), _problem(P, variant, transposed=True)
        live, live_t = P["live"], P["pairs"].any(0)
        x, y, w, go = (P[k].to(DEV) for k in ("x", "y", "w", "go"))
        center = ops.default_center(x, y)
        for kind in KINDS:
            for unclamped in (False, True):
                for blur in ((0.05, 0.5) if kind != "energy" else (0.5,)):
                    what = f"D={D} {variant} {kind}{' unclamped' if unclamped else ''} blur={blur}" + (
                        " self" if self_problem else "")
                    kid = ops.KERNEL_KINDS[kind] | (ops.KERNEL_UNCLAMPED if unclamped else 0)
                    ref, rx, ry, rw, ax, ay = _ref_conv(D, kind, unclamped, blur, self_problem)
                    xg, yg, wg = (t.clone().requires_grad_(True) for t in (x, y, w))
                    out = ranges.kernel_conv_ranges(kid, xg, yg, wg, blur, prob, prob_t, center=center)
                    gx, gy, gw = torch.autograd.grad(out, [xg, yg, wg], go)
                    _check("C", what + " value", out[live.to(DEV)], ref[live], _conv_bar(ref[live], P["w"]))
                    _check("C", what + " grad x", gx[live.to(DEV)], rx[live], _grad_bar(rx[live], CONV_GRAD_BAR) + ax[live])
                    _check("C", what + " grad y", gy[live_t.to(DEV)], ry[live_t], _grad_bar(ry[live_t], CONV_GRAD_BAR)
                           + ay[live_t])
                    _check("C", what + " grad w", gw[live_t.to(DEV)], rw[live_t], _grad_bar(rw[live_t], CONV_GRAD_BAR))
                    # rows without a kept column: exactly zero, value and gradient
                    assert bool((out[~live.to(DEV)] == 0).all() and (gx[~live.to(DEV)] == 0).all()), what


# ------------------------------------------------------------------------------------------------------
# D. batched problems
# ------------------------------------------------------------------------------------------------------
BATCH = [(B, N, M) for B in (1, 2, 9) for (N, M) in ((1, 1), (31, 17), (700, 450), (2049, 2050))]
BATCH = [(B, N, M, 1 + i % 8) for i, (B, N, M) in enumerate(BATCH)]  # every D in 1 ... 8


@pytest.mark.parametrize("B,N,M,D", BATCH, ids=[f"B{b}-{n}x{m}-D{d}" for b, n, m, d in BATCH])
def test_batched_problems_element_by_element(B, N, M, D):
    from geomloss_b200 import ops, ranges

    g = torch.Generator().manual_seed(B * 10000 + N + D)
    x, y = torch.rand(B, N, D, generator=g), torch.rand(B, M, D, generator=g) * 1.1 - 0.05
    h = torch.randn(B, M, generator=g) * 0.5 - math.log(M)
    w, go = torch.randn(B, M, generator=g), torch.randn(B, N, generator=g)
    xf, yf = x.reshape(B * N, D).to(DEV), y.reshape(B * M, D).to(DEV)
    hf, wf, gof = h.reshape(-1).to(DEV), w.reshape(-1).to(DEV), go.reshape(-1).to(DEV)
    center = ops.default_center(xf, yf)
    prob, prob_t = ranges.batch_problem(B, N, M, DEV), ranges.batch_problem(B, M, N, DEV)
    assert prob.variant == (ranges.BIG if min(N, M) >= 2048 else ranges.SMALL)
    eps, blur = 0.05, 0.2

    def run(ycols):
        res = {}
        for conv in CONVS:
            res[conv] = ranges.softmin_ranges_raw(eps, xf, ycols, hf, None, 0.0, prob, p=_pv(conv), center=center)[0]
        xg = xf.clone().requires_grad_(True)
        (res["grad"],) = torch.autograd.grad(ranges.softmin_ranges(eps, xg, ycols, hf, None, 0.0, prob, p=2,
                                                                    center=center), xg, gof)
        for kind in KINDS:
            res[kind] = ranges.kernel_conv_ranges(ops.KERNEL_KINDS[kind], xf, ycols, wf, blur, prob, prob_t,
                                                  center=center)
        return {k: v.view(B, N, -1) for k, v in res.items()}

    got = run(yf)
    for k in range(B):
        what = f"B={B} N={N} M={M} D={D} element {k}"
        for conv in CONVS:
            ref, gref, _ = softmin64(eps, x[k], y[k], h[k], None, conv, go=go[k] if conv == "p2" else None)
            _check("D", f"{what} {conv}", got[conv][k, :, 0], ref, _softmin_bar(ref))
            if gref is not None:
                _check("D", f"{what} row gradient", got["grad"][k], gref, _grad_bar(gref, GRAD_BAR))
        for kind in KINDS:
            ref = O.kernel_conv_points(kind, x[k].double(), y[k].double(), w[k].double(), blur)
            _check("D", f"{what} {kind}", got[kind][k, :, 0], ref, _conv_bar(ref, w[k]))
    if B > 1:
        # new columns for one element: with the same centre, every other element's output is bit for bit the same
        b0 = B // 2
        y2 = yf.clone().view(B, M, D)
        y2[b0] = torch.rand(M, D, generator=g).to(DEV)
        moved = run(y2.view(B * M, D))
        others = [k for k in range(B) if k != b0]
        for key in got:
            assert torch.equal(got[key][others], moved[key][others]), key
            assert not torch.equal(got[key][b0], moved[key][b0]), key


LOSSES = [dict(loss="sinkhorn", p=2, blur=0.05), dict(loss="sinkhorn", p=1, blur=0.1, reach=0.5),
          dict(loss="gaussian", blur=0.2), dict(loss="laplacian", blur=0.2), dict(loss="energy")]


@pytest.mark.parametrize("D", [2, 5, 8])
def test_batched_samples_loss_on_the_ranges_path(D, monkeypatch):
    """Batches above the small-cloud limit run every softmin / kernel product as one block-diagonal ranges problem:
    values and x, y gradients per element against the fp64 oracle (bars of test_sinkhorn_cases)."""
    from geomloss_b200 import SamplesLoss, sinkhorn_small

    monkeypatch.setattr(sinkhorn_small, "SMALL_MAX", 0)
    B, N, M = 3, 700, 450
    g = torch.Generator().manual_seed(300 + D)
    x, y = torch.rand(B, N, D, generator=g), torch.rand(B, M, D, generator=g)
    a, b = torch.rand(B, N, generator=g) + 0.2, torch.rand(B, M, generator=g) + 0.2
    a, b = a / a.sum(1, keepdim=True), b / b.sum(1, keepdim=True)
    diameter = math.sqrt(D)  # both sides on the same eps-schedule
    for kw in LOSSES:
        kw = dict(kw, diameter=diameter) if kw["loss"] == "sinkhorn" else kw
        what = f"D={D} {kw}"
        xg, yg = x.to(DEV).requires_grad_(True), y.to(DEV).requires_grad_(True)
        vals = SamplesLoss(**kw)(a.to(DEV), xg, b.to(DEV), yg)
        gx, gy = torch.autograd.grad(vals.sum(), [xg, yg])
        xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
        ref = O.samples_loss(a.double(), xr, b.double(), yr, **kw)
        rx, ry = torch.autograd.grad(ref.sum(), [xr, yr])
        assert vals.shape == (B,)
        for k in range(B):
            _check("D", f"{what} value {k}", vals[k], ref[k].detach(), 1e-4 * abs(ref[k].item()) + 1e-7)
            _check("D", f"{what} grad x {k}", gx[k], rx[k], 1e-4 * max(rx[k].abs().max().item(), 1e-3))
            _check("D", f"{what} grad y {k}", gy[k], ry[k], 1e-4 * max(ry[k].abs().max().item(), 1e-3))


# ------------------------------------------------------------------------------------------------------
# E. column shards merged on one GPU
# ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _dense_case(D, M):
    g = torch.Generator().manual_seed(500 + 7 * D + M)
    N = 600
    x, y = torch.rand(N, D, generator=g), torch.rand(M, D, generator=g) * 1.1 - 0.05
    return dict(x=x, y=y, h_a=torch.randn(M, generator=g) * 0.5 - math.log(M), pot=0.2 * torch.rand(M, generator=g),
                old=torch.rand(N, generator=g), go=torch.randn(N, generator=g), w=torch.randn(M, generator=g))


@functools.lru_cache(maxsize=None)
def _ref_dense_softmin(D, M, conv, eps):
    P = _dense_case(D, M)
    return softmin64(eps, P["x"], P["y"], P["h_a"].double() + P["pot"].double() / eps, None, conv, go=P["go"],
                      center=mid(P["x"], P["y"]))


@functools.lru_cache(maxsize=None)
def _ref_dense_conv(D, M, kind, unclamped, blur):
    P = _dense_case(D, M)
    return conv64(kind, unclamped, P["x"], P["y"], P["w"], blur, None, P["go"], mid(P["x"], P["y"]))


def _shard_softmin(st, eps, P, p, center, W, skip=None):
    """Every rank's merged (m, s) partial over its column shard, stacked (ranks without a column: empty_shard)."""
    from geomloss_b200.distributed import shard_bounds

    x, y, ha, pot = (P[k].to(DEV) for k in ("x", "y", "h_a", "pot"))
    M, N = y.shape[0], x.shape[0]
    parts = []
    for r in range(W):
        if r == skip:
            continue
        lo, hi = shard_bounds(M, r, W)
        parts.append(st.softmin_shard(eps, x, y[lo:hi], ha[lo:hi], pot[lo:hi], 1.0 / eps, p, center) if hi > lo
                     else st.empty_shard(N, x.device))
    return torch.stack(parts).contiguous()


@pytest.mark.parametrize("splits", ["default", "1", "3"])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6, 7, 8, 16])
def test_dense_column_shards(D, splits, monkeypatch):
    """One GPU computes every rank's shard in turn: the merged partials (b200ot_softmin_finalize, n_part = W), the
    summed row-gradient sums and the summed kernel products equal the one-problem fp64 results.  At D = 16 the shard
    is the tensor-core softmin's (lse2, 1), held to the bars of the dense tensor-core path
    (test_softmin_tensor_core_path: 5e-6 values, 5e-5 row gradients)."""
    from geomloss_b200 import ops
    from geomloss_b200.distributed import CudaStages, shard_bounds

    if splits != "default":
        monkeypatch.setenv("B200OT_FORCE_SPLITS", splits)
    st = CudaStages()
    vbar, gbar = (5e-6, 5e-5) if D > 8 else (SOFTMIN_BAR, GRAD_BAR)
    eps = 0.05
    for M, worlds in ((2000, (2, 3, 7)), (5, (7,))):
        P = _dense_case(D, M)
        x, y, ha, pot, old, go = (P[k].to(DEV) for k in ("x", "y", "h_a", "pot", "old", "go"))
        center = ops.default_center(x, y)
        for conv in (CONVS if D <= 8 else ("p2",)):
            p = _pv(conv)
            ref, gref, allow = _ref_dense_softmin(D, M, conv, eps)
            want = 0.5 * P["old"].double() + 0.7 * ref
            one, _ = ops.softmin_raw(eps, x, y, ha, pot, 1.0 / eps, p=p, center=center, out_old=old, alpha_old=0.5,
                                     beta=0.7)
            for W in worlds:
                what = f"D={D} M={M} W={W} {conv} splits={splits}"
                parts = _shard_softmin(st, eps, P, p, center, W)
                if M < W:
                    assert any(shard_bounds(M, r, W)[0] == shard_bounds(M, r, W)[1] for r in range(W))
                out, lse2 = st.softmin_finalize(parts, eps, old, 0.5, 0.7, True)
                _check("E", what, out, want, vbar * max(1.0, want.abs().max().item()))
                _check("E", what + " vs one call", out, one, vbar * max(1.0, want.abs().max().item()))
                sums = torch.zeros(x.shape[0], D + 1, device=DEV)
                for r in range(W):
                    lo, hi = shard_bounds(M, r, W)
                    if hi > lo:
                        sums += st.softmin_bwd_shard(eps, x, y[lo:hi], ha[lo:hi], pot[lo:hi], 1.0 / eps, p, center,
                                                     lse2)
                gx = st.softmin_bwd_finalize(sums, eps, x, center, go, p)
                _check("E", what + " row gradient", gx, gref, _grad_bar(gref, gbar) + allow)
                if W == 3:
                    # F: a merge without rank 1 misses the bar by far
                    miss, _ = st.softmin_finalize(_shard_softmin(st, eps, P, p, center, W, skip=1), eps, old, 0.5, 0.7,
                                                  False)
                    err = (miss.double().cpu() - want).abs().max().item()
                    assert err >= 10 * vbar * max(1.0, want.abs().max().item()), (what, err)
        if D > 8:
            continue
        w = P["w"].to(DEV)
        for kind in KINDS:
            for unclamped in (False, True):
                kid = ops.KERNEL_KINDS[kind] | (ops.KERNEL_UNCLAMPED if unclamped else 0)
                ref, rx, _, _, ax, _ = _ref_dense_conv(D, M, kind, unclamped, 0.3)
                for W in worlds:
                    what = f"D={D} M={M} W={W} {kind}{' unclamped' if unclamped else ''} splits={splits}"
                    out = torch.zeros(x.shape[0], device=DEV)
                    gx = torch.zeros_like(x)
                    for r in range(W):
                        lo, hi = shard_bounds(M, r, W)
                        if hi > lo:
                            out += st.conv_shard(kid, x, y[lo:hi], w[lo:hi], 0.3, center)
                            gx += st.conv_grad_shard(kid, x, y[lo:hi], w[lo:hi], 0.3, go, center)
                    _check("E", what + " product", out, ref, _conv_bar(ref, P["w"]))
                    _check("E", what + " row gradient", gx, rx, _grad_bar(rx, CONV_GRAD_BAR) + ax)


@pytest.mark.parametrize("D,variant", [(d, v) for d in (1, 3, 8) for v in ("BIG", "SMALL")],
                         ids=[f"D{d}-{v}" for d in (1, 3, 8) for v in ("BIG", "SMALL")])
def test_ranges_column_shards(D, variant):
    """build_problem(..., rank=r, world=3): each rank reduces its slab of column clusters; the stacked partials merge
    to the masked fp64 softmin (a rank with nothing for a row merges as neutral) and the summed row-gradient sums give
    its row gradient."""
    from geomloss_b200 import ranges

    P = _clusters(D)
    live = P["live"]
    ld = live.to(DEV)
    x, y, ha, pot, old, go = (P[k].to(DEV) for k in ("x", "y", "h_a", "pot", "old", "go"))
    W = 3
    probs = [ranges.build_problem(P["keep"].to(DEV), P["rc"].to(DEV), ranges.ColumnLayout(P["cc"].to(DEV)),
                                  variant=getattr(ranges, variant), rank=r, world=W) for r in range(W)]
    for conv in CONVS:
        p = _pv(conv)
        for eps in (0.5, 0.02):
            what = f"D={D} {variant} {conv} eps={eps} W={W}"
            parts = torch.stack([ranges.softmin_shard_ranges(eps, x, y, ha, pot, 1.0 / eps, pr, p=p) for pr in probs])
            # some live rows have nothing in some rank's slab: their partial is the neutral (s = 0)
            assert bool((parts[:, ld, 1] == 0).any()), what
            out, lse2 = ranges.softmin_finalize(parts, W, eps, old, 0.5, 0.7, True)
            ref, gref, allow = _ref_softmin(D, conv, eps, grad=True)
            want = 0.5 * P["old"].double() + 0.7 * ref
            _check("E", what, out[ld], want[live], _softmin_bar(want[live]))
            assert bool(torch.isinf(out[~ld]).all()), what
            sums = sum(ranges.softmin_bwd_shard_ranges(eps, x, y, ha, pot, 1.0 / eps, pr, lse2, p=p) for pr in probs)
            gx = ranges.softmin_bwd_finalize(sums, eps, x, None, go, p)
            _check("E", what + " row gradient", gx[ld], gref[live], _grad_bar(gref[live], GRAD_BAR) + allow[live])


# ------------------------------------------------------------------------------------------------------
# F. negative controls: one wrong block is far outside the bars
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,variant", [(3, "BIG"), (6, "SMALL")], ids=["D3-BIG", "D6-SMALL"])
def test_one_flipped_block_misses_the_bars(D, variant):
    """The reference of a keep matrix with one kept block dropped — the 15-column cluster of the keep-all row cluster,
    0.4 % of its columns — misses the kernels' results by at least 10x the bar, softmin and kernel product alike."""
    from geomloss_b200 import ops, ranges

    P = _clusters(D)
    prob = _problem(P, variant)
    flipped = P["keep"].clone()
    assert bool(flipped[FULL_ROW, 1])
    flipped[FULL_ROW, 1] = False
    wrong = _expand(flipped, P["rc"], P["cc"])
    live = P["live"]
    x, y, ha, pot, w = (P[k].to(DEV) for k in ("x", "y", "h_a", "pot", "w"))
    eps = 0.5
    out, _ = ranges.softmin_ranges_raw(eps, x, y, ha, pot, 1.0 / eps, prob, p=2)
    h = P["h_a"].double() + P["pot"].double() / eps
    ref = softmin64(eps, P["x"], P["y"], h, P["pairs"], "p2")[0]
    bad = softmin64(eps, P["x"], P["y"], h, wrong, "p2")[0]
    bar = _softmin_bar(ref[live])
    _check("F", f"D={D} {variant} softmin, right keep", out[live.to(DEV)], ref[live], bar)
    assert (out[live.to(DEV)].double().cpu() - bad[live]).abs().max().item() >= 10 * bar
    prob_t = _problem(P, variant, transposed=True)
    conv = ranges.kernel_conv_ranges(0, x, y, w, 0.5, prob, prob_t, center=ops.default_center(x, y))
    ref = _ref_conv(D, "gaussian", False, 0.5)[0]
    bad = conv64("gaussian", False, P["x"], P["y"], P["w"], 0.5, wrong, P["go"], mid(P["x"], P["y"]))[0]
    bar = _conv_bar(ref[live], P["w"])
    _check("F", f"D={D} {variant} gaussian, right keep", conv[live.to(DEV)], ref[live], bar)
    assert (conv[live.to(DEV)].double().cpu() - bad[live]).abs().max().item() >= 10 * bar

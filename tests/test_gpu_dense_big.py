"""The dense CUDA-core reductions of one problem in their big tile shape, against fp64 references of the same operators.

csrc/plan.cuh runs softmin_partial_kernel and rowsum_partial_kernel in the big shape (512 rows per CTA, 1024-column
tiles) whenever N >= 4096 and M >= 4096.  That shape is what large clouds at D <= 8 take for every softmin, softmin row
gradient, kernel product and kernel-product gradient, and its CTA layouts differ per D and per convention:
  softmin (b200ot_softmin.cu, Variants<D, P, DIRECT>::Big): D = 3 4 rows x 128 threads, 32-pair chunks; D = 4 2 x 256,
    32-pair chunks, a 2-stage ring; D = 1, 2 2 x 256, 8-pair chunks whose pair 0 takes the FMA-pipe ex2_poly2;
    D >= 5 8-pair chunks; p = 1 16-pair chunks;
  row sums (rowsum_launch.cuh): D <= 4 2 x 256; D >= 5 1 row x 512 threads.

  A. softmin values, p = 2, 1 and 1 | P_UNCLAMPED at D = 1 ... 8: last CTAs partly empty under each layout, last tiles
     of 1, 2, 16 and 32 chunks and the D = 3, 4 read past last_pairs, four temperatures, a cloud translated by +50, the
     h_b / h_scale_b columns, the fused epilogue and lse2;
  B. a term far above a row's lazy running max planted at every pair position of a chunk, for each instantiation's
     own chunk length (the ex2_poly2 pair included), 70, 140 and 300 log2 units up;
  C. softmin row gradients (ops.softmin_grad_rows and ops.softmin autograd), also on a self problem with duplicated
     points and pairs inside the 1e-8 clamp;
  D. kernel products, their row gradients, the gaussian one-pass value and gradient, and the x, y, w gradients of
     ops.kernel_conv with and without the one-pass gradient, three kernels in both conventions, cross and self problems;
  E. whole SamplesLoss values, potentials and gradients on the tiled path;
  F. negative controls: a reference without one column misses by 10x.

Every D <= 8 operator is pinned to the CUDA cores ($B200OT_TC_MIN_D = 9), and the column splits vary
($B200OT_FORCE_SPLITS).  The references run in fp64 on the GPU (fp64_refs.py, cross-checked against the CPU oracle
at a small shape); the bars are those of test_gpu_parity.py / test_gpu_ranges.py, with the rounding allowances of the
p = 1, laplacian and energy pair directions (fp64_refs.direction_slack) and of the cancelling sums of the gaussian row
gradient (fp64_refs.conv64, expansion_slack: a self problem at blur = 0.05 needs it).  The largest error-to-bar ratio
per section is printed when the module ends.
"""
import functools
import math

import pytest
import torch

from fp64_refs import check, conv64, cost64, mid, softmin64
from oracle import geomloss_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CONVS = ("p2", "p1", "p1u")  # p = 2; p = 1 with the clamp of the tensorized cost; p = 1 | P_UNCLAMPED (pykeops)
KINDS = ("gaussian", "laplacian", "energy")
DIMS = range(1, 9)
BLOCK = 1024  # rows per block of the fp64 references

# bars of the dense CUDA-core operators (test_gpu_parity.py)
SOFTMIN_BAR = 3e-6  # test_softmin_vs_oracle_shapes
GRAD_BAR = 2e-5  # test_softmin_gradient_vs_oracle, test_row_reductions_last_tile_lengths
CONV_REL, CONV_W = 5e-6, 2e-7  # test_kernel_conv_vs_oracle
CONV_GRAD_BAR = 3e-5  # test_kernel_conv_gradients_vs_autograd

# (N, M, column splits).  Rows: 4096 fill 8 CTAs; 4097 and 4609 leave one row in the last CTA; 4400 leaves 304 rows,
# which fill the 2 x 256 layout's first row slot and 48 of the second, the 4 x 128 layout's first two slots and 48 of
# the third, and 304 of the 512 threads of the 1 x 512 layout.  Columns: 4096 end on a whole tile; 4097 and 5121 on a
# last tile of 1 column and 4127 of 31 (16 pairs: 2 chunks of 8, 1 of 16, and half a 32-pair chunk, whose other half
# the D = 3, 4 softmin reads as padding); 4129 on 33 columns (32 pairs: 4, 2, 1 chunks); 5120 on a whole second tile
# (64, 32, 16 chunks).  Default splits give one tile per split; 1 streams every tile through one CTA; 3 cuts 5 tiles
# 2 + 2 + 1.
SHAPES = [(4096, 4096, "default"), (4097, 4097, "1"), (4609, 4127, "3"), (4400, 4129, "default"), (4097, 5120, "3"),
          (4609, 5121, "1")]
assert all(min(n, m) >= 4096 for n, m, _ in SHAPES)  # the big tile shape of make_plan
GRAD_SHAPES = [SHAPES[1], SHAPES[3], SHAPES[4]]
CONV_SHAPES = [SHAPES[2], SHAPES[5]]

RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    yield
    for sec in sorted(RATIOS):
        what, r = RATIOS[sec]
        print(f"\n[dense big] section {sec}: largest error / bar = {r:.3g} ({what})")


@pytest.fixture(autouse=True)
def _cuda_cores(monkeypatch):
    """Every D <= 8 operator on the CUDA-core kernels, whatever the default routing (tc_routed reads these per call)."""
    monkeypatch.setenv("B200OT_TC_MIN_D", "9")
    monkeypatch.setenv("B200OT_TC_MIN_PAIRS", "0")


def _splits(monkeypatch, splits):
    if splits == "default":
        monkeypatch.delenv("B200OT_FORCE_SPLITS", raising=False)
    else:
        monkeypatch.setenv("B200OT_FORCE_SPLITS", splits)


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
# problems (on the GPU)
# ------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _case(D, N, M):
    """x in the unit cube, y a little wider; normalised log-weights (softmin values of the order of the cost, so that
    the bar is close to absolute) with zero-weight columns; potentials, old values, upstream gradients, signed
    weights."""
    g = torch.Generator().manual_seed(100 * D + 7 * N + M)
    x, y = torch.rand(N, D, generator=g), torch.rand(M, D, generator=g) * 1.1 - 0.05
    b = torch.rand(M, generator=g) + 0.5
    h_a = (b / b.sum()).log()
    h_a[3::7] = -1e5  # zero-weight columns (log_weights of a zero mass)
    P = dict(x=x, y=y, h_a=h_a, pot=0.2 * torch.rand(M, generator=g), old=torch.rand(N, generator=g),
             go=torch.randn(N, generator=g), w=torch.randn(M, generator=g))
    return {k: v.to(DEV) for k, v in P.items()}


@functools.lru_cache(maxsize=None)
def _self_case(D):
    """A cloud against itself (x is y), with 64 points duplicated exactly and 64 pairs 1e-6 apart: inside the 1e-8
    clamp on |x - y|^2, and for the laplacian inside the clamp on |x/blur - y/blur|^2 for every blur >= 0.05 (fp32
    rounding of x + 1e-6 u moves the distance by < 2e-7)."""
    N = 4400
    g = torch.Generator().manual_seed(9000 + D)
    x = torch.rand(N, D, generator=g)
    x[100:164] = x[1000:1064]
    u = torch.randn(64, D, generator=g)
    x[200:264] = x[2000:2064] + 1e-6 * u / u.norm(dim=1, keepdim=True)
    d = (x[200:264].double() - x[2000:2064].double()).norm(dim=1)
    assert bool((d > 5e-7).all() and (d < 1.5e-6).all())
    P = dict(x=x, h_a=torch.randn(N, generator=g) * 0.5 - math.log(N), pot=0.2 * torch.rand(N, generator=g),
             go=torch.randn(N, generator=g), w=torch.randn(N, generator=g))
    return {k: v.to(DEV) for k, v in P.items()}


# ------------------------------------------------------------------------------------------------------
# the references themselves, once against the CPU oracle
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("part", ["softmin", "kernel", "loss"])
def test_gpu_references_match_the_cpu_oracle(part):
    """The fp64 references on the GPU equal the oracle's CPU results at a small shape (softmin_points, keops_softmin,
    softmin_grad_rows, kernel_conv_points, keops_kernel_matrix and autograd, samples_loss), to fp64 rounding."""
    g = torch.Generator().manual_seed(77)
    D, eps, blur = 3, 0.5, 0.3
    x, y = torch.rand(300, D, generator=g).double(), torch.rand(200, D, generator=g).double()
    h, go, w = (torch.randn(n, generator=g).double() for n in (200, 300, 200))

    def close(got, ref, what):
        err = (got.cpu() - ref).abs().max().item()
        assert err <= 1e-11 * max(1.0, ref.abs().max().item()), (what, err)

    if part == "softmin":
        for conv in CONVS:
            out, gx, _ = softmin64(eps, x, y, h, None, conv, go=go, center=mid(x, y), block=128, device=DEV)
            xr = x.clone().requires_grad_(True)
            if conv == "p1u":
                ref = O.keops_softmin(eps, xr, y, h, p=1)  # 1/eps = 2 is exact in fp32
                (gref,) = torch.autograd.grad(ref, xr, go)
            else:
                p = 2 if conv == "p2" else 1
                ref = O.softmin_points(eps, x, y, h, p=p)
                gref = O.softmin_grad_rows(eps, x, y, h, go, p=p)
            close(out, ref.detach(), f"{conv} value")
            close(gx, gref, f"{conv} row gradient")
    elif part == "kernel":
        for kind in KINDS:
            for unclamped in (False, True):
                out, rx, ry, rw, _, _ = conv64(kind, unclamped, x, y, w, blur, None, go, mid(x, y), block=128,
                                               device=DEV)
                xr, yr, wr = (t.clone().requires_grad_(True) for t in (x, y, w))
                K = (O.keops_kernel_matrix if unclamped else O.kernel_matrix)(kind, xr, yr, blur)
                ref = K @ wr
                grads = torch.autograd.grad(ref, [xr, yr, wr], go)
                if not unclamped:
                    close(ref.detach(), O.kernel_conv_points(kind, x, y, w, blur), f"{kind} oracle")
                for got, r, what in zip((out, rx, ry, rw), (ref.detach(),) + grads, ("value", "x", "y", "w")):
                    close(got, r, f"{kind} unclamped={unclamped} {what}")
    else:
        for kw in LOSSES:
            ref = O.samples_loss(x, y, **kw)
            got = O.samples_loss(x.to(DEV), y.to(DEV), **kw)
            close(got, ref, kw)


# ------------------------------------------------------------------------------------------------------
# A. softmin values
# ------------------------------------------------------------------------------------------------------
# 2.0: normalised weights keep the values near the mean cost, so that the bar is absolute and a relative error r of the
# row sums shows as 2 r (the FMA-pipe exponentials of D = 1, 2 are one term in eight)
EPS_A = (2.0, 0.5, 0.01, 5e-4)


@pytest.mark.parametrize("conv", CONVS)
@pytest.mark.parametrize("D", DIMS)
def test_softmin_values(D, conv, monkeypatch):
    """Values with h_b / h_scale_b and lse2, and the fused epilogue with the potentials folded into h_a, on every shape
    of SHAPES at four temperatures, and at eps = 0.01 with both clouds translated by +50 (default_center)."""
    from geomloss_b200 import ops

    p = _pv(conv)
    for N, M, splits in SHAPES:
        _splits(monkeypatch, splits)
        P = _case(D, N, M)
        for eps in EPS_A:
            for shifted in ((False, True) if eps == 0.01 else (False,)):
                what = f"D={D} {conv} N={N} M={M} splits={splits} eps={eps}{' +50' if shifted else ''}"
                xd, yd = (P["x"] + 50.0, P["y"] + 50.0) if shifted else (P["x"], P["y"])
                center = ops.default_center(xd, yd)
                # the fp32 translated clouds, translated back exactly in fp64
                x64, y64 = xd.double() - (50.0 if shifted else 0.0), yd.double() - (50.0 if shifted else 0.0)
                ref = softmin64(eps, x64, y64, P["h_a"].double() + P["pot"].double() / eps, None, conv, block=BLOCK,
                                device=DEV)[0]
                out, lse2 = ops.softmin_raw(eps, xd, yd, P["h_a"], P["pot"], 1.0 / eps, p=p, center=center,
                                            want_lse2=True)
                _check("A", what, out, ref, _softmin_bar(ref))
                o, l2 = out.double(), lse2.double()
                assert (-eps * math.log(2.0) * l2 - o).abs().max().item() <= 1e-6 * o.abs().max().item() + 1e-7, what
                # the same potentials folded into h_a (no h_b), with the fused epilogue
                fused, none = ops.softmin_raw(eps, xd, yd, P["h_a"] + P["pot"] / eps, p=p, center=center,
                                              out_old=P["old"], alpha_old=0.5, beta=0.7)
                assert none is None
                want = 0.5 * P["old"].double() + 0.7 * ref
                _check("A", what + " fused epilogue", fused, want, _softmin_bar(want))


# ------------------------------------------------------------------------------------------------------
# B. stale max at every pair position of a chunk
# ------------------------------------------------------------------------------------------------------
PRE_PAIRS = 256  # column pairs of a split that the max pre-pass reads (softmin.cuh)


def _chunk_pairs(D, conv):
    """Column pairs per chunk of the dense big softmin (Variants::kCH)."""
    return 16 if conv != "p2" else (32 if D in (3, 4) else 8)


# p = 2 at D = 3, 4: test_gpu_softmin_sm90_shape.py::test_stale_max_every_chunk_position
B_GRID = [(d, c) for d in DIMS for c in CONVS if not (c == "p2" and d in (3, 4))]


@pytest.mark.parametrize("D,conv", B_GRID, ids=[f"D{d}-{c}" for d, c in B_GRID])
def test_stale_max_every_chunk_position(D, conv, monkeypatch):
    """One column whose log2-domain exponent exceeds every row's running max by more than ``jump`` is planted past the
    pre-pass, once per pair position of a chunk (alternating the column within the pair; both columns at position 0,
    the ex2_poly2 pair of D = 1, 2 at p = 2).  jump = 70 clears the 2^64 chunk-sum guard; 140 takes ex2_poly2 to its
    clamp at 2^127 (and the MUFU exponential to +inf), which the guard must still see; 300 makes the rescale factor
    2^(m - cm) of the row's earlier sums underflow to zero.  One column split, so the plant is never absorbed by the
    pre-pass of another split.  Negative control: the reference without the plant misses by 10x."""
    from geomloss_b200 import ops

    _splits(monkeypatch, "1")
    p, ch = _pv(conv), _chunk_pairs(D, conv)
    N, M, eps = 4609, 4129, 0.5
    g = torch.Generator().manual_seed(500 + 10 * D + len(conv))
    x, y = torch.rand(N, D, generator=g).to(DEV), torch.rand(M, D, generator=g).to(DEV)
    h = (torch.rand(M, generator=g) - 0.5).to(DEV)
    center = ops.default_center(x, y)
    base = softmin64(eps, x, y, h, None, conv, block=BLOCK, device=DEV)[0]
    cmax = D / 2 if conv == "p2" else math.sqrt(D)  # the largest cost on the unit cube
    for jump in (70.0, 140.0, 300.0):
        # every other term is below max(h) in natural units: the plant clears the running max by more than `jump`
        h_plant = float(h.max()) + cmax / eps + (jump + 1.0) * math.log(2.0)
        for pos in range(ch):
            for lane in ((0, 1) if pos == 0 else (pos & 1,)):
                j = 2 * (2 * PRE_PAIRS + 3 * ch + pos) + lane
                what = f"D={D} {conv} jump={jump} pair position {pos} column {lane}"
                hp = h.clone()
                hp[j] = h_plant
                # fp64: the base row sums with column j's term replaced by the planted one
                cj = cost64(x.double(), y[j:j + 1].double(), conv)[:, 0] / eps
                lse = torch.logaddexp(-base / eps, h_plant - cj)
                lse = lse + torch.log1p(-torch.exp(float(h[j]) - cj - lse))
                ref = -eps * lse
                out, _ = ops.softmin_raw(eps, x, y, hp, p=p, center=center)
                bar = _softmin_bar(ref)
                _check("B", what, out, ref, bar)
                assert (out.double() - base).abs().max().item() >= 10 * bar, what  # F: the plant matters


# ------------------------------------------------------------------------------------------------------
# C. softmin row gradients
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("conv", CONVS)
@pytest.mark.parametrize("D", DIMS)
def test_softmin_row_gradients(D, conv, monkeypatch):
    """ops.softmin_grad_rows with lse2 from the forward, and ops.softmin's autograd (scale_out 0.7), on cross problems
    and on the self problem, whose duplicated points and pairs inside the clamp must contribute exactly zero (p = 1,
    clamped) or only their rounding allowance (p = 1 | P_UNCLAMPED)."""
    from geomloss_b200 import ops

    p = _pv(conv)
    problems = [(f"N={n} M={m} splits={s}", s, _case(D, n, m)) for n, m, s in GRAD_SHAPES]
    S = _self_case(D)
    problems.append(("self", "default", dict(S, y=S["x"])))
    for name, splits, P in problems:
        _splits(monkeypatch, splits)
        x, y, h_a, pot, go = (P[k] for k in ("x", "y", "h_a", "pot", "go"))
        center = ops.default_center(x, y)
        for eps in (0.5, 0.02):
            what = f"D={D} {conv} {name} eps={eps}"
            _, gref, allow = softmin64(eps, x, y, h_a.double() + pot.double() / eps, None, conv, go=go,
                                       center=mid(x, y), block=BLOCK, device=DEV)
            _, lse2 = ops.softmin_raw(eps, x, y, h_a, pot, 1.0 / eps, p=p, center=center, want_lse2=True)
            gx = ops.softmin_grad_rows(eps, x, y, h_a, pot, 1.0 / eps, lse2, go, p=p, center=center)
            _check("C", what + " grad_rows", gx, gref, _grad_bar(gref, GRAD_BAR) + allow)
            xg = x.clone().requires_grad_(True)
            val = ops.softmin(eps, xg, y, h_a, pot, 1.0 / eps, p=p, center=center, scale_out=0.7)
            (g2,) = torch.autograd.grad(val, xg, go)
            _check("C", what + " autograd", g2, 0.7 * gref, _grad_bar(0.7 * gref, GRAD_BAR) + 0.7 * allow)


# ------------------------------------------------------------------------------------------------------
# D. kernel products and their gradients
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", DIMS)
def test_kernel_products_and_gradients(D, kind, monkeypatch):
    """kernel_conv_raw, kernel_conv_grad_rows, the gaussian kernel_conv_value_and_grad_rows (value, and the unit
    gradient against the fp64 gradient of sum(out)) and the x, y, w gradients of ops.kernel_conv with the one-pass
    gradient on and off, in both conventions, on cross problems (the y and w gradients reduce the M x N transpose) and
    on the self problem."""
    from geomloss_b200 import ops

    problems = [(f"N={n} M={m} splits={s}", s, _case(D, n, m)) for n, m, s in CONV_SHAPES]
    S = _self_case(D)
    problems.append(("self", "default", dict(S, y=S["x"])))
    for name, splits, P in problems:
        _splits(monkeypatch, splits)
        x, y, w, go = P["x"], P["y"], P["w"], P["go"]
        center = ops.default_center(x, y)
        for unclamped in (False, True):
            kid = ops.KERNEL_KINDS[kind] | (ops.KERNEL_UNCLAMPED if unclamped else 0)
            for blur in ((0.05, 0.5) if kind != "energy" else (0.5,)):
                what = f"D={D} {kind}{' unclamped' if unclamped else ''} {name} blur={blur}"
                ref, rx, ry, rw, ax, ay = conv64(kind, unclamped, x, y, w, blur, None, go, mid(x, y), block=BLOCK,
                                                 device=DEV, expansion_slack=True)
                vbar, xbar = _conv_bar(ref, w), _grad_bar(rx, CONV_GRAD_BAR) + ax
                _check("D", what + " value", ops.kernel_conv_raw(kid, x, y, w, blur, center=center), ref, vbar)
                _check("D", what + " grad_rows", ops.kernel_conv_grad_rows(kid, x, y, w, blur, go, center=center), rx,
                       xbar)
                if kind == "gaussian":
                    ones = torch.ones_like(go)
                    _, r1, _, _, a1, _ = conv64(kind, unclamped, x, y, w, blur, None, ones, mid(x, y), block=BLOCK,
                                                device=DEV, expansion_slack=True)
                    val, gunit = ops.kernel_conv_value_and_grad_rows(kid, x, y, w, blur, center=center)
                    _check("D", what + " one-pass value", val, ref, vbar)
                    _check("D", what + " one-pass unit gradient", gunit, r1, _grad_bar(r1, CONV_GRAD_BAR) + a1)
                for fused in (False, True):
                    monkeypatch.setattr(ops, "FUSED_CONV_GRAD", fused)
                    xg, yg, wg = (t.clone().requires_grad_(True) for t in (x, y, w))
                    out = ops.kernel_conv(kid, xg, yg, wg, blur, center=center)
                    gx, gy, gw = torch.autograd.grad(out, [xg, yg, wg], go)
                    tag = f"{what} fused={fused}"
                    _check("D", tag + " kernel_conv value", out, ref, vbar)
                    _check("D", tag + " grad x", gx, rx, xbar)
                    _check("D", tag + " grad y", gy, ry, _grad_bar(ry, CONV_GRAD_BAR) + ay)
                    # K(y, x) go: a kernel product of the transpose, held to the product bar (per unit weight of go)
                    _check("D", tag + " grad w", gw, rw, _conv_bar(rw, go))


# ------------------------------------------------------------------------------------------------------
# E. whole losses on the tiled path
# ------------------------------------------------------------------------------------------------------
LOSSES = [dict(loss="sinkhorn", p=2, blur=0.05), dict(loss="sinkhorn", p=1, blur=0.1),
          dict(loss="gaussian", blur=0.2), dict(loss="laplacian", blur=0.2), dict(loss="energy")]


@pytest.mark.parametrize("D", [1, 5, 8])
def test_whole_losses_on_the_tiled_path(D, monkeypatch):
    """SamplesLoss above the small-cloud limit (SMALL_MAX = 0): value, potentials and x, y gradients against the fp64
    oracle on the GPU, at the bars of test_sinkhorn_cases / test_kernel_losses."""
    from geomloss_b200 import SamplesLoss, sinkhorn_small

    monkeypatch.setattr(sinkhorn_small, "SMALL_MAX", 0)
    N, M = 4133, 4100
    g = torch.Generator().manual_seed(700 + D)
    x, y = torch.rand(N, D, generator=g), 0.8 * torch.rand(M, D, generator=g) + 0.3
    a, b = torch.rand(N, generator=g) + 0.2, torch.rand(M, generator=g) + 0.2
    a, b = (a / a.sum()).to(DEV), (b / b.sum()).to(DEV)
    x, y = x.to(DEV), y.to(DEV)
    for kw in LOSSES:
        kw = dict(kw, diameter=2.0 * math.sqrt(D)) if kw["loss"] == "sinkhorn" else kw  # one eps-schedule for both
        sinkhorn = kw["loss"] == "sinkhorn"
        what = f"D={D} {kw}"
        xg, yg = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        val = SamplesLoss(**kw)(a, xg, b, yg)
        gx, gy = torch.autograd.grad(val, [xg, yg])
        F, G = SamplesLoss(potentials=True, **kw)(a, x, b, y)
        xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
        ref = O.samples_loss(a.double(), xr, b.double(), yr, **kw)
        rx, ry = torch.autograd.grad(ref, [xr, yr])
        RF, RG = (t.reshape(-1) for t in O.samples_loss(a.double(), x.double(), b.double(), y.double(), potentials=True,
                                                          **kw))
        _check("E", what + " value", val, ref.detach(), 1e-4 * abs(ref.item()) + (1e-7 if sinkhorn else 2e-7))
        _check("E", what + " grad x", gx, rx, 1e-4 * max(rx.abs().max().item(), 1e-3))
        _check("E", what + " grad y", gy, ry, 1e-4 * max(ry.abs().max().item(), 1e-3))
        for got, r, side in ((F, RF, "F"), (G, RG, "G")):
            pbar = 1e-5 * max(1.0, r.abs().max().item()) if sinkhorn else 2e-5 * r.abs().max().item()
            _check("E", f"{what} potential {side}", got.reshape(-1), r, pbar)


# ------------------------------------------------------------------------------------------------------
# F. negative controls
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [1, 3, 6])
def test_dropping_the_last_tile_misses_the_bars(D):
    """M = 4097: the last tile holds one column.  A reference without it misses the kernels' results by at least 10x
    the bar (p = 2 and p = 1 softmins, gaussian product), while the reference with it meets the bar."""
    from geomloss_b200 import ops

    P = _case(D, 4097, 4097)
    x, y, h, w = P["x"], P["y"], P["h_a"].clone(), P["w"].clone()
    h[-1], w[-1] = 0.0, 1.0  # a column of mass 1, where the others share 1: it leads the rows near it
    center = ops.default_center(x, y)
    eps, blur = 0.05, 0.5
    for conv in ("p2", "p1"):
        out, _ = ops.softmin_raw(eps, x, y, h, p=_pv(conv), center=center)
        ref = softmin64(eps, x, y, h, None, conv, block=BLOCK, device=DEV)[0]
        bad = softmin64(eps, x, y[:-1], h[:-1], None, conv, block=BLOCK, device=DEV)[0]
        bar = _softmin_bar(ref)
        _check("F", f"D={D} {conv} softmin, every column", out, ref, bar)
        assert (out.double() - bad).abs().max().item() >= 10 * bar, (D, conv)
    out = ops.kernel_conv_raw("gaussian", x, y, w, blur, center=center)
    ref = conv64("gaussian", False, x, y, w, blur, None, P["go"], mid(x, y), block=BLOCK, device=DEV)[0]
    bad = conv64("gaussian", False, x, y[:-1], w[:-1], blur, None, P["go"], mid(x, y), block=BLOCK, device=DEV)[0]
    bar = _conv_bar(ref, w)
    _check("F", f"D={D} gaussian product, every column", out, ref, bar)
    assert (out.double() - bad).abs().max().item() >= 10 * bar, D

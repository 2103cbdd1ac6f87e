"""The small-cloud kernels (csrc/b200ot_small.cu: N, M <= 6000, D <= 8, batched or not) against the fp64 oracle, at every
dimension they are instantiated for, around their tile edges, on both warp variants of the iteration kernel, with
per-element upstream gradients, at the routing boundary, on translated clouds and on batches above 65535 elements.

Tolerances are the suite's (tests/test_gpu_parity.py, BASELINE.md section 3 item 7): softmin 3e-6 max(1, |ref|), row
gradients 2e-5 of the largest entry, kernel products 5e-6 max(1e-3, |ref|) + 2e-7 sum|w|, loss 1e-4 relative,
potentials 1e-5 absolute on unit-cube data, loss gradients 1e-4 of the largest entry."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
LN2 = float(np.log(2.0))
UNCLAMPED = 0x100
KERNEL_IDS = {"gaussian": 0, "laplacian": 1, "energy": 2}


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()  # fails loudly if libb200ot.so is missing: there is no fallback to test
    yield


def _P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _L():
    from geomloss_b200 import _lib

    return _lib.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cu(t):
    return t.float().contiguous().to(DEV)


# ------------------------------------------------------------------------------------------------------------------
# fp64 references of one operator (unbatched clouds)
# ------------------------------------------------------------------------------------------------------------------
def _softmin_ref(eps, x, y, h, p):
    """-eps log sum_j exp(h_j - C(x_i, y_j)/eps); p = 1 | UNCLAMPED is the pykeops convention (exact zero distance)."""
    from oracle import geomloss_oracle as O

    if p & UNCLAMPED:
        return O.keops_softmin(eps, x, y, h, p=p & 0xff)
    return O.softmin_points(eps, x, y, h, p=p, row_block=512)


def _grad_rows_ref(eps, x, y, h, go, p):
    from oracle import geomloss_oracle as O

    if not p & UNCLAMPED:
        return O.softmin_grad_rows(eps, x, y, h, go, p=p)
    xr = x.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad((O.keops_softmin(eps, xr, y, h, p=p & 0xff) * go).sum(), xr)
    return g


def _conv_ref(kind, x, y, w, blur, unclamped):
    from oracle import geomloss_oracle as O

    if unclamped:
        return O.keops_kernel_matrix(kind, x, y, blur) @ w
    return O.kernel_conv_points(kind, x, y, w, blur)


def _clouds(g, B, N, M, D, dup=0):
    """Unit-cube x, slightly larger y; the first `dup` points of x are exact copies of points of y."""
    x = torch.rand(B, N, D, generator=g)
    y = torch.rand(B, M, D, generator=g) * 1.1 - 0.05
    k = min(dup, N, M)
    if k:
        x[:, :k] = y[:, M - k:]
    return x, y


# ------------------------------------------------------------------------------------------------------------------
# b200ot_sinkhorn_iteration_small
# ------------------------------------------------------------------------------------------------------------------
def _box(x, y):
    """(2, D) bounding box of a batch of clouds: the coordinate origin of the small Sinkhorn kernels."""
    from geomloss_b200 import ops

    return ops.cloud_extent(x.reshape(-1, x.shape[-1]), y.reshape(-1, y.shape[-1]))


def _iteration(x, y, wa, wb, pots, p, eps, alpha_old, beta, debias, w_linear, lo_hi=None):
    """One call; returns the four outputs (None when not debiased) and the lse2 buffer, on the host."""
    B, N, D = x.shape
    M = y.shape[1]
    outs = [torch.full((B, n), float("nan"), device=DEV) for n in (N, M, N, M)]
    if not debias:
        outs[2] = outs[3] = None
    lse2 = torch.full((B * (2 * N + 2 * M),), float("nan"), device=DEV)
    f_ba, g_ab, f_aa, g_bb = pots if pots is not None else (None,) * 4
    rc = _L().b200ot_sinkhorn_iteration_small(_P(x), _P(y), _P(wa), _P(wb), _P(f_ba), _P(g_ab), _P(f_aa), _P(g_bb),
                                              *[_P(o) for o in outs], _P(lse2), B, N, M, D, p, eps, alpha_old, beta,
                                              w_linear, _P(lo_hi), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    return [None if o is None else o.cpu().double() for o in outs], lse2.cpu().double()


def _iteration_refs(x, y, wa, wb, pots, p, eps, w_linear):
    """fp64 softmins of element k: [xy, yx, xx, yy] with h = log w + pot/eps (log_weights' -100000 floor)."""
    from oracle import geomloss_oracle as O

    la = O.log_weights(wa) if w_linear else wa
    lb = O.log_weights(wb) if w_linear else wb
    hs = [lb, la, la, lb]
    if pots is not None:
        hs = [h + q / eps for h, q in zip(hs, (pots[1], pots[0], pots[2], pots[3]))]
    rows, cols = (x, y, x, y), (y, x, x, y)
    return [_softmin_ref(eps, r, c, h, p) for r, c, h in zip(rows, cols, hs)]


def _check_iteration(g, B, N, M, D, p, eps, *, averaged, debias, w_linear, dup=0, centred=True, shift=0.0):
    x, y = _clouds(g, B, N, M, D, dup)
    x, y = x + shift, y + shift
    wa, wb = torch.rand(B, N, generator=g) + 0.1, torch.rand(B, M, generator=g) + 0.1
    if w_linear:  # zero weights take the -100000 floor (the first point keeps a positive mass)
        wa[:, 1::3] = 0.0
        wb[:, 2::4] = 0.0
        wa, wb = wa / wa.sum(1, keepdim=True), wb / wb.sum(1, keepdim=True)
    else:
        wa, wb = (wa / wa.sum(1, keepdim=True)).log(), (wb / wb.sum(1, keepdim=True)).log()
    pots, alpha, lam = None, 0.0, 1.0
    if averaged:
        pots = [torch.randn(B, n, generator=g) * 0.1 for n in (N, M, N, M)]
        alpha, lam = 0.5, 0.8
    beta = 0.5 * lam if averaged else lam
    xd, yd = _cu(x), _cu(y)
    got, lse2 = _iteration(xd, yd, _cu(wa), _cu(wb), None if pots is None else [_cu(t) for t in pots], p, eps, alpha,
                           beta, debias, w_linear, _box(xd, yd) if centred else None)
    offs = np.cumsum([0, B * N, B * M, B * N])
    for k in range(B):
        refs = _iteration_refs(x[k].double(), y[k].double(), wa[k].double(), wb[k].double(),
                               None if pots is None else [t[k].double() for t in pots], p, eps, w_linear)
        for q in range(4 if debias else 2):
            n = N if q % 2 == 0 else M
            ref = beta * refs[q] + (alpha * pots[q][k].double() if averaged else 0.0)
            out = got[q][k]
            tol = 3e-6 * max(1.0, refs[q].abs().max().item())
            err = (out - ref).abs().max().item()
            assert err <= tol, (f"B={B} N={N} M={M} D={D} p={p} eps={eps} averaged={averaged} debias={debias} "
                                f"w_linear={w_linear} element {k} problem {q}: {err:.3e} > {tol:.3e}")
            # lse2 is the log2-domain log-sum-exp behind the output: out = alpha old - beta eps ln2 lse2
            l2 = lse2[offs[q] + k * n: offs[q] + (k + 1) * n]
            back = -beta * eps * LN2 * l2 + (alpha * pots[q][k].double() if averaged else 0.0)
            assert (back - out).abs().max().item() <= 1e-6 * max(1.0, out.abs().max().item()), (k, q)
    return got


# row counts around the 32-row CTA x column counts around the 8-column chunk and the 256-column tile, plus a few shapes
# with far more rows than columns (the column problems' CTAs beyond ceil(M/32) return at once)
SHAPES = [(n, m) for n in (1, 31, 32, 33) for m in (1, 7, 8, 9, 255, 256, 257, 1000)] + [(1000, 9), (257, 31), (300, 1)]
PS = [1, 2, 1 | UNCLAMPED]


@pytest.mark.parametrize("p", PS, ids=["p1", "p2", "p1u"])
@pytest.mark.parametrize("D", range(1, 9))
def test_iteration_small_vs_oracle(D, p):
    """Every instantiation of sinkhorn_iteration_small_kernel (8-warp variant: B = 2 and at most 32 row tiles x 4
    problems x 2 = 256 CTAs); the initialisation and the averaged form, debias on and off, natural-log and linear
    weights with zeros, coordinates taken from the bounding box's mid-point or from the origin, all cycled over the
    shapes."""
    g = torch.Generator().manual_seed(100 * D + p)
    for s, (N, M) in enumerate(SHAPES):
        _check_iteration(g, 2, N, M, D, p, 0.5 if s % 3 else 0.02, averaged=bool(s % 2), debias=bool((s // 2) % 2),
                         w_linear=(s // 4) % 2, centred=bool((s // 8) % 2))


@pytest.mark.parametrize("p", PS, ids=["p1", "p2", "p1u"])
@pytest.mark.parametrize("D", range(1, 9))
def test_iteration_small_warp_variants(D, p):
    """launch_iter_p takes 8 warps up to 1024 CTAs and 4 above.  N = 64, M = 250 is ceil(250/32) = 8 row tiles, and
    250 columns give every warp of either variant some columns of the tile:
      B = 32, debias (4 problems): 8 * 4 * 32 = 1024 CTAs -> 8 warps (the last count on that side)
      B = 33, debias:              8 * 4 * 33 = 1056 CTAs -> 4 warps
      B = 64, no debias (2):       8 * 2 * 64 = 1024 CTAs -> 8 warps
      B = 65, no debias:           8 * 2 * 65 = 1040 CTAs -> 4 warps"""
    g = torch.Generator().manual_seed(7 * D + p)
    for B, debias in ((32, True), (33, True), (64, False), (65, False)):
        _check_iteration(g, B, 64, 250, D, p, 0.05, averaged=True, debias=debias, w_linear=1, dup=5)


# ------------------------------------------------------------------------------------------------------------------
# b200ot_sinkhorn_final_bwd_small
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", PS, ids=["p1", "p2", "p1u"])
@pytest.mark.parametrize("D", [1, 3, 5, 8])
def test_final_bwd_small_vs_oracle(D, p):
    """grad_x = scale_out go_scale[b] (sum over the problems sharing the row cloud of go_q . d softmin_q / d x), with
    n_terms = 1 and 2, a non-uniform go_scale, and x holding exact copies of points of y (and the x <-> x diagonal):
    the clamped tensorized cost and the unclamped zero-distance rule must both match the oracle there."""
    g = torch.Generator().manual_seed(31 * D + p)
    B, N, M, eps, lam = 3, 300, 517, 0.05, 0.7
    x, y = _clouds(g, B, N, M, D, dup=40)
    wa, wb = torch.rand(B, N, generator=g) + 0.1, torch.rand(B, M, generator=g) + 0.1
    wa, wb = wa / wa.sum(1, keepdim=True), wb / wb.sum(1, keepdim=True)
    pots = [torch.randn(B, n, generator=g) * 0.05 for n in (N, M, N, M)]
    go_scale = torch.tensor([0.7, -1.9, 3.1])
    xd, yd, ad, bd = map(_cu, (x, y, wa, wb))
    potd = [_cu(t) for t in pots]
    lo_hi = _box(xd, yd)
    _, lse2 = _iteration(xd, yd, ad, bd, potd, p, eps, 0.0, lam, True, 1, lo_hi)
    lse2d = _cu(lse2)
    for n_terms in (1, 2):
        gos = [torch.randn(B, n, generator=g) for n in (N, M, N, M)]
        if n_terms == 1:
            gos[2] = gos[3] = None
        gx, gy = torch.empty(B, N, D, device=DEV), torch.empty(B, M, D, device=DEV)
        gosd, go_scaled = [None if t is None else _cu(t) for t in gos], _cu(go_scale)  # (held until the launch)
        rc = _L().b200ot_sinkhorn_final_bwd_small(_P(xd), _P(yd), _P(ad), _P(bd), *[_P(t) for t in potd], _P(lse2d),
                                                  *[_P(t) for t in gosd], _P(gx), _P(gy), B, N, M, D, p, eps, lam,
                                                  _P(go_scaled), 1, _P(lo_hi), _stream())
        assert rc == 0
        torch.cuda.synchronize()
        for k in range(B):
            refs = [torch.zeros(N, D, dtype=torch.float64), torch.zeros(M, D, dtype=torch.float64)]
            la, lb = torch.log(wa[k].double()), torch.log(wb[k].double())
            xk, yk = x[k].double(), y[k].double()
            terms = [(0, xk, yk, lb + pots[1][k].double() / eps), (1, yk, xk, la + pots[0][k].double() / eps),
                     (0, xk, xk, la + pots[2][k].double() / eps), (1, yk, yk, lb + pots[3][k].double() / eps)]
            for q, (side, r, c, h) in enumerate(terms[: 2 * n_terms]):
                refs[side] += _grad_rows_ref(eps, r, c, h, gos[q][k].double(), p)
            for side, got in ((0, gx), (1, gy)):
                ref = lam * go_scale[k].item() * refs[side]
                err = (got[k].cpu().double() - ref).abs().max().item()
                tol = 2e-5 * ref.abs().max().item()
                assert err <= tol, (n_terms, k, side, err, tol)


# ------------------------------------------------------------------------------------------------------------------
# b200ot_sinkhorn_loop_small
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("reach", [None, 0.4])
@pytest.mark.parametrize("debias", [True, False])
@pytest.mark.parametrize("D", [4, 8])
def test_loop_small_vs_oracle(D, debias, reach):
    """The whole eps-descent in one call (B = 2, N = 600, M = 530: three column tiles), followed by the final
    non-averaged update, against the oracle's sinkhorn_loop on the same eps_list."""
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(D + 10 * debias + (reach is not None))
    B, N, M, p, blur = 2, 600, 530, 2, 0.05
    x, y = _clouds(g, B, N, M, D)
    a, b = torch.rand(B, N, generator=g) + 0.2, torch.rand(B, M, generator=g) + 0.2
    a, b = a / a.sum(1, keepdim=True), b / b.sum(1, keepdim=True)
    diameter, eps_final, eps_list, rho = O.scaling_parameters(x, y, p, blur, reach, None, 0.5)
    xd, yd, ad, bd = map(_cu, (x, y, a, b))
    lo_hi = _box(xd, yd)
    bufs = torch.empty(2, B * (2 * N + 2 * M), device=DEV)
    arr = (ctypes.c_double * len(eps_list))(*eps_list)
    which = ctypes.c_int32(-1)
    rc = _L().b200ot_sinkhorn_loop_small(_P(xd), _P(yd), _P(ad), _P(bd), 1, arr, len(eps_list),
                                         -1.0 if rho is None else rho, int(debias), _P(bufs[0]), _P(bufs[1]),
                                         ctypes.byref(which), B, N, M, D, p, _P(lo_hi), _stream())
    assert rc == 0 and which.value in (0, 1)
    buf = bufs[0] if which.value else bufs[1]
    pots = [buf[: B * N].view(B, N), buf[B * N: B * (N + M)].view(B, M)]
    pots += [buf[B * (N + M): B * (2 * N + M)].view(B, N), buf[B * (2 * N + M):].view(B, M)] if debias else [None] * 2
    lam = O.damping(eps_list[-1], rho)
    got, _ = _iteration(xd, yd, ad, bd, pots, p, eps_list[-1], 0.0, lam, debias, 1, lo_hi)
    xx, yy = x.double(), y.double()
    C = [O.cost_matrix(xx, yy, p), O.cost_matrix(yy, xx, p), O.cost_matrix(xx, xx, p), O.cost_matrix(yy, yy, p)]
    f_aa, g_bb, g_ab, f_ba = O.sinkhorn_loop(O.softmin_dense, O.log_weights(a.double()), O.log_weights(b.double()),
                                             C[2], C[3], C[0], C[1], eps_list, rho, debias=debias)
    refs = [f_ba, g_ab, f_aa, g_bb]
    for q in range(4 if debias else 2):
        err = (got[q] - refs[q].detach()).abs().max().item()
        assert err <= 1e-5 * max(1.0, refs[q].abs().max().item()), (q, err)


# ------------------------------------------------------------------------------------------------------------------
# b200ot_kernel_mmd_small, _bwd_small, _value_small
# ------------------------------------------------------------------------------------------------------------------
def _mmd_call(x, y, a, b, kind_id, blur, grad_value):
    B, N, D = x.shape
    M = y.shape[1]
    outs = [torch.full((B, n), float("nan"), device=DEV) for n in (N, M, N, M)]
    L = _L()
    assert L.b200ot_kernel_mmd_small(_P(x), _P(y), _P(a), _P(b), *[_P(o) for o in outs], B, N, M, D, kind_id, blur,
                                     _stream()) == 0
    val = torch.empty(B, device=DEV)
    assert L.b200ot_kernel_mmd_value_small(_P(a), _P(b), _P(outs[0]), _P(outs[1]), _P(outs[2]), B, N, M, _P(val),
                                           _stream()) == 0
    gx, gy = torch.empty_like(x), torch.empty_like(y)
    assert L.b200ot_kernel_mmd_bwd_small(_P(x), _P(y), _P(a), _P(b), _P(grad_value), _P(gx), _P(gy), B, N, M, D,
                                         kind_id, blur, _stream()) == 0
    torch.cuda.synchronize()
    return [o.cpu().double() for o in outs], val.cpu().double(), gx.cpu().double(), gy.cpu().double()


def _conv_tol(ref, w):
    """test_kernel_conv_vs_oracle's bar for one kernel product out = K w."""
    return 5e-6 * max(1e-3, ref.abs().max().item()) + 2e-7 * w.abs().sum().item()


MMD_SHAPES = [(1, 1), (31, 7), (32, 8), (33, 9), (1, 257), (33, 256), (257, 255), (300, 1000), (1000, 31)]


@pytest.mark.parametrize("unclamped", [False, True], ids=["tensorized", "online"])
@pytest.mark.parametrize("kind", ["gaussian", "laplacian", "energy"])
@pytest.mark.parametrize("D", range(1, 9))
def test_kernel_mmd_small_vs_oracle(D, kind, unclamped):
    """The four kernel products, the value and both cloud gradients (per-element, non-uniform grad_value) against
    kernel_conv_points and fp64 autograd of mmd_dense (tensorized convention) / mmd_online (pykeops convention), over
    the row / column edges, with duplicated points, and once on identical clouds with different weights."""
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(D * 17 + KERNEL_IDS[kind] + 5 * unclamped)
    kid = KERNEL_IDS[kind] | (UNCLAMPED if unclamped else 0)
    blur = 0.3
    B = 3
    go = torch.tensor([1.3, -0.4, 2.2])
    for s, (N, M) in enumerate(MMD_SHAPES + [(200, 200)]):
        same = s == len(MMD_SHAPES)
        # coordinates on a 2^-12 grid: points are either equal or at least 2^-12 apart, so that the fp32 scaled
        # coordinates of distinct points stay distinct and the laplacian / energy gradients, discontinuous at
        # coincident points, are decided there exactly as in fp64
        x, y = (torch.round(t * 4096) / 4096 for t in _clouds(g, B, N, M, D, dup=N // 3))
        if same:
            y = x.clone()
        a, b = torch.rand(B, N, generator=g) + 0.1, torch.rand(B, M, generator=g) + 0.1
        a, b = a / a.sum(1, keepdim=True), b / b.sum(1, keepdim=True)
        outs, val, gx, gy = _mmd_call(*map(_cu, (x, y, a, b)), kid, blur, _cu(go))
        xr, yr = x.double().requires_grad_(True), y.double().requires_grad_(True)
        ad, bd = a.double(), b.double()
        fn = O.mmd_online if unclamped else O.mmd_dense
        vr = fn(ad, xr, bd, yr, kind, blur=blur)
        rx, ry = torch.autograd.grad((vr * go.double()).sum(), [xr, yr])
        for k in range(B):
            xk, yk = x[k].double(), y[k].double()
            prods = [(xk, xk, ad[k]), (yk, yk, bd[k]), (xk, yk, bd[k]), (yk, xk, ad[k])]
            tols = []
            for q, (r, c, w) in enumerate(prods):
                ref = _conv_ref(kind, r, c, w, blur, unclamped)
                tols.append(_conv_tol(ref, w))
                err = (outs[q][k] - ref).abs().max().item()
                assert err <= tols[q], (N, M, k, q, err, tols[q])
            # the value from the three products: each product's bar, weighted as the value weighs it
            vtol = 1e-4 * abs(vr[k].item()) + 0.5 * tols[0] + 0.5 * tols[1] + tols[2]
            assert abs(val[k].item() - vr[k].item()) <= vtol, (N, M, k, val[k].item(), vr[k].item())
            for got, ref in ((gx[k], rx[k]), (gy[k], ry[k])):
                err = (got - ref).abs().max().item()
                assert err <= 1e-4 * ref.abs().max().item(), (N, M, k, same, err, ref.abs().max().item())


# ------------------------------------------------------------------------------------------------------------------
# SamplesLoss on the small route
# ------------------------------------------------------------------------------------------------------------------
def _rand_weights(g, *shape):
    w = torch.rand(*shape, generator=g) + 0.2
    return w / w.sum(-1, keepdim=True)


def _grads_close(grads, refs, names):
    for got, ref, name in zip(grads, refs, names):
        ref = ref.detach()
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= 1e-4 * max(ref.abs().max().item(), 1e-3), (name, err, ref.abs().max().item())


SINKHORN_CASES = [
    dict(D=4, N=700, M=1300, p=2, backend="tensorized"),
    dict(D=6, N=500, M=900, p=1, backend="tensorized", reach=0.5),
    dict(D=7, N=1500, M=2000, p=2, backend="tensorized", debias=False),
    dict(D=8, N=600, M=400, p=1, backend="online"),
    dict(D=8, N=900, M=700, p=2, backend="online", reach=0.3, debias=False),
    dict(D=6, N=300, M=800, p=2, backend="online", reach=0.5),
    dict(D=7, N=333, M=280, p=1, backend="online", debias=False),
    dict(D=4, N=1100, M=257, p=1, backend="tensorized", reach=0.7, debias=False),
]


@pytest.mark.parametrize("case", SINKHORN_CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_samples_loss_sinkhorn_small_route(case):
    """Value, potentials and the four gradients against the fp64 oracle, D = 4..8 over several column tiles."""
    from geomloss_b200 import SamplesLoss, sinkhorn_small
    from oracle import geomloss_oracle as O

    c = dict(case)
    D, N, M, backend = c.pop("D"), c.pop("N"), c.pop("M"), c.pop("backend")
    assert sinkhorn_small.eligible(N, M, D)
    kw = dict(loss="sinkhorn", blur=0.05, **c)
    g = torch.Generator().manual_seed(N + M + D)
    x, y = _clouds(g, 1, N, M, D, dup=10)
    x, y = x[0], y[0]
    a, b = _rand_weights(g, N), _rand_weights(g, M)
    leaves = [t.to(DEV).requires_grad_(True) for t in (a, x, b, y)]
    val = SamplesLoss(backend=backend, **kw)(*leaves)
    grads = torch.autograd.grad(val, leaves)
    F, G = SamplesLoss(backend=backend, potentials=True, **kw)(*map(_cu, (a, x, b, y)))
    refl = [t.double().requires_grad_(True) for t in (a, x, b, y)]
    if backend == "online":
        sq = [t.unsqueeze(0) for t in refl]
        ref = O.sinkhorn_online(*sq, **c, blur=0.05)[0]
        Fr, Gr = O.sinkhorn_online(*[t.detach().unsqueeze(0) for t in refl], **c, blur=0.05, potentials=True)
    else:
        ref = O.samples_loss(*refl, **kw)
        Fr, Gr = O.samples_loss(*[t.detach() for t in refl], potentials=True, **kw)
    assert abs(val.item() - ref.item()) <= 1e-4 * abs(ref.item()), (val.item(), ref.item())
    for got, r in ((F, Fr), (G, Gr)):
        err = (got.cpu().double().reshape(-1) - r.reshape(-1)).abs().max().item()
        assert err <= 1e-5 * max(1.0, r.abs().max().item()), err
    _grads_close(grads, torch.autograd.grad(ref, refl), ("a", "x", "b", "y"))


def _per_element_refs(loss, a, x, b, y, w, **kw):
    """fp64 value and the four gradients of (vals * w).sum(), one batch element at a time (the Sinkhorn elements share
    the batch's diameter, as the reference measures one over the flattened batch)."""
    from oracle import geomloss_oracle as O

    if loss == "sinkhorn":
        kw = dict(kw, diameter=O.max_diameter(x.reshape(-1, x.shape[-1]).double(), y.reshape(-1, y.shape[-1]).double()))
    vals, grads = [], [[], [], [], []]
    for k in range(x.shape[0]):
        leaves = [t[k].double().requires_grad_(True) for t in (a, x, b, y)]
        v = O.samples_loss(*leaves, loss=loss, **kw)
        for lst, gk in zip(grads, torch.autograd.grad(v * w[k].item(), leaves)):
            lst.append(gk)
        vals.append(v.item())
    return torch.tensor(vals, dtype=torch.float64), [torch.stack(t) for t in grads]


@pytest.mark.parametrize("loss", ["sinkhorn", "gaussian", "laplacian", "energy"])
def test_samples_loss_bench_batch(loss):
    """The bench's small_and_batched workload, B = 64 x N = 500 x D = 3: ceil(500/32) = 16 row tiles x 4 problems x 64
    = 4096 CTAs, the 4-warp iteration kernel.  (vals * w).sum() with distinct w[k]: every element's gradient carries
    its own upstream factor (go_scale[b] / grad_value[b] in the kernels)."""
    from geomloss_b200 import SamplesLoss

    g = torch.Generator().manual_seed(64)
    B, N, D = 64, 500, 3
    x, y = torch.rand(B, N, D, generator=g), torch.rand(B, N, D, generator=g) * 0.9 + 0.1
    a, b = _rand_weights(g, B, N), _rand_weights(g, B, N)
    w = torch.linspace(-1.5, 2.5, B)[torch.randperm(B, generator=g)]
    kw = dict(p=2, blur=0.05) if loss == "sinkhorn" else dict(blur=0.1)
    leaves = [t.to(DEV).requires_grad_(True) for t in (a, x, b, y)]
    vals = SamplesLoss(loss, **kw)(*leaves)
    grads = torch.autograd.grad((vals * w.to(DEV)).sum(), leaves)
    rv, rg = _per_element_refs(loss, a, x, b, y, w, **kw)
    err = (vals.detach().cpu().double() - rv).abs()
    # (kernel losses: + 2e-7 absolute, as test_kernel_losses)
    assert (err <= 1e-4 * rv.abs() + (0.0 if loss == "sinkhorn" else 2e-7)).all(), (err / rv.abs()).max().item()
    for got, ref, name in zip(grads, rg, "axby"):
        err = (got.cpu().double() - ref).abs().flatten(1).max(1).values
        bar = 1e-4 * ref.abs().flatten(1).max(1).values
        assert (err <= bar).all(), (name, (err / bar).max().item())


def _points_sinkhorn_ref(a, x, b, y, p, blur, reach=None, debias=True):
    """fp64 value and potentials of one large problem with row-blocked softmins (no (N, M) matrix is ever formed)."""
    from oracle import geomloss_oracle as O

    diameter, eps, eps_list, rho = O.scaling_parameters(x, y, p, blur, reach, None, 0.5)

    def sm(e, C, h):
        return O.softmin_points(e, C[0], C[1], h.reshape(-1), p=p, row_block=1024)

    f_aa, g_bb, g_ab, f_ba = O.sinkhorn_loop(sm, O.log_weights(a), O.log_weights(b), (x, x), (y, y), (x, y), (y, x),
                                             eps_list, rho, debias=debias)
    pots = [None if t is None else t.reshape(1, -1) for t in (f_aa, g_bb, g_ab, f_ba)]
    value = O.sinkhorn_value(eps, rho, a.reshape(1, -1), b.reshape(1, -1), *pots, debias=debias)
    F, G = O.sinkhorn_value(eps, rho, a, b, *pots, debias=debias, potentials=True)
    return value.item(), F.reshape(-1), G.reshape(-1)


def _check_route(monkeypatch, tiled, a, x, b, y, p, blur, ref, route_ok):
    from geomloss_b200 import SamplesLoss, sinkhorn_small

    if tiled:
        monkeypatch.setattr(sinkhorn_small, "SMALL_MAX", 0)
    N, D = x.shape
    assert sinkhorn_small.eligible(N, y.shape[0], D) == route_ok
    val = SamplesLoss("sinkhorn", p=p, blur=blur)(*map(_cu, (a, x, b, y))).item()
    F, G = SamplesLoss("sinkhorn", p=p, blur=blur, potentials=True)(*map(_cu, (a, x, b, y)))
    monkeypatch.undo()
    rv, Fr, Gr = ref
    errs = [(F.cpu().double().reshape(-1) - Fr).abs().max().item(), (G.cpu().double().reshape(-1) - Gr).abs().max().item()]
    return abs(val - rv) / abs(rv), max(errs)


@pytest.mark.parametrize("D", [3, 8])
def test_routing_boundary(monkeypatch, D):
    """N = 6000 is the last size on the small route, N = 6001 the first on the tiled one: both against fp64."""
    g = torch.Generator().manual_seed(6000 + D)
    x, y = torch.rand(6001, D, generator=g), torch.rand(3000, D, generator=g) * 0.9 + 0.05
    a, b = _rand_weights(g, 6001), _rand_weights(g, 3000)
    for n, small in ((6000, True), (6001, False)):
        an = a[:n] / a[:n].sum()
        ref = _points_sinkhorn_ref(an.double(), x[:n].double(), b.double(), y.double(), 2, 0.05)
        rel, perr = _check_route(monkeypatch, False, an, x[:n].contiguous(), b, y, 2, 0.05, ref, small)
        assert rel <= 1e-4 and perr <= 1e-5, (n, rel, perr)


@pytest.mark.parametrize("shift", [1e2, 1e3])
def test_translated_clouds(monkeypatch, shift):
    """Unit-cube clouds shifted by `shift` in every coordinate (same blur): the Sinkhorn problem is the same, only the
    fp32 coordinates are large.  Both routes must meet the unit-cube bars against fp64 on the same fp32 inputs."""
    g = torch.Generator().manual_seed(int(shift))
    N, M, D = 1000, 900, 3
    x = torch.rand(N, D, generator=g) + shift
    y = torch.rand(M, D, generator=g) * 0.9 + 0.05 + shift
    a, b = _rand_weights(g, N), _rand_weights(g, M)
    ref = _points_sinkhorn_ref(a.double(), x.double(), b.double(), y.double(), 2, 0.05)
    for tiled in (False, True):
        rel, perr = _check_route(monkeypatch, tiled, a, x, b, y, 2, 0.05, ref, not tiled)
        print(f"shift {shift:g} {'tiled' if tiled else 'small'} route: value rel err {rel:.2e}, potentials {perr:.2e}")
        assert rel <= 1e-4 and perr <= 1e-5, ("tiled" if tiled else "small", rel, perr)


# ------------------------------------------------------------------------------------------------------------------
# batches above 65535 (the grid's z limit)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [65536, 70000])
def test_batches_above_grid_limit(B):
    """SamplesLoss on B tiny problems: the Sinkhorn value and per-element-weighted x gradient, and the gaussian value,
    against the batched fp64 oracle."""
    from geomloss_b200 import SamplesLoss
    from oracle import geomloss_oracle as O

    g = torch.Generator().manual_seed(B)
    N, M, D = 5, 8, 3
    x, y = torch.rand(B, N, D, generator=g), torch.rand(B, M, D, generator=g)
    a, b = _rand_weights(g, B, N), _rand_weights(g, B, M)
    w = torch.rand(B, generator=g) * 2 - 0.5
    xg = x.to(DEV).requires_grad_(True)
    vals = SamplesLoss("sinkhorn", p=2, blur=0.1)(_cu(a), xg, _cu(b), _cu(y))
    (gx,) = torch.autograd.grad((vals * w.to(DEV)).sum(), xg)
    xr = x.double().requires_grad_(True)
    ref = O.samples_loss(a.double(), xr, b.double(), y.double(), loss="sinkhorn", p=2, blur=0.1)
    (rx,) = torch.autograd.grad((ref * w.double()).sum(), xr)
    assert vals.shape == (B,)
    err = (vals.detach().cpu().double() - ref.detach()).abs()
    assert (err <= 1e-4 * ref.detach().abs()).all(), (err / ref.detach().abs()).max().item()
    err = (gx.cpu().double() - rx).abs().flatten(1).max(1).values
    assert (err <= 1e-4 * rx.abs().flatten(1).max(1).values).all()
    vg = SamplesLoss("gaussian", blur=0.3)(*map(_cu, (a, x, b, y)))
    rg = O.samples_loss(a.double(), x.double(), b.double(), y.double(), loss="gaussian", blur=0.3)
    tol = 1e-4 * rg.abs() + 2e-7  # 2e-7: the products' 2e-7 sum|w| bar, the weights summing to one
    assert ((vg.cpu().double() - rg).abs() <= tol).all()

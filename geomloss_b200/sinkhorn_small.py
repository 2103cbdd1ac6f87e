"""Sinkhorn divergence on SMALL point clouds (N, M up to a few thousand, batched or not): one kernel launch per
symmetric Sinkhorn iteration instead of twelve.

Same algorithm and autograd contract as sinkhorn.sinkhorn_points / the reference's sinkhorn_tensorized and
sinkhorn_online (src/geomloss/_legacy/sinkhorn_samples.py:74-221, :349-424; loop sinkhorn_divergence.py:258-628),
driven through ``b200ot_sinkhorn_iteration_small`` (csrc/b200ot_small.cu): the four softmins of an iteration — which
all read the OLD potentials — are the y-slices of one grid, batch elements its z-slices; initialisation, every
eps-scaling step and the final gradient-carrying step are one launch each, the gradient w.r.t. both clouds one more.
The reference's own benchmark protocol at N = 1 000 (blur = .05: 8 temperatures) is then 10 + 1 launches.
"""
from __future__ import annotations

import ctypes

import torch

from . import ops
from .sinkhorn import damping, extent_diameter, scaling_parameters, sinkhorn_cost

# largest cloud served by the one-launch-per-iteration kernels; beyond, the tiled TMA kernels win
SMALL_MAX = 6000


def eligible(N, M, D):
    return max(N, M) <= SMALL_MAX and D <= ops.MAX_D


def _views(buf, B, N, M, debias):
    f_ba = buf[: B * N].view(B, N)
    g_ab = buf[B * N: B * (N + M)].view(B, M)
    if not debias:
        return f_ba, g_ab, None, None
    return f_ba, g_ab, buf[B * (N + M): B * (2 * N + M)].view(B, N), buf[B * (2 * N + M):].view(B, M)


def _descent(x, y, a, b, eps_list, rho, p, debias, lh):
    """Initialisation + every eps-scaling step in ONE C call (n_eps + 1 launches enqueued back to back); weights are
    passed as they are, their logarithm (with the reference's -100000 floor) is taken inside the kernel."""
    B, N, D = x.shape
    M = y.shape[1]
    dev = x.device
    bufs = torch.empty(2, B * (2 * N + 2 * M), dtype=torch.float32, device=dev)
    eps_arr = (ctypes.c_double * len(eps_list))(*[float(e) for e in eps_list])
    which = ctypes.c_int32(0)
    ops._call(dev, "b200ot_sinkhorn_loop_small", x, y, a, b, 1, eps_arr, len(eps_list),
              -1.0 if rho is None else float(rho), 1 if debias else 0, bufs[0], bufs[1], ctypes.byref(which), B, N, M,
              D, int(p), lh, launches=len(eps_list) + 1)
    return _views(bufs[0] if which.value else bufs[1], B, N, M, debias)


class _FinalStep(torch.autograd.Function):
    """The last, non-averaged update (sinkhorn_divergence.py:612-623): potentials detached, gradient to x and y only."""

    @staticmethod
    def forward(ctx, x, y, a, b, f_ba, g_ab, f_aa, g_bb, eps, lam, p, debias, lh):
        B, N, D = x.shape
        M = y.shape[1]
        dev = x.device
        new = torch.empty(B * (2 * N + 2 * M), dtype=torch.float32, device=dev)
        n_f_ba, n_g_ab, n_f_aa, n_g_bb = _views(new, B, N, M, debias)
        need = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        lse2 = torch.empty(B * (2 * N + 2 * M), device=dev) if need else None
        ops._call(dev, "b200ot_sinkhorn_iteration_small", x, y, a, b, f_ba, g_ab, f_aa, g_bb, n_f_ba, n_g_ab, n_f_aa,
                  n_g_bb, lse2, B, N, M, D, int(p), float(eps), 0.0, float(lam), 1, lh, launches=1)
        if need:
            ctx.save_for_backward(x, y, a, b, f_ba, g_ab, f_aa if debias else f_ba, g_bb if debias else g_ab, lse2, lh)
            ctx.meta = (float(eps), float(lam), int(p), bool(debias))
        if debias:
            return n_f_ba, n_g_ab, n_f_aa, n_g_bb
        return n_f_ba, n_g_ab

    @staticmethod
    def backward(ctx, *gos):
        x, y, a, b, f_ba, g_ab, f_aa, g_bb, lse2, lh = ctx.saved_tensors
        eps, lam, p, debias = ctx.meta
        B, N, D = x.shape
        M = y.shape[1]
        gos = [None if g is None else g.contiguous() for g in gos] + [None] * (4 - len(gos))
        gx, gy = torch.empty_like(x), torch.empty_like(y)
        ops._call(x.device, "b200ot_sinkhorn_final_bwd_small", x, y, a, b, f_ba, g_ab, f_aa if debias else None,
                  g_bb if debias else None, lse2, *gos, gx, gy, B, N, M, D, p, eps, lam, None, 1, lh, launches=1)
        return (gx, gy) + (None,) * 11


class _FinalValue(torch.autograd.Function):
    """Final update + sinkhorn_cost (sinkhorn_divergence.py:612-623, :165-255) as TWO launches forward and ONE backward:
    the (B,) loss values come from b200ot_sinkhorn_cost_small, which also leaves d value / d potential for the backward
    kernel — no elementwise torch kernels, no autograd graph between the potentials and the value."""

    @staticmethod
    def forward(ctx, x, y, a, b, f_ba, g_ab, f_aa, g_bb, eps, lam, p, debias, rho, eps_final, lh):
        B, N, D = x.shape
        M = y.shape[1]
        dev = x.device
        tot = B * (2 * N + 2 * M)
        need_xy = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        need_w = ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        # one allocation: new potentials | lse2 | d value / d potential | phi, psi
        work = torch.empty(3 * tot + B * (N + M), dtype=torch.float32, device=dev)
        new, lse2, gos, terms = work[:tot], work[tot: 2 * tot], work[2 * tot: 3 * tot], work[3 * tot:]
        value = torch.empty(B, dtype=torch.float32, device=dev)
        n_f_ba, n_g_ab, n_f_aa, n_g_bb = _views(new, B, N, M, debias)
        go_f_ba, go_g_ab, go_f_aa, go_g_bb = _views(gos, B, N, M, debias)
        ad, bd = a.detach(), b.detach()
        ops._call(dev, "b200ot_sinkhorn_iteration_small", x, y, ad, bd, f_ba, g_ab, f_aa, g_bb, n_f_ba, n_g_ab, n_f_aa,
                  n_g_bb, lse2 if need_xy else None, B, N, M, D, int(p), float(eps), 0.0, float(lam), 1, lh,
                  launches=1)
        ops._call(dev, "b200ot_sinkhorn_cost_small", ad, bd, n_f_ba, n_g_ab, n_f_aa, n_g_bb, B, N, M,
                  -1.0 if rho is None else float(rho), float(eps_final), value, go_f_ba if need_xy else None,
                  go_g_ab if need_xy else None, go_f_aa if need_xy and debias else None,
                  go_g_bb if need_xy and debias else None, terms[: B * N] if need_w else None,
                  terms[B * N:] if need_w else None, launches=1)
        if need_xy or need_w:
            ctx.save_for_backward(x, y, ad, bd, f_ba, g_ab, f_aa if debias else f_ba, g_bb if debias else g_ab, work,
                                  lh)
            ctx.meta = (float(eps), float(lam), int(p), bool(debias), need_xy, need_w)
        return value

    @staticmethod
    def backward(ctx, gv):
        x, y, a, b, f_ba, g_ab, f_aa, g_bb, work, lh = ctx.saved_tensors
        eps, lam, p, debias, need_xy, need_w = ctx.meta
        B, N, D = x.shape
        M = y.shape[1]
        tot = B * (2 * N + 2 * M)
        gv = gv.contiguous().float()
        gx = gy = ga = gb = None
        if need_xy:
            lse2, gos = work[tot: 2 * tot], work[2 * tot: 3 * tot]
            go_f_ba, go_g_ab, go_f_aa, go_g_bb = _views(gos, B, N, M, debias)
            gx, gy = torch.empty_like(x), torch.empty_like(y)
            ops._call(x.device, "b200ot_sinkhorn_final_bwd_small", x, y, a, b, f_ba, g_ab, f_aa if debias else None,
                      g_bb if debias else None, lse2, go_f_ba, go_g_ab, go_f_aa, go_g_bb, gx, gy, B, N, M, D, p, eps,
                      lam, gv, 1, lh, launches=1)
        if need_w:
            terms = work[3 * tot:]
            if ctx.needs_input_grad[2]:
                ga = terms[: B * N].view(B, N) * gv[:, None]
            if ctx.needs_input_grad[3]:
                gb = terms[B * N:].view(B, M) * gv[:, None]
        return (gx, gy, ga, gb) + (None,) * 11


def sinkhorn_small(a, x, b, y, p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, debias=True, potentials=False,
                   keops=False, **_ignored):
    """a:(B,N) x:(B,N,D) b:(B,M) y:(B,M,D) float32 CUDA tensors -> (B,) values or the (B,N), (B,M) potentials."""
    if p not in (1, 2):
        raise KeyError(p)
    x, y = ops._f32c(x, "x"), ops._f32c(y, "y")
    a, b = ops._f32c(a, "a"), ops._f32c(b, "b")
    D = x.shape[-1]
    # the batch's bounding box, in one launch: its mid-point is the origin of the kernels' coordinates (whatever the
    # diameter), its diagonal the default diameter (one over the flattened batch, as the reference measures it)
    lh = ops.cloud_extent(x.view(-1, D), y.view(-1, D))
    if diameter is None:
        diameter = extent_diameter(lh)
    diameter, eps_final, eps_list, rho = scaling_parameters(x, y, p, blur, reach, diameter, scaling)
    pk = (p | ops.P_UNCLAMPED) if keops else p
    ad, bd = a.detach(), b.detach()
    with torch.no_grad():
        f_ba, g_ab, f_aa, g_bb = _descent(x.detach(), y.detach(), ad, bd, eps_list, rho, pk, debias, lh)
    eps = eps_list[-1]
    lam = damping(eps, rho)
    if not potentials:
        return _FinalValue.apply(x, y, a, b, f_ba, g_ab, f_aa, g_bb, eps, lam, pk, debias, rho, eps_final, lh)
    outs = _FinalStep.apply(x, y, ad, bd, f_ba, g_ab, f_aa, g_bb, eps, lam, pk, debias, lh)
    n_f_ba, n_g_ab, n_f_aa, n_g_bb = outs if debias else outs + (None, None)
    return sinkhorn_cost(eps_final, rho, a, b, n_f_aa, n_g_bb, n_g_ab, n_f_ba, debias=debias, potentials=True)

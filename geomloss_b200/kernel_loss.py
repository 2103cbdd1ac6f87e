"""Kernel MMD losses (gaussian / laplacian / energy) on point clouds; every matvec is a fused
on-the-fly reduction in libb200ot.so.  Reference: src/geomloss/_legacy/kernel_samples.py:43-146."""
from __future__ import annotations

import torch

from . import ops


class _TwiceGrad(torch.autograd.Function):
    """Identity in forward, doubles the gradient in backward: compensates for the detached right-hand
    side of the two symmetric terms (kernel_samples.py:43-54)."""

    @staticmethod
    def forward(ctx, t):
        return t.view_as(t)

    @staticmethod
    def backward(ctx, g):
        return 2 * g


def kernel_points(a, x, b, y, name=None, blur=0.05, potentials=False, kernel=None, conv=None, keops=False,
                  **_ignored):
    """1/2 |a - b|_k^2 for unbatched a:(N,) x:(N,D) b:(M,) y:(M,D).        kernel_samples.py:92-146

    ``conv(kind, x, y, w, blur, center=)`` defaults to the single-GPU kernel ``ops.kernel_conv_operator`` names for
    D; distributed.py injects the column-sharded one.  ``keops``:
    the reference's use_keops=True convention (backend "online" / "multiscale"): laplacian and energy take
    sqrt(|x-y|^2) without the 1e-8 clamp of the tensorized `distances` (utils.py:56-61 vs kernel_samples.py:71-82)."""
    if kernel is not None:
        raise NotImplementedError("user-supplied kernel callables are outside the CUDA hot path")
    if name not in ops.KERNEL_KINDS:
        # the reference maps loss="hausdorff" to kernel_loss(name=None) and dies with KeyError(None)
        # (samples_loss.py:22-26, kernel_samples.py:107-108): keep the error type, say why.
        raise KeyError(name)
    conv = conv or ops.kernel_conv_operator(x.shape[-1])
    if keops:
        name = ops.KERNEL_KINDS[name] | ops.KERNEL_UNCLAMPED
    dg = _TwiceGrad.apply
    center = ops.default_center(x.detach(), y.detach())
    a_x = conv(name, dg(x), x.detach(), a.detach(), blur, center=center)
    b_y = conv(name, dg(y), y.detach(), b.detach(), blur, center=center)
    b_x = conv(name, x, y, b, blur, center=center)
    if potentials:
        a_y = conv(name, y, x, a, blur, center=center)
        return a_x - b_x, b_y - a_y
    return 0.5 * (dg(a) * a_x).sum() + 0.5 * (dg(b) * b_y).sum() - (a * b_x).sum()


def kernel_points_batched(a, x, b, y, name=None, blur=0.05, potentials=False, kernel=None, keops=False, **_ignored):
    """Batched kernel norms a:(B,N) x:(B,N,D) b:(B,M) y:(B,M,D): the three (four) matvecs take one launch group each
    for the whole batch — the batched operator ``ops.kernel_conv_operator`` names for D, and for D <= 8, where it
    names none, ranges-mode reductions over the block-diagonal stacked problem.
    Reference: kernel_loss on (B, ...) inputs (kernel_samples.py:92-146)."""
    from . import ranges

    if kernel is not None:
        raise NotImplementedError("user-supplied kernel callables are outside the CUDA hot path")
    if name not in ops.KERNEL_KINDS:
        raise KeyError(name)
    B, N, D = x.shape
    M = y.shape[1]
    dev = x.device
    kid = ops.KERNEL_KINDS[name] | (ops.KERNEL_UNCLAMPED if keops else 0)
    xf, yf, af, bf = x.reshape(B * N, D), y.reshape(B * M, D), a.reshape(B * N), b.reshape(B * M)
    center = ops.default_center(xf.detach(), yf.detach())
    dg = _TwiceGrad.apply
    cv = ops.kernel_conv_operator(D, batched=True)
    if cv is not None:
        a_x = cv(kid, dg(x), x.detach(), a.detach(), blur, center=center)
        b_y = cv(kid, dg(y), y.detach(), b.detach(), blur, center=center)
        b_x = cv(kid, x, y, b, blur, center=center)
        if potentials:
            a_y = cv(kid, y, x, a, blur, center=center)
            return a_x - b_x, b_y - a_y
        return 0.5 * (dg(a) * a_x).sum(1) + 0.5 * (dg(b) * b_y).sum(1) - (a * b_x).sum(1)
    p_xx, p_yy = ranges.batch_problem(B, N, N, dev), ranges.batch_problem(B, M, M, dev)
    p_xy, p_yx = ranges.batch_problem(B, N, M, dev), ranges.batch_problem(B, M, N, dev)
    cv = ranges.kernel_conv_ranges
    a_x = cv(kid, dg(xf), xf.detach(), af.detach(), blur, p_xx, None, center=center)
    b_y = cv(kid, dg(yf), yf.detach(), bf.detach(), blur, p_yy, None, center=center)
    b_x = cv(kid, xf, yf, bf, blur, p_xy, p_yx, center=center)
    if potentials:
        a_y = cv(kid, yf, xf, af, blur, p_yx, p_xy, center=center)
        return (a_x - b_x).view(B, N), (b_y - a_y).view(B, M)
    return (0.5 * (dg(af) * a_x).view(B, N).sum(1) + 0.5 * (dg(bf) * b_y).view(B, M).sum(1)
            - (af * b_x).view(B, N).sum(1))

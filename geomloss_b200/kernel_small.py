"""Kernel norms (gaussian / laplacian / energy) on SMALL point clouds, batched or not: the three matvecs of
``kernel_loss`` (src/geomloss/_legacy/kernel_samples.py:92-146) are one launch, the gradient w.r.t. both clouds one
more (csrc/b200ot_small.cu: b200ot_kernel_mmd_small / _bwd_small).  Same autograd result as kernel_loss.kernel_points:
DoubleGrad on the symmetric terms, detached right-hand sides, d value / d a = a_x - b_x, d value / d b = b_y - a_y."""
from __future__ import annotations

import torch

from . import ops
from .sinkhorn_small import SMALL_MAX  # noqa: F401  (one threshold for both small paths)


def _forward(kid, a, x, b, y, blur, want_ay):
    B, N, D = x.shape
    M = y.shape[1]
    dev = x.device
    a_x, b_y, b_x = torch.empty(B, N, device=dev), torch.empty(B, M, device=dev), torch.empty(B, N, device=dev)
    a_y = torch.empty(B, M, device=dev) if want_ay else None
    ops._call(dev, "b200ot_kernel_mmd_small", x, y, a, b, a_x, b_y, b_x, a_y, B, N, M, D, int(kid), float(blur),
              launches=1)
    return a_x, b_y, b_x, a_y


class _MMDValue(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, x, b, y, kid, blur):
        need_b = ctx.needs_input_grad[2]
        a_x, b_y, b_x, a_y = _forward(kid, a, x, b, y, blur, want_ay=need_b)
        B, N, _ = x.shape
        val = torch.empty(B, dtype=torch.float32, device=x.device)
        ops._call(x.device, "b200ot_kernel_mmd_value_small", a, b, a_x, b_y, b_x, B, N, y.shape[1], val, launches=1)
        ctx.save_for_backward(a, x, b, y, a_x, b_y, b_x, a_y if need_b else a_x)
        ctx.meta = (int(kid), float(blur), need_b)
        return val

    @staticmethod
    def backward(ctx, go):
        a, x, b, y, a_x, b_y, b_x, a_y = ctx.saved_tensors
        kid, blur, need_b = ctx.meta
        go = go.contiguous()
        ga = gx = gb = gy = None
        if ctx.needs_input_grad[0]:
            ga = go[:, None] * (a_x - b_x)
        if need_b:
            gb = go[:, None] * (b_y - a_y)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[3]:
            B, N, D = x.shape
            M = y.shape[1]
            gx, gy = torch.empty_like(x), torch.empty_like(y)
            ops._call(x.device, "b200ot_kernel_mmd_bwd_small", x, y, a, b, go, gx, gy, B, N, M, D, kid, blur,
                      launches=1)
        return ga, gx, gb, gy, None, None


def kernel_small(a, x, b, y, name=None, blur=0.05, potentials=False, kernel=None, keops=False, **_ignored):
    """a:(B,N) x:(B,N,D) b:(B,M) y:(B,M,D) float32 CUDA tensors -> (B,) values, or the potentials (B,N), (B,M)."""
    if kernel is not None:
        raise NotImplementedError("user-supplied kernel callables are outside the CUDA hot path")
    if name not in ops.KERNEL_KINDS:
        raise KeyError(name)
    kid = ops.KERNEL_KINDS[name] | (ops.KERNEL_UNCLAMPED if keops else 0)
    x, y, a, b = ops._f32c(x, "x"), ops._f32c(y, "y"), ops._f32c(a, "a"), ops._f32c(b, "b")
    if potentials:
        a_x, b_y, b_x, a_y = _forward(kid, a.detach(), x.detach(), b.detach(), y.detach(), blur, want_ay=True)
        return a_x - b_x, b_y - a_y
    return _MMDValue.apply(a, x, b, y, kid, blur)

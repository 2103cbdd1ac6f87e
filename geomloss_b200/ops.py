"""Torch-facing wrappers of the C-ABI kernels: device buffers in, device buffers out, autograd wired.

Mirrors the reference's operator seam — ``softmin(eps, C_xy, h_y) -> f_x`` with ``C_xy = (x, y)``
(src/geomloss/_legacy/sinkhorn_samples.py:337-346, sinkhorn_divergence.py:291-303) and the kernel
matvecs of ``kernel_loss`` (kernel_samples.py:128-137) — but every call lands in libb200ot.so.
PyTorch is used for memory, streams and autograd bookkeeping only.
"""
from __future__ import annotations

import ctypes
from typing import Callable, NamedTuple, Optional

import torch

from . import _lib

KERNEL_KINDS = {"gaussian": 0, "laplacian": 1, "energy": 2}
# flags of include/b200ot.h: the pykeops convention for sqrt(|x-y|^2) (no 1e-8 clamp, zero gradient at 0), used by
# the reference's "online" / "multiscale" backends; the plain values are the "tensorized" convention
P_UNCLAMPED = 0x100
KERNEL_UNCLAMPED = 0x100
MAX_D = 8  # dimensions instantiated in this build of libb200ot.so (supported_simt_dim in csrc/host_util.cuh)

# Number of kernels of libb200ot.so enqueued so far by this process (bench.py reports the delta over its
# timed region as `gpu_launches`).  Every one-call entry point is pack + partial reduction + finalize.
_launches = 0


def count_launches(n: int):
    global _launches
    _launches += n


# NVTX ranges around every reduction (SURVEY.md section 5: the reference's only tracing hook is the torch profiler in
# examples/performances/plot_profile.py).  Off by default; B200OT_NVTX=1 brackets each softmin / kernel matvec so that a
# timeline (nsys, or ncu --nvtx --nvtx-include) shows the Sinkhorn loop iteration by iteration.
import os as _os

NVTX = _os.environ.get("B200OT_NVTX", "0") == "1"


class nvtx_range:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if NVTX:
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if NVTX:
            torch.cuda.nvtx.range_pop()


def launches() -> int:
    return _launches


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _call(dev, name, *args, launches):
    """Enqueue the C entry ``name`` on the current stream of ``dev``: tensors travel as device pointers, every other
    argument (None, numbers, ctypes objects) as it is, the stream last.  A failure raises ``B200OTError``; the entry's
    ``launches`` kernels are counted."""
    fn = getattr(_lib.lib(), name)
    ptrs = [_ptr(a) if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(dev):
        rc = fn(*ptrs, _stream(dev))
    _lib.check(rc, name)
    count_launches(launches)


def _query(dev, name, *args):
    """The answer of the size query ``name`` for ``dev``: split counts, and so scratch sizes, follow the SM count of
    the current device, so the query runs with ``dev`` current."""
    with torch.cuda.device(dev):
        return getattr(_lib.lib(), name)(*args)


def _f32c(t, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.B200OTError(f"{name} must live on a CUDA device (geomloss_b200 has no CPU path), got {t.device}")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32 (the engine computes in fp32), got {t.dtype}")
    return t.contiguous()


MAX_D_TC = 64  # softmin (p = 2, and p = 1 through softmin_l1) and the three kernel convolutions, forward + row
# gradients: tensor-core path, 8 < D <= 64


def _check_clouds(x, y, max_d=None):
    max_d = MAX_D if max_d is None else max_d
    if x.dim() != 2 or y.dim() != 2 or x.shape[1] != y.shape[1]:
        raise ValueError(f"expected x:(N,D), y:(M,D); got {tuple(x.shape)}, {tuple(y.shape)}")
    if x.shape[0] == 0 or y.shape[0] == 0:
        raise ValueError("empty point cloud")
    if x.shape[1] > max_d:
        raise NotImplementedError(f"D = {x.shape[1]} > {max_d}: not instantiated in this build (CUDA-core kernels "
                                  f"serve every operator for D <= {MAX_D}; the tensor-core kernels serve the p = 2 "
                                  f"softmin and the gaussian, laplacian and energy kernel convolutions, forward and row "
                                  f"gradients, up to D = {MAX_D_TC}; the p = 1 softmin above D = {MAX_D} is "
                                  f"ops.softmin_l1 / softmin_l1_raw)")
    if x.device != y.device:
        raise ValueError("x and y must be on the same device")


_scratch_cache: dict = {}


def _scratch(nbytes: int, dev, tag: str):
    """Per-(device, stream, tag) scratch buffer, grown geometrically; stream-ordered reuse is safe because
    every kernel that touches it is enqueued on that same stream."""
    key = (dev, torch.cuda.current_stream(dev).cuda_stream, tag)
    buf = _scratch_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=dev)
        _scratch_cache[key] = buf
    return buf


_extent_scratch: dict = {}


def cloud_extent(x, y=None):
    """(2, D) device tensor [minima; maxima] over the rows of x (and y) in ONE launch (b200ot_cloud_extent), or None
    when the clouds are not float32 CUDA tensors with D <= MAX_D (callers then use torch reductions)."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and 1 <= x.shape[1] <= MAX_D and x.shape[0] > 0):
        return None
    if y is not None and not (y.is_cuda and y.dtype == torch.float32 and y.dim() == 2 and y.shape[1] == x.shape[1]
                              and y.device == x.device):
        return None
    x = x.detach().contiguous()
    y = None if y is None or y.shape[0] == 0 else y.detach().contiguous()
    dev = x.device
    key = (dev, torch.cuda.current_stream(dev).cuda_stream)
    scratch = _extent_scratch.get(key)
    if scratch is None:  # zero once: the kernel's ticket counter returns to zero after every launch
        scratch = _extent_scratch[key] = torch.zeros(_lib.lib().b200ot_cloud_extent_scratch_bytes(), dtype=torch.uint8,
                                                     device=dev)
    out = torch.empty(2, x.shape[1], dtype=torch.float32, device=dev)
    _call(dev, "b200ot_cloud_extent", x, x.shape[0], y, 0 if y is None else y.shape[0], x.shape[1], out, scratch,
          scratch.numel(), launches=1)
    return out


def default_center(x, y):
    """Mid-point of the joint bounding box: the origin of the |x|^2 - 2x.y + |y|^2 expansion."""
    lh = cloud_extent(x, y)
    if lh is not None:
        return (0.5 * (lh[0] + lh[1])).contiguous()
    lo = torch.minimum(x.min(0).values, y.min(0).values)
    hi = torch.maximum(x.max(0).values, y.max(0).values)
    return (0.5 * (lo + hi)).float().contiguous()


# ------------------------------------------------------------------------------------------------
# softmin
# ------------------------------------------------------------------------------------------------


def softmin_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                beta=1.0, out=None, want_lse2=False):
    """One fused launch group: ``out <- alpha_old*out_old + beta*softmin(eps, (x, y), h_a + h_scale_b*h_b)``.

    No autograd.  Returns ``(out, lse2 | None)``.
    """
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, out_old = _f32c(center, "center"), _f32c(out_old, "out_old")
    _check_clouds(x, y, MAX_D_TC if (p & 0xFF) == 2 else MAX_D)
    N, D = x.shape
    M = y.shape[0]
    if h_a.numel() != M or (h_b is not None and h_b.numel() != M):
        raise ValueError("h must have one entry per column")
    dev = x.device
    with nvtx_range(f"b200ot.softmin N={N} M={M} D={D} eps={float(eps):.3g}"):
        if out is None:
            out = torch.empty(N, dtype=torch.float32, device=dev)
        lse2 = torch.empty(N, dtype=torch.float32, device=dev) if want_lse2 else None
        scratch = _scratch(_query(dev, "b200ot_softmin_scratch_bytes", N, M, D), dev, "softmin")
        _call(dev, "b200ot_softmin_fwd", x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, N, M, D, int(p), float(eps), scratch, scratch.numel(), launches=3)
    return out, lse2


def softmin_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x of <grad_out, softmin(eps, (x, y), h)> with y, h constant (b200ot_softmin_bwd_x)."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, grad_out = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(grad_out, "grad_out")
    _check_clouds(x, y, MAX_D_TC if (p & 0xFF) == 2 else MAX_D)
    N, D = x.shape
    M = y.shape[0]
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _scratch(_query(dev, "b200ot_softmin_scratch_bytes", N, M, D), dev, "softmin")
    _call(dev, "b200ot_softmin_bwd_x", x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, N, M, D, int(p),
          float(eps), scratch, scratch.numel(), launches=3)
    return gx


def plan_apply_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    """``out[i, k] = row_factor_i * sum_j w_ij v[j, k]`` with ``w_ij = softmax_j(h_j - |x_i - y_j|^2 / (2 eps))`` and
    ``h = h_a + h_scale_b * h_b`` (b200ot_plan_apply): the softmin's weights applied to a value matrix without ever
    forming them.  ``lse2`` is ``softmin_raw(..., want_lse2=True)[1]`` for the same arguments; ``v`` is (M,) or (M, K),
    any sign, any strides.  p = 2, D <= 64.  One pass over the pairs per slab of value columns (8 for D <= 8, 64
    above).  No autograd.  Returns (N,) or (N, K)."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, v = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(v, "v")
    row_factor = _f32c(row_factor, "row_factor")
    _check_clouds(x, y, MAX_D_TC)
    N, D = x.shape
    M = y.shape[0]
    if v.dim() not in (1, 2) or v.shape[0] != M or v.numel() == 0:
        raise ValueError(f"v must be (M,) or (M, K) with M = {M} and K >= 1, got {tuple(v.shape)}")
    if h_a.numel() != M or (h_b is not None and h_b.numel() != M):
        raise ValueError("h must have one entry per column")
    if lse2.numel() != N or (row_factor is not None and row_factor.numel() != N):
        raise ValueError("lse2 and row_factor must have one entry per row")
    K = 1 if v.dim() == 1 else v.shape[1]
    dev = x.device
    with nvtx_range(f"b200ot.plan_apply N={N} M={M} D={D} K={K}"):
        out = torch.empty((N,) if v.dim() == 1 else (N, K), dtype=torch.float32, device=dev)
        scratch = _scratch(_query(dev, "b200ot_plan_apply_scratch_bytes", N, M, D, K), dev, "plan_apply")
        slabs = -(-K // (8 if D <= MAX_D else 64))
        _call(dev, "b200ot_plan_apply", x, y, h_a, h_b, float(h_scale_b), center, lse2, v, row_factor, out, N, M, D, K,
              2, float(eps), scratch, scratch.numel(), launches=1 + 3 * slabs)
    return out


class _Softmin(torch.autograd.Function):
    """``scale_out * softmin(eps, (x, y), h_a + h_scale_b*h_b)`` with the reference's autograd contract: the gradient
    flows to the row cloud x only; y and h are treated as constants (they are ``.detach()``-ed at every call site of
    the reference: sinkhorn_samples.py:392-393, sinkhorn_divergence.py:616-623).

    ``fwd`` and ``bwd`` are the forward and row-gradient operators of one kind of problem (one problem, a batch, the
    p = 1 cost, ranges, column shards):
        fwd(eps, x, y, h_a, h_b, h_scale_b, *, p, center, beta, want_lse2) -> (out, lse2)
        bwd(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p, center) -> grad_x"""

    @staticmethod
    def forward(ctx, fwd, bwd, x, y, h_a, h_b, h_scale_b, eps, p, center, scale_out):
        need_grad = ctx.needs_input_grad[2]
        out, lse2 = fwd(eps, x, y, h_a, h_b, h_scale_b, p=p, center=center, beta=scale_out, want_lse2=need_grad)
        if need_grad:
            ctx.bwd = bwd
            ctx.save_for_backward(x, y, h_a, h_b, center, lse2)
            ctx.meta = (float(h_scale_b), float(eps), int(p), float(scale_out))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, y, h_a, h_b, center, lse2 = ctx.saved_tensors
        h_scale_b, eps, p, scale_out = ctx.meta
        gx = ctx.bwd(eps, x, y, h_a, h_b, h_scale_b, lse2, (grad_out * scale_out).contiguous(), p=p, center=center)
        return (None, None, gx) + (None,) * 8


def _softmin_apply(fwd, bwd, eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out):
    """``_Softmin`` on the row cloud x, the columns and their potentials detached."""
    return _Softmin.apply(fwd, bwd, x, y.detach(), h_a.detach(), None if h_b is None else h_b.detach(), h_scale_b, eps,
                          p, center, scale_out)


def softmin(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) ``scale_out * softmin(eps, (x, y.detach()), (h_a + h_scale_b*h_b).detach())``."""
    return _softmin_apply(softmin_raw, softmin_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out)


# ------------------------------------------------------------------------------------------------
# kernel convolutions
# ------------------------------------------------------------------------------------------------


def kind_id(kind):
    """Kernel name (tensorized convention) or an integer kind, possibly or-ed with KERNEL_UNCLAMPED."""
    return KERNEL_KINDS[kind] if isinstance(kind, str) else int(kind)


def kernel_conv_raw(kind, x, y, w, blur, *, center=None):
    """out_i = sum_j k(x_i, y_j) w_j, no autograd."""
    x, y, w, center = _f32c(x, "x"), _f32c(y, "y"), _f32c(w, "w"), _f32c(center, "center")
    _check_clouds(x, y, MAX_D_TC)
    N, D = x.shape
    M = y.shape[0]
    if w.numel() != M:
        raise ValueError("w must have one entry per column")
    dev = x.device
    with nvtx_range(f"b200ot.kernel_conv kind={kind} N={N} M={M} D={D}"):
        out = torch.empty(N, dtype=torch.float32, device=dev)
        scratch = _scratch(_query(dev, "b200ot_kernel_conv_scratch_bytes", N, M, D), dev, "conv")
        _call(dev, "b200ot_kernel_conv_fwd", x, y, w, center, out, N, M, D, kind_id(kind), float(blur), scratch,
              scratch.numel(), launches=3)
    return out


def kernel_conv_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    x, y, w, center = _f32c(x, "x"), _f32c(y, "y"), _f32c(w, "w"), _f32c(center, "center")
    grad_out = _f32c(grad_out, "grad_out")
    _check_clouds(x, y, MAX_D_TC)
    N, D = x.shape
    M = y.shape[0]
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _scratch(_query(dev, "b200ot_kernel_conv_scratch_bytes", N, M, D), dev, "conv")
    _call(dev, "b200ot_kernel_conv_bwd_x", x, y, w, center, grad_out, gx, N, M, D, kind_id(kind), float(blur), scratch,
          scratch.numel(), launches=3)
    return gx


def kernel_conv_value_and_grad_rows(kind, x, y, w, blur, *, center=None):
    """(out, grad_unit) with out_i = sum_j k(x_i, y_j) w_j and grad_unit[i] = sum_j w_j dk(x_i, y_j)/dx_i from ONE
    pass over the pairs (gaussian kernel; b200ot_kernel_conv_fwd_bwd_x).  No autograd."""
    x, y, w, center = _f32c(x, "x"), _f32c(y, "y"), _f32c(w, "w"), _f32c(center, "center")
    if (kind_id(kind) & 0xFF) != 0:
        raise ValueError("the one-pass value + row gradient exists for the gaussian kernel only")
    _check_clouds(x, y, MAX_D_TC)
    N, D = x.shape
    M = y.shape[0]
    if w.numel() != M:
        raise ValueError("w must have one entry per column")
    dev = x.device
    with nvtx_range(f"b200ot.kernel_conv value+grad kind={kind} N={N} M={M} D={D}"):
        out = torch.empty(N, dtype=torch.float32, device=dev)
        gunit = torch.empty_like(x)
        scratch = _scratch(_query(dev, "b200ot_kernel_conv_scratch_bytes", N, M, D), dev, "conv")
        _call(dev, "b200ot_kernel_conv_fwd_bwd_x", x, y, w, center, out, gunit, N, M, D, kind_id(kind), float(blur),
              scratch, scratch.numel(), launches=3)
    return out, gunit


# A gaussian matvec whose ROW cloud requires a gradient is evaluated by the row-gradient reduction, which accumulates
# sum_j w_j k_ij next to sum_j w_j k_ij y_j anyway: value and unit gradient come from one pass over the N x M pairs and
# backward() is an N x D elementwise product — 3 reductions instead of 5 for SamplesLoss("gaussian")(x, y) + grad w.r.t.
# x (tools/ab_tc_route.py part C times both evaluations).  The price: a forward whose result is never differentiated although x requires a
# gradient pays the (slower) gradient reduction, and (N, D) floats are kept until backward.
# B200OT_FUSED_CONV_GRAD=0 restores the two-pass evaluation.
FUSED_CONV_GRAD = _os.environ.get("B200OT_FUSED_CONV_GRAD", "1") == "1"


class _ConvOps(NamedTuple):
    """The operators of one kind of kernel matvec problem:
        raw(kind, x, y, w, blur, *, center) -> out
        grad_rows(kind, x, y, w, blur, grad_out, *, center) -> grad_x
        value_and_grad_rows(kind, x, y, w, blur, *, center) -> (out, grad_unit), or None"""
    raw: Callable
    grad_rows: Callable
    value_and_grad_rows: Optional[Callable] = None


class _KernelConv(torch.autograd.Function):
    """out = K(x, y) @ w, differentiable w.r.t. x, y and w.  ``rows`` holds the operators of the problem (x against
    y), ``cols`` those of its transpose (y against x): kernels are symmetric, so the y- and w-gradients are the same
    reductions with the roles of the clouds swapped.  ``cols`` is None when the transpose is not available (ranges
    problems built without it); ``fused``: value and unit row gradient from one pass (``rows.value_and_grad_rows``)."""

    @staticmethod
    def forward(ctx, rows, cols, x, y, w, kind, blur, center, fused):
        if fused:
            out, gunit = rows.value_and_grad_rows(kind, x, y, w, blur, center=center)
        else:
            out, gunit = rows.raw(kind, x, y, w, blur, center=center), None
        ctx.ops = (rows, cols)
        ctx.save_for_backward(x, y, w, center, gunit)
        ctx.meta = (kind, float(blur))
        return out

    @staticmethod
    def backward(ctx, go):
        x, y, w, center, gunit = ctx.saved_tensors
        rows, cols = ctx.ops
        kind, blur = ctx.meta
        go = go.contiguous()
        gx = gy = gw = None
        if ctx.needs_input_grad[2]:
            if gunit is not None:
                gx = go.unsqueeze(-1) * gunit
            else:
                gx = rows.grad_rows(kind, x, y, w, blur, go, center=center)
        if (ctx.needs_input_grad[3] or ctx.needs_input_grad[4]) and cols is None:
            raise RuntimeError("the transposed ranges problem is needed for gradients w.r.t. y / w")
        if ctx.needs_input_grad[3]:
            # d/dy_j sum_i go_i k(x_i, y_j) w_j = w_j * sum_i go_i dk(y_j, x_i)/dy_j
            gy = cols.grad_rows(kind, y, x, go, blur, w, center=center)
        if ctx.needs_input_grad[4]:
            gw = cols.raw(kind, y, x, go, blur, center=center).view_as(w)
        return None, None, gx, gy, gw, None, None, None, None


def _fused(kind, x):
    return bool(FUSED_CONV_GRAD and torch.is_grad_enabled() and x.requires_grad and (kind_id(kind) & 0xFF) == 0)


def kernel_conv(kind, x, y, w, blur, *, center=None):
    dense = _ConvOps(kernel_conv_raw, kernel_conv_grad_rows, kernel_conv_value_and_grad_rows)
    return _KernelConv.apply(dense, dense, x, y, w, kind, blur, center, _fused(kind, x))


# ------------------------------------------------------------------------------------------------
# batches of B problems in the tensor-core dimensions (8 < D <= 64): x (B,N,D), y (B,M,D), per-column vectors (B,M),
# per-row vectors (B,N); element b of the rows is reduced over element b of the columns only, the whole batch in one
# launch group per call (b200ot_*_batched).  Same contracts as the one-problem operators above.
# ------------------------------------------------------------------------------------------------
def _check_batch(x, y):
    if x.dim() != 3 or y.dim() != 3 or x.shape[0] != y.shape[0] or x.shape[2] != y.shape[2]:
        raise ValueError(f"expected x:(B,N,D), y:(B,M,D); got {tuple(x.shape)}, {tuple(y.shape)}")
    B, N, D = x.shape
    M = y.shape[1]
    if B == 0 or N == 0 or M == 0:
        raise ValueError("empty batch or point cloud")
    if not MAX_D < D <= MAX_D_TC:
        raise NotImplementedError(f"the batched tensor-core operators serve {MAX_D} < D <= {MAX_D_TC}, got D = {D} "
                                  f"(batches with D <= {MAX_D} run as block-diagonal ranges problems, ranges.py)")
    if x.device != y.device:
        raise ValueError("x and y must be on the same device")
    return B, N, M, D


def _per_point(t, n, name):
    if t is not None and t.numel() != n:
        raise ValueError(f"{name} must have one entry per point of its cloud ({n}), got {tuple(t.shape)}")


def _batched_scratch(B, N, M, D, dev):
    return _scratch(_query(dev, "b200ot_batched_scratch_bytes", B, N, M, D), dev, "batched")


def softmin_batched_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                        beta=1.0, out=None, want_lse2=False):
    """``softmin_raw`` on a batch: out (B,N) <- alpha_old*out_old + beta*softmin(eps, (x[b], y[b]), h[b]).  p = 2 only.
    No autograd.  Returns ``(out, lse2 | None)``."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, out_old = _f32c(center, "center"), _f32c(out_old, "out_old")
    B, N, M, D = _check_batch(x, y)
    if (p & 0xFF) != 2:
        raise NotImplementedError(f"p = {p & 0xFF}: the batched softmin exists for p = 2 only (tensor cores)")
    _per_point(h_a, B * M, "h_a")
    _per_point(h_b, B * M, "h_b")
    _per_point(out_old, B * N, "out_old")
    dev = x.device
    with nvtx_range(f"b200ot.softmin_batched B={B} N={N} M={M} D={D} eps={float(eps):.3g}"):
        if out is None:
            out = torch.empty(B, N, dtype=torch.float32, device=dev)
        lse2 = torch.empty(B, N, dtype=torch.float32, device=dev) if want_lse2 else None
        scratch = _batched_scratch(B, N, M, D, dev)
        _call(dev, "b200ot_softmin_fwd_batched", x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, B, N, M, D, int(p), float(eps), scratch, scratch.numel(), launches=3)
    return out, lse2


def softmin_batched_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x (B,N,D) of <grad_out, softmin_batched(eps, x, y, h)> with y, h constant (b200ot_softmin_bwd_x_batched)."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, grad_out = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(grad_out, "grad_out")
    B, N, M, D = _check_batch(x, y)
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _batched_scratch(B, N, M, D, dev)
    _call(dev, "b200ot_softmin_bwd_x_batched", x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, B, N, M,
          D, int(p), float(eps), scratch, scratch.numel(), launches=3)
    return gx


def softmin_batched(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) batched softmin, (B,N): ``softmin`` element by element."""
    return _softmin_apply(softmin_batched_raw, softmin_batched_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center,
                          scale_out)


def _conv_batched_args(x, y, w, center):
    x, y, w, center = _f32c(x, "x"), _f32c(y, "y"), _f32c(w, "w"), _f32c(center, "center")
    B, N, M, D = _check_batch(x, y)
    _per_point(w, B * M, "w")
    return x, y, w, center, B, N, M, D


def kernel_conv_batched_raw(kind, x, y, w, blur, *, center=None):
    """out (B,N), out[b, i] = sum_j k(x[b, i], y[b, j]) w[b, j], no autograd."""
    x, y, w, center, B, N, M, D = _conv_batched_args(x, y, w, center)
    dev = x.device
    with nvtx_range(f"b200ot.kernel_conv_batched kind={kind} B={B} N={N} M={M} D={D}"):
        out = torch.empty(B, N, dtype=torch.float32, device=dev)
        scratch = _batched_scratch(B, N, M, D, dev)
        _call(dev, "b200ot_kernel_conv_fwd_batched", x, y, w, center, out, B, N, M, D, kind_id(kind), float(blur),
              scratch, scratch.numel(), launches=3)
    return out


def kernel_conv_batched_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    x, y, w, center, B, N, M, D = _conv_batched_args(x, y, w, center)
    grad_out = _f32c(grad_out, "grad_out")
    _per_point(grad_out, B * N, "grad_out")
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _batched_scratch(B, N, M, D, dev)
    _call(dev, "b200ot_kernel_conv_bwd_x_batched", x, y, w, center, grad_out, gx, B, N, M, D, kind_id(kind),
          float(blur), scratch, scratch.numel(), launches=3)
    return gx


def kernel_conv_batched_value_and_grad_rows(kind, x, y, w, blur, *, center=None):
    """``kernel_conv_value_and_grad_rows`` on a batch (gaussian only): (out (B,N), grad_unit (B,N,D))."""
    if (kind_id(kind) & 0xFF) != 0:
        raise ValueError("the one-pass value + row gradient exists for the gaussian kernel only")
    x, y, w, center, B, N, M, D = _conv_batched_args(x, y, w, center)
    dev = x.device
    with nvtx_range(f"b200ot.kernel_conv_batched value+grad B={B} N={N} M={M} D={D}"):
        out = torch.empty(B, N, dtype=torch.float32, device=dev)
        gunit = torch.empty_like(x)
        scratch = _batched_scratch(B, N, M, D, dev)
        _call(dev, "b200ot_kernel_conv_fwd_bwd_x_batched", x, y, w, center, out, gunit, B, N, M, D, kind_id(kind),
              float(blur), scratch, scratch.numel(), launches=3)
    return out, gunit


def kernel_conv_batched(kind, x, y, w, blur, *, center=None):
    """out (B,N) = K(x[b], y[b]) @ w[b] for every b, differentiable w.r.t. x, y and w."""
    batched = _ConvOps(kernel_conv_batched_raw, kernel_conv_batched_grad_rows, kernel_conv_batched_value_and_grad_rows)
    return _KernelConv.apply(batched, batched, x, y, w, kind, blur, center, _fused(kind, x))


# ------------------------------------------------------------------------------------------------
# the p = 1 softmin in the tensor-core dimensions (8 < D <= 64): f_i = -eps log sum_j exp(h_j - |x_i - y_j| / eps), one
# problem (N,D) / (M,D) or a batch (B,N,D) / (B,M,D) in one launch group per call (b200ot_softmin_l1_*).
# ------------------------------------------------------------------------------------------------
def _l1_args(x, y, p):
    if (p & 0xFF) != 1 or (p & ~(0xFF | P_UNCLAMPED)) != 0:
        raise ValueError(f"softmin_l1 computes the p = 1 softmin (p = 1 or 1 | P_UNCLAMPED), got p = {p}")
    if x.dim() == 2 and y.dim() == 2:
        return False, _check_batch(x.unsqueeze(0), y.unsqueeze(0))
    return True, _check_batch(x, y)


def softmin_l1_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=1, center=None, out_old=None, alpha_old=0.0,
                   beta=1.0, out=None, want_lse2=False):
    """``softmin_batched_raw`` for the cost |x - y|: out <- alpha_old*out_old + beta*softmin(eps, (x, y), h), (N,) for
    (N,D) clouds, (B,N) for (B,N,D) ones.  No autograd.  Returns ``(out, lse2 | None)``."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, out_old = _f32c(center, "center"), _f32c(out_old, "out_old")
    batched, (B, N, M, D) = _l1_args(x, y, p)
    _per_point(h_a, B * M, "h_a")
    _per_point(h_b, B * M, "h_b")
    _per_point(out_old, B * N, "out_old")
    shape = (B, N) if batched else (N,)
    dev = x.device
    with nvtx_range(f"b200ot.softmin_l1 B={B} N={N} M={M} D={D} eps={float(eps):.3g}"):
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=dev)
        lse2 = torch.empty(shape, dtype=torch.float32, device=dev) if want_lse2 else None
        scratch = _scratch(_query(dev, "b200ot_softmin_l1_scratch_bytes", B, N, M, D), dev, "softmin_l1")
        # coordinate maximum, two packs, reduction, finalize
        _call(dev, "b200ot_softmin_l1_fwd", x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, B, N, M, D, int(p), float(eps), scratch, scratch.numel(), launches=5)
    return out, lse2


def softmin_l1_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=1, center=None):
    """grad_x, shaped like x, of <grad_out, softmin_l1(eps, x, y, h)> with y, h constant (b200ot_softmin_l1_bwd_x)."""
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, grad_out = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(grad_out, "grad_out")
    _, (B, N, M, D) = _l1_args(x, y, p)
    _per_point(grad_out, B * N, "grad_out")
    _per_point(lse2, B * N, "lse2")
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _scratch(_query(dev, "b200ot_softmin_l1_scratch_bytes", B, N, M, D), dev, "softmin_l1")
    # coordinate maximum, two packs, reduction, finalize
    _call(dev, "b200ot_softmin_l1_bwd_x", x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, B, N, M, D,
          int(p), float(eps), scratch, scratch.numel(), launches=5)
    return gx


def softmin_l1(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=1, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) ``scale_out * softmin_l1_raw(...)``, for (N,D) or (B,N,D) clouds."""
    return _softmin_apply(softmin_l1_raw, softmin_l1_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out)


# ------------------------------------------------------------------------------------------------
# above D = 64 (64 < D <= MAX_D_WIDE): the p = 2 and p = 1 softmins and the three kernel convolutions on the K-slab
# tensor-core kernels (csrc/tcwide.cuh, b200ot_wide_*), one problem (N,D) / (M,D) or a batch (B,N,D) / (B,M,D) in one
# launch group per call.  Same contracts as the one-problem and batched operators above.
# ------------------------------------------------------------------------------------------------
MAX_D_WIDE = 1024  # B200OT_MAX_D_WIDE


def _wide_args(x, y):
    """(batched, (B, N, M, D)) of (N,D) / (M,D) or (B,N,D) / (B,M,D) clouds in the wide dimensions."""
    batched = not (x.dim() == 2 and y.dim() == 2)
    xb, yb = (x, y) if batched else (x.unsqueeze(0), y.unsqueeze(0))
    if xb.dim() != 3 or yb.dim() != 3 or xb.shape[0] != yb.shape[0] or xb.shape[2] != yb.shape[2]:
        raise ValueError(f"expected x:(N,D), y:(M,D) or x:(B,N,D), y:(B,M,D); got {tuple(x.shape)}, {tuple(y.shape)}")
    B, N, D = xb.shape
    M = yb.shape[1]
    if B == 0 or N == 0 or M == 0:
        raise ValueError("empty batch or point cloud")
    if not MAX_D_TC < D <= MAX_D_WIDE:
        raise NotImplementedError(f"the wide tensor-core operators serve {MAX_D_TC} < D <= {MAX_D_WIDE}, got D = {D} "
                                  f"(no kernel of this build reduces clouds above D = {MAX_D_WIDE})")
    if x.device != y.device:
        raise ValueError("x and y must be on the same device")
    return batched, (B, N, M, D)


def _wide_scratch(B, N, M, D, dev):
    return _scratch(_query(dev, "b200ot_wide_scratch_bytes", B, N, M, D), dev, "wide")


def softmin_wide_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                     beta=1.0, out=None, want_lse2=False):
    """``softmin_raw`` above D = 64 for p = 1 or 2 (| P_UNCLAMPED): out <- alpha_old*out_old + beta*softmin(eps, (x, y),
    h), (N,) for (N,D) clouds, (B,N) for (B,N,D) ones.  No autograd.  Returns ``(out, lse2 | None)``."""
    batched, (B, N, M, D) = _wide_args(x, y)
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, out_old = _f32c(center, "center"), _f32c(out_old, "out_old")
    _per_point(h_a, B * M, "h_a")
    _per_point(h_b, B * M, "h_b")
    _per_point(out_old, B * N, "out_old")
    shape = (B, N) if batched else (N,)
    dev = x.device
    with nvtx_range(f"b200ot.softmin_wide B={B} N={N} M={M} D={D} eps={float(eps):.3g}"):
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=dev)
        lse2 = torch.empty(shape, dtype=torch.float32, device=dev) if want_lse2 else None
        scratch = _wide_scratch(B, N, M, D, dev)
        # two packs, reduction, finalize (p = 1: and the coordinate maximum)
        _call(dev, "b200ot_wide_softmin_fwd", x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, B, N, M, D, int(p), float(eps), scratch, scratch.numel(),
              launches=5 if (p & 0xFF) == 1 else 4)
    return out, lse2


def softmin_wide_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x, shaped like x, of <grad_out, softmin_wide(eps, x, y, h)> with y, h constant
    (b200ot_wide_softmin_bwd_x)."""
    _, (B, N, M, D) = _wide_args(x, y)
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, grad_out = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(grad_out, "grad_out")
    _per_point(grad_out, B * N, "grad_out")
    _per_point(lse2, B * N, "lse2")
    dev = x.device
    gx = torch.empty_like(x)
    scratch = _wide_scratch(B, N, M, D, dev)
    _call(dev, "b200ot_wide_softmin_bwd_x", x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, B, N, M, D,
          int(p), float(eps), scratch, scratch.numel(), launches=5 if (p & 0xFF) == 1 else 4)
    return gx


def plan_apply_wide_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    """``plan_apply_raw`` above D = 64 (b200ot_wide_plan_apply): ``out[i, k] = row_factor_i * sum_j w_ij v[j, k]`` for
    (N,D) / (M,D) clouds, ``lse2`` from ``softmin_wide_raw(..., want_lse2=True)`` with the same arguments.  ``v`` is
    (M,) or (M, K), any sign, any strides; p = 2.  One pass over the pairs per slab of 64 value columns, each
    recomputing the full-K exponent.  No autograd.  Returns (N,) or (N, K)."""
    if x.dim() != 2 or y.dim() != 2:
        raise ValueError(f"expected x:(N,D), y:(M,D); got {tuple(x.shape)}, {tuple(y.shape)}")
    _, (_, N, M, D) = _wide_args(x, y)
    x, y, h_a, h_b = _f32c(x, "x"), _f32c(y, "y"), _f32c(h_a, "h_a"), _f32c(h_b, "h_b")
    center, lse2, v = _f32c(center, "center"), _f32c(lse2, "lse2"), _f32c(v, "v")
    row_factor = _f32c(row_factor, "row_factor")
    if v.dim() not in (1, 2) or v.shape[0] != M or v.numel() == 0:
        raise ValueError(f"v must be (M,) or (M, K) with M = {M} and K >= 1, got {tuple(v.shape)}")
    _per_point(h_a, M, "h_a")
    _per_point(h_b, M, "h_b")
    if lse2.numel() != N or (row_factor is not None and row_factor.numel() != N):
        raise ValueError("lse2 and row_factor must have one entry per row")
    K = 1 if v.dim() == 1 else v.shape[1]
    dev = x.device
    with nvtx_range(f"b200ot.plan_apply_wide N={N} M={M} D={D} K={K}"):
        out = torch.empty((N,) if v.dim() == 1 else (N, K), dtype=torch.float32, device=dev)
        scratch = _scratch(_query(dev, "b200ot_wide_plan_apply_scratch_bytes", N, M, D, K), dev, "plan_apply")
        # two packs, the column maxima of v, then value pack, reduction and finalize per slab of 64 columns
        _call(dev, "b200ot_wide_plan_apply", x, y, h_a, h_b, float(h_scale_b), center, lse2, v, row_factor, out, N, M,
              D, K, 2, float(eps), scratch, scratch.numel(), launches=3 + 3 * -(-K // 64))
    return out


def softmin_wide(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) ``scale_out * softmin_wide_raw(...)``, for (N,D) or (B,N,D) clouds."""
    return _softmin_apply(softmin_wide_raw, softmin_wide_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center,
                          scale_out)


def _conv_wide_args(x, y, w, center):
    batched, (B, N, M, D) = _wide_args(x, y)  # the shape check first: D > MAX_D_WIDE is refused on any device
    x, y, w, center = _f32c(x, "x"), _f32c(y, "y"), _f32c(w, "w"), _f32c(center, "center")
    _per_point(w, B * M, "w")
    return x, y, w, center, batched, B, N, M, D


def kernel_conv_wide_raw(kind, x, y, w, blur, *, center=None):
    """out_i = sum_j k(x_i, y_j) w_j above D = 64, (N,) or (B,N); no autograd."""
    x, y, w, center, batched, B, N, M, D = _conv_wide_args(x, y, w, center)
    dev = x.device
    energy = (kind_id(kind) & 0xFF) == KERNEL_KINDS["energy"]
    with nvtx_range(f"b200ot.kernel_conv_wide kind={kind} B={B} N={N} M={M} D={D}"):
        out = torch.empty((B, N) if batched else (N,), dtype=torch.float32, device=dev)
        scratch = _wide_scratch(B, N, M, D, dev)
        # two packs, reduction, finalize (energy: and the coordinate maximum)
        _call(dev, "b200ot_wide_kernel_conv_fwd", x, y, w, center, out, B, N, M, D, kind_id(kind), float(blur), scratch,
              scratch.numel(), launches=5 if energy else 4)
    return out


def kernel_conv_wide_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    """grad_x, shaped like x, of <grad_out, kernel_conv_wide_raw(kind, x, y, w, blur)>
    (b200ot_wide_kernel_conv_bwd_x)."""
    x, y, w, center, _, B, N, M, D = _conv_wide_args(x, y, w, center)
    grad_out = _f32c(grad_out, "grad_out")
    _per_point(grad_out, B * N, "grad_out")
    dev = x.device
    energy = (kind_id(kind) & 0xFF) == KERNEL_KINDS["energy"]
    gx = torch.empty_like(x)
    scratch = _wide_scratch(B, N, M, D, dev)
    # weight maximum, two packs, reduction, finalize (energy: and the coordinate maximum)
    _call(dev, "b200ot_wide_kernel_conv_bwd_x", x, y, w, center, grad_out, gx, B, N, M, D, kind_id(kind), float(blur),
          scratch, scratch.numel(), launches=6 if energy else 5)
    return gx


def kernel_conv_wide(kind, x, y, w, blur, *, center=None):
    """out = K(x, y) @ w above D = 64, (N,) or (B,N), differentiable w.r.t. x, y and w (no one-pass value + gradient:
    the forward and the row gradient are separate launches)."""
    wide = _ConvOps(kernel_conv_wide_raw, kernel_conv_wide_grad_rows, None)
    return _KernelConv.apply(wide, wide, x, y, w, kind, blur, center, False)

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
    """The NVTX range ``fmt.format(*args)``: the name is formatted only when ranges are on, off the enqueue path."""

    def __init__(self, fmt, *args):
        self.fmt, self.args = fmt, args

    def __enter__(self):
        if NVTX:
            torch.cuda.nvtx.range_push(self.fmt.format(*self.args))

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
MAX_D_WIDE = 1024  # B200OT_MAX_D_WIDE: the K-slab tensor-core kernels above MAX_D_TC


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


# ---- the operator families, and one body per kind of operator that serves every family ------------------------
class _Family(NamedTuple):
    """What one family of library operators serves for one kind of operator, and the C entries that serve it."""
    label: str  # in NVTX ranges and errors
    ranks: tuple  # 2: (N,D) / (M,D) clouds, 3: (B,N,D) / (B,M,D) ones (the C entries then take B)
    dims: tuple  # (lo, hi): lo < D <= hi; lo = 0 is the one-problem family, checked by _check_clouds
    entries: tuple  # C entries: forward, row gradient, one-pass value + row gradient
    scratch: str  # the scratch-size query, and the _scratch tag of the buffer it sizes
    tag: str
    launches: Callable  # kernels per call, from p (softmins), (kind id, row gradient?) (matvecs) or (K, D) (plans)
    p: tuple = ()  # softmins that serve one p & 0xFF only: (that p, the error class for another)


_SOFTMIN = _Family("softmin", ranks=(2,), dims=(0, MAX_D_TC), scratch="b200ot_softmin_scratch_bytes", tag="softmin",
                   entries=("b200ot_softmin_fwd", "b200ot_softmin_bwd_x"), launches=lambda p: 3)
_SOFTMIN_BATCHED = _Family("softmin_batched", ranks=(3,), dims=(MAX_D, MAX_D_TC), p=(2, NotImplementedError),
                           scratch="b200ot_batched_scratch_bytes", tag="batched", launches=lambda p: 3,
                           entries=("b200ot_softmin_fwd_batched", "b200ot_softmin_bwd_x_batched"))
# the coordinate maximum, two packs, reduction, finalize
_SOFTMIN_L1 = _Family("softmin_l1", ranks=(2, 3), dims=(MAX_D, MAX_D_TC), p=(1, ValueError), launches=lambda p: 5,
                      scratch="b200ot_softmin_l1_scratch_bytes", tag="softmin_l1",
                      entries=("b200ot_softmin_l1_fwd", "b200ot_softmin_l1_bwd_x"))
# two packs, reduction, finalize, and for p = 1 the coordinate maximum
_SOFTMIN_WIDE = _Family("softmin_wide", ranks=(2, 3), dims=(MAX_D_TC, MAX_D_WIDE), scratch="b200ot_wide_scratch_bytes",
                        tag="wide", entries=("b200ot_wide_softmin_fwd", "b200ot_wide_softmin_bwd_x"),
                        launches=lambda p: 5 if (p & 0xFF) == 1 else 4)
_CONV = _Family("kernel_conv", ranks=(2,), dims=(0, MAX_D_TC), scratch="b200ot_kernel_conv_scratch_bytes", tag="conv",
                entries=("b200ot_kernel_conv_fwd", "b200ot_kernel_conv_bwd_x", "b200ot_kernel_conv_fwd_bwd_x"),
                launches=lambda kind, bwd: 3)
_CONV_BATCHED = _Family("kernel_conv_batched", ranks=(3,), dims=(MAX_D, MAX_D_TC), launches=lambda kind, bwd: 3,
                        scratch="b200ot_batched_scratch_bytes", tag="batched",
                        entries=("b200ot_kernel_conv_fwd_batched", "b200ot_kernel_conv_bwd_x_batched",
                                 "b200ot_kernel_conv_fwd_bwd_x_batched"))
# (the row gradient's weight maximum,) two packs, reduction, finalize, and for energy the coordinate maximum
_CONV_WIDE = _Family("kernel_conv_wide", ranks=(2, 3), dims=(MAX_D_TC, MAX_D_WIDE), scratch="b200ot_wide_scratch_bytes",
                     tag="wide", entries=("b200ot_wide_kernel_conv_fwd", "b200ot_wide_kernel_conv_bwd_x"),
                     launches=lambda kind, bwd: 4 + bwd + ((kind & 0xFF) == KERNEL_KINDS["energy"]))
# a pack (and the value maxima), then value pack, reduction, finalize per slab of 8 (D <= 8) or 64 value columns
_PLAN = _Family("plan_apply", ranks=(2,), dims=(0, MAX_D_TC), tag="plan_apply", entries=("b200ot_plan_apply",),
                scratch="b200ot_plan_apply_scratch_bytes", launches=lambda K, D: 1 + 3 * -(-K // (8 if D <= 8 else 64)))
# two packs, the column maxima of v, then value pack, reduction, finalize per slab of 64 value columns
_PLAN_WIDE = _Family("plan_apply_wide", ranks=(2,), dims=(MAX_D_TC, MAX_D_WIDE), tag="plan_apply",
                     scratch="b200ot_wide_plan_apply_scratch_bytes", entries=("b200ot_wide_plan_apply",),
                     launches=lambda K, D: 3 + 3 * -(-K // 64))


def _inputs(fam, p, x, y, cols, rows, *more, v=None):
    """Every operator's checks, in order: (1) the clouds' shapes and D, and p, against ``fam``; (2) one entry per point
    for each vector of ``cols`` and ``rows`` ((vector, name), ...), and M rows for a value matrix ``v``; (3) device and
    dtype of every tensor, ``more`` given like ``cols``.  Returns (B, N, M, D), the sizes the family's C entries take,
    and x, y, the vectors, ``more`` and ``v`` as contiguous float32 CUDA tensors."""
    lo, hi = fam.dims
    if lo == 0:  # the one-problem family serves D from 1: _check_clouds' checks, p = 1 up to MAX_D
        _check_clouds(x, y, hi if (p & 0xFF) == 2 else MAX_D)
        B, (N, D), M = 1, x.shape, y.shape[0]
    else:
        if x.dim() not in fam.ranks or y.dim() != x.dim() or x.shape[:-2] != y.shape[:-2] or x.shape[-1] != y.shape[-1]:
            shapes = " or ".join({2: "x:(N,D), y:(M,D)", 3: "x:(B,N,D), y:(B,M,D)"}[r] for r in fam.ranks)
            raise ValueError(f"expected {shapes}; got {tuple(x.shape)}, {tuple(y.shape)}")
        B, (N, D), M = (x.shape[0] if x.dim() == 3 else 1), x.shape[-2:], y.shape[-2]
        if B == 0 or N == 0 or M == 0:
            raise ValueError("empty batch or point cloud")
        if fam.p and ((p & 0xFF) != fam.p[0] or (p & ~(0xFF | P_UNCLAMPED)) != 0):
            raise fam.p[1](f"ops.{fam.label} computes the p = {fam.p[0]} softmin (p = {fam.p[0]} or {fam.p[0]} | "
                           f"P_UNCLAMPED), got p = {p}")
        if not lo < D <= hi:
            raise NotImplementedError(f"the {fam.label} operators serve {lo} < D <= {hi}, got D = {D}")
        if x.device != y.device:
            raise ValueError("x and y must be on the same device")
    for vectors, n in ((cols, B * M), (rows, B * N)):
        for t, name in vectors:
            if t is not None and t.numel() != n:
                raise ValueError(f"{name} must have one entry per point of its cloud ({n}), got {tuple(t.shape)}")
    if v is not None and (v.dim() not in (1, 2) or v.shape[0] != M or v.numel() == 0):
        raise ValueError(f"v must be (M,) or (M, K) with M = {M} and K >= 1, got {tuple(v.shape)}")
    ready = [_f32c(x, "x"), _f32c(y, "y")] + [_f32c(t, name) for t, name in cols + rows + more]
    ready += [] if v is None else [_f32c(v, "v")]
    return (B, N, M, D), ((B, N, M, D) if 3 in fam.ranks else (N, M, D)), ready


def _softmin(fam, eps, x, y, h_a, h_b, h_scale_b, p, center, out_old, alpha_old, beta, out, want_lse2):
    (B, N, M, D), sizes, (x, y, h_a, h_b, out_old, out_f32, center) = _inputs(
        fam, p, x, y, ((h_a, "h_a"), (h_b, "h_b")), ((out_old, "out_old"), (out, "out")), (center, "center"))
    dev = x.device
    if out is not None and (out_f32 is not out or out.device != dev):  # written in place: refused if it needs a copy
        raise ValueError(f"out must be contiguous and on {dev}, got strides {out.stride()} on {out.device}")
    with nvtx_range("b200ot.{} B={} N={} M={} D={} eps={:.3g}", fam.label, B, N, M, D, float(eps)):
        shape = (B, N) if x.dim() == 3 else N
        out = torch.empty(shape, dtype=torch.float32, device=dev) if out is None else out
        lse2 = torch.empty(shape, dtype=torch.float32, device=dev) if want_lse2 else None
        scratch = _scratch(_query(dev, fam.scratch, *sizes), dev, fam.tag)
        _call(dev, fam.entries[0], x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, *sizes, int(p), float(eps), scratch, scratch.numel(), launches=fam.launches(p))
    return out, lse2


def _softmin_grad_rows(fam, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, p, center):
    (B, N, M, D), sizes, (x, y, h_a, h_b, lse2, grad_out, center) = _inputs(
        fam, p, x, y, ((h_a, "h_a"), (h_b, "h_b")), ((lse2, "lse2"), (grad_out, "grad_out")), (center, "center"))
    dev = x.device
    with nvtx_range("b200ot.{} grad_rows B={} N={} M={} D={} eps={:.3g}", fam.label, B, N, M, D, float(eps)):
        gx = torch.empty_like(x)
        scratch = _scratch(_query(dev, fam.scratch, *sizes), dev, fam.tag)
        _call(dev, fam.entries[1], x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, *sizes, int(p),
              float(eps), scratch, scratch.numel(), launches=fam.launches(p))
    return gx


def _kernel_conv(fam, mode, kind, x, y, w, blur, center, grad_out=None):
    """``mode`` 0: the matvec; 1: its row gradient against ``grad_out``; 2: both from one pass (gaussian kernel)."""
    kid = kind_id(kind)
    if mode == 2 and (kid & 0xFF) != 0:
        raise ValueError("the one-pass value + row gradient exists for the gaussian kernel only")
    (B, N, M, D), sizes, (x, y, w, grad_out, center) = _inputs(
        fam, 2, x, y, ((w, "w"),), ((grad_out, "grad_out"),), (center, "center"))
    dev = x.device
    with nvtx_range("b200ot.{} mode={} kind={} B={} N={} M={} D={}", fam.label, mode, kind, B, N, M, D):
        out = None if mode == 1 else torch.empty((B, N) if x.dim() == 3 else N, dtype=torch.float32, device=dev)
        gx = None if mode == 0 else torch.empty_like(x)
        scratch = _scratch(_query(dev, fam.scratch, *sizes), dev, fam.tag)
        results = ((out,), (grad_out, gx), (out, gx))[mode]  # what each entry takes after the inputs
        _call(dev, fam.entries[mode], x, y, w, center, *results, *sizes, kid, float(blur), scratch, scratch.numel(),
              launches=fam.launches(kid, mode == 1))
    return (out, gx, (out, gx))[mode]


def _plan_apply(fam, eps, x, y, h_a, h_b, h_scale_b, lse2, v, row_factor, center):
    """``out[i, k] = row_factor_i * sum_j w_ij v[j, k]`` with ``w_ij = softmax_j(h_j - |x_i - y_j|^2 / (2 eps))`` and
    ``h = h_a + h_scale_b * h_b``: the softmin's weights applied to a value matrix without ever forming them.  ``lse2``
    is the forward softmin's for the same arguments; ``v`` is (M,) or (M, K), any sign, any strides; p = 2.  One pass
    over the pairs per slab of value columns.  No autograd.  Returns (N,) or (N, K)."""
    (_, N, M, D), _, (x, y, h_a, h_b, lse2, row_factor, center, v) = _inputs(fam, 2, x, y,
        ((h_a, "h_a"), (h_b, "h_b")), ((lse2, "lse2"), (row_factor, "row_factor")), (center, "center"), v=v)
    dev = x.device
    K = 1 if v.dim() == 1 else v.shape[1]
    with nvtx_range("b200ot.{} N={} M={} D={} K={}", fam.label, N, M, D, K):
        out = torch.empty((N, *v.shape[1:]), dtype=torch.float32, device=dev)
        scratch = _scratch(_query(dev, fam.scratch, N, M, D, K), dev, fam.tag)
        _call(dev, fam.entries[0], x, y, h_a, h_b, float(h_scale_b), center, lse2, v, row_factor, out, N, M, D,
              K, 2, float(eps), scratch, scratch.numel(), launches=fam.launches(K, D))
    return out


def softmin_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                beta=1.0, out=None, want_lse2=False):
    """One fused launch group: ``out <- alpha_old*out_old + beta*softmin(eps, (x, y), h_a + h_scale_b*h_b)``.  No
    autograd.  Returns ``(out, lse2 | None)``."""
    return _softmin(_SOFTMIN, eps, x, y, h_a, h_b, h_scale_b, p, center, out_old, alpha_old, beta, out, want_lse2)


# Two softmins of one Jacobi iteration that mirror each other (A's rows are B's columns and A's columns B's rows, same
# eps, p and center) share their exponentials: b200ot_softmin_fwd_pair, or, with the symmetric softmins of both
# clouds, b200ot_softmin_fwd_step.  B200OT_PAIR=0, read on every call, runs every
# call on its own (the library's symmetric xx / yy kernel follows the same switch).
def _same(s, t):
    """The same tensor data: one object, or views such as two ``.detach()`` of one cloud."""
    if s is None or t is None:
        return s is t
    return s is t or (s.data_ptr() == t.data_ptr() and s.shape == t.shape and s.stride() == t.stride()
                      and s.dtype == t.dtype and s.device == t.device)


def _mirrors(a, b):
    """Whether the ``softmin_raw`` calls ``a``, ``b`` (each ``(args, kwargs)``) can run as one paired launch group."""
    (ea, xa, ya, *_), ka = a
    (eb, xb, yb, *_), kb = b
    if _same(xa, ya) or not _same(xa, yb) or not _same(ya, xb) or float(ea) != float(eb):
        return False
    if ka.get("p", 2) != 2 or kb.get("p", 2) != 2 or not _same(ka.get("center"), kb.get("center")):
        return False
    if xa.dim() != 2 or xa.shape[-1] != 3 or ya.dim() != 2 or ya.shape[-1] != 3:
        return False
    return _disjoint((a, b))


def _disjoint(calls):
    """No output of ``calls`` shares storage with an input of any of them or with another output: the recomputation
    of a softmin whose sums leave the paired range reads every input after the outputs are written."""
    ins = [t for args, kw in calls for t in (*args[1:], kw.get("out_old"), kw.get("center")) if torch.is_tensor(t)]
    outs = [kw["out"] for _, kw in calls if kw.get("out") is not None]
    shared = lambda s, t: s.untyped_storage().data_ptr() == t.untyped_storage().data_ptr()  # noqa: E731
    return not any(shared(o, t) for o in outs for t in ins) and not any(
        shared(o, q) for i, o in enumerate(outs) for q in outs[i + 1:])


def pair_plan(calls):
    """The launch groups of ``softmin_raw_many(calls)``: ``(i, j)`` for two calls that run paired, ``(k,)`` for one
    that runs alone, in the order of the first call of each group."""
    plan, used = [], set()
    for i in range(len(calls)):
        if i in used:
            continue
        j = next((j for j in range(i + 1, len(calls)) if j not in used and _mirrors(calls[i], calls[j])), None)
        if j is None:
            plan.append((i,))
        else:
            plan.append((i, j))
            used.add(j)
    return plan


def _self_call(c, cloud, eps, kw):
    """Whether the ``softmin_raw`` call ``c`` is the symmetric softmin of ``cloud`` at ``eps``, p = 2 and the center
    of ``kw``."""
    (e, rows, cols, *_), kc = c
    return (_same(rows, cloud) and _same(cols, cloud) and float(e) == float(eps) and kc.get("p", 2) == 2
            and _same(kc.get("center"), kw.get("center")))


def step_plan(calls):
    """``pair_plan(calls)`` with each pair ``(i, j)`` that has self calls ``k`` on its rows' cloud and ``l`` on its
    columns' cloud (same eps, p = 2 and center; no output of the four overlapping an input or another output) merged
    into one step group ``(i, j, k, l)``: the four softmins of a symmetric Jacobi iteration as one launch group
    (b200ot_softmin_fwd_step).  Groups in the order of their first call."""
    plan = pair_plan(calls)
    free = {g[0] for g in plan if len(g) == 1}
    steps = {}
    for g in plan:
        if len(g) == 2:
            (eps, x, y, *_), kw = calls[g[0]]
            kx = next((k for k in sorted(free) if _self_call(calls[k], x, eps, kw)), None)
            ky = next((k for k in sorted(free - {kx}) if _self_call(calls[k], y, eps, kw)), None)
            if kx is not None and ky is not None and _disjoint([calls[c] for c in (*g, kx, ky)]):
                steps[g] = (*g, kx, ky)
                free -= {kx, ky}
    taken = {c for st in steps.values() for c in st[2:]}
    return [steps.get(g, g) for g in plan if len(g) == 2 or g[0] not in taken]


def _softmin_pair(a, b):
    """``softmin_raw(*a)`` and ``softmin_raw(*b)`` from one pass over the pairs (``_mirrors(a, b)`` holds), or None
    when the library does not pair this shape."""
    (eps, x, y, h_a, *ha_more), ka = a
    (_, _, _, g_a, *hb_more), kb = b
    h_b, h_scale_b = (ha_more + [None, 0.0])[:2]
    g_b, g_scale_b = (hb_more + [None, 0.0])[:2]
    p, center = ka.get("p", 2), ka.get("center")
    (_, N, M, D), sizes, (x, y, h_a, h_b, g_a, g_b, out_a_old, out_a, out_b_old, out_b, center) = _inputs(
        _SOFTMIN, p, x, y, ((h_a, "h_a"), (h_b, "h_b")), ((g_a, "h_a"), (g_b, "h_b"), (ka.get("out_old"), "out_old"),
                                                          (ka.get("out"), "out")),
        (kb.get("out_old"), "out_old"), (kb.get("out"), "out"), (center, "center"))
    if (out_b_old is not None and out_b_old.numel() != M) or (out_b is not None and out_b.numel() != M):
        raise ValueError(f"out_old / out of the columns' softmin must have {M} entries")
    dev = x.device
    nbytes = _query(dev, "b200ot_softmin_pair_scratch_bytes", N, M, D)
    if nbytes == 0:
        return None
    for o, given in ((out_a, ka.get("out")), (out_b, kb.get("out"))):
        if given is not None and (o is not given or given.device != dev):
            raise ValueError(f"out must be contiguous and on {dev}, got strides {given.stride()} on {given.device}")
    with nvtx_range("b200ot.softmin_pair N={} M={} D={} eps={:.3g}", N, M, D, float(eps)):
        out_a = torch.empty(N, dtype=torch.float32, device=dev) if out_a is None else out_a
        out_b = torch.empty(M, dtype=torch.float32, device=dev) if out_b is None else out_b
        lse2_a = torch.empty(N, dtype=torch.float32, device=dev) if ka.get("want_lse2") else None
        lse2_b = torch.empty(M, dtype=torch.float32, device=dev) if kb.get("want_lse2") else None
        scratch = _scratch(nbytes, dev, "softmin_pair")
        # two packs, the paired pass, two checked finalizes, and the gated pack, partial and finalize of each softmin
        _call(dev, "b200ot_softmin_fwd_pair", x, y, h_a, h_b, float(h_scale_b), out_a_old, float(ka.get("alpha_old", 0.0)),
              float(ka.get("beta", 1.0)), out_a, lse2_a, g_a, g_b, float(g_scale_b), out_b_old,
              float(kb.get("alpha_old", 0.0)), float(kb.get("beta", 1.0)), out_b, lse2_b, center, N, M, D, int(p),
              float(eps), scratch, scratch.numel(), launches=11)
    return (out_a, lse2_a), (out_b, lse2_b)


def _softmin_step(cs):
    """``softmin_raw(*c)`` for the four calls ``cs`` of a step group (xy, yx, xx, yy; ``step_plan``) from one launch
    group, or None when the library does not run this shape as one."""
    (eps, x, y, *_), k0 = cs[0]
    p, center = k0.get("p", 2), k0.get("center")
    hs = [(args[3], *(list(args[4:]) + [None, 0.0])[:2]) for args, _ in cs]  # h_a, h_b, h_scale_b of each softmin
    vecs = lambda k: ((hs[k][0], "h_a"), (hs[k][1], "h_b"), (cs[k][1].get("out_old"), "out_old"),  # noqa: E731
                      (cs[k][1].get("out"), "out"))
    # on the columns' cloud (M entries): the potentials of xy and yy, the epilogues of yx and yy; the rest on the rows'
    on_y = ((hs[0][0], "h_a"), (hs[0][1], "h_b"), *vecs(1)[2:], *vecs(3))
    on_x = ((hs[1][0], "h_a"), (hs[1][1], "h_b"), *vecs(0)[2:], *vecs(2))
    (_, N, M, D), sizes, (x, y, *ready) = _inputs(_SOFTMIN, p, x, y, on_y, on_x, (center, "center"))
    ry, rx, center = ready[:8], ready[8:16], ready[16]
    dev = x.device
    nbytes = _query(dev, "b200ot_softmin_step_scratch_bytes", *sizes)
    if nbytes == 0:
        return None
    # per softmin: h_a, h_b, out_old, out as checked, and its row count
    got = [(ry[0], ry[1], rx[2], rx[3], N), (rx[0], rx[1], ry[2], ry[3], M), (rx[4], rx[5], rx[6], rx[7], N),
           (ry[4], ry[5], ry[6], ry[7], M)]
    for (*_, o, _), (_, kw) in zip(got, cs):
        given = kw.get("out")
        if given is not None and (o is not given or given.device != dev):
            raise ValueError(f"out must be contiguous and on {dev}, got strides {given.stride()} on {given.device}")
    with nvtx_range("b200ot.softmin_step N={} M={} D={} eps={:.3g}", N, M, D, float(eps)):
        slots, res = (_lib.SoftminSlot * 4)(), []
        for slot, (h_a, h_b, out_old, out, n), (_, h_scale_b), (_, kw) in zip(slots, got, [h[1:] for h in hs], cs):
            out = torch.empty(n, dtype=torch.float32, device=dev) if out is None else out
            lse2 = torch.empty(n, dtype=torch.float32, device=dev) if kw.get("want_lse2") else None
            slot.h_a, slot.h_b, slot.out_old, slot.out, slot.lse2 = (None if t is None else t.data_ptr()
                                                                     for t in (h_a, h_b, out_old, out, lse2))
            slot.h_scale_b, slot.alpha_old, slot.beta = float(h_scale_b), float(kw.get("alpha_old", 0.0)), float(
                kw.get("beta", 1.0))
            res.append((out, lse2))
        scratch = _scratch(nbytes, dev, "softmin_pair")
        # four packs, the paired pass, four checked finalizes, and the gated pack, partial and finalize of each softmin
        _call(dev, "b200ot_softmin_fwd_step", x, y, slots, center, *sizes, int(p), float(eps), scratch,
              scratch.numel(), launches=21)
    return res


def softmin_raw_many(calls):
    """``[softmin_raw(*args, **kw) for args, kw in calls]``, the groups of ``step_plan(calls)`` each from one launch
    group: a step group through b200ot_softmin_fwd_step, a mirrored pair through b200ot_softmin_fwd_pair (also the
    pair of a step group whose shape the step entry does not serve, its self calls then on their own)."""
    res = [None] * len(calls)
    paired = _os.environ.get("B200OT_PAIR", "1") != "0"
    for group in (step_plan(calls) if paired else [(k,) for k in range(len(calls))]):
        got = _softmin_step([calls[k] for k in group]) if len(group) == 4 else None
        if got is None and len(group) >= 2:
            got = _softmin_pair(calls[group[0]], calls[group[1]])
        got = list(got or ())
        for k, r in zip(group, got):
            res[k] = r
        for k in group[len(got):]:
            args, kw = calls[k]
            res[k] = softmin_raw(*args, **kw)
    return res


# what sinkhorn.softmin_many looks up on the operator it is handed: the library's softmin_raw, not a stand-in for it
softmin_raw.softmin_raw_many = softmin_raw_many


def softmin_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x of <grad_out, softmin(eps, (x, y), h)> with y, h constant (b200ot_softmin_bwd_x)."""
    return _softmin_grad_rows(_SOFTMIN, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, p, center)


def plan_apply_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    """``_plan_apply`` for D <= 64 (b200ot_plan_apply), ``lse2`` from ``softmin_raw(..., want_lse2=True)``."""
    return _plan_apply(_PLAN, eps, x, y, h_a, h_b, h_scale_b, lse2, v, row_factor, center)


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


# ---- kernel convolutions ----------------------------------------------------------------------------------------
def kind_id(kind):
    """Kernel name (tensorized convention) or an integer kind, possibly or-ed with KERNEL_UNCLAMPED."""
    return KERNEL_KINDS[kind] if isinstance(kind, str) else int(kind)


def kernel_conv_raw(kind, x, y, w, blur, *, center=None):
    """out_i = sum_j k(x_i, y_j) w_j, no autograd."""
    return _kernel_conv(_CONV, 0, kind, x, y, w, blur, center)


def kernel_conv_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    """grad_x of <grad_out, kernel_conv_raw(kind, x, y, w, blur)> (b200ot_kernel_conv_bwd_x)."""
    return _kernel_conv(_CONV, 1, kind, x, y, w, blur, center, grad_out)


def kernel_conv_value_and_grad_rows(kind, x, y, w, blur, *, center=None):
    """(out, grad_unit) with out_i = sum_j k(x_i, y_j) w_j and grad_unit[i] = sum_j w_j dk(x_i, y_j)/dx_i from ONE
    pass over the pairs (gaussian kernel; b200ot_kernel_conv_fwd_bwd_x).  No autograd."""
    return _kernel_conv(_CONV, 2, kind, x, y, w, blur, center)


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
# the other families, with the contracts of the one-problem operators above: batches (B,N,D) / (B,M,D) with per-column
# vectors (B,M) and per-row vectors (B,N), element b of the rows reduced over element b of the columns only; the p = 1
# softmin; above D = 64, the K-slab tensor-core kernels (csrc/tcwide.cuh).  One launch group per call.
# ------------------------------------------------------------------------------------------------
def softmin_batched_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                        beta=1.0, out=None, want_lse2=False):
    """``softmin_raw`` on a batch: out[b] (B,N) is the softmin of (x[b], y[b], h[b]).  p = 2 only."""
    return _softmin(_SOFTMIN_BATCHED, eps, x, y, h_a, h_b, h_scale_b, p, center, out_old, alpha_old, beta, out,
                    want_lse2)


def softmin_batched_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x (B,N,D) of <grad_out, softmin_batched(eps, x, y, h)> with y, h constant (b200ot_softmin_bwd_x_batched)."""
    return _softmin_grad_rows(_SOFTMIN_BATCHED, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, p, center)


def softmin_batched(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) batched softmin, (B,N): ``softmin`` element by element."""
    return _softmin_apply(softmin_batched_raw, softmin_batched_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center,
                          scale_out)


def kernel_conv_batched_raw(kind, x, y, w, blur, *, center=None):
    """out (B,N), out[b, i] = sum_j k(x[b, i], y[b, j]) w[b, j], no autograd."""
    return _kernel_conv(_CONV_BATCHED, 0, kind, x, y, w, blur, center)


def kernel_conv_batched_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    """grad_x (B,N,D) of <grad_out, kernel_conv_batched_raw(kind, x, y, w, blur)> (b200ot_kernel_conv_bwd_x_batched)."""
    return _kernel_conv(_CONV_BATCHED, 1, kind, x, y, w, blur, center, grad_out)


def kernel_conv_batched_value_and_grad_rows(kind, x, y, w, blur, *, center=None):
    """``kernel_conv_value_and_grad_rows`` on a batch (gaussian only): (out (B,N), grad_unit (B,N,D))."""
    return _kernel_conv(_CONV_BATCHED, 2, kind, x, y, w, blur, center)


def kernel_conv_batched(kind, x, y, w, blur, *, center=None):
    """out (B,N) = K(x[b], y[b]) @ w[b] for every b, differentiable w.r.t. x, y and w."""
    batched = _ConvOps(kernel_conv_batched_raw, kernel_conv_batched_grad_rows, kernel_conv_batched_value_and_grad_rows)
    return _KernelConv.apply(batched, batched, x, y, w, kind, blur, center, _fused(kind, x))


def softmin_l1_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=1, center=None, out_old=None, alpha_old=0.0,
                   beta=1.0, out=None, want_lse2=False):
    """``softmin_raw`` for the cost |x - y|, (N,) for (N,D) clouds, (B,N) for (B,N,D) ones."""
    return _softmin(_SOFTMIN_L1, eps, x, y, h_a, h_b, h_scale_b, p, center, out_old, alpha_old, beta, out, want_lse2)


def softmin_l1_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=1, center=None):
    """grad_x, shaped like x, of <grad_out, softmin_l1(eps, x, y, h)> with y, h constant (b200ot_softmin_l1_bwd_x)."""
    return _softmin_grad_rows(_SOFTMIN_L1, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, p, center)


def softmin_l1(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=1, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) ``scale_out * softmin_l1_raw(...)``, for (N,D) or (B,N,D) clouds."""
    return _softmin_apply(softmin_l1_raw, softmin_l1_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out)


def softmin_wide_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                     beta=1.0, out=None, want_lse2=False):
    """``softmin_raw`` above D = 64 for p = 1 or 2, (N,) for (N,D) clouds, (B,N) for (B,N,D) ones."""
    return _softmin(_SOFTMIN_WIDE, eps, x, y, h_a, h_b, h_scale_b, p, center, out_old, alpha_old, beta, out, want_lse2)


def softmin_wide_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    """grad_x, shaped like x, of <grad_out, softmin_wide(eps, x, y, h)> with y, h constant."""
    return _softmin_grad_rows(_SOFTMIN_WIDE, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, p, center)


def plan_apply_wide_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    """``_plan_apply`` above D = 64 (b200ot_wide_plan_apply), lse2 from ``softmin_wide_raw(..., want_lse2=True)``."""
    return _plan_apply(_PLAN_WIDE, eps, x, y, h_a, h_b, h_scale_b, lse2, v, row_factor, center)


def softmin_wide(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0):
    """Differentiable (w.r.t. x) ``scale_out * softmin_wide_raw(...)``, for (N,D) or (B,N,D) clouds."""
    return _softmin_apply(softmin_wide_raw, softmin_wide_grad_rows, eps, x, y, h_a, h_b, h_scale_b, p, center,
                          scale_out)


def kernel_conv_wide_raw(kind, x, y, w, blur, *, center=None):
    """out_i = sum_j k(x_i, y_j) w_j above D = 64, (N,) or (B,N); no autograd."""
    return _kernel_conv(_CONV_WIDE, 0, kind, x, y, w, blur, center)


def kernel_conv_wide_grad_rows(kind, x, y, w, blur, grad_out, *, center=None):
    """grad_x, shaped like x, of <grad_out, kernel_conv_wide_raw(kind, x, y, w, blur)>."""
    return _kernel_conv(_CONV_WIDE, 1, kind, x, y, w, blur, center, grad_out)


def kernel_conv_wide(kind, x, y, w, blur, *, center=None):
    """out = K(x, y) @ w above D = 64, (N,) or (B,N), differentiable w.r.t. x, y and w, in two passes."""
    wide = _ConvOps(kernel_conv_wide_raw, kernel_conv_wide_grad_rows, None)
    return _KernelConv.apply(wide, wide, x, y, w, kind, blur, center, False)


# ------------------------------------------------------------------------------------------------
# explicit cost matrices C (N, M) or (B, N, M): both softmins of a symmetric Sinkhorn update from one pass over C
# (b200ot_dense_*, csrc/b200ot_dense.cu).  No clouds, so no _Family: one body per operator.
# ------------------------------------------------------------------------------------------------
def _dense_inputs(C, rows, cols):
    """The dense operators' checks, in ``_inputs``' order: (1) C is (N, M) or (B, N, M) and not empty; (2) one entry
    per row (B N) / column (B M) for each vector of ``rows`` / ``cols`` ((vector, name), ...); (3) device and dtype of
    every tensor.  Returns (B, N, M), the shape of a row / column vector, and C then the vectors as contiguous float32
    CUDA tensors."""
    if C.dim() not in (2, 3) or C.numel() == 0:
        raise ValueError(f"expected a non-empty cost matrix C:(N,M) or (B,N,M); got {tuple(C.shape)}")
    B, N, M = (1, *C.shape) if C.dim() == 2 else tuple(C.shape)
    for vectors, n in ((rows, B * N), (cols, B * M)):
        for t, name in vectors:
            if t is not None and t.numel() != n:
                raise ValueError(f"{name} must have one entry per {'row' if n == B * N else 'column'} of C ({n}), "
                                 f"got {tuple(t.shape)}")
    ready = [_f32c(C, "C")] + [_f32c(t, name) for t, name in rows + cols]
    if any(t is not None and t.device != C.device for t in ready):
        raise ValueError(f"every tensor must live on C's device ({C.device})")
    lead = (B,) if C.dim() == 3 else ()
    return (B, N, M), (lead + (N,), lead + (M,)), ready


def dense_softmin_pair_raw(eps, C, log_a, log_b, f_old, g_old, *, alpha_old=0.0, beta=1.0, want_lse2=False):
    """One pass over C for both softmins of a symmetric Sinkhorn update, each averaged / damped like ``softmin_raw``:
        f <- alpha_old f_old + beta (-eps log sum_j exp(log_b_j + (g_old_j - C_ij) / eps)),
        g <- alpha_old g_old + beta (-eps log sum_i exp(log_a_i + (f_old_i - C_ij) / eps)).
    C (N, M) or (B, N, M); the vectors (N,) / (M,) or (B, N) / (B, M).  No autograd.
    Returns ``(f, g, lse2_row | None, lse2_col | None)``."""
    (B, N, M), (rshape, cshape), (C, log_a, f_old, log_b, g_old) = _dense_inputs(
        C, ((log_a, "log_a"), (f_old, "f_old")), ((log_b, "log_b"), (g_old, "g_old")))
    dev = C.device
    with nvtx_range("b200ot.dense_pair B={} N={} M={} eps={:.3g}", B, N, M, float(eps)):
        f, lse2_row = torch.empty(rshape, dtype=torch.float32, device=dev), None
        g, lse2_col = torch.empty(cshape, dtype=torch.float32, device=dev), None
        if want_lse2:
            lse2_row, lse2_col = torch.empty_like(f), torch.empty_like(g)
        scratch = _scratch(_query(dev, "b200ot_dense_scratch_bytes", B, N, M), dev, "dense")
        _call(dev, "b200ot_dense_softmin_pair", C, log_a, log_b, f_old, g_old, 1.0 / float(eps), float(alpha_old),
              float(beta), f, g, lse2_row, lse2_col, B, N, M, float(eps), scratch, scratch.numel(), launches=3)
    return f, g, lse2_row, lse2_col


def dense_softmin_pair_grad(eps, C, log_a, log_b, f, g, lse2_row, lse2_col, go_f, go_g):
    """grad_C of ``<go_f, f~> + <go_g, g~>`` for ``f~, g~ = dense_softmin_pair_raw(eps, C, log_a, log_b, f, g)``
    (alpha_old = 0, beta = 1: fold a damping factor into go_f, go_g), lse2_* from that call; one pass over C."""
    (B, N, M), _, (C, log_a, f, lse2_row, go_f, log_b, g, lse2_col, go_g) = _dense_inputs(
        C, ((log_a, "log_a"), (f, "f"), (lse2_row, "lse2_row"), (go_f, "go_f")),
        ((log_b, "log_b"), (g, "g"), (lse2_col, "lse2_col"), (go_g, "go_g")))
    dev = C.device
    with nvtx_range("b200ot.dense_pair grad B={} N={} M={} eps={:.3g}", B, N, M, float(eps)):
        grad_C = torch.empty_like(C)
        _call(dev, "b200ot_dense_softmin_pair_bwd", C, log_a, log_b, f, g, 1.0 / float(eps), lse2_row, lse2_col,
              go_f, go_g, grad_C, B, N, M, launches=1)
    return grad_C


DENSE_ROWS_MAX = 4  # B200OT_DENSE_ROWS_MAX: matrices per dense_softmin_rows_raw call


def dense_softmin_rows_raw(eps, problems, *, alpha_old=0.0, beta=1.0, want_lse2=False):
    """The row softmins of 1 to 4 cost matrices in one partials launch (b200ot_dense_softmin_rows), each averaged /
    damped like ``softmin_raw``:
        out <- alpha_old out_old + beta (-eps log sum_j exp(log_w_j + (pot_j - C_ij) / eps)).
    ``problems``: ``[(C, log_w, pot | None, out_old | None), ...]``, C (N, M) or (B, N, M), log_w and pot (M,) / (B, M),
    out_old (N,) / (B, N); the matrices may differ in shape.  No autograd.  Returns ``[(out, lse2 | None), ...]``."""
    if not 1 <= len(problems) <= DENSE_ROWS_MAX:
        raise ValueError(f"expected 1 to {DENSE_ROWS_MAX} problems, got {len(problems)}")
    checked = [_dense_inputs(C, ((out_old, "out_old"),), ((log_w, "log_w"), (pot, "pot")))
               for C, log_w, pot, out_old in problems]
    dev = checked[0][2][0].device
    if any(ready[0].device != dev for _, _, ready in checked):
        raise ValueError(f"every problem must live on one device ({dev})")
    with nvtx_range("b200ot.dense_rows n={} eps={:.3g}", len(problems), float(eps)):
        descs, results = (_lib.DenseRows * len(problems))(), []
        for d, ((B, N, M), (rshape, _), (C, out_old, log_w, pot)) in zip(descs, checked):
            out = torch.empty(rshape, dtype=torch.float32, device=dev)
            lse2 = torch.empty_like(out) if want_lse2 else None
            d.C, d.log_w, d.pot, d.out_old, d.out, d.lse2 = (None if t is None else t.data_ptr()
                                                             for t in (C, log_w, pot, out_old, out, lse2))
            d.B, d.n_rows, d.n_cols = B, N, M
            results.append((out, lse2))
        scratch = _scratch(_query(dev, "b200ot_dense_rows_scratch_bytes", descs, len(descs)), dev, "dense_rows")
        _call(dev, "b200ot_dense_softmin_rows", descs, len(descs), float(eps), float(alpha_old), float(beta), scratch,
              scratch.numel(), launches=1 + len(problems))
    return results


def dense_softmin_rows_grad(eps, C, log_w, pot, lse2, go):
    """grad_C of ``<go, out~>`` for ``out~, lse2 = dense_softmin_rows_raw(eps, [(C, log_w, pot, None)],
    want_lse2=True)[0]`` (alpha_old = 0, beta = 1: fold a damping factor into go); one pass over C."""
    (B, N, M), _, (C, lse2, go, log_w, pot) = _dense_inputs(C, ((lse2, "lse2"), (go, "go")),
                                                            ((log_w, "log_w"), (pot, "pot")))
    dev = C.device
    with nvtx_range("b200ot.dense_rows grad B={} N={} M={} eps={:.3g}", B, N, M, float(eps)):
        grad_C = torch.empty_like(C)
        _call(dev, "b200ot_dense_softmin_rows_bwd", C, log_w, pot, 1.0 / float(eps), lse2, go, grad_C, B, N, M,
              launches=1)
    return grad_C


# ------------------------------------------------------------------------------------------------
# regular grids with their own side, pitch and periodicity per axis (b200ot_softmin_grid_axes, b200ot_grid_plan_apply,
# csrc/b200ot_grid.cu): one launch per axis, one chain of them per slab of GRID_APPLY_SLAB value channels
# ------------------------------------------------------------------------------------------------
GRID_MAX_SIDE = 1024
GRID_APPLY_SLAB = 4  # kGridApplyKS: value channels per launch of b200ot_grid_plan_apply


def _grid_geometry(shape, pitch, periodic):
    """(batch, dim, sides, pitch, periodic) of a (B, *grid) tensor as the host arrays of the grid entries."""
    dim = len(shape) - 1
    if not 1 <= dim <= 3 or len(pitch) != dim or len(periodic) != dim:
        raise ValueError(f"expected a (B, N1[, N2[, N3]]) grid with one pitch and one periodic flag per axis; got "
                         f"{tuple(shape)}, pitch {tuple(pitch)}, periodic {tuple(periodic)}")
    if any(not 1 <= n <= GRID_MAX_SIDE for n in shape[1:]):
        raise ValueError(f"grid sides must be in 1..{GRID_MAX_SIDE}, got {tuple(shape[1:])}")
    return (shape[0], dim, (ctypes.c_int32 * dim)(*shape[1:]), (ctypes.c_float * dim)(*map(float, pitch)),
            (ctypes.c_int32 * dim)(*(int(bool(p)) for p in periodic)))


def softmin_grid_axes_raw(eps, h_a, h_b=None, h_scale_b=0.0, *, pitch, periodic, out_old=None, alpha_old=0.0,
                          beta=1.0):
    """``alpha_old out_old + beta (-eps log sum_j exp(h_j - |x_i - x_j|^2 / (2 eps)))`` over a (B, *grid) grid with
    pixel pitch ``pitch[d]`` and wrap-around on the axes where ``periodic[d]``; h = h_a + h_scale_b h_b.
    No autograd."""
    h_a, h_b, out_old = _f32c(h_a, "h_a"), _f32c(h_b, "h_b"), _f32c(out_old, "out_old")
    for t, name in ((h_b, "h_b"), (out_old, "out_old")):
        if t is not None and (t.shape != h_a.shape or t.device != h_a.device):
            raise ValueError(f"{name} must match h_a ({tuple(h_a.shape)} on {h_a.device}), got {tuple(t.shape)}")
    B, dim, sides, pitch_c, periodic_c = _grid_geometry(h_a.shape, pitch, periodic)
    dev = h_a.device
    with nvtx_range("b200ot.softmin_grid_axes shape={} eps={:.3g}", tuple(h_a.shape), float(eps)):
        out = torch.empty_like(h_a)
        _call(dev, "b200ot_softmin_grid_axes", h_a, h_b, float(h_scale_b), out_old, float(alpha_old), float(beta), out,
              B, dim, sides, pitch_c, periodic_c, float(eps), launches=dim)
    return out


def grid_plan_apply_raw(eps, h_a, h_b, h_scale_b, v, *, pitch, periodic):
    """The weights ``w_ij = exp(h_j - |x_i - x_j|^2 / (2 eps))`` of that softmin applied to K channels, v (K, B, *grid)
    channel-major: returns ``(ell, s)`` with ``ell = log2 sum_j w_ij`` (B, *grid) and ``s = sum_j w_ij v_j / sum_j
    w_ij`` (K, B, *grid), s = 0 where every weight is 0.  No autograd."""
    h_a, h_b, v = _f32c(h_a, "h_a"), _f32c(h_b, "h_b"), _f32c(v, "v")
    if h_b is not None and (h_b.shape != h_a.shape or h_b.device != h_a.device):
        raise ValueError(f"h_b must match h_a ({tuple(h_a.shape)} on {h_a.device}), got {tuple(h_b.shape)}")
    if v.dim() != h_a.dim() + 1 or v.shape[1:] != h_a.shape or v.shape[0] == 0 or v.device != h_a.device:
        raise ValueError(f"v must be (K, *h_a.shape) = (K, {', '.join(map(str, h_a.shape))}) with K >= 1 on "
                         f"{h_a.device}, got {tuple(v.shape)}")
    B, dim, sides, pitch_c, periodic_c = _grid_geometry(h_a.shape, pitch, periodic)
    K, dev = v.shape[0], h_a.device
    with nvtx_range("b200ot.grid_plan_apply shape={} K={} eps={:.3g}", tuple(h_a.shape), K, float(eps)):
        ell, s = torch.empty_like(h_a), torch.empty_like(v)
        _call(dev, "b200ot_grid_plan_apply", h_a, h_b, float(h_scale_b), v, ell, s, B, K, dim, sides, pitch_c,
              periodic_c, float(eps), launches=dim * -(-K // GRID_APPLY_SLAB))
    return ell, s


# which operators serve which clouds: the one place that compares D with MAX_D / MAX_D_TC.  The operators are module
# globals read at every call, so a replaced operator is the one returned.
def softmin_operators(D, p=2, batched=False):
    """(raw, differentiable) softmins for one problem of dimension D and cost |x - y|^p / p, or a batch; None for a
    batch with D <= MAX_D (a block-diagonal ranges problem, ranges.py).  Above MAX_D_WIDE the wide ones refuse."""
    if D > MAX_D_TC:
        return softmin_wide_raw, softmin_wide
    if D <= MAX_D:
        return None if batched else (softmin_raw, softmin)
    if (p & 0xFF) == 1:
        return softmin_l1_raw, softmin_l1
    return (softmin_batched_raw, softmin_batched) if batched else (softmin_raw, softmin)


def kernel_conv_operator(D, batched=False):
    """The differentiable kernel matvec for one problem of dimension D or a batch; None for a batch with D <= MAX_D."""
    if D > MAX_D_TC:
        return kernel_conv_wide
    return (None if D <= MAX_D else kernel_conv_batched) if batched else kernel_conv


def ot_operators(D):
    """(forward, row gradient, plan apply) of the p = 2 softmin on one problem of dimension D: the operators the
    entropic OT solver (ot.solve_sample) runs."""
    if D > MAX_D_TC:
        return softmin_wide_raw, softmin_wide_grad_rows, plan_apply_wide_raw
    return softmin_raw, softmin_grad_rows, plan_apply_raw

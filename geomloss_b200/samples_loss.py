"""``SamplesLoss`` — drop-in for ``geomloss.SamplesLoss`` on CUDA point clouds.

Same constructor keywords, same 2 / 4 / 6 positional-tensor call forms, same shape rules, error types
and output shapes as the reference module (src/geomloss/_legacy/samples_loss.py:45-474), including
its quirks that user code may rely on:
  * ``potentials=True`` on unbatched input returns ``(1, N)`` / ``(1, M)`` tensors (SURVEY.md A-12);
  * ``loss="hausdorff"`` is accepted by the constructor and fails with ``KeyError(None)`` at call
    time, exactly like the reference at this commit (SURVEY.md A-13);
  * unknown ``p`` raises ``KeyError`` (the reference's cost table only has p = 1, 2).

``backend`` keeps the reference's routing rules (samples_loss.py:220-257: labels need "auto"/"multiscale"; "auto"
picks "multiscale" for Sinkhorn, p = 2, D <= 3 above 1e8 pairs; a batched multiscale call warns and falls back to
the dense path).  "tensorized" and "online" are ONE engine — the never-materialised sm_90a reductions, evaluated
exactly — and differ only where the reference's two backends differ numerically: for p = 1 / laplacian / energy
"tensorized" clamps |x-y|^2 at 1e-8 under the square root (utils.py:56-61) while "online" and "multiscale" use the
pykeops norm (no clamp).  "multiscale" is the two-scale Sinkhorn with kernel truncation / the truncated kernel
norms (multiscale.py) on the ranges mode of the same kernels, with exactly the reference's cluster blocks.  With
explicit labels for both clouds (the 6-tensor call form) the two-scale Sinkhorn also runs for 3 < D <= 64, like the
reference, whose ``clusterize`` takes labels in any dimension: the CUDA-core ranges kernels up to D = 8, the
tensor-core block-sparse softmins above (p = 2; p = 1 above D = 8 raises NotImplementedError).  Column-sharded
multi-GPU engines keep the single-scale route for such calls.
The Sinkhorn loss with p = 1 above D = 8 runs on the tensor-core p = 1 softmin (ops.softmin_l1), batched or not, in
both cost conventions; column-sharded multi-GPU engines have no such operator and raise NotImplementedError there.
Batched inputs (B, N, D) run as ONE launch group per reduction for the whole batch: a block-diagonal ranges problem
for D <= 8 (ranges.py), the batched tensor-core operators for 8 < D <= 64 (ops.softmin_batched, ops.softmin_l1,
kernel_conv_batched) and the wide ones for 64 < D <= 1024 (ops.softmin_wide, kernel_conv_wide).  Column-sharded
multi-GPU engines solve the batch element by element.
Above D = 64 every loss runs on the wide tensor-core operators (K-slab kernels, DESIGN.md section 3.5d), up to
D = 1024; above that, and for labelled two-scale calls or column-sharded engines above D = 64, NotImplementedError.
``cost=`` (a callable taking (B,N,D), (B,M,D) clouds and returning the (B,N,M) cost matrix) runs for the Sinkhorn loss
where the reference runs it, on the "tensorized" backend (chosen, picked by "auto" for N*M <= 5000**2, or reached by the
batched multiscale fallback), for any p > 0 and any D: the four matrices are formed by the user's function and each
Jacobi iteration's row softmins are one sm_90a launch (sinkhorn.sinkhorn_cost_matrices).  KeOps formula strings, the
"online" and "multiscale" backends, labels, column-sharded engines and the kernel losses raise NotImplementedError
with a cost.
Inputs must be float32 CUDA tensors: there is no CPU path.
"""
from __future__ import annotations

import torch
from torch.nn import Module

import warnings

from .kernel_loss import kernel_points, kernel_points_batched
from .multiscale import kernel_multiscale, sinkhorn_multiscale
from .ops import MAX_D, MAX_D_TC, MAX_D_WIDE
from . import kernel_small, sinkhorn_small
from .sinkhorn import sinkhorn_cost_matrices, sinkhorn_points, sinkhorn_points_batched

_LOSSES = ("sinkhorn", "hausdorff", "energy", "gaussian", "laplacian")

# Batches above D = 8 take the batched tensor-core operators while one element has at most this many pairs.  A larger
# element fills the GPU on its own, and the batched launch (B elements' column images streamed at once) is then no
# faster than the per-element loop.  Measured with tools/bench_batched_tc.py (DESIGN.md section 3.5b).
BATCHED_TC_MAX_PAIRS = 1e9
_BACKENDS = ("auto", "tensorized", "online", "multiscale")


def _route(loss):
    """Per-loss routine taking one unbatched problem (reference: the ``routines`` table, samples_loss.py:16-42)."""
    if loss == "sinkhorn":
        return sinkhorn_points
    if loss == "hausdorff":
        return lambda *args, **kw: kernel_points(*args, name=None, **kw)
    if loss in ("energy", "gaussian", "laplacian"):
        return lambda *args, **kw: kernel_points(*args, name=loss, **kw)
    raise KeyError(loss)


def _cuda_f32(*tensors):
    return all(t.is_cuda and t.dtype == torch.float32 for t in tensors)


_uniform_weights: dict = {}


class SamplesLoss(Module):
    """Geometric loss between two weighted point clouds (see the module docstring).

    Args mirror ``geomloss.SamplesLoss`` (samples_loss.py:178-194): loss, p, blur, reach, diameter,
    scaling, truncate, cost, kernel, cluster_scale, debias, potentials, verbose, backend.
    """

    def __init__(self, loss="sinkhorn", p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, truncate=5,
                 cost=None, kernel=None, cluster_scale=None, debias=True, potentials=False, verbose=False,
                 backend="auto"):
        super().__init__()
        self.loss = loss
        self.backend = backend
        self.p = p
        self.blur = blur
        self.reach = reach
        self.truncate = truncate
        self.diameter = diameter
        self.scaling = scaling
        self.cost = cost
        self.kernel = kernel
        self.cluster_scale = cluster_scale
        self.debias = debias
        self.potentials = potentials
        self.verbose = verbose
        # injected by geomloss_b200.distributed.shard_columns(): column-sharded reduction operators
        self._engine = {}
        self._multiscale_engine = None

    # ------------------------------------------------------------------------------------------
    def forward(self, *args):
        l_x, a, x, l_y, b, y = self.process_args(*args)
        B, N, M, D, l_x, a, l_y, b = self.check_shapes(l_x, a, x, l_y, b, y)

        backend = self.backend
        if backend not in _BACKENDS:
            raise KeyError(backend)
        if l_x is not None or l_y is not None:
            if backend not in ("auto", "multiscale"):
                raise ValueError(
                    'Explicit cluster labels are only supported with the "auto" and "multiscale" backends.')
            backend = "multiscale"
        elif backend == "auto":
            if M * N <= 5000**2:
                backend = "tensorized"
            elif D <= 3 and self.loss == "sinkhorn" and M * N > 10000**2 and self.p == 2:
                backend = "multiscale"
            else:
                backend = "online"
        if backend == "multiscale" and B > 1:
            warnings.warn("The 'multiscale' backend do not support batchsize > 1. Using 'tensorized' instead: "
                          "beware of memory overflows!")
            backend = "tensorized"
        if self.cost is not None:
            if (self.loss == "sinkhorn" and backend == "tensorized" and callable(self.cost) and not self._engine
                    and self._multiscale_engine is None and _cuda_f32(a, x, b, y)):
                # the user's cost matrices, row softmins on the GPU (sinkhorn.sinkhorn_cost_matrices)
                values = sinkhorn_cost_matrices(a, x, b, y, self.cost, p=self.p, blur=self.blur, reach=self.reach,
                                                diameter=self.diameter, scaling=self.scaling, debias=self.debias,
                                                potentials=self.potentials)
                if self.potentials:
                    return values[0].view(-1, N), values[1].view(-1, M)
                return values
            raise NotImplementedError(
                "a custom cost (a callable returning the (B,N,M) cost matrix) runs with loss='sinkhorn' and "
                "backend='tensorized' (chosen, or picked by 'auto' for "
                "N*M <= 5000**2) on float32 CUDA clouds, without labels or column-sharded engines: the engine forms "
                "the user's (B,N,M) cost matrices there; KeOps formulas, the 'online' and 'multiscale' backends "
                "and the kernel losses evaluate only |x-y|^p/p, p in {1,2}, on the fly")
        routine = _route(self.loss)
        kw = dict(p=self.p, blur=self.blur, reach=self.reach, diameter=self.diameter, scaling=self.scaling,
                  debias=self.debias, potentials=self.potentials, kernel=self.kernel,
                  keops=(backend != "tensorized"), **self._engine)
        if backend == "multiscale" and self.loss != "sinkhorn":
            # kernel_multiscale (kernel_samples.py:177-271); "hausdorff" dies with KeyError(None) like the reference
            sq = (lambda t: t[0]) if B == 1 else (lambda t: t)
            name = None if self.loss == "hausdorff" else self.loss
            values = kernel_multiscale(sq(a), sq(x), sq(b), sq(y), name=name, blur=self.blur, truncate=self.truncate,
                                       diameter=self.diameter, cluster_scale=self.cluster_scale,
                                       potentials=self.potentials, kernel=self.kernel, verbose=self.verbose,
                                       conv=self._engine.get("conv"))
            if self.potentials:
                F, G = values
                return F.view_as(a), G.view_as(b)
            return values if B == 0 else values.view(-1)
        # user labels above D = 3 (the voxel grid stops there): the two-scale Sinkhorn on one GPU, up to D = 64
        labelled = (l_x is not None and l_y is not None and D <= MAX_D_TC and not self._engine
                    and self._multiscale_engine is None)
        if backend == "multiscale" and self.loss == "sinkhorn" and l_x is not None and l_y is not None and D > MAX_D_TC:
            # no block-sparse kernel above D = 64: refuse rather than return the single-scale value
            raise NotImplementedError(f"the labelled two-scale Sinkhorn serves D <= {MAX_D_TC}, got D = {D} (the "
                                      f"single-scale backends 'tensorized' / 'online' serve D <= {MAX_D_WIDE})")
        if self._engine and D > MAX_D_TC:
            raise NotImplementedError(f"column-sharded engines serve D <= {MAX_D_TC}, got D = {D} (one GPU serves "
                                      f"D <= {MAX_D_WIDE})")
        if backend == "multiscale" and self.loss == "sinkhorn" and (D <= 3 or labelled):
            # single problem (B == 0, or B == 1 squeezed like the reference does, samples_loss.py:249-251)
            sq = (lambda t: t[0]) if B == 1 else (lambda t: t)
            values = sinkhorn_multiscale(sq(a), sq(x), sq(b), sq(y), p=self.p, blur=self.blur, reach=self.reach,
                                         diameter=self.diameter, scaling=self.scaling, truncate=self.truncate,
                                         cluster_scale=self.cluster_scale, debias=self.debias,
                                         potentials=self.potentials, labels_x=l_x, labels_y=l_y,
                                         verbose=self.verbose, engine=self._multiscale_engine)
            if self.potentials:
                F, G = values
                return F.view_as(a), G.view_as(b)
            return values if B == 0 else values.view(-1)

        if self.loss == "sinkhorn" and not self._engine and sinkhorn_small.eligible(N, M, D):
            # small clouds (batched or not): one launch per Sinkhorn iteration (csrc/b200ot_small.cu)
            lift = (lambda t: t.unsqueeze(0)) if B == 0 else (lambda t: t)
            values = sinkhorn_small.sinkhorn_small(lift(a), lift(x), lift(b), lift(y), **kw)
            if self.potentials:
                F, G = values
                return (F.view(1, -1), G.view(1, -1)) if B == 0 else (F.view_as(a), G.view_as(b))
            return values[0] if B == 0 else values
        if (self.loss in ("gaussian", "laplacian", "energy") and not self._engine and self.kernel is None
                and not self.potentials and sinkhorn_small.eligible(N, M, D)):
            # small clouds: the matvecs of kernel_loss in one launch, the cloud gradients in one more
            lift = (lambda t: t.unsqueeze(0)) if B == 0 else (lambda t: t)
            values = kernel_small.kernel_small(lift(a), lift(x), lift(b), lift(y), name=self.loss, blur=self.blur,
                                               potentials=self.potentials, keops=kw["keops"])
            if self.potentials:
                F, G = values
                return (F.view(1, -1), G.view(1, -1)) if B == 0 else (F.view_as(a), G.view_as(b))
            return values[0] if B == 0 else values
        if B == 0:
            values = routine(a, x, b, y, **kw)
            if self.potentials:
                F, G = values
                return F.view(1, -1), G.view(1, -1)  # the reference's (1,N) shape for unbatched input
            return values
        if self.loss == "sinkhorn" and kw["diameter"] is None:
            # the reference measures ONE diameter over the flattened batch (sinkhorn_divergence.py:156-158),
            # so all batch elements share the same eps-schedule
            from .sinkhorn import max_diameter

            kw["diameter"] = max_diameter(x.reshape(-1, D), y.reshape(-1, D))
        one_group = D <= MAX_D or (D <= MAX_D_WIDE and N * M <= BATCHED_TC_MAX_PAIRS)
        if B > 1 and one_group and not self._engine and self.loss != "hausdorff":
            # the whole batch in one launch group per reduction (D <= 8: block-diagonal ranges problem; above: the
            # batched tensor-core operators)
            batched = sinkhorn_points_batched if self.loss == "sinkhorn" else kernel_points_batched
            if self.loss != "sinkhorn":
                kw["name"] = self.loss
            values = batched(a, x, b, y, **kw)
            if self.potentials:
                return values[0].view_as(a), values[1].view_as(b)
            return values
        per_batch = [routine(a[k], x[k], b[k], y[k], **kw) for k in range(B)]
        if self.potentials:
            F = torch.stack([f for f, _ in per_batch])
            G = torch.stack([g for _, g in per_batch])
            return F.view_as(a), G.view_as(b)
        return torch.stack(per_batch)

    # ------------------------------------------------------------------------------------------
    def process_args(self, *args):
        """2 tensors: (x, y) with uniform weights; 4: (a, x, b, y); 6: (l_x, a, x, l_y, b, y)."""
        if len(args) == 6:
            return args
        if len(args) == 4:
            a, x, b, y = args
            return None, a, x, None, b, y
        if len(args) == 2:
            x, y = args
            return None, self.generate_weights(x), x, None, self.generate_weights(y), y
        raise ValueError(
            "A SamplesLoss accepts two (x, y), four (α, x, β, y) or six (l_x, α, x, l_y, β, y)  arguments.")

    def generate_weights(self, x):
        """Uniform weights 1/N (samples_loss.py:328-335); read-only, so one tensor per (shape, device, dtype) is kept
        instead of three tiny launches per cloud and call."""
        if x.dim() not in (2, 3):
            raise ValueError("Input samples 'x' and 'y' should be encoded as (N,D) or (B,N,D) (batch) tensors.")
        key = (tuple(x.shape[:-1]), x.device, x.dtype)
        w = _uniform_weights.get(key)
        if w is None:
            if len(_uniform_weights) >= 64:
                _uniform_weights.clear()
            w = _uniform_weights[key] = torch.ones(x.shape[:-1]).type_as(x) / x.shape[-2]
        return w

    @staticmethod
    def _check_labels(l, n, which):
        if l is None:
            return None
        if l.dim() not in (1, 2) or (l.dim() == 2 and l.shape[1] > 1):
            raise ValueError(f"Without batches, the vector of labels '{which}' should be encoded as an "
                             f"({'N' if which == 'l_x' else 'M'},) or ({'N' if which == 'l_x' else 'M'},1) tensor.")
        l = l.view(-1)
        if len(l) != n:
            raise ValueError(f"The vector of labels '{which}' should have the same length as the point cloud "
                             f"'{'x' if which == 'l_x' else 'y'}'.")
        return l

    def check_shapes(self, l_x, a, x, l_y, b, y):
        """Validation rules of samples_loss.py:337-474; returns (B, N, M, D, l_x, a, l_y, b), B = 0 unbatched."""
        if a.dim() != b.dim():
            raise ValueError("Input weights 'α' and 'β' should have the same number of dimensions.")
        if x.dim() != y.dim():
            raise ValueError("Input samples 'x' and 'y' should have the same number of dimensions.")
        if x.shape[-1] != y.shape[-1]:
            raise ValueError("Input samples 'x' and 'y' should have the same last dimension.")

        if x.dim() == 2:
            B = 0
            N, D = x.shape
            M = y.shape[0]
            if a.dim() not in (1, 2):
                raise ValueError(
                    "Without batches, input weights 'α' and 'β' should be encoded as (N,) or (N,1) tensors.")
            if a.dim() == 2:
                if a.shape[1] > 1:
                    raise ValueError(
                        "Without batches, input weights 'α' should be encoded as (N,) or (N,1) tensors.")
                if b.shape[1] > 1:
                    raise ValueError(
                        "Without batches, input weights 'β' should be encoded as (M,) or (M,1) tensors.")
                a, b = a.view(-1), b.view(-1)
            l_x = self._check_labels(l_x, N, "l_x")
            l_y = self._check_labels(l_y, M, "l_y")
            N2, M2 = a.shape[0], b.shape[0]
        elif x.dim() == 3:
            B, N, D = x.shape
            B2, M, _ = y.shape
            if B != B2:
                raise ValueError("Samples 'x' and 'y' should have the same batchsize.")
            if a.dim() not in (2, 3):
                raise ValueError(
                    "With batches, input weights 'α' and 'β' should be encoded as (B,N) or (B,N,1) tensors.")
            if a.dim() == 3:
                if a.shape[2] > 1:
                    raise ValueError(
                        "With batches, input weights 'α' should be encoded as (B,N) or (B,N,1) tensors.")
                if b.shape[2] > 1:
                    raise ValueError(
                        "With batches, input weights 'β' should be encoded as (B,M) or (B,M,1) tensors.")
                a, b = a.squeeze(-1), b.squeeze(-1)
            if l_x is not None or l_y is not None:
                raise NotImplementedError('The "multiscale" backend has not been implemented with batches.')
            B2, N2 = a.shape
            B3, M2 = b.shape
            if B != B2:
                raise ValueError("Samples 'x' and weights 'α' should have the same batchsize.")
            if B != B3:
                raise ValueError("Samples 'y' and weights 'β' should have the same batchsize.")
        else:
            raise ValueError("Input samples 'x' and 'y' should be encoded as (N,D) or (B,N,D) (batch) tensors.")

        if N != N2:
            raise ValueError("Weights 'α' and samples 'x' should have compatible shapes.")
        if M != M2:
            raise ValueError("Weights 'β' and samples 'y' should have compatible shapes.")
        return B, N, M, D, l_x, a, l_y, b

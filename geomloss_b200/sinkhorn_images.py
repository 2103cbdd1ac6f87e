"""Sinkhorn divergence between measures on regular 2-D / 3-D grids (images, volumes).

Host-side counterpart of src/geomloss/_legacy/sinkhorn_images.py:26-202 and of the grid helpers of
src/geomloss/_legacy/utils.py:69-108: a multiscale (pyramid) epsilon-scaling Sinkhorn loop whose only
heavy operator is the separable grid softmin — here ``b200ot_softmin_grid`` (csrc/b200ot_grid.cu) instead of
three pykeops LazyTensor reductions and two permutes.  The pyramid (2x sum-pooling), the log-densities
(floor -10000) and the bi/tri-linear upsampling of the potentials at a scale jump are cheap elementwise
torch ops on the device, exactly as in the reference.

Inputs follow the reference's actual contract (SURVEY.md appendix A-20): ``(B, C, N, N)`` or
``(B, C, N, N, N)`` float32 CUDA tensors with equal power-of-two sides.  Autograd: like the reference,
only the weights receive gradients (the potentials), through the final value formula.
"""
from __future__ import annotations


import numpy as np
import torch
from torch.nn.functional import avg_pool2d, avg_pool3d, interpolate

from . import ops
from .sinkhorn import damping, descend, epsilon_schedule, potential_reads, sinkhorn_cost


def _dimension(t):
    return t.dim() - 2


def pyramid(t):
    """[coarsest (1 pixel), ..., t]: repeated 2x sum-pooling.                              utils.py:77-97"""
    d = _dimension(t)
    levels = [t]
    for _ in range(int(np.log2(t.shape[2]))):
        t = 4 * avg_pool2d(t, 2) if d == 2 else 8 * avg_pool3d(t, 2)
        levels.append(t)
    levels.reverse()
    return levels


def upsample(t):
    """2x bi/tri-linear interpolation, align_corners=False.                               utils.py:100-102"""
    return interpolate(t, scale_factor=2, mode="bilinear" if _dimension(t) == 2 else "trilinear",
                       align_corners=False)


def log_dens(a):
    """log-density with empty pixels pinned to -10000.                                    utils.py:105-108"""
    return torch.where(a > 0, a.clamp_min(1e-45).log(), torch.full_like(a, -10000.0))


def softmin_grid(eps, p, h_a, h_b=None, h_scale_b=0.0, *, out_old=None, alpha_old=0.0, beta=1.0):
    """``alpha_old*out_old + beta*softmin_grid(eps, p, h_a + h_scale_b*h_b)`` on a (B, C, N, .., N) grid
    (reference operator: softmin_grid, utils.py:190-279).  One C-ABI call = one launch per axis."""
    h_a = ops._f32c(h_a, "h_a")
    h_b = ops._f32c(h_b, "h_b")
    out_old = ops._f32c(out_old, "out_old")
    d = _dimension(h_a)
    if d not in (2, 3):
        raise ValueError("grids must be (B, C, N, N) or (B, C, N, N, N)")
    N = h_a.shape[-1]
    if any(s != N for s in h_a.shape[2:]):
        raise ValueError("grid sides must be equal")
    dev = h_a.device
    out = torch.empty_like(h_a)
    ops._call(dev, "b200ot_softmin_grid", h_a, h_b, float(h_scale_b), out_old, float(alpha_old), float(beta), out,
              h_a.shape[0] * h_a.shape[1], N, d, int(p), float(eps), launches=d)
    return out


def sinkhorn_divergence(a, b, p=2, blur=None, reach=None, axes=None, scaling=0.5, cost=None, debias=True,
                        potentials=False, verbose=False, **kwargs):
    """Sinkhorn divergence between two batches of images / volumes.        sinkhorn_images.py:26-202

    Returns a ``(B,)`` tensor, or the pair of dual potentials (same shape as the inputs) if
    ``potentials=True``.
    """
    if a.shape != b.shape:
        raise ValueError("a and b must have the same shape")
    if cost is not None:
        raise NotImplementedError()
    if blur is None:
        blur = 1 / a.shape[-1]
    if scaling < 0.5:
        raise ValueError(f"Scaling value of {scaling} is too small: please use a number in [0.5, 1).")

    a_s, b_s = pyramid(a)[1:], pyramid(b)[1:]  # the 1-pixel level is dropped (:110)
    a_logs = [log_dens(t.detach()) for t in a_s]
    b_logs = [log_dens(t.detach()) for t in b_s]
    diameter = 1
    eps_final = blur**p
    rho = None if reach is None else reach**p
    eps_list = epsilon_schedule(p, diameter, blur, scaling)

    # jump to the next (finer) level as soon as its pixels are resolved by the temperature (:152-170)
    scales = [diameter / t.shape[-1] for t in a_s]
    current = scales.pop(0)
    jumps = []
    for i, eps in enumerate(eps_list[1:]):
        if current**p > eps:
            jumps.append(i + 1)
            current = scales.pop(0)
    if verbose:
        print("Pyramid scales:", [diameter / t.shape[-1] for t in a_s])
        print("Temperatures: ", eps_list)
        print("Jumps: ", jumps)
    assert len(jumps) == len(a_s) - 1, "There's a bug in the multicale pre-processing..."

    def level_step(k):
        """``descend``'s step on pyramid level k, its slots (f_ba, g_ab, f_aa, g_bb) the log-weights of the columns."""
        logs = [b_logs[k], a_logs[k], a_logs[k], b_logs[k]][:4 if debias else 2]
        none = [None] * len(logs)

        def step(eps, reads, olds, alpha_old, beta):
            inv = 0.0 if reads is None else 1.0 / eps
            return [softmin_grid(eps, p, log_w, h, inv, out_old=old, alpha_old=alpha_old, beta=beta)
                    for log_w, h, old in zip(logs, reads or none, olds or none)]
        return step

    # one descent per level on the temperatures up to its jump, the potentials up-sampled between levels
    bounds = [0] + [i + 1 for i in jumps] + [len(eps_list)]
    pots = None
    for k in range(len(a_s)):
        pots = descend(level_step(k), eps_list[bounds[k]:bounds[k + 1]], rho, pots)
        if k + 1 < len(a_s):
            pots = [upsample(t) for t in pots]
    if len(eps_list) - 1 not in jumps:  # else the up-sampling was the last step (:520-526)
        eps = eps_list[-1]
        with torch.no_grad():
            pots = level_step(len(a_s) - 1)(eps, potential_reads(pots), None, 0.0, damping(eps, rho))

    B = a.shape[0]
    f_ba, g_ab, f_aa, g_bb = [t.reshape(B, -1) for t in pots] + [None] * (4 - len(pots))
    out = sinkhorn_cost(eps_final, rho, a.reshape(B, -1), b.reshape(B, -1), f_aa, g_bb, g_ab, f_ba, debias=debias,
                        potentials=potentials)
    return tuple(t.view(a.shape) for t in out) if potentials else out

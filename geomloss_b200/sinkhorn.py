"""Host side of the Sinkhorn divergence on point clouds: epsilon-scaling schedule, the symmetric
Sinkhorn loop and the dual-to-value formulas.  Every softmin lands in libb200ot.so (see ops.py).

This follows the control flow of the reference because the control flow *is* the specification
(src/geomloss/_legacy/sinkhorn_divergence.py:56-163 schedule/scalars, :171-250 value, :258-628 loop;
driver src/geomloss/_legacy/sinkhorn_samples.py:349-424), with three changes:
  * the "cost matrix" is the pair of point clouds — nothing of size N x M is ever stored;
  * ``h = log_w + pot/eps``, the damping factor and the ``1/2 (f + f~)`` averaging are fused into the
    softmin launch (prologue / epilogue) instead of separate elementwise kernels;
  * the autograd switch is a context manager, not the reference's global ``set_grad_enabled`` toggle.
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def damping(eps, rho):
    """1 for balanced OT, 1/(1+eps/rho) with a KL marginal penalty.          sinkhorn_divergence.py:56-58"""
    return 1.0 if rho is None else 1.0 / (1.0 + eps / rho)


def log_weights(a):
    """log(a) with the log of non-positive weights pinned to -1e5.           sinkhorn_divergence.py:61-65"""
    return torch.where(a > 0, a.clamp_min(1e-45).log(), torch.full_like(a, -100000.0))


def max_diameter(x, y):
    """Length of the diagonal of the joint bounding box (one host sync).     sinkhorn_divergence.py:96-112"""
    lh = ops.cloud_extent(x, y)
    if lh is not None:  # one launch + one 2D-float copy; the norm of D numbers is taken on the host
        return extent_diameter(lh)
    lo = torch.minimum(x.min(0).values, y.min(0).values)
    hi = torch.maximum(x.max(0).values, y.max(0).values)
    return (hi - lo).norm().item()


def extent_diameter(lh):
    """Diagonal of a (2, D) [minima; maxima] box from ops.cloud_extent."""
    lo, hi = lh.cpu().double().unbind(0)
    return float(torch.sqrt(((hi - lo) ** 2).sum()).float())


def epsilon_schedule(p, diameter, blur, scaling):
    """Temperatures diam^p -> blur^p, geometric with ratio scaling^p; the first value appears twice
    (the arange starts at p log diam) exactly as in the reference.          sinkhorn_divergence.py:115-151"""
    steps = np.arange(p * np.log(diameter), p * np.log(blur), p * np.log(scaling))
    return [diameter**p] + [float(np.exp(e)) for e in steps] + [blur**p]


def scaling_parameters(x, y, p, blur, reach, diameter, scaling):
    """(diameter, eps, eps_list, rho).                                      sinkhorn_divergence.py:154-163"""
    if diameter is None:
        d = x.shape[-1]
        diameter = max_diameter(x.reshape(-1, d), y.reshape(-1, d))
    rho = None if reach is None else reach**p
    return diameter, blur**p, epsilon_schedule(p, diameter, blur, scaling), rho


def softmin_many(sm, calls):
    """Run the independent softmins ``calls = [(args, kwargs), ...]`` of one Jacobi iteration through ``sm``; an engine
    that can overlap their collectives (distributed.ColumnShardedEngine.softmin_raw_many) gets them all at once, and
    ``ops.softmin_raw`` runs mirrored calls (the xy and yx updates) as one paired launch group (ops.softmin_raw_many).
    An operator that offers neither (an injected or recording one) gets the calls one by one."""
    owner = getattr(sm, "__self__", None)
    many = getattr(sm if owner is None else owner, "softmin_raw_many", None)
    if many is not None:
        return many(calls)
    return [sm(*args, **kw) for args, kw in calls]


def potential_reads(pots):
    """The potential each slot (f_ba, g_ab, f_aa, g_bb) reads: C_xy reads g_ab, C_yx f_ba, the debias ones their own."""
    return [pots[1], pots[0]] + list(pots[2:])


def descend(step, eps_list, rho, pots=None):
    """The no-grad part of the reference's loop (sinkhorn_divergence.py:461-493) over the 2 (no debias) or 4 slots
    (f_ba, g_ab, f_aa, g_bb): without starting ``pots``, the initialisation at ``eps_list[0]``; then one averaged
    Jacobi step per temperature of ``eps_list``, every slot reading the OLD potentials.  ``step(eps, reads, olds,
    alpha_old, beta)`` returns the slots' ``alpha_old * olds[k] + beta * softmin(eps, slot k, reads[k])``, ``reads``
    and ``olds`` None at the initialisation.  The extrapolations and the last, gradient-carrying step stay with the
    drivers: each runs its own operator there."""
    with torch.no_grad():
        if pots is None:
            pots = step(eps_list[0], None, None, 0.0, damping(eps_list[0], rho))
        for eps in eps_list:
            pots = step(eps, potential_reads(pots), pots, 0.5, 0.5 * damping(eps, rho))
    return pots


def slot_calls(slots, eps, reads, olds, alpha_old, beta, **kw):
    """The calls ``[(args, kwargs), ...]`` of one ``descend`` step of a point-cloud softmin (``ops.softmin_raw``'s
    signature): slot k is (rows, columns, log-weights of the columns, operands after ``h_scale_b``)."""
    n = len(slots)
    inv = 0.0 if reads is None else 1.0 / eps
    return [((eps, rows, cols, log_w, h, inv, *more), dict(out_old=old, alpha_old=alpha_old, beta=beta, **kw))
            for (rows, cols, log_w, *more), h, old in zip(slots, reads or [None] * n, olds or [None] * n)]


def sinkhorn_loop_points(a_log, b_log, x, y, eps_list, rho, *, p=2, debias=True, center=None, softmin_raw=None,
                         softmin_grad=None, problems=None):
    """Symmetric Sinkhorn iterations with eps-scaling on one pair of clouds.   sinkhorn_divergence.py:258-628

    The iterations (``descend``) run without autograd on detached clouds, each one fused launch group per update.
    The last update is not averaged, takes ``x`` / ``y`` with autograd and detached right-hand sides,
    and therefore carries the whole gradient (envelope theorem).  Returns (f_aa, g_bb, g_ab, f_ba).

    ``softmin_raw`` / ``softmin_grad`` default to the single-GPU kernels; the column-sharded
    multi-GPU engine (distributed.py) injects its own pair with the same signatures, and gets the updates of one
    iteration at once (``softmin_many``).
    ``problems`` (batched inputs): ranges-mode descriptors of the block-diagonal problems (f_ba, g_ab[, f_aa, g_bb])
    obtained by stacking the B batch elements along the point axis — the whole batch then runs in ONE launch group
    per softmin, like the reference's batched LazyTensor reduction (sinkhorn_samples.py:229-290).
    """
    # the (f_ba, g_ab, f_aa, g_bb) slots: rows, columns, log-weights of the columns (, ranges problem)
    slots = [(x, y, b_log), (y, x, a_log), (x, x, a_log), (y, y, b_log)][:4 if debias else 2]
    if problems is None:
        sm, smg = softmin_raw or ops.softmin_raw, softmin_grad or ops.softmin
    else:
        from . import ranges

        sm, smg = ranges.softmin_ranges_raw, ranges.softmin_ranges
        slots = [slot + (prob,) for slot, prob in zip(slots, problems)]
    detached = [(rows.detach(), cols.detach(), *rest) for rows, cols, *rest in slots]

    def step(*args):
        return [out for out, _ in softmin_many(sm, slot_calls(detached, *args, p=p, center=center))]

    pots = descend(step, eps_list, rho)
    # final extrapolation: eps / lam are the last values of the schedule (reference: leaked loop variables)
    eps = eps_list[-1]
    lam, inv = damping(eps, rho), 1.0 / eps
    new = [smg(eps, rows, cols.detach(), log_w, h, inv, *more, p=p, center=center, scale_out=lam)
           for (rows, cols, log_w, *more), h in zip(slots, potential_reads(pots))]
    f_ba, g_ab, f_aa, g_bb = new + [None] * (4 - len(new))
    return f_aa, g_bb, g_ab, f_ba


def sinkhorn_cost(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=True, potentials=False):
    """Value of the divergence (or the dual potentials) from the four potentials, reduced over the last axis: (N,)
    vectors give a scalar, B problems as (B, n) rows give (B,) (scal(batch=True), utils.py:13-18).
    sinkhorn_divergence.py:171-250.  The unbalanced weight is (rho + eps/2) in both passes — the
    reference's UnbalancedWeight.backward is dead code (SURVEY.md appendix A-11).  Elementwise products and sums
    (plain reduction kernels: no cuBLAS on the value path)."""
    if potentials:
        return (f_ba - f_aa, g_ab - g_bb) if debias else (f_ba, g_ab)
    if rho is None:
        f, g = (f_ba - f_aa, g_ab - g_bb) if debias else (f_ba, g_ab)
    else:
        w = rho + eps / 2
        if debias:
            f, g = w * ((-f_aa / rho).exp() - (-f_ba / rho).exp()), w * ((-g_bb / rho).exp() - (-g_ab / rho).exp())
        else:
            f, g = w * (1 - (-f_ba / rho).exp()), w * (1 - (-g_ab / rho).exp())
    return (a * f).sum(-1) + (b * g).sum(-1)


def sinkhorn_points(a, x, b, y, p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, debias=True,
                    potentials=False, softmin_raw=None, softmin_grad=None, keops=False, **_ignored):
    """Sinkhorn divergence between two weighted clouds a:(N,) x:(N,D) b:(M,) y:(M,D) on one CUDA device.
    Counterpart of sinkhorn_tensorized / sinkhorn_online (sinkhorn_samples.py:74-221, :349-424) for a single batch
    element.  ``keops``: the "online" cost convention — for p = 1, Norm2(x-y) without the 1e-8 clamp of the
    tensorized `distances` (sinkhorn_samples.py:303-306 vs utils.py:56-61).  The softmins are the ones
    ``ops.softmin_operators`` names for D and p, unless the caller injected its own operators."""
    if p not in (1, 2):
        raise KeyError(p)  # the reference's cost table only knows p = 1, 2 (sinkhorn_samples.py:26-29)
    diameter, eps, eps_list, rho = scaling_parameters(x, y, p, blur, reach, diameter, scaling)
    center = ops.default_center(x.detach(), y.detach())
    pk = (p | ops.P_UNCLAMPED) if keops else p
    if softmin_raw is None and softmin_grad is None:
        softmin_raw, softmin_grad = ops.softmin_operators(x.shape[-1], p)
    f_aa, g_bb, g_ab, f_ba = sinkhorn_loop_points(log_weights(a.detach()), log_weights(b.detach()), x, y, eps_list,
                                                  rho, p=pk, debias=debias, center=center, softmin_raw=softmin_raw,
                                                  softmin_grad=softmin_grad)
    return sinkhorn_cost(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=debias, potentials=potentials)


def sinkhorn_points_batched(a, x, b, y, p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, debias=True,
                            potentials=False, keops=False, **_ignored):
    """Batched Sinkhorn divergence a:(B,N) x:(B,N,D) b:(B,M) y:(B,M,D): every softmin of the loop is ONE launch group
    over the whole batch, not B launches — the batched operators ``ops.softmin_operators`` names for D and p, and for
    D <= 8, where it names none, a ranges-mode block-diagonal problem.
    Reference: sinkhorn_tensorized / sinkhorn_online on (B, ...) inputs, softmin_online_lazytensor
    (sinkhorn_samples.py:74-221, :229-290, :349-424); one shared eps-schedule (diameter over the flattened batch)."""
    from . import ranges

    if p not in (1, 2):
        raise KeyError(p)
    B, N, D = x.shape
    M = y.shape[1]
    diameter, eps, eps_list, rho = scaling_parameters(x, y, p, blur, reach, diameter, scaling)
    xf, yf = x.reshape(B * N, D), y.reshape(B * M, D)
    center = ops.default_center(xf.detach(), yf.detach())
    pk = (p | ops.P_UNCLAMPED) if keops else p
    a_log, b_log = log_weights(a.detach()), log_weights(b.detach())
    batched_ops = ops.softmin_operators(D, p, batched=True)
    if batched_ops is not None:  # the operators take the (B, n, D) clouds and (B, n) potentials
        raw, grad = batched_ops
        inputs = (a_log, b_log, xf.view(B, N, D), yf.view(B, M, D))
        loop = dict(softmin_raw=raw, softmin_grad=grad)
    else:  # the B problems stacked along the point axis: one block-diagonal ranges problem per pair of clouds
        sizes = [(N, M), (M, N), (N, N), (M, M)][:4 if debias else 2]
        inputs = (a_log.reshape(B * N), b_log.reshape(B * M), xf, yf)
        loop = dict(problems=[ranges.batch_problem(B, r, c, x.device) for r, c in sizes])
    pots = sinkhorn_loop_points(*inputs, eps_list, rho, p=pk, debias=debias, center=center, **loop)
    f_aa, g_bb, g_ab, f_ba = (None if t is None else t.view(B, -1) for t in pots)
    return sinkhorn_cost(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=debias, potentials=potentials)


class _LastRows(torch.autograd.Function):
    """The last, non-averaged update ``lam * softmin(eps, C_k, log_w_k + pot_k / eps)`` of the 2 or 4 cost matrices
    in one group, differentiable w.r.t. each C_k; log-weights and potentials are constants, as the reference's
    detached right-hand sides make them (sinkhorn_divergence.py:612-623).  ``rest`` is the k matrices (each carrying
    the caller's graph, contiguous) followed by their k log-weights and k potentials."""

    @staticmethod
    def forward(ctx, eps, lam, *rest):
        k = len(rest) // 3
        Cs, logs, pots = rest[:k], rest[k:2 * k], rest[2 * k:]
        res = ops.dense_softmin_rows_raw(eps, [(C, lw, pot, None) for C, lw, pot in zip(Cs, logs, pots)], beta=lam,
                                         want_lse2=True)
        ctx.save_for_backward(*Cs, *logs, *pots, *(lse2 for _, lse2 in res))
        ctx.meta = (k, float(eps), float(lam))
        return tuple(out for out, _ in res)

    @staticmethod
    def backward(ctx, *gos):
        k, eps, lam = ctx.meta
        saved = ctx.saved_tensors
        grads = [None] * k
        for i in range(k):
            if ctx.needs_input_grad[2 + i] and gos[i] is not None:
                grads[i] = ops.dense_softmin_rows_grad(eps, saved[i], saved[k + i], saved[2 * k + i], saved[3 * k + i],
                                                       (lam * gos[i]).contiguous())
        return (None, None, *grads) + (None,) * (2 * k)


def _cost_matrix(cost, u, v, name, rows, cols, like):
    """``cost(u, v)`` checked like an operator input: (B, rows, cols), of ``like``'s dtype (float32 for the kernels)
    and on its device; a non-contiguous result (a transposed view, ...) is copied once."""
    C = cost(u, v)
    B = u.shape[0]
    if not torch.is_tensor(C) or tuple(C.shape) != (B, rows, cols):
        shape = tuple(C.shape) if torch.is_tensor(C) else type(C).__name__
        raise ValueError(f"cost(x, y) must return the (B, N, M) = {(B, rows, cols)} matrix {name}, got {shape}")
    if C.dtype != like.dtype or C.device != like.device:
        raise TypeError(f"cost(x, y) must return a {like.dtype} tensor on {like.device} ({name}), got {C.dtype} on "
                        f"{C.device}")
    return C.contiguous()


def sinkhorn_cost_matrices(a, x, b, y, cost, p=2, blur=0.05, reach=None, diameter=None, scaling=0.5, debias=True,
                           potentials=False):
    """Sinkhorn divergence with a user-supplied cost: the reference's "tensorized" backend with ``cost=``
    (sinkhorn_samples.py:74-221), for a:(N,) x:(N,D) b:(M,) y:(M,D) or a batch a:(B,N) x:(B,N,D) b:(B,M) y:(B,M,D).

    ``cost`` is called exactly as the reference calls it, on (B, n, D) clouds (B = 1 for unbatched input) with detached
    right-hand sides: C_xy = cost(x, y), C_yx = cost(y, x), then with ``debias`` C_xx = cost(x, x), C_yy = cost(y, y).
    C_yx need not be C_xy^T.  Every update of the loop is a row softmin of one of these matrices, and all those of one
    iteration are ONE ``ops.dense_softmin_rows_raw`` call (1 + k launches for k softmins).  The last update carries the
    gradient to the matrices, and through ``cost`` to x and y; a and b get theirs through the value formula.
    Returns the (B,) values (a scalar for unbatched input) or the potentials (1, N) / (1, M), (B, N) / (B, M)."""
    batched = x.dim() == 3
    if not batched:
        a, x, b, y = a.unsqueeze(0), x.unsqueeze(0), b.unsqueeze(0), y.unsqueeze(0)
    B, N, _ = x.shape
    M = y.shape[1]
    xd, yd = x.detach(), y.detach()
    mats = [_cost_matrix(cost, x, yd, "C_xy", N, M, x), _cost_matrix(cost, y, xd, "C_yx", M, N, x)]
    if debias:
        mats += [_cost_matrix(cost, x, xd, "C_xx", N, N, x), _cost_matrix(cost, y, yd, "C_yy", M, M, x)]
    diameter, eps, eps_list, rho = scaling_parameters(x, y, p, blur, reach, diameter, scaling)
    a_log, b_log = log_weights(a.detach()), log_weights(b.detach())
    logs = [b_log, a_log, a_log, b_log][:len(mats)]  # the columns of C_xy are y's, of C_yx x's, ...
    Cd = [C.detach() for C in mats]

    def step(eps, reads, olds, alpha_old, beta):
        none = [None] * len(Cd)
        problems = list(zip(Cd, logs, reads or none, olds or none))
        return [out for out, _ in ops.dense_softmin_rows_raw(eps, problems, alpha_old=alpha_old, beta=beta)]

    pots = descend(step, eps_list, rho)
    # final extrapolation: eps / lam are the last values of the schedule (reference: leaked loop variables)
    eps = eps_list[-1]
    lam = damping(eps, rho)
    reads = potential_reads(pots)
    if torch.is_grad_enabled() and any(C.requires_grad for C in mats):
        new = list(_LastRows.apply(eps, lam, *mats, *logs, *reads))
    else:
        new = step(eps, reads, None, 0.0, lam)
    f_ba, g_ab, f_aa, g_bb = new + [None] * (4 - len(new))
    out = sinkhorn_cost(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=debias, potentials=potentials)
    return out if batched or potentials else out[0]

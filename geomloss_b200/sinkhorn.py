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
    that can overlap their collectives (distributed.ColumnShardedEngine.softmin_raw_many) gets them all at once."""
    owner = getattr(sm, "__self__", None)
    many = getattr(owner, "softmin_raw_many", None) if owner is not None else None
    if many is not None:
        return many(calls)
    return [sm(*args, **kw) for args, kw in calls]


def sinkhorn_loop_points(a_log, b_log, x, y, eps_list, rho, *, p=2, debias=True, center=None, softmin_raw=None,
                         softmin_grad=None, problems=None):
    """Symmetric Sinkhorn iterations with eps-scaling on one pair of clouds.   sinkhorn_divergence.py:258-628

    The iterations run without autograd on detached clouds.  All four updates of an iteration read the
    OLD potentials (Jacobi), then  f <- 1/2 f + 1/2 lam softmin(...)  — one fused launch each.
    The last update is not averaged, takes ``x`` / ``y`` with autograd and detached right-hand sides,
    and therefore carries the whole gradient (envelope theorem).  Returns (f_aa, g_bb, g_ab, f_ba).

    ``softmin_raw`` / ``softmin_grad`` default to the single-GPU kernels; the column-sharded
    multi-GPU engine (distributed.py) injects its own pair with the same signatures.
    ``problems`` (batched inputs): ranges-mode descriptors {"xy", "yx", "xx", "yy"} of the block-diagonal problems
    obtained by stacking the B batch elements along the point axis — the whole batch then runs in ONE launch group
    per softmin, like the reference's batched LazyTensor reduction (sinkhorn_samples.py:229-290).
    """
    if problems is None:
        sm = softmin_raw or ops.softmin_raw
        smg = softmin_grad or ops.softmin
    else:
        from . import ranges

        def _prob(rows, cols):
            key = ("x" if rows is x or rows is xd else "y") + ("x" if cols is x or cols is xd else "y")
            # (x is y: every key reads "xx", and the four problems have the same shape)
            return problems[key] if key in problems else problems["xy"]

        def sm(eps, rows, cols, h_a, h_b=None, h_scale_b=0.0, **kw):
            return ranges.softmin_ranges_raw(eps, rows, cols, h_a, h_b, h_scale_b, _prob(rows, cols), **kw)

        def smg(eps, rows, cols, h_a, h_b=None, h_scale_b=0.0, **kw):
            return ranges.softmin_ranges(eps, rows, cols, h_a, h_b, h_scale_b, _prob(rows, cols), **kw)

    xd, yd = x.detach(), y.detach()
    with torch.no_grad():
        eps = eps_list[0]
        lam = damping(eps, rho)
        g_ab = sm(eps, yd, xd, a_log, p=p, center=center, beta=lam)[0]
        f_ba = sm(eps, xd, yd, b_log, p=p, center=center, beta=lam)[0]
        if debias:
            f_aa = sm(eps, xd, xd, a_log, p=p, center=center, beta=lam)[0]
            g_bb = sm(eps, yd, yd, b_log, p=p, center=center, beta=lam)[0]
        for eps in eps_list:
            lam = damping(eps, rho)
            inv = 1.0 / eps
            ukw = dict(p=p, center=center, alpha_old=0.5, beta=0.5 * lam)
            calls = [((eps, xd, yd, b_log, g_ab, inv), dict(out_old=f_ba, **ukw)),
                     ((eps, yd, xd, a_log, f_ba, inv), dict(out_old=g_ab, **ukw))]
            if debias:
                calls += [((eps, xd, xd, a_log, f_aa, inv), dict(out_old=f_aa, **ukw)),
                          ((eps, yd, yd, b_log, g_bb, inv), dict(out_old=g_bb, **ukw))]
            res = softmin_many(sm, calls)  # all four read the OLD potentials (Jacobi): independent
            f_ba, g_ab = res[0][0], res[1][0]
            if debias:
                f_aa, g_bb = res[2][0], res[3][0]
    # final extrapolation: eps / lam are the last values of the schedule (reference: leaked loop variables)
    inv = 1.0 / eps
    new_f_ba = smg(eps, x, yd, b_log, g_ab, inv, p=p, center=center, scale_out=lam)
    new_g_ab = smg(eps, y, xd, a_log, f_ba, inv, p=p, center=center, scale_out=lam)
    if debias:
        new_f_aa = smg(eps, x, xd, a_log, f_aa, inv, p=p, center=center, scale_out=lam)
        new_g_bb = smg(eps, y, yd, b_log, g_bb, inv, p=p, center=center, scale_out=lam)
        return new_f_aa, new_g_bb, new_g_ab, new_f_ba
    return None, None, new_g_ab, new_f_ba


def _dot(w, f):
    """<w, f> as an elementwise product + sum (a plain reduction kernel: no cuBLAS on the value path)."""
    return (w * f).sum()


def sinkhorn_cost(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, debias=True, potentials=False):
    """Value of the divergence (or the dual potentials) from the four potentials, unbatched vectors.
    sinkhorn_divergence.py:171-250.  The unbalanced weight is (rho + eps/2) in both passes — the
    reference's UnbalancedWeight.backward is dead code (SURVEY.md appendix A-11)."""
    if potentials:
        return (f_ba - f_aa, g_ab - g_bb) if debias else (f_ba, g_ab)
    if rho is None:
        if debias:
            return _dot(a, f_ba - f_aa) + _dot(b, g_ab - g_bb)
        return _dot(a, f_ba) + _dot(b, g_ab)
    w = rho + eps / 2
    if debias:
        return _dot(a, w * ((-f_aa / rho).exp() - (-f_ba / rho).exp())) + _dot(
            b, w * ((-g_bb / rho).exp() - (-g_ab / rho).exp()))
    return _dot(a, w * (1 - (-f_ba / rho).exp())) + _dot(b, w * (1 - (-g_ab / rho).exp()))


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


def _bsum(w, f, B):
    return (w * f).view(B, -1).sum(1)


def sinkhorn_cost_batched(eps, rho, a, b, f_aa, g_bb, g_ab, f_ba, B, debias=True, potentials=False):
    """sinkhorn_cost on B problems stacked along the point axis: one value per batch element (scal(batch=True),
    utils.py:13-18)."""
    if potentials:
        return (f_ba - f_aa, g_ab - g_bb) if debias else (f_ba, g_ab)
    if rho is None:
        if debias:
            return _bsum(a, f_ba - f_aa, B) + _bsum(b, g_ab - g_bb, B)
        return _bsum(a, f_ba, B) + _bsum(b, g_ab, B)
    w = rho + eps / 2
    if debias:
        return _bsum(a, w * ((-f_aa / rho).exp() - (-f_ba / rho).exp()), B) + _bsum(
            b, w * ((-g_bb / rho).exp() - (-g_ab / rho).exp()), B)
    return _bsum(a, w * (1 - (-f_ba / rho).exp()), B) + _bsum(b, w * (1 - (-g_ab / rho).exp()), B)


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
    xf, yf, af, bf = x.reshape(B * N, D), y.reshape(B * M, D), a.reshape(B * N), b.reshape(B * M)
    center = ops.default_center(xf.detach(), yf.detach())
    dev = x.device
    pk = (p | ops.P_UNCLAMPED) if keops else p
    loop = dict(p=pk, debias=debias, center=center)
    batched_ops = ops.softmin_operators(D, p, batched=True)
    if batched_ops is not None:
        raw, grad = batched_ops

        # the loop runs on the flattened clouds and potentials; the operators see the (B, n, D) views
        def sm(eps, rows, cols, h_a, h_b=None, h_scale_b=0.0, **kw):
            out, lse2 = raw(eps, rows.view(B, -1, D), cols.view(B, -1, D), h_a, h_b, h_scale_b, **kw)
            return out.view(-1), None if lse2 is None else lse2.view(-1)

        def smg(eps, rows, cols, h_a, h_b=None, h_scale_b=0.0, **kw):
            return grad(eps, rows.view(B, -1, D), cols.view(B, -1, D), h_a, h_b, h_scale_b, **kw).view(-1)

        loop.update(softmin_raw=sm, softmin_grad=smg)
    else:
        problems = {"xy": ranges.batch_problem(B, N, M, dev), "yx": ranges.batch_problem(B, M, N, dev)}
        if debias:
            problems["xx"] = ranges.batch_problem(B, N, N, dev)
            problems["yy"] = ranges.batch_problem(B, M, M, dev)
        loop.update(problems=problems)
    f_aa, g_bb, g_ab, f_ba = sinkhorn_loop_points(log_weights(af.detach()), log_weights(bf.detach()), xf, yf,
                                                  eps_list, rho, **loop)
    out = sinkhorn_cost_batched(eps, rho, af, bf, f_aa, g_bb, g_ab, f_ba, B, debias=debias, potentials=potentials)
    if potentials:
        return out[0].view(B, N), out[1].view(B, M)
    return out


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
    with torch.no_grad():
        eps = eps_list[0]
        lam = damping(eps, rho)
        pots = [out for out, _ in ops.dense_softmin_rows_raw(eps, [(C, lw, None, None) for C, lw in zip(Cd, logs)],
                                                              beta=lam)]
        for eps in eps_list:
            lam = damping(eps, rho)
            # (f_ba, g_ab, f_aa, g_bb): C_xy reads g_ab, C_yx reads f_ba, each debias matrix its own potential
            reads = [pots[1], pots[0]] + pots[2:]
            pots = [out for out, _ in ops.dense_softmin_rows_raw(
                eps, [(C, lw, h, old) for C, lw, h, old in zip(Cd, logs, reads, pots)], alpha_old=0.5, beta=0.5 * lam)]
    # final extrapolation: eps / lam are the last values of the schedule (reference: leaked loop variables)
    reads = [pots[1], pots[0]] + pots[2:]
    if torch.is_grad_enabled() and any(C.requires_grad for C in mats):
        new = _LastRows.apply(eps, lam, *mats, *logs, *reads)
    else:
        new = [out for out, _ in ops.dense_softmin_rows_raw(eps, [(C, lw, h, None) for C, lw, h in zip(Cd, logs, reads)],
                                                             beta=lam)]
    f_ba, g_ab = new[0].reshape(-1), new[1].reshape(-1)
    f_aa, g_bb = (new[2].reshape(-1), new[3].reshape(-1)) if debias else (None, None)
    out = sinkhorn_cost_batched(eps, rho, a.reshape(-1), b.reshape(-1), f_aa, g_bb, g_ab, f_ba, B, debias=debias,
                                potentials=potentials)
    if potentials:
        return out[0].view(B, N), out[1].view(B, M)
    return out if batched else out[0]

"""``geomloss.ot.solve_sample``, ``solve``, ``solve_batch`` and ``solve_grid`` over the CUDA kernels (SURVEY.md
section 8, row f-3; ``solve_grid`` and its result object are at the end of this file).

The reference's "new API" for point clouds (src/geomloss/ot/_implementations/sample.py:190-395) builds dense (N, M)
cost matrices and runs ``sinkhorn_loop`` (ot/_abstract_solvers/sinkhorn_ot.py:240-447) on them.  Here the same
iteration runs on the fused on-the-fly softmin of ``ops.softmin_raw`` (``ops.softmin_wide_raw`` for 64 < D <= 1024;
never an N x M matrix), so the facade works at N = M = 1e6 like the rest of the engine.  Conventions of THIS API (they
differ from ``SamplesLoss``):

* cost ``"sqeuclidean"`` is ``C(x, y) = |x - y|^2`` — no 1/2 (sample.py:38-66); ``reg`` is the temperature eps and
  ``unbalanced`` the marginal penalty rho, used as given; ``blur`` / ``reach`` are shortcuts for ``2 blur^2`` /
  ``2 reach^2`` (sample.py:283-297);
* the eps ladder is ``geomspace(diameter^2, reg, max_iter)`` (annealing.py:131-170), one symmetric averaged update
  per value and one final non-averaged update (sinkhorn_ot.py:262-288, :419-436);
* the first iterate is the eps = +inf softmin (cost averages), minus the per-point ``0.5 a_i f_i`` — the
  reference's ``bk.dot_products`` treats the N axis of un-batched vectors as a batch axis (sinkhorn_ot.py:17-29,
  _backends/torch.py:28-32); kept, the goldens pin it.

Mapping onto the kernel (which evaluates ``-e log sum_j exp(h_j - (|x-y|^2/2)/e)``): with ``e = reg/2``,
``-reg log sum_j b_j exp((g_j - |x-y|^2)/reg) = 2 * softmin_kernel(e; h = log b + g/reg)``.

Autograd: like the reference, ``result.value`` is differentiable w.r.t. ``X_a``, ``X_b`` (through the cost in the
LAST update only — log-weights and incoming potentials are detached, sinkhorn_ot.py:419-436) and w.r.t. ``a``, ``b``
(their direct appearance in the value formula).  Unlike ``SamplesLoss`` the last update is differentiated w.r.t.
BOTH clouds of every softmin: the column gradient  sum_i u_i p_ij 2 (y_j - x_i)  is the row-gradient kernel run on
the swapped problem with column "log-weights" log u_i + softmin_i/eps (see ``_LastUpdate``).  The other attributes
(potentials, marginals, plan) are returned detached.  Inputs: float32 CUDA tensors; no CPU path.
Parity: pinned — ``tests/golden/ot_sample_case*.npz`` hold fp32 and fp64 runs of the real reference.
"""
from __future__ import annotations

import math
from functools import cached_property

import numpy as np
import torch

from . import ops
from .sinkhorn import log_weights, max_diameter

__all__ = ["solve", "solve_batch", "solve_grid", "solve_sample", "solve_sample_batch", "OTResultGrid",
           "OTResultMatrix", "OTResultSample", "LinearOperator"]

_DENSE_LIMIT = 1 << 27  # entries of a dense (N, M) plan we are willing to materialise on request


# ----------------------------------------------------------------------------------------------------
# argument checks                                            src/geomloss/_arguments.py:14-154
# ----------------------------------------------------------------------------------------------------
def _check_regularization(reg, unbalanced, unbalanced_type, method, tol, max_iter):
    if reg is None:
        raise TypeError("'<' not supported between instances of 'NoneType' and 'int'")  # the reference's own failure
    if reg < 0:
        raise ValueError(f"Parameter 'reg' should be >= 0. Received {reg}.")
    if reg == 0:
        raise NotImplementedError("Currently, we require that reg > 0.")
    if unbalanced is not None and unbalanced <= 0:
        raise ValueError(f"Parameter 'unbalanced' should be None (= +infty) or > 0. Received {unbalanced}.")
    if unbalanced_type != "KL":
        raise NotImplementedError("Currently, we only support unbalanced OT with a 'KL' penalty on the marginal "
                                  "constraints.")
    if method != "auto":
        raise NotImplementedError("Currently, we only support a single method.")
    if max_iter is None:
        raise ValueError("The 'max_iter' parameter should be a positive integer.")
    if tol is not None:
        raise NotImplementedError("Currently, we do not support rigorous stopping criteria.")


def _check_marginal(m, like, size, name):
    if m is None:
        return torch.full_like(like, 1.0 / size)
    if m.shape != like.shape:
        raise ValueError(f"The marginal '{name}' should be of shape {like.shape}. Instead, received an array of "
                         f"shape {m.shape}.")
    if bool((m < 0).any()):
        raise ValueError(f"The marginal '{name}' contains negative values. We require that {name} >= 0.")
    return m


def _check_masses(sums_a, sums_b):
    """Balanced problems: the (B,) total masses of a and b agree to 1e-3 relative (_arguments.py:126-156)."""
    sa, sb = sums_a.double(), sums_b.double()
    if bool(((sa - sb).abs() / (sa + sb) > 1e-3).any()):
        which = ("do not sum up to the same value." if sa.numel() == 1 else
                 "have rows that do not sum up to the same values.")
        raise ValueError(f"The two arrays of marginal weights 'a' and 'b' {which} As a consequence, the balanced OT "
                         "problem is not feasible. To fix this error, you may either normalize the two marginals or "
                         "use UNbalanced optimal transport with the 'unbalanced' keyword argument.")


def annealing_eps(maxmin_cost, eps, n_iter):
    """The eps ladder of ``annealing_parameters(maxmin_cost=, eps=, n_iter=)``, scaling=None (annealing.py:114-170)."""
    if n_iter <= 0:
        raise ValueError(f"The number of iterations should be >= 1. Received n_iter={n_iter}.")
    maxmin_cost = max(float(maxmin_cost), eps)
    if n_iter == 1:
        return [eps]
    return [float(e) for e in np.geomspace(maxmin_cost, eps, n_iter)]


# ----------------------------------------------------------------------------------------------------
# the solver
# ----------------------------------------------------------------------------------------------------
class _Softmin:
    """``softmin_sample`` (sample.py:91-182) for the four (rows, columns) pairs of one problem, on the kernel.

    It also holds the three operators every pass of the facade runs, as ``ops.ot_operators`` names them for D when
    the solver starts: the forward softmin (``fwd``), its row gradient (``grad_rows``) and the plan applied to a value
    matrix (``apply``)."""

    def __init__(self, X_a, X_b):
        self.D = X_a.shape[1]
        if self.D > ops.MAX_D_WIDE:
            raise NotImplementedError(f"solve_sample serves D <= {ops.MAX_D_WIDE}, got D = {self.D} (no kernel of this "
                                      f"build reduces clouds above D = {ops.MAX_D_WIDE})")
        self.center = ops.default_center(X_a, X_b)
        self.X_a, self.X_b = X_a, X_b
        self.fwd, self.grad_rows, self.apply = ops.ot_operators(self.D)

    def __call__(self, eps, x, y, log_w, pot, *, damp=1.0, old=None):
        """damp * softmin(eps, log_w, C(x, y), pot), or its average with ``old`` (the symmetric Sinkhorn update)."""
        if old is None:
            return self.fwd(0.5 * eps, x, y, log_w, pot, 1.0 / eps, p=2, center=self.center, beta=2.0 * damp)[0]
        return self.fwd(0.5 * eps, x, y, log_w, pot, 1.0 / eps, p=2, center=self.center, out_old=old, alpha_old=0.5,
                        beta=damp)[0]

    def at_infinity(self, x, y, w_rows, w_cols, damp):
        """eps = +inf: f_i = sum_j w_j |x_i - y_j|^2 / sum_j w_j by moments (fp64, centred), then the reference's
        offset and dampening (sinkhorn_ot.py:17-29)."""
        c = self.center.double()
        xc, yc, w = x.double() - c, y.double() - c, w_cols.double()
        W = w.sum()
        ybar = (w[:, None] * yc).sum(0) / W
        f = (xc * xc).sum(1) - 2.0 * (xc @ ybar) + (w * (yc * yc).sum(1)).sum() / W
        return (damp * (f - 0.5 * w_rows.double() * f)).float()


class _LastUpdate(torch.autograd.Function):
    """``damp * softmin(eps, log_w, C(rows, cols), pot)`` of the new API, differentiable w.r.t. rows AND cols.

    With p_ij the softmax weights of row i over the columns and u = damp * grad_output:
      d/d rows_i = u_i 2 (rows_i - sum_j p_ij cols_j)                    -> b200ot_softmin_bwd_x as is;
      d/d cols_j = sum_i u_i p_ij 2 (cols_j - rows_i) = 2 W_j (cols_j - sum_i q_ji rows_i),
         W_j = sum_i u_i p_ij = exp(log_w_j + pot_j/eps) sum_i exp(log u_i + softmin_i/eps - C_ij/eps),
      i.e. the SAME row-gradient kernel on the swapped problem (rows <- cols, column log-weights log u_i, column
      potential softmin_i), one extra softmin for its normaliser W; signed u is split into its two parts."""

    @staticmethod
    def forward(ctx, rows, cols, log_w, pot, eps, damp, sm):
        out, lse2 = sm.fwd(0.5 * eps, rows.detach(), cols.detach(), log_w, pot, 1.0 / eps, p=2, center=sm.center,
                           beta=2.0 * damp, want_lse2=True)
        ctx.save_for_backward(rows.detach(), cols.detach(), log_w, pot, out, lse2)
        ctx.meta = (float(eps), float(damp), sm)
        return out

    @staticmethod
    def backward(ctx, go):
        rows, cols, log_w, pot, out, lse2 = ctx.saved_tensors
        eps, damp, sm = ctx.meta
        center = sm.center
        e2, inv = 0.5 * eps, 1.0 / eps
        u_all = (damp * go).float().contiguous()
        g_rows = g_cols = None
        if ctx.needs_input_grad[0]:
            g_rows = sm.grad_rows(e2, rows, cols, log_w, pot, inv, lse2, 2.0 * u_all, p=2, center=center)
        if ctx.needs_input_grad[1]:
            sm_und = out / damp  # undamped softmin values, new-API scale
            g_cols = torch.zeros_like(cols)
            for sign in (1.0, -1.0):
                u = (sign * u_all).clamp_min(0.0)
                if not bool((u > 0).any()):
                    continue
                lu = log_weights(u)
                sm_t, lse2_t = sm.fwd(e2, cols, rows, lu, sm_und, inv, p=2, center=center, want_lse2=True)
                W = torch.exp((log_w.double() + pot.double() * inv - sm_t.double() / e2)).float()
                g_cols = g_cols + sign * sm.grad_rows(e2, cols, rows, lu, sm_und, inv, lse2_t, (2.0 * W).contiguous(),
                                                      p=2, center=center)
        return g_rows, g_cols, None, None, None, None, None


def solve_sample(X_a, X_b, a=None, b=None, cost="sqeuclidean", debias=False, reg=None, unbalanced=None,
                 unbalanced_type="KL", method="auto", max_iter=None, tol=None, blur=None, reach=None):
    """Entropic (un)balanced OT between two point clouds; mirrors ``geomloss.ot.solve_sample`` (sample.py:190-395).

    X_a: (N, D), X_b: (M, D) float32 CUDA tensors; a: (N,), b: (M,) non-negative weights (uniform 1/N, 1/M if None).
    Returns an :class:`OTResultSample`.
    """
    p = 2 if cost == "sqeuclidean" else 1
    if blur is not None:
        if reg is not None:
            raise ValueError("Parameters 'reg' and 'blur' are redundant. Please specify only one of them.")
        reg = p * (blur**p)
    if reach is not None:
        if unbalanced is not None:
            raise ValueError("Parameters 'unbalanced' and 'reach' are redundant. Please specify only one of them.")
        unbalanced = p * (reach**p)
    _check_regularization(reg, unbalanced, unbalanced_type, method, tol, max_iter)
    if not (torch.is_tensor(X_a) and torch.is_tensor(X_b)):
        raise TypeError("X_a and X_b must be torch CUDA tensors (this engine has no NumPy / CPU path)")
    if X_a.dim() != 2:
        raise ValueError(f"Expected X_a to be a (N, D) array. Received {tuple(X_a.shape)}.")
    if X_b.dim() != 2:
        raise ValueError(f"Expected X_b to be a (M, D) array. Received {tuple(X_b.shape)}.")
    N, D = X_a.shape
    M, D_ = X_b.shape
    if D != D_:
        raise ValueError("Expected X_a and X_b to have the same number of coordinates per sample. "
                         f"Received D={D} for X_a and D={D_} for X_b.")
    a = _check_marginal(a, X_a[:, 0], N, "a")
    b = _check_marginal(b, X_b[:, 0], M, "b")
    if unbalanced is None:
        _check_masses(a.detach().sum()[None], b.detach().sum()[None])
    if cost != "sqeuclidean":
        raise NotImplementedError()  # as the reference (sample.py:76-88)
    reg = float(reg)
    rho = None if unbalanced is None else float(unbalanced)

    live = (X_a, X_b, a, b)  # the caller's tensors: the value stays attached to them when they require grad
    want_grad = torch.is_grad_enabled() and any(t.requires_grad for t in live)
    with torch.no_grad():
        X_a, X_b, a, b = X_a.detach(), X_b.detach(), a.detach(), b.detach()
        eps_list = annealing_eps(max_diameter(X_a, X_b) ** p, reg, int(max_iter))
        sm = _Softmin(X_a, X_b)
        log_a, log_b = log_weights(a), log_weights(b)

        def damp(eps):
            return 1.0 if rho is None else 1.0 / (1.0 + eps / rho)

        lam = damp(eps_list[0])
        f_ba = sm.at_infinity(X_a, X_b, a, b, lam)
        g_ab = sm.at_infinity(X_b, X_a, b, a, lam)
        if debias:
            f_aa = sm.at_infinity(X_a, X_a, a, a, lam)
            g_bb = sm.at_infinity(X_b, X_b, b, b, lam)
        for eps in eps_list:
            lam = damp(eps)
            ft_ba = sm(eps, X_a, X_b, log_b, g_ab, damp=lam, old=f_ba)
            gt_ab = sm(eps, X_b, X_a, log_a, f_ba, damp=lam, old=g_ab)
            if debias:
                f_aa = sm(eps, X_a, X_a, log_a, f_aa, damp=lam, old=f_aa)
                g_bb = sm(eps, X_b, X_b, log_b, g_bb, damp=lam, old=g_bb)
            f_ba, g_ab = ft_ba, gt_ab
        if not want_grad:
            # last, non-averaged update (last_extrapolation=True, sinkhorn_ot.py:419-436)
            new_f = sm(eps, X_a, X_b, log_b, g_ab, damp=lam)
            new_g = sm(eps, X_b, X_a, log_a, f_ba, damp=lam)
            f_ba, g_ab = new_f, new_g
            if debias:
                f_aa = sm(eps, X_a, X_a, log_a, f_aa, damp=lam)
                g_bb = sm(eps, X_b, X_b, log_b, g_bb, damp=lam)
    if want_grad:
        # the same update, attached to the caller's clouds through the cost (both arguments of every softmin)
        xa, xb = live[0], live[1]
        last = lambda rows, cols, lw, pot: _LastUpdate.apply(rows, cols, lw, pot, eps, lam, sm)  # noqa: E731
        new_f, new_g = last(xa, xb, log_b, g_ab), last(xb, xa, log_a, f_ba)
        f_ba, g_ab = new_f, new_g
        if debias:
            f_aa, g_bb = last(xa, xa, log_a, f_aa), last(xb, xb, log_b, g_bb)
        a, b = live[2], live[3]
    if not debias:
        f_aa = g_bb = None
    return OTResultSample(X_a=X_a, X_b=X_b, a=a, b=b, reg=reg, unbalanced=rho, debias=bool(debias),
                          potentials=(f_aa, g_bb, g_ab, f_ba), softmin=sm)


def solve_sample_batch(*args, **kwargs):
    raise NotImplementedError("This function is not implemented yet.")  # as the reference (sample.py:405-431)


# ----------------------------------------------------------------------------------------------------
# results                                       ot/_ot_result.py:164-440, sample.py:444-641
# ----------------------------------------------------------------------------------------------------
def _ot_value(a, b, f_ba, g_ab, eps, rho, f_aa=None, g_bb=None):
    """The transport cost of dual potentials (unbalanced_ot.py:25-185), debiased when f_aa, g_bb are given, summed over
    the last axis: a scalar for (N,) / (M,) vectors, (B,) for (B, N) / (B, M) ones.  fp64 inside, float32 out."""
    a, b, f_ba, g_ab = a.double(), b.double(), f_ba.double(), g_ab.double()
    debias = f_aa is not None
    if debias:
        f_aa, g_bb = f_aa.double(), g_bb.double()
    if rho is None:
        F, G = (f_ba - f_aa, g_ab - g_bb) if debias else (f_ba, g_ab)
    elif not debias:
        F = (rho + eps / 2 * b.sum(-1, keepdim=True)) - (rho + eps / 2) * torch.exp(-f_ba / rho)
        G = (rho + eps / 2 * a.sum(-1, keepdim=True)) - (rho + eps / 2) * torch.exp(-g_ab / rho)
    else:
        F = (rho + eps / 2) * (torch.exp(-f_aa / rho) - torch.exp(-f_ba / rho))
        G = (rho + eps / 2) * (torch.exp(-g_bb / rho) - torch.exp(-g_ab / rho))
    return ((a * F).sum(-1) + (b * G).sum(-1)).float()


def _fused_operator(s):
    """Whether ``operator @ s`` runs on the fused kernel (``ops.plan_apply_raw``): every CUDA tensor.  The engine has no
    CPU path; a host tensor is evaluated through ``ops.softmin_raw`` alone, where the real operator refuses it, so that
    a stand-in for that one operator drives the whole facade on the CPU (tests/test_host_logic.py)."""
    return s.is_cuda


class LinearOperator:
    """``x -> A @ x`` without the matrix (ot/_ot_result.py:9-160): ``op @ x``, ``op.T``, ``op.shape``."""

    def __init__(self, *, matmat, rmatmat, input_shape, output_shape):
        self._matmat, self._rmatmat = matmat, rmatmat
        self._input_shape, self._output_shape = tuple(input_shape), tuple(output_shape)

    def __matmul__(self, x):
        k = len(self._input_shape)
        if x.dim() < k or tuple(x.shape[:k]) != self._input_shape:
            raise ValueError(f"Expects an input of shape {self._input_shape} with, maybe, additional trailing "
                             f"dimensions, but found an array of shape {tuple(x.shape)}.")
        trailing = tuple(x.shape[k:])
        out = self._matmat(x.reshape(self._input_shape + (-1,)))
        return out.reshape(self._output_shape + trailing)

    @property
    def shape(self):
        return (math.prod(self._output_shape), math.prod(self._input_shape))

    def transpose(self):
        return LinearOperator(matmat=self._rmatmat, rmatmat=self._matmat, input_shape=self._output_shape,
                              output_shape=self._input_shape)

    @property
    def T(self):
        return self.transpose()

    def rescale(self, *, input_scaling, output_scaling):
        def matmat(s):
            return output_scaling[:, None] * (self._matmat(input_scaling[:, None] * s))

        def rmatmat(s):
            return input_scaling[:, None] * (self._rmatmat(output_scaling[:, None] * s))

        return LinearOperator(matmat=matmat, rmatmat=rmatmat, input_shape=self._input_shape,
                              output_shape=self._output_shape)


class OTResultSample:
    """Result of :func:`solve_sample`; lazily evaluated, cached attributes named like the reference's
    (``value``, ``potential_a/b/aa/bb``, ``marginal_a/b``, ``plan``, ``density``, ``plan_operator``,
    ``density_operator``; ``lazy_plan``, ``lazy_density`` are ``None`` as in the reference without KeOps).  ``a_to_b``
    / ``b_to_a``, documented and unimplemented in the reference (ot/_ot_result.py:408-418), are the barycentric
    displacement fields of the plan."""

    def __init__(self, *, X_a, X_b, a, b, reg, unbalanced, debias, potentials, softmin):
        self._X_a, self._X_b, self._a, self._b = X_a, X_b, a.detach(), b.detach()
        self._reg, self._unbalanced, self._debias = reg, unbalanced, debias
        self._live = (a, b) + tuple(potentials)  # possibly attached to the caller's graph: used by `value` only
        self._f_aa, self._g_bb, self._g_ab, self._f_ba = (None if t is None else t.detach() for t in potentials)
        self._sm = softmin

    # ---- dual potentials --------------------------------------------------------------------------
    @property
    def potential_a(self):
        return self._f_ba

    @property
    def potential_b(self):
        return self._g_ab

    @property
    def potential_aa(self):
        if self._f_aa is None:
            raise ValueError("The self-interaction potential `f_aa` is not defined. To fix this issue, run your OT "
                             "solver with `debias = True`.")
        return self._f_aa

    @property
    def potential_bb(self):
        if self._g_bb is None:
            raise ValueError("The self-interaction potential `g_bb` is not defined. To fix this issue, run your OT "
                             "solver with `debias = True`.")
        return self._g_bb

    # ---- value                                                   unbalanced_ot.py:25-185 ----------
    @cached_property
    def value(self):
        a, b, f_aa, g_bb, g_ab, f_ba = self._live
        return _ot_value(a, b, f_ba, g_ab, self._reg, self._unbalanced, f_aa, g_bb)

    # ---- the plan as an operator ---------------------------------------------------------------------
    # With w_ij = softmax_j(h_j - C_ij / reg), h = log_w + g / reg, and sm the softmin of the same h:
    #   sum_j w_j exp((f_i + g_j - C_ij) / reg) s_jk = exp((f_i - sm_i) / reg) * sum_j w_ij s_jk      (w = exp(log_w))
    # so (density @ s) takes log_w = 0 and (plan @ s) takes w = b and the row factor a_i exp((f_i - sm_i) / reg), which
    # is the plan's marginal.  One forward softmin per (direction, weighting) gives lse2 and the row factor; after
    # that every application is ONE call of ops.plan_apply_raw (plan_apply_wide_raw above D = 64), for any number of
    # columns and any signs.
    def _apply_state(self, transpose, weighted):
        """(log_w, lse2, row_factor) of the operator's direction, cached until ``cache_clear``."""
        cache = self.__dict__.setdefault("_apply_cache", {})
        key = (bool(transpose), bool(weighted))
        if key not in cache:
            eps = self._reg
            rows, cols = (self._X_b, self._X_a) if transpose else (self._X_a, self._X_b)
            f, g = (self._g_ab, self._f_ba) if transpose else (self._f_ba, self._g_ab)
            w_rows, w_cols = (self._b, self._a) if transpose else (self._a, self._b)
            with torch.no_grad():
                log_w = log_weights(w_cols) if weighted else torch.zeros_like(w_cols)
                smv, lse2 = self._sm.fwd(0.5 * eps, rows, cols, log_w, g, 1.0 / eps, p=2, center=self._sm.center,
                                         beta=2.0, want_lse2=True)
                factor = torch.exp((f - smv) / eps)
                if weighted:
                    factor = w_rows * factor
            cache[key] = (log_w, lse2, factor.contiguous())
        return cache[key]

    def _apply(self, s, transpose, weighted, *, normalized=False):
        """plan @ s (weighted) or density @ s for s of shape (M, K) [``.T @ s`` with ``transpose``, s (N, K)];
        ``normalized``: rows of weights summing to one (no row factor).  Detached."""
        rows, cols = (self._X_b, self._X_a) if transpose else (self._X_a, self._X_b)
        g = self._f_ba if transpose else self._g_ab
        log_w, lse2, factor = self._apply_state(transpose, weighted)
        with torch.no_grad():
            return self._sm.apply(0.5 * self._reg, rows, cols, log_w, g, 1.0 / self._reg, lse2, s.detach().float(),
                                  row_factor=None if normalized else factor, center=self._sm.center)

    def _density_matmat(self, s, transpose, weighted=False):
        """(density @ s), or (plan @ s) when ``weighted``; differentiable w.r.t. s when it requires a gradient."""
        if not _fused_operator(s):
            return self._matmat_by_softmins(s, transpose, weighted)
        if torch.is_grad_enabled() and s.requires_grad:
            return _PlanApply.apply(self, s, transpose, weighted)
        return self._apply(s, transpose, weighted)

    def _matmat_by_softmins(self, s, transpose, weighted):
        """The same product through ``ops.softmin_raw`` alone, P s = exp((f - softmin(eps, log s, C, g)) / eps) for
        s >= 0: one softmin per column and sign.  Host tensors only (see ``_fused_operator``)."""
        eps = self._reg
        rows, cols = (self._X_b, self._X_a) if transpose else (self._X_a, self._X_b)
        f, g = (self._g_ab, self._f_ba) if transpose else (self._f_ba, self._g_ab)
        w_rows, w_cols = (self._b, self._a) if transpose else (self._a, self._b)
        out = []
        with torch.no_grad():
            for v in range(s.shape[1]):
                col = s[:, v].float() * w_cols if weighted else s[:, v].float()
                acc = torch.zeros(rows.shape[0], dtype=torch.float32, device=rows.device)
                for sign in (1.0, -1.0):
                    part = (sign * col).clamp_min(0.0)
                    if bool((part > 0).any()):
                        acc = acc + sign * torch.exp((f - self._sm(eps, rows, cols, log_weights(part), g)) / eps)
                out.append(w_rows * acc if weighted else acc)
        return torch.stack(out, 1)

    def _operator(self, weighted):
        N, M = self._X_a.shape[0], self._X_b.shape[0]
        return LinearOperator(matmat=lambda s: self._density_matmat(s, False, weighted),
                              rmatmat=lambda s: self._density_matmat(s, True, weighted), input_shape=(M,),
                              output_shape=(N,))

    @cached_property
    def density_operator(self):
        return self._operator(False)

    @cached_property
    def plan_operator(self):
        return self._operator(True)

    # (the plan's marginals are the row factors of the two directions: a_i sum_j b_j density_ij)
    @cached_property
    def marginal_a(self):
        return self._apply_state(False, True)[2]

    @cached_property
    def marginal_b(self):
        return self._apply_state(True, True)[2]

    # ---- barycentric maps: displacement of each point to the conditional mean of its row of the plan ------
    def _barycentric(self, transpose):
        src, dst = (self._X_b, self._X_a) if transpose else (self._X_a, self._X_b)
        c = self._sm.center
        return self._apply(dst - c, transpose, True, normalized=True) + c - src

    @cached_property
    def a_to_b(self):
        """(N, D): sum_j P_ij X_b[j] / sum_j P_ij - X_a[i] (also defined for unbalanced problems); detached."""
        return self._barycentric(False)

    @cached_property
    def b_to_a(self):
        """(M, D): the same on the transposed plan; detached."""
        return self._barycentric(True)

    # ---- dense accessors (small problems only) --------------------------------------------------------
    @cached_property
    def density(self):
        N, M = self._X_a.shape[0], self._X_b.shape[0]
        if N * M > _DENSE_LIMIT:
            raise MemoryError(f"a dense ({N}, {M}) density does not fit the budget of this accessor; use "
                              "density_operator / plan_operator, which never build the matrix")
        C = torch.cdist(self._X_a, self._X_b, compute_mode="donot_use_mm_for_euclid_dist") ** 2
        return torch.exp((self._f_ba[:, None] + self._g_ab[None, :] - C) / self._reg)

    @cached_property
    def plan(self):
        return self.density * self._a[:, None] * self._b[None, :]

    lazy_density = None
    lazy_plan = None

    def cache_clear(self):
        for k in ("value", "density_operator", "plan_operator", "marginal_a", "marginal_b", "density", "plan",
                  "a_to_b", "b_to_a", "_apply_cache"):
            self.__dict__.pop(k, None)


class _PlanApply(torch.autograd.Function):
    """``plan @ s`` / ``density @ s`` (or their transposes) as a function of s alone: the operator is linear in s,
    so the gradient is the transposed operator applied to the upstream gradient.  Clouds and potentials are constants,
    as for every other accessor of the result."""

    @staticmethod
    def forward(ctx, res, s, transpose, weighted):
        ctx.res, ctx.meta = res, (transpose, weighted)
        return res._apply(s, transpose, weighted)

    @staticmethod
    def backward(ctx, go):
        transpose, weighted = ctx.meta
        return None, ctx.res._apply(go, not transpose, weighted), None, None


# ----------------------------------------------------------------------------------------------------
# explicit cost matrices                               ot/_implementations/matrix.py:97-660
# ----------------------------------------------------------------------------------------------------
class _fp32_matmul:
    """Full-precision fp32 matmuls (no TF32) inside the block, the caller's setting restored after it."""

    def __enter__(self):
        self.prev = torch.get_float32_matmul_precision()
        torch.set_float32_matmul_precision("highest")

    def __exit__(self, *exc):
        torch.set_float32_matmul_precision(self.prev)


def _dense_at_infinity(C, a, b, damp):
    """eps = +inf: f_i = sum_j b_j C_ij / sum_j b_j and g_j = sum_i a_i C_ij / sum_i a_i as two matvecs on C (no
    transpose, no C-sized temporary), minus the per-problem offsets 0.5 <a, f>, 0.5 <b, g>, then damped
    (sinkhorn_ot.py:17-29, matrix.py:72-81)."""
    with _fp32_matmul():
        f = (C @ b.unsqueeze(-1)).squeeze(-1) / b.sum(-1, keepdim=True)
        g = (a.unsqueeze(-2) @ C).squeeze(-2) / a.sum(-1, keepdim=True)
    f = damp * (f - 0.5 * (a * f).sum(-1, keepdim=True))
    g = damp * (g - 0.5 * (b * g).sum(-1, keepdim=True))
    return f.contiguous(), g.contiguous()


class _LastPair(torch.autograd.Function):
    """The last, non-averaged update ``(f, g) = damp * (softmin rows, softmin columns)`` of C, differentiable w.r.t. C
    through both softmins; log-weights and incoming potentials are constants (sinkhorn_ot.py:419-436).  ``C`` carries
    the caller's graph, ``Cd`` is its detached contiguous copy the kernels read."""

    @staticmethod
    def forward(ctx, C, Cd, log_a, log_b, f, g, eps, damp):
        f_new, g_new, lse2_row, lse2_col = ops.dense_softmin_pair_raw(eps, Cd, log_a, log_b, f, g, beta=damp,
                                                                      want_lse2=True)
        ctx.save_for_backward(Cd, log_a, log_b, f, g, lse2_row, lse2_col)
        ctx.meta = (float(eps), float(damp))
        return f_new, g_new

    @staticmethod
    def backward(ctx, go_f, go_g):
        Cd, log_a, log_b, f, g, lse2_row, lse2_col = ctx.saved_tensors
        eps, damp = ctx.meta
        grad_C = ops.dense_softmin_pair_grad(eps, Cd, log_a, log_b, f, g, lse2_row, lse2_col,
                                             (damp * go_f).contiguous(), (damp * go_g).contiguous())
        return grad_C, None, None, None, None, None, None, None


def solve(C, *, reg, a=None, b=None, unbalanced=None, unbalanced_type="KL", method="auto", max_iter=None, tol=None):
    """Entropic (un)balanced OT on an explicit (N, M) cost matrix; mirrors ``geomloss.ot.solve`` (matrix.py:348-512).

    C: (N, M), a: (N,), b: (M,) float32 CUDA tensors (a, b non-negative, uniform 1/N, 1/M if None); ``reg`` is the
    temperature eps, ``unbalanced`` the marginal penalty rho (None: balanced).  Use this for any cost that is not
    ``|x - y|^p`` on point clouds: build C, then solve.  A non-contiguous C is copied once.  Returns an
    :class:`OTResultMatrix` without batch axis."""
    if not torch.is_tensor(C):
        raise TypeError("C must be a torch CUDA tensor (this engine has no NumPy / CPU path)")
    if C.dim() != 2:
        raise ValueError("The 'cost' matrix should be an array with 2 dimensions. "
                         f"Instead, ot.solve received an array of shape {C.shape}.")
    N, M = C.shape
    a = _check_marginal(a, C[:, 0], N, "a")
    b = _check_marginal(b, C[0, :], M, "b")
    res = solve_batch(C[None], reg=reg, a=a[None], b=b[None], unbalanced=unbalanced, unbalanced_type=unbalanced_type,
                      method=method, max_iter=max_iter, tol=tol)
    res._batched = False
    return res


def solve_batch(C, *, reg, a=None, b=None, unbalanced=None, unbalanced_type="KL", method="auto", max_iter=None,
                tol=None):
    """B independent problems of :func:`solve` in one solver, C: (B, N, M), a: (B, N), b: (B, M); mirrors
    ``geomloss.ot.solve_batch`` (matrix.py:515-660).  The eps ladder starts from max(C) - min(C) over the whole batch.

    Each iteration is ONE pass over C for both potentials (``ops.dense_softmin_pair_raw``): no transposed copy and
    no (B, N, M) temporary.  ``result.value`` is differentiable w.r.t. C through the last update (both softmins) and
    w.r.t. a and b through the value formula."""
    _check_regularization(reg, unbalanced, unbalanced_type, method, tol, max_iter)
    if not torch.is_tensor(C):
        raise TypeError("C must be a torch CUDA tensor (this engine has no NumPy / CPU path)")
    if C.dim() != 3:
        raise ValueError("The 'cost' matrix should be an array with 3 dimensions (batch, N, M). "
                         f"Instead, ot.solve received an array of shape {C.shape}.")
    B, N, M = C.shape
    a = _check_marginal(a, C[:, :, 0], N, "a")
    b = _check_marginal(b, C[:, 0, :], M, "b")
    if unbalanced is None:
        _check_masses(a.detach().sum(-1), b.detach().sum(-1))
    for t, name in ((C, "C"), (a, "a"), (b, "b")):
        if not (t.is_cuda and t.dtype == torch.float32):
            raise TypeError(f"{name} must be a float32 CUDA tensor (this engine computes in fp32 on the GPU), got "
                            f"{t.dtype} on {t.device}")
    reg = float(reg)
    rho = None if unbalanced is None else float(unbalanced)

    def damp(eps):
        return 1.0 if rho is None else 1.0 / (1.0 + eps / rho)

    want_grad = torch.is_grad_enabled() and any(t.requires_grad for t in (C, a, b))
    with torch.no_grad():
        Cd = C.detach().contiguous()
        a_d, b_d = a.detach().contiguous(), b.detach().contiguous()
        eps_list = annealing_eps(float(Cd.amax() - Cd.amin()), reg, int(max_iter))
        log_a, log_b = log_weights(a_d), log_weights(b_d)
        lam = damp(eps_list[0])
        f, g = _dense_at_infinity(Cd, a_d, b_d, lam)
        for eps in eps_list:
            lam = damp(eps)
            f, g, _, _ = ops.dense_softmin_pair_raw(eps, Cd, log_a, log_b, f, g, alpha_old=0.5, beta=0.5 * lam)
        if not want_grad:  # last, non-averaged update (last_extrapolation=True, sinkhorn_ot.py:419-436)
            f, g, _, _ = ops.dense_softmin_pair_raw(eps, Cd, log_a, log_b, f, g, beta=lam)
    if want_grad:
        f, g = _LastPair.apply(C, Cd, log_a, log_b, f, g, eps, lam)
    return OTResultMatrix(C=Cd, a=a, b=b, reg=reg, unbalanced=rho, potentials=(f, g))


class OTResultMatrix:
    """Result of :func:`solve` / :func:`solve_batch`; lazily evaluated, cached attributes named like the reference's
    (matrix.py:97-345): ``value``, ``potential_a``, ``potential_b``, ``marginal_a``, ``marginal_b``, ``density``,
    ``plan``, ``density_operator``, ``plan_operator``; ``lazy_plan``, ``lazy_density`` are ``None``.  Shapes follow
    the solver: (N,) / (M,) / (N, M) for :func:`solve`, with a leading batch axis B for :func:`solve_batch`.

    Only ``value`` is attached to the caller's graph; every other attribute is returned detached.  ``density`` and
    ``plan`` are dense (N, M) tensors, as in the reference, built once and cached; the operators apply them."""

    def __init__(self, *, C, a, b, reg, unbalanced, potentials):
        self._C, self._a, self._b = C, a.detach(), b.detach()
        self._reg, self._unbalanced = reg, unbalanced
        self._live = (a, b) + tuple(potentials)  # possibly attached to the caller's graph: used by `value` only
        self._f, self._g = (t.detach() for t in potentials)
        self._batched = True

    def _out(self, t):
        return t if self._batched else t[0]

    @property
    def potential_a(self):
        return self._out(self._f)

    @property
    def potential_b(self):
        return self._out(self._g)

    @cached_property
    def value(self):
        a, b, f, g = self._live
        return self._out(_ot_value(a, b, f, g, self._reg, self._unbalanced))

    # (the plan's marginals: a_i sum_j b_j density_ij = a_i exp((f_i - softmin_i) / eps), and the same on columns,
    # from one pass over C)
    @cached_property
    def _marginals(self):
        eps = self._reg
        with torch.no_grad():
            sm_f, sm_g, _, _ = ops.dense_softmin_pair_raw(eps, self._C, log_weights(self._a), log_weights(self._b),
                                                          self._f, self._g)
            return self._a * torch.exp((self._f - sm_f) / eps), self._b * torch.exp((self._g - sm_g) / eps)

    @cached_property
    def marginal_a(self):
        return self._out(self._marginals[0])

    @cached_property
    def marginal_b(self):
        return self._out(self._marginals[1])

    @cached_property
    def density(self):
        with torch.no_grad():
            return self._out(torch.exp((self._f[:, :, None] + self._g[:, None, :] - self._C) / self._reg))

    @cached_property
    def plan(self):
        a, b = self._out(self._a), self._out(self._b)
        return self.density * a[..., :, None] * b[..., None, :]

    def _operator(self, P):
        def matmat(s):  # (M, K) -> (N, K), or (B, M, K) -> (B, N, K)
            with _fp32_matmul():
                return P @ s.to(P.dtype)

        def rmatmat(s):
            with _fp32_matmul():
                return P.transpose(-1, -2) @ s.to(P.dtype)

        B, N, M = self._C.shape
        lead = (B,) if self._batched else ()
        return LinearOperator(matmat=matmat, rmatmat=rmatmat, input_shape=lead + (M,), output_shape=lead + (N,))

    @cached_property
    def density_operator(self):
        return self._operator(self.density)

    @cached_property
    def plan_operator(self):
        return self._operator(self.plan)

    lazy_density = None
    lazy_plan = None

    def cache_clear(self):
        for k in ("value", "_marginals", "marginal_a", "marginal_b", "density", "plan", "density_operator",
                  "plan_operator"):
            self.__dict__.pop(k, None)


# ----------------------------------------------------------------------------------------------------
# regular grids (images, volumes)                       ot/_implementations/grid.py:215-242 (a stub there)
# ----------------------------------------------------------------------------------------------------
class _Grid:
    """The pixel grid shared by ``a`` and ``b``: side N_d, extent [lo_d, hi_d), pitch h_d = (hi_d - lo_d) / N_d and
    pixel centres lo_d + (k + 1/2) h_d on every axis d; offsets on a periodic axis go the shorter way round."""

    def __init__(self, sides, axes, periodic):
        self.sides, self.D = tuple(int(n) for n in sides), len(sides)
        D = self.D
        if axes is None:
            pairs = [(0.0, 1.0)] * D
        elif torch.is_tensor(axes) or isinstance(axes, np.ndarray) or (
                isinstance(axes, (tuple, list)) and any(torch.is_tensor(t) or isinstance(t, np.ndarray) for t in axes)):
            raise NotImplementedError("solve_grid serves uniform grids given by (lo, hi) extents; explicit pixel "
                                      "coordinates (non-uniform spacing) are not supported.")
        elif isinstance(axes, (tuple, list)) and len(axes) == 2 and all(_is_real(t) for t in axes):
            pairs = [tuple(axes)] * D
        elif (isinstance(axes, (tuple, list)) and len(axes) == D
              and all(isinstance(t, (tuple, list)) and len(t) == 2 and all(_is_real(u) for u in t) for t in axes)):
            pairs = [tuple(t) for t in axes]
        else:
            raise ValueError(f"'axes' should be None, one (lo, hi) pair for every axis or a tuple of {D} (lo, hi) "
                             f"pairs, one per axis. Received {axes!r}.")
        for lo, hi in pairs:
            if not (math.isfinite(lo) and math.isfinite(hi) and hi > lo):
                raise ValueError(f"Every axis extent (lo, hi) should satisfy lo < hi. Received {(lo, hi)}.")
        if isinstance(periodic, (bool, np.bool_)):
            periodic = (bool(periodic),) * D
        elif not (isinstance(periodic, (tuple, list)) and len(periodic) == D
                  and all(isinstance(t, (bool, np.bool_)) for t in periodic)):
            raise ValueError(f"'periodic' should be a bool or a tuple of {D} bools, one per axis. Received "
                             f"{periodic!r}.")
        self.lo = tuple(float(lo) for lo, _ in pairs)
        self.pitch = tuple((float(hi) - float(lo)) / n for (lo, hi), n in zip(pairs, self.sides))
        self.periodic = tuple(bool(t) for t in periodic)

    @property
    def diameter(self):
        """Diagonal of the box of pixel centres; half the side on a periodic axis, its largest offset."""
        ext = [(n // 2 if per else n - 1) * h for n, h, per in zip(self.sides, self.pitch, self.periodic)]
        return math.sqrt(sum(e * e for e in ext))

    def center(self, d):
        return self.lo[d] + 0.5 * self.sides[d] * self.pitch[d]

    def coords(self, d, device):
        """(N_d,) fp64 pixel centres of axis d, relative to the middle of the axis."""
        k = torch.arange(self.sides[d], dtype=torch.float64, device=device)
        return (k + 0.5 - 0.5 * self.sides[d]) * self.pitch[d]

    def axis_cost(self, d, device):
        """(N_d, N_d) fp64 squared distances along axis d."""
        k = torch.arange(self.sides[d], dtype=torch.float64, device=device)
        n = (k[:, None] - k[None, :]).abs()
        if self.periodic[d]:
            n = torch.minimum(n, self.sides[d] - n)
        return (n * self.pitch[d]) ** 2

    def _along(self, t, d):
        """(B, N_d) -> (B, 1, .., N_d, .., 1), broadcastable over the grid."""
        shape = [t.shape[0]] + [1] * self.D
        shape[1 + d] = self.sides[d]
        return t.reshape(shape)

    def points(self, device):
        """(P, D) fp32 pixel centres in the order of a flattened grid."""
        cs = torch.meshgrid(*[self.coords(d, device) + self.center(d) for d in range(self.D)], indexing="ij")
        return torch.stack([c.reshape(-1) for c in cs], 1).float()

    def cost(self, device):
        """(P, P) fp64 cost matrix sum_d dist_d^2 between pixels (small grids only)."""
        idx = torch.meshgrid(*[torch.arange(n, device=device) for n in self.sides], indexing="ij")
        return sum(self.axis_cost(d, device)[k.reshape(-1)][:, k.reshape(-1)] for d, k in enumerate(idx))

    def at_infinity(self, w_rows, w_cols, damp):
        """eps = +inf: f_i = sum_j w_j C_ij / sum_j w_j, separably in fp64 (sum_d of the axis cost applied to the axis
        marginal of w), then the per-point offset and dampening of ``_Softmin.at_infinity``."""
        w = w_cols.double()
        dims = tuple(range(1, self.D + 1))
        W = w.sum(dims)
        f = torch.zeros_like(w)
        for d in range(self.D):
            other = tuple(e for e in dims if e != 1 + d)
            m = w.sum(other) if other else w  # (B, N_d) marginal along axis d
            fd = (m[:, None, :] * self.axis_cost(d, w.device)[None]).sum(-1)  # one row reduction per output
            f = f + self._along(fd / W[:, None], d)
        return (damp * (f - 0.5 * w_rows.double() * f)).float()

    def softmin(self, eps, log_w, pot, *, damp=1.0, old=None):
        """damp * softmin(eps, log_w, C, pot) of the new API on the grid, or its average with ``old``; with e = eps / 2
        the kernel's -e log sum exp(h - |x-y|^2 / (2e)) is half of it, as in ``_Softmin``."""
        kw = dict(pitch=self.pitch, periodic=self.periodic)
        if old is None:
            return ops.softmin_grid_axes_raw(0.5 * eps, log_w, pot, 1.0 / eps, beta=2.0 * damp, **kw)
        return ops.softmin_grid_axes_raw(0.5 * eps, log_w, pot, 1.0 / eps, out_old=old, alpha_old=0.5, beta=damp, **kw)


def _is_real(t):
    return isinstance(t, (int, float, np.integer, np.floating)) and not isinstance(t, bool)


def solve_grid(a, b, cost="sqeuclidean", axes=None, periodic=False, debias=False, reg=None, unbalanced=None,
               unbalanced_type="KL", method="auto", max_iter=None, tol=None, p=None, blur=None, reach=None):
    """Entropic (un)balanced OT between B pairs of images or volumes on one regular grid (the new API's
    ``solve_grid``, a stub in the reference: ot/_implementations/grid.py:215-242).

    a, b: (B, N1[, N2[, N3]]) non-negative float32 CUDA tensors, axis 0 the batch, sides up to 1024.  ``axes``: None
    ([0, 1) on every axis), one (lo, hi) pair for every axis, or one pair per axis; pixel centres lo + (k + 1/2) h_d
    with h_d = (hi - lo) / N_d.  ``periodic``: a bool or one per axis.  Conventions of :func:`solve_sample`: cost
    ``|x - y|^2`` (no 1/2; wrapped around on periodic axes), ``reg`` the temperature, ``unbalanced`` the KL penalty,
    ``blur`` / ``reach`` shortcuts for ``2 blur^2`` / ``2 reach^2``, the same eps ladder, start and updates.  Element k
    of the result is ``solve_sample(X, X, a[k].flatten(), b[k].flatten(), ...)`` with X the pixel centres; the softmins
    run on the separable grid kernel (one launch per axis) and never form a (P, P) matrix.  Returns an
    :class:`OTResultGrid`; ``value`` is differentiable w.r.t. a and b."""
    if p is not None and p != 2:
        raise NotImplementedError(f"solve_grid serves the squared Euclidean cost (p = 2) only. Received p={p}.")
    if cost != "sqeuclidean":
        raise NotImplementedError(f"solve_grid serves cost='sqeuclidean' only. Received cost={cost!r}.")
    if blur is not None:
        if reg is not None:
            raise ValueError("Parameters 'reg' and 'blur' are redundant. Please specify only one of them.")
        reg = 2 * blur**2
    if reach is not None:
        if unbalanced is not None:
            raise ValueError("Parameters 'unbalanced' and 'reach' are redundant. Please specify only one of them.")
        unbalanced = 2 * reach**2
    _check_regularization(reg, unbalanced, unbalanced_type, method, tol, max_iter)
    if not (torch.is_tensor(a) and torch.is_tensor(b)):
        raise TypeError("a and b must be torch CUDA tensors (this engine has no NumPy / CPU path)")
    if not 2 <= a.dim() <= 4:
        raise ValueError(f"Expected a to be a (B, N1[, N2[, N3]]) batch of 1-, 2- or 3-D grids. Received "
                         f"{tuple(a.shape)}.")
    if any(n > ops.GRID_MAX_SIDE for n in a.shape[1:]) or a.numel() == 0:
        raise ValueError(f"solve_grid serves non-empty grids with sides up to {ops.GRID_MAX_SIDE}. Received "
                         f"{tuple(a.shape)}.")
    a = _check_marginal(a, a, None, "a")
    b = _check_marginal(b, a, None, "b")
    geo = _Grid(a.shape[1:], axes, periodic)
    dims = tuple(range(1, a.dim()))
    if unbalanced is None:
        _check_masses(a.detach().sum(dims), b.detach().sum(dims))
    for t, name in ((a, "a"), (b, "b")):
        if not (t.is_cuda and t.dtype == torch.float32):
            raise TypeError(f"{name} must be a float32 CUDA tensor (this engine computes in fp32 on the GPU), got "
                            f"{t.dtype} on {t.device}")
    reg = float(reg)
    rho = None if unbalanced is None else float(unbalanced)

    def damp(eps):
        return 1.0 if rho is None else 1.0 / (1.0 + eps / rho)

    with torch.no_grad():
        a_d, b_d = a.detach().contiguous(), b.detach().contiguous()
        eps_list = annealing_eps(geo.diameter ** 2, reg, int(max_iter))
        log_a, log_b = log_weights(a_d), log_weights(b_d)
        sm = geo.softmin
        lam = damp(eps_list[0])
        f_ba, g_ab = geo.at_infinity(a_d, b_d, lam), geo.at_infinity(b_d, a_d, lam)
        if debias:
            f_aa, g_bb = geo.at_infinity(a_d, a_d, lam), geo.at_infinity(b_d, b_d, lam)
        for eps in eps_list:
            lam = damp(eps)
            ft_ba = sm(eps, log_b, g_ab, damp=lam, old=f_ba)
            gt_ab = sm(eps, log_a, f_ba, damp=lam, old=g_ab)
            if debias:
                f_aa = sm(eps, log_a, f_aa, damp=lam, old=f_aa)
                g_bb = sm(eps, log_b, g_bb, damp=lam, old=g_bb)
            f_ba, g_ab = ft_ba, gt_ab
        # last, non-averaged update (last_extrapolation=True, sinkhorn_ot.py:419-436)
        f_ba, g_ab = sm(eps, log_b, g_ab, damp=lam), sm(eps, log_a, f_ba, damp=lam)
        if debias:
            f_aa, g_bb = sm(eps, log_a, f_aa, damp=lam), sm(eps, log_b, g_bb, damp=lam)
    if not debias:
        f_aa = g_bb = None
    return OTResultGrid(a=a, b=b, grid=geo, reg=reg, unbalanced=rho, potentials=(f_aa, g_bb, g_ab, f_ba))


class OTResultGrid(OTResultSample):
    """Result of :func:`solve_grid`, with the attributes of :class:`OTResultSample` shaped like the grids:
    ``potential_a/b/aa/bb`` and ``marginal_a/b`` (B, *grid), ``value`` (B,), ``a_to_b`` / ``b_to_a`` (B, *grid, D)
    displacement fields, ``plan_operator`` / ``density_operator`` from ``b.shape`` to ``a.shape`` with trailing channels
    (and ``.T``), dense ``plan`` / ``density`` (B, P, P) for small grids only.

    Every operator application is ONE ``b200ot_grid_plan_apply`` call (``ops.grid_plan_apply_raw``: the normalised
    weights of each row applied to all the channels), then the row factor ``w_i exp((f_i - sm_i) / reg)``, whose
    softmin sm comes from the same call; it is differentiable w.r.t. its input through the transposed operator."""

    def __init__(self, *, a, b, grid, reg, unbalanced, potentials):
        super().__init__(X_a=None, X_b=None, a=a, b=b, reg=reg, unbalanced=unbalanced, debias=potentials[0] is not None,
                         potentials=potentials, softmin=None)
        self._grid = grid

    @cached_property
    def value(self):
        B = self._a.shape[0]
        a, b, f_aa, g_bb, g_ab, f_ba = (None if t is None else t.reshape(B, -1) for t in self._live)
        return _ot_value(a, b, f_ba, g_ab, self._reg, self._unbalanced, f_aa, g_bb)

    def _weights(self, transpose):
        """(f, g, w_rows, w_cols) of the operator's direction."""
        if transpose:
            return self._g_ab, self._f_ba, self._b, self._a
        return self._f_ba, self._g_ab, self._a, self._b

    def _apply_state(self, transpose, weighted):
        """(None, None, row factor): w_rows exp((f - sm) / reg), sm the softmin of log w_cols + g / reg (the marginal
        when ``weighted``), cached until ``cache_clear``."""
        cache = self.__dict__.setdefault("_apply_cache", {})
        key = (bool(transpose), bool(weighted))
        if key not in cache:
            f, g, w_rows, w_cols = self._weights(transpose)
            with torch.no_grad():
                log_w = log_weights(w_cols) if weighted else torch.zeros_like(w_cols)
                factor = torch.exp((f - self._grid.softmin(self._reg, log_w, g)) / self._reg)
                cache[key] = (None, None, (w_rows * factor if weighted else factor).contiguous())
        return cache[key]

    def _apply(self, s, transpose, weighted, *, normalized=False):
        """plan @ s (weighted) or density @ s for s of shape (B, *grid, K) [``.T @ s`` with ``transpose``];
        ``normalized``: rows of weights summing to one (no row factor).  Detached."""
        f, g, w_rows, w_cols = self._weights(transpose)
        eps, geo = self._reg, self._grid
        with torch.no_grad():
            log_w = log_weights(w_cols) if weighted else torch.zeros_like(w_cols)
            v = s.detach().float().movedim(-1, 0).contiguous()
            ell, out = ops.grid_plan_apply_raw(0.5 * eps, log_w, g, 1.0 / eps, v, pitch=geo.pitch,
                                               periodic=geo.periodic)
            out = out.movedim(0, -1)
            if normalized:
                return out
            factor = torch.exp((f - (-eps * math.log(2.0)) * ell) / eps)  # sm = -eps ln2 ell, new-API scale
            return ((w_rows * factor) if weighted else factor)[..., None] * out

    def _density_matmat(self, s, transpose, weighted=False):
        if torch.is_grad_enabled() and s.requires_grad:
            return _PlanApply.apply(self, s, transpose, weighted)
        return self._apply(s, transpose, weighted)

    def _operator(self, weighted):
        shape = tuple(self._a.shape)
        return LinearOperator(matmat=lambda s: self._density_matmat(s, False, weighted),
                              rmatmat=lambda s: self._density_matmat(s, True, weighted), input_shape=shape,
                              output_shape=shape)

    def _barycentric(self, transpose):
        geo, dev = self._grid, self._a.device
        B = self._a.shape[0]
        cs = torch.meshgrid(*[geo.coords(d, dev) for d in range(geo.D)], indexing="ij")
        x = torch.stack(cs, -1).float().expand((B,) + geo.sides + (geo.D,))  # centred pixel coordinates
        return self._apply(x, transpose, True, normalized=True) - x

    @cached_property
    def a_to_b(self):
        """(B, *grid, D): sum_j P_ij y_j / sum_j P_ij - x_i (also defined for unbalanced problems); detached."""
        return self._barycentric(False)

    @cached_property
    def b_to_a(self):
        """(B, *grid, D): the same on the transposed plan; detached."""
        return self._barycentric(True)

    @cached_property
    def density(self):
        B, P = self._a.shape[0], self._a[0].numel()
        if B * P * P > _DENSE_LIMIT:
            raise MemoryError(f"a dense ({B}, {P}, {P}) density does not fit the budget of this accessor; use "
                              "density_operator / plan_operator, which never build the matrix")
        C = self._grid.cost(self._a.device).float()
        f, g = self._f_ba.reshape(B, P), self._g_ab.reshape(B, P)
        return torch.exp((f[:, :, None] + g[:, None, :] - C) / self._reg)

    @cached_property
    def plan(self):
        B = self._a.shape[0]
        return self.density * self._a.reshape(B, -1, 1) * self._b.reshape(B, 1, -1)

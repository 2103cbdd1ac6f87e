"""Column-sharded (multi-GPU) reductions: one process per GPU, ``torch.distributed`` for the plumbing.

SURVEY.md section 8(e): every softmin of the Sinkhorn loop reduces over the *column* cloud, so the
column axis is partitioned across the ranks while the row cloud and all potentials stay replicated
(2 x 12 MB at N = 1e6 — storage is not the constraint, work is).  Per softmin:

    rank r:  pack(y[lo_r:hi_r], h[lo_r:hi_r]) -> partial (m_i, s_i) over its columns for ALL rows
             -> merge its own splits to one (m, s) per row                      [libb200ot.so]
    all ranks: all_gather of the (N, 2) fp32 partials  (8 MB per rank at N = 1e6)   [NCCL / NVLink]
    every rank: online log-sum-exp merge of the W partials + the fused Sinkhorn epilogue  [libb200ot.so]

After the merge every rank holds the full new potential, so the next softmin's ``h`` for any shard is
a local slice: exactly ONE collective per softmin.  The backward pass shards the same way; its
partial sums simply add (one all_reduce of (N, D+1) floats).

The exchange is orders of magnitude cheaper than the reduction it follows (8 MB against an eighth of a
~0.3 s softmin per shard at N = M = 1e6 on 8 GPUs), so a plain NCCL collective on the compute stream is
used rather than a fused peer-memory epilogue.

``stages`` is injectable so that the sharding / merging logic can be exercised on CPU with the
``gloo`` backend in tests (tests/test_distributed_gloo.py supplies an oracle-backed stand-in); the
default is the CUDA implementation and it refuses non-CUDA tensors.
"""
from __future__ import annotations

from functools import partial

import torch
import torch.distributed as dist

from . import _lib, ops, ranges


def shard_bounds(M: int, rank: int, world: int):
    """Contiguous, balanced partition of range(M): sizes differ by at most one."""
    return (M * rank) // world, (M * (rank + 1)) // world


class CudaStages:
    """The staged C-ABI calls (pack -> partial -> merge | finalize) on the current CUDA stream."""

    def softmin_shard(self, eps, x, y, h_a, h_b, h_scale_b, p, center):
        """(N, 2) merged (m, s) partial of the softmin of rows x over the column shard (y, h)."""
        x, y, h_a, h_b, center = (ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"),
                                                               (center, "center")))
        N, D = x.shape
        M = y.shape[0]
        dev = x.device
        L = _lib.lib()
        if D > ops.MAX_D:
            # tensor-core dimensions (8 < D <= 64, p = 2): the one-call forward leaves the shard's log2-domain
            # log-sum-exp, which IS a merged partial (m = lse2, s = 1)
            lse2 = ops.softmin_raw(eps, x, y, h_a, h_b, h_scale_b, p=p, center=center, want_lse2=True)[1]
            return torch.stack([lse2, torch.ones_like(lse2)], dim=1).contiguous()
        merged = torch.empty(N, 2, dtype=torch.float32, device=dev)
        nsplit = ops._query(dev, "b200ot_softmin_num_splits", N, M, D)
        cols = ops._scratch(L.b200ot_packed_cols_floats(M, D, 1) * 4, dev, "shard_cols")
        part = ops._scratch(nsplit * N * 8, dev, "shard_part")
        ops._call(dev, "b200ot_softmin_pack", y, h_a, h_b, float(h_scale_b), center, M, D, int(p), float(eps), cols,
                  launches=1)
        ops._call(dev, "b200ot_softmin_partial", x, center, cols, part, nsplit, N, M, D, int(p), float(eps), launches=1)
        ops._call(dev, "b200ot_softmin_merge", part, nsplit, merged, N, launches=1)
        return merged

    def empty_shard(self, N, dev):
        """Neutral (m, s) partial for a rank that owns no column."""
        out = torch.zeros(N, 2, dtype=torch.float32, device=dev)
        out[:, 0] = -1.0e30
        return out

    def softmin_finalize(self, parts, eps, out_old, alpha_old, beta, want_lse2):
        return ranges.softmin_finalize(parts, parts.shape[0], eps, out_old, alpha_old, beta, want_lse2)

    def softmin_bwd_shard(self, eps, x, y, h_a, h_b, h_scale_b, p, center, lse2):
        """(N, D+1) partial sums of the backward pass over the column shard (any supported D)."""
        x, y, h_a, h_b, center, lse2 = (ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"),
                                                                     (center, "center"), (lse2, "lse2")))
        N, D = x.shape
        M = y.shape[0]
        dev = x.device
        sums = torch.empty(N, D + 1, dtype=torch.float32, device=dev)
        scratch = ops._scratch(ops._query(dev, "b200ot_softmin_scratch_bytes", N, M, D), dev, "softmin")
        ops._call(dev, "b200ot_softmin_bwd_sums", x, y, h_a, h_b, float(h_scale_b), center, lse2, sums, N, M, D, int(p),
                  float(eps), scratch, scratch.numel(), launches=3)
        return sums

    def softmin_bwd_finalize(self, sums, eps, x, center, grad_out, p):
        return ranges.softmin_bwd_finalize(sums, eps, x, center, grad_out, p)

    # -- ranges mode (multiscale fine phase): ALL columns are packed, the pieces select this rank's clusters --
    def softmin_sparse_shard(self, eps, x, y, h_a, h_b, h_scale_b, p, center, prob):
        """(N, 2) partial (m, s) over the column pieces listed for this rank."""
        return ranges.softmin_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, p=p, center=center)

    def softmin_bwd_sparse_shard(self, eps, x, y, h_a, h_b, h_scale_b, p, center, lse2, prob):
        """(N, D+1) partial backward sums over the column pieces listed for this rank."""
        return ranges.softmin_bwd_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, lse2, p=p, center=center)

    # -- kernel convolutions (plain sums: partial results simply add across shards) --
    def conv_shard(self, kind, x, y, w, blur, center):
        return ops.kernel_conv_raw(kind, x, y, w, blur, center=center)

    def conv_grad_shard(self, kind, x, y, w, blur, grad_out, center):
        return ops.kernel_conv_grad_rows(kind, x, y, w, blur, grad_out, center=center)


class ColumnShardedEngine:
    """Drop-in replacements for ``ops.softmin_raw`` / ``ops.softmin`` whose column reduction is spread over
    the ranks of ``group``.  Every rank must pass identical (replicated) tensors."""

    def __init__(self, group=None, stages=None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised (launch with torchrun / init_process_group)")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.stages = stages or CudaStages()
        self.collectives = 0

    # -- forward -------------------------------------------------------------------------------
    def softmin_raw(self, eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None,
                    alpha_old=0.0, beta=1.0, out=None, want_lse2=False, local=False):
        M = y.shape[0]
        N = x.shape[0]
        if local:  # replicated (un-sharded) reduction: every rank computes the whole thing, no collective
            mine = self.stages.softmin_shard(eps, x, y, h_a, h_b, h_scale_b, p, center)
            return self.stages.softmin_finalize(mine[None], eps, out_old, alpha_old, beta, want_lse2)
        lo, hi = shard_bounds(M, self.rank, self.world)
        if hi > lo:
            mine = self.stages.softmin_shard(eps, x, y[lo:hi], h_a[lo:hi], None if h_b is None else h_b[lo:hi],
                                             h_scale_b, p, center)
        else:
            mine = self.stages.empty_shard(N, x.device)
        parts = torch.empty(self.world, N, 2, dtype=mine.dtype, device=mine.device)
        dist.all_gather_into_tensor(parts.view(self.world * N, 2), mine, group=self.group)
        self.collectives += 1
        return self.stages.softmin_finalize(parts, eps, out_old, alpha_old, beta, want_lse2)

    def softmin_raw_many(self, calls):
        """The independent softmins of one Jacobi iteration, ``calls = [(args, kwargs), ...]`` of ``softmin_raw``:
        every shard reduction is enqueued first, each followed by an ASYNCHRONOUS all_gather of its (N, 2) partials,
        and the merges come last — so the exchange of softmin k travels over NVLink while the partial-reduction
        kernel of softmin k+1 runs (the collectives of an iteration are off the critical path except the last)."""
        pending = []
        for args, kw in calls:
            kw = dict(kw)
            eps, x, y, h_a = args[:4]
            h_b = args[4] if len(args) > 4 else kw.pop("h_b", None)
            h_scale_b = args[5] if len(args) > 5 else kw.pop("h_scale_b", 0.0)
            p, center = kw.pop("p", 2), kw.pop("center", None)
            M, N = y.shape[0], x.shape[0]
            lo, hi = shard_bounds(M, self.rank, self.world)
            if hi > lo:
                mine = self.stages.softmin_shard(eps, x, y[lo:hi], h_a[lo:hi], None if h_b is None else h_b[lo:hi],
                                                 h_scale_b, p, center)
            else:
                mine = self.stages.empty_shard(N, x.device)
            parts = torch.empty(self.world, N, 2, dtype=mine.dtype, device=mine.device)
            work = dist.all_gather_into_tensor(parts.view(self.world * N, 2), mine, group=self.group, async_op=True)
            self.collectives += 1
            pending.append((work, parts, mine, eps, kw))
        out = []
        for work, parts, _mine, eps, kw in pending:
            work.wait()  # stream-level wait: the host does not block
            out.append(self.stages.softmin_finalize(parts, eps, kw.get("out_old"), kw.get("alpha_old", 0.0),
                                                    kw.get("beta", 1.0), kw.get("want_lse2", False)))
        return out

    # -- forward + backward (the final, gradient-carrying Sinkhorn step) --------------------------
    def softmin(self, eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, scale_out=1.0, local=False):
        return ops._softmin_apply(partial(self.softmin_raw, local=local), partial(self.softmin_grad_rows, local=local),
                                  eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out)

    def softmin_grad_rows(self, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None, local=False,
                          prob=None):
        """grad_x of <grad_out, softmin_raw(...)> (``prob`` None) or of <grad_out, sparse_raw(..., prob)>, with y, h
        constant: the shards' partial sums, added over the ranks unless ``local``, then finalized."""
        M = y.shape[0]
        lo, hi = (0, M) if local else shard_bounds(M, self.rank, self.world)
        if prob is not None:
            sums = self.stages.softmin_bwd_sparse_shard(eps, x, y, h_a, h_b, h_scale_b, p, center, lse2, prob)
        elif hi > lo:
            sums = self.stages.softmin_bwd_shard(eps, x, y[lo:hi], h_a[lo:hi], None if h_b is None else h_b[lo:hi],
                                                 h_scale_b, p, center, lse2)
        else:
            sums = torch.zeros(x.shape[0], x.shape[1] + 1, dtype=x.dtype, device=x.device)
        if not local:
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self.group)
            self.collectives += 1
        return self.stages.softmin_bwd_finalize(sums, eps, x, center, grad_out, p)

    # -- the operator set of multiscale.sinkhorn_multiscale (same names as multiscale.LocalEngine) ----
    def build(self, keep, row_counts, layout, variant=None):
        """Ranges problem restricted to THIS rank's slab of column clusters (balanced by kept pairs)."""
        if variant is None:
            variant = getattr(self.stages, "ranges_variant", None)
        return ranges.build_problem(keep, row_counts, layout, variant=variant, rank=self.rank, world=self.world)

    def broadcast(self, t):
        t = t.contiguous()
        dist.broadcast(t, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0, group=self.group)
        self.collectives += 1
        return t

    def dense_raw(self, *args, **kw):
        return self.softmin_raw(*args, local=True, **kw)

    def dense(self, *args, **kw):
        return self.softmin(*args, local=True, **kw)

    def sparse_raw(self, eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, out_old=None, alpha_old=0.0,
                   beta=1.0, want_lse2=False):
        """Block-sparse softmin; ``prob`` holds THIS rank's column tiles (multiscale.tiles_from_cluster_mask)."""
        mine = self.stages.softmin_sparse_shard(eps, x, y, h_a, h_b, h_scale_b, p, center, prob)
        N = x.shape[0]
        parts = torch.empty(self.world, N, 2, dtype=mine.dtype, device=mine.device)
        dist.all_gather_into_tensor(parts.view(self.world * N, 2), mine, group=self.group)
        self.collectives += 1
        return self.stages.softmin_finalize(parts, eps, out_old, alpha_old, beta, want_lse2)

    def sparse(self, eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, scale_out=1.0):
        return ops._softmin_apply(partial(self.sparse_raw, prob=prob), partial(self.softmin_grad_rows, prob=prob), eps,
                                  x, y, h_a, h_b, h_scale_b, p, center, scale_out)

    # -- kernel MMD matvec: out = K(x, y) @ w with the columns sharded, one all_reduce(SUM) --------
    def kernel_conv(self, kind, x, y, w, blur, *, center=None):
        return _ShardedConv.apply(self, x, y, w, kind, blur, center)

    def attach(self, loss_module):
        """Make a ``SamplesLoss`` module run its reductions (Sinkhorn softmins, kernel matvecs) through this
        engine."""
        loss_module._engine = dict(softmin_raw=self.softmin_raw, softmin_grad=self.softmin, conv=self.kernel_conv)
        loss_module._multiscale_engine = self
        return loss_module


class _ShardedConv(torch.autograd.Function):
    """out = K(x, y) @ w, columns sharded.  Gradients: rows by a sharded reduction + all_reduce; columns and
    weights are computed for the local shard (full row reduction, kernels are symmetric) and all_gathered."""

    @staticmethod
    def forward(ctx, eng, x, y, w, kind, blur, center):
        lo, hi = shard_bounds(y.shape[0], eng.rank, eng.world)
        if hi > lo:
            out = eng.stages.conv_shard(kind, x, y[lo:hi], w[lo:hi], blur, center)
        else:
            out = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device)
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=eng.group)
        eng.collectives += 1
        ctx.eng = eng
        ctx.save_for_backward(x, y, w, center if center is not None else w)
        ctx.meta = (kind, float(blur), center is not None)
        return out

    @staticmethod
    def backward(ctx, go):
        eng = ctx.eng
        x, y, w, center = ctx.saved_tensors
        kind, blur, has_center = ctx.meta
        center = center if has_center else None
        go = go.contiguous()
        M = y.shape[0]
        lo, hi = shard_bounds(M, eng.rank, eng.world)
        gx = gy = gw = None
        if ctx.needs_input_grad[1]:
            if hi > lo:
                gx = eng.stages.conv_grad_shard(kind, x, y[lo:hi], w[lo:hi], blur, go, center)
            else:
                gx = torch.zeros_like(x)
            dist.all_reduce(gx, op=dist.ReduceOp.SUM, group=eng.group)
            eng.collectives += 1
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            # shard-local rows y[lo:hi] against ALL of x; ragged shards -> pad to the largest, gather, trim
            size = -(-M // eng.world)
            sizes = [shard_bounds(M, r, eng.world) for r in range(eng.world)]
            if ctx.needs_input_grad[2]:
                loc = torch.zeros(size, y.shape[1], dtype=y.dtype, device=y.device)
                if hi > lo:
                    loc[: hi - lo] = eng.stages.conv_grad_shard(kind, y[lo:hi], x, go, blur, w[lo:hi], center)
                buf = torch.empty(eng.world * size, y.shape[1], dtype=y.dtype, device=y.device)
                dist.all_gather_into_tensor(buf, loc, group=eng.group)
                gy = torch.cat([buf[r * size: r * size + (b - a)] for r, (a, b) in enumerate(sizes)])
                eng.collectives += 1
            if ctx.needs_input_grad[3]:
                loc = torch.zeros(size, dtype=w.dtype, device=w.device)
                if hi > lo:
                    loc[: hi - lo] = eng.stages.conv_shard(kind, y[lo:hi], x, go, blur, center)
                buf = torch.empty(eng.world * size, dtype=w.dtype, device=w.device)
                dist.all_gather_into_tensor(buf, loc, group=eng.group)
                gw = torch.cat([buf[r * size: r * size + (b - a)] for r, (a, b) in enumerate(sizes)])
                eng.collectives += 1
        return None, gx, gy, gw, None, None, None

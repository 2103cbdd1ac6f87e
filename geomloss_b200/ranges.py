"""Ranges mode of the reductions: block-sparse and batched problems in ONE launch group.

Host side of the reference's ``ranges=`` machinery — pykeops' ``from_matrix`` / ``cluster_ranges`` tuples consumed by
``softmin_multiscale`` (src/geomloss/_legacy/sinkhorn_samples.py:445-450, built by ``kernel_truncation`` :493-530) and
``kernel_multiscale`` (src/geomloss/_legacy/kernel_samples.py:246-271) — and of the batched LazyTensor reduction
(``softmin_online_lazytensor``, sinkhorn_samples.py:229-290), which is the block-diagonal special case.

A problem is described to libb200ot.so (include/b200ot.h, "ranges mode") by
  * a ``ColumnLayout``: the column cloud is grouped (clusters of a label-sorted cloud, or batch elements); every
    group is padded to a multiple of 16 column SLOTS so that it starts on a chunk boundary of the kernels; the pack
    kernel gathers ``slot -> column`` through ``src`` (padding slots are neutral columns);
  * segments ``(row_start, row_count, piece_begin, piece_end)``: runs of rows of ONE row group, at most one CTA tall;
  * pieces ``(col_start, col_count)``: runs of consecutive kept column groups, cut to at most one tile.
The kernels then visit exactly the (row group, column group) pairs of the boolean ``keep`` matrix — the same blocks
as the reference, not a tile-level superset.  Everything below is vectorised torch on the device (no Python loop
over clusters); the only host syncs are the sizes of the descriptor arrays.

These are the CUDA-core kernels, D <= 8.  For 8 < D <= 64 the same ``keep`` matrix is run by the tensor-core kernels
(``variant=TC``, the b200ot_*_blocks entries): every row cluster AND every column cluster is padded to whole 128-point
tiles, segments are single 128-row tiles of one row cluster and pieces runs of whole column tiles.  Padding slots cost
computation (a cluster of 1 point fills a tile) but no accuracy: padding columns vanish from the log-sum-exp and
padding rows write nothing.
"""
from __future__ import annotations

import ctypes
from functools import partial

import torch

from . import _lib, ops

BIG, SMALL = 0, 1
TC = 2  # block-sparse tensor-core problems, 8 < D <= 64


def shape(variant):
    r, c, al = ctypes.c_int32(0), ctypes.c_int32(0), ctypes.c_int32(0)
    _lib.lib().b200ot_ranges_shape(int(variant), ctypes.byref(r), ctypes.byref(c), ctypes.byref(al))
    return r.value, c.value, al.value


def blocks_shape():
    """(rows per segment, column alignment) of the tensor-core block-sparse problems: both 128."""
    r, al = ctypes.c_int32(0), ctypes.c_int32(0)
    _lib.lib().b200ot_blocks_shape(ctypes.byref(r), ctypes.byref(al))
    return r.value, al.value


def _excl_cumsum(t):
    out = torch.zeros(t.numel() + 1, dtype=torch.int64, device=t.device)
    out[1:] = t.cumsum(0)
    return out


class ColumnLayout:
    """Slot layout of a grouped column cloud: ``counts[g]`` consecutive columns belong to group g."""

    def __init__(self, counts, align=16):
        counts = counts.to(torch.int64)
        dev = counts.device
        self.align = align
        self.counts = counts
        self.padded = (counts + align - 1) // align * align
        self.col_start = _excl_cumsum(counts)
        self.slot_start = _excl_cumsum(self.padded)
        self.n_cols = int(self.col_start[-1].item())
        self.n_slots = int(self.slot_start[-1].item())
        grp = torch.repeat_interleave(torch.arange(counts.numel(), device=dev), counts)
        cols = torch.arange(self.n_cols, device=dev)
        slot_of_col = self.slot_start[grp] + (cols - self.col_start[grp])
        src = torch.full((max(self.n_slots, 1),), -1, dtype=torch.int32, device=dev)
        src[slot_of_col] = cols.to(torch.int32)
        self.src = src.contiguous()


class RangesProblem:
    """Descriptor arrays of one reduction problem (rows x grouped columns restricted to ``keep``)."""

    def __init__(self, seg, pieces, layout, variant, n_rows, density, row_layout=None, computed=None):
        self.seg, self.pieces, self.layout, self.variant = seg, pieces, layout, variant
        self.n_seg = int(seg.shape[0])
        self.n_rows = n_rows
        self.density = density  # kept (row, column) pairs / all pairs
        # TC: the row slot layout, and the (row slot, column slot) pairs the kernels compute / all pairs
        self.row_layout = row_layout
        self.computed = density if computed is None else computed
        self._scratch_bytes = {}


def pick_variant(row_counts, col_counts):
    """Big tiles (512-row segments, 1024-column pieces) pay off once groups hold a few hundred points."""
    rows = float(row_counts.double().mean().item())
    cols = float(col_counts.double().mean().item())
    return BIG if (rows >= 192 and cols >= 192) else SMALL


def build_problem(keep, row_counts, layout, variant=None, rank=0, world=1):
    """``keep``: (R, C) bool over (row groups, column groups), or None for all pairs.  ``row_counts``: (R,) rows per
    row group (consecutive).  ``world > 1``: column-sharded run — this rank keeps a contiguous slab of column groups,
    cut so that every rank reduces about the same number of pairs (SURVEY.md section 8e)."""
    dev = row_counts.device
    row_counts = row_counts.to(torch.int64)
    R, C = row_counts.numel(), layout.counts.numel()
    if variant is None:
        variant = pick_variant(row_counts, layout.counts)
    tc = variant == TC
    if tc:
        max_rows, align = blocks_shape()
        if layout.align != align or world > 1:
            raise ValueError(f"tensor-core block problems need a ColumnLayout(counts, align={align}) and one GPU")
        max_cols = max(layout.n_slots, 1)  # a run of kept column clusters is one piece
    else:
        max_rows, max_cols, _ = shape(variant)
    if keep is None:
        keep = torch.ones(R, C, dtype=torch.bool, device=dev)
    keep = keep.to(torch.bool)
    pairs_all = float(row_counts.sum().item()) * float(layout.counts.sum().item())
    w_pairs = (keep.double() * row_counts.double()[:, None] * layout.counts.double()[None, :])
    density = float(w_pairs.sum().item()) / max(pairs_all, 1.0)
    if world > 1:
        load = w_pairs.sum(0).cumsum(0)
        total = load[-1]
        cuts = torch.searchsorted(load, total * torch.arange(1, world, device=dev, dtype=torch.float64) / world)
        cuts = [0] + [min(int(c) + 1, C) for c in cuts.tolist()] + [C]
        lo, hi = cuts[rank], max(cuts[rank], cuts[rank + 1])
        keep = keep.clone()
        keep[:, :lo] = False
        keep[:, hi:] = False
    # maximal runs of consecutive kept column groups, row group by row group
    false_col = torch.zeros(R, 1, dtype=torch.bool, device=dev)
    start = keep & ~torch.cat([false_col, keep[:, :-1]], dim=1)
    end = keep & ~torch.cat([keep[:, 1:], false_col], dim=1)
    s_idx, e_idx = start.nonzero(), end.nonzero()  # row-major order: the k-th start pairs with the k-th end
    run_row = s_idx[:, 0]
    run_lo = layout.slot_start[s_idx[:, 1]]
    run_hi = layout.slot_start[e_idx[:, 1] + 1]
    n_piece = (run_hi - run_lo + max_cols - 1) // max_cols
    n_runs = run_row.numel()
    piece_run = torch.repeat_interleave(torch.arange(n_runs, device=dev), n_piece)
    first = n_piece.cumsum(0) - n_piece
    k_in = torch.arange(piece_run.numel(), device=dev) - first[piece_run]
    col_start = run_lo[piece_run] + k_in * max_cols
    col_count = torch.minimum(torch.full_like(col_start, max_cols), run_hi[piece_run] - col_start)
    pieces = torch.stack([col_start, col_count], dim=1).to(torch.int32).contiguous()
    per_row = torch.zeros(R, dtype=torch.int64, device=dev).index_add_(0, run_row, n_piece)
    piece_ptr = _excl_cumsum(per_row)
    # segments: every row group is cut into CTA-sized runs of rows sharing its piece list (TC: whole row tiles of the
    # row slot layout, every row cluster padded to a multiple of 128 rows on its own)
    row_layout = ColumnLayout(row_counts, align=max_rows) if tc else None
    row_off = _excl_cumsum(row_counts)
    n_seg_r = (row_counts + max_rows - 1) // max_rows
    seg_grp = torch.repeat_interleave(torch.arange(R, device=dev), n_seg_r)
    k_seg = torch.arange(seg_grp.numel(), device=dev) - (n_seg_r.cumsum(0) - n_seg_r)[seg_grp]
    row_base = row_layout.slot_start if tc else row_off
    row_start = row_base[seg_grp] + k_seg * max_rows
    row_count = torch.minimum(torch.full_like(row_start, max_rows), row_off[seg_grp + 1] - (row_off[seg_grp] +
                                                                                             k_seg * max_rows))
    seg = torch.stack([row_start, row_count, piece_ptr[seg_grp], piece_ptr[seg_grp + 1]], dim=1)
    # heaviest segments first: shortens the tail of the last wave
    if tc:
        slots = torch.zeros(R, dtype=torch.int64, device=dev).index_add_(0, run_row, run_hi - run_lo)
        work = slots[seg_grp]
    else:
        work = (seg[:, 3] - seg[:, 2]) * max_cols
    seg = seg[torch.argsort(work, descending=True, stable=True)].to(torch.int32).contiguous()
    if pieces.shape[0] == 0:
        pieces = torch.zeros(1, 2, dtype=torch.int32, device=dev)
    if not tc:
        return RangesProblem(seg, pieces, layout, variant, int(row_off[-1].item()), density)
    # the tensor-core entries read the descriptors on the host
    computed = float((slots.double() * max_rows * n_seg_r.double()).sum().item()) / max(pairs_all, 1.0)
    return RangesProblem(seg.cpu(), pieces.cpu(), layout, variant, int(row_off[-1].item()), density,
                         row_layout=row_layout, computed=computed)


def batch_problem(B, N, M, device, variant=None):
    """B independent (N rows) x (M columns) problems stacked along the row / column axes (block-diagonal keep)."""
    layout = ColumnLayout(torch.full((B,), M, dtype=torch.int64, device=device))
    rows = torch.full((B,), N, dtype=torch.int64, device=device)
    if variant is None:
        variant = BIG if (N >= 2048 and M >= 2048) else SMALL
    return build_problem(torch.eye(B, dtype=torch.bool, device=device), rows, layout, variant=variant)


# ------------------------------------------------------------------------------------------------------
# softmin
# ------------------------------------------------------------------------------------------------------
def _check_path(prob, D):
    """A problem is built for one family of kernels: CUDA-core ranges (BIG / SMALL, D <= 8) or tensor-core blocks
    (TC, 8 < D <= 64).  The other one refuses it."""
    if prob.variant == TC:
        if not ops.MAX_D < D <= ops.MAX_D_TC:
            raise ValueError(f"a tensor-core block problem (variant TC) serves {ops.MAX_D} < D <= {ops.MAX_D_TC}, "
                             f"got D = {D}")
    elif D > ops.MAX_D:
        raise ValueError(f"a ranges problem (variant BIG / SMALL) serves D <= {ops.MAX_D}, got D = {D}: build it with "
                         "variant=ranges.TC and ColumnLayout(counts, align=128)")


def softmin_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, part=None):
    """pack (gather) + partial reduction: the (N, 2) (m, s) partials of this problem's pieces."""
    x, y, h_a, h_b, center = (ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"),
                                                           (center, "center")))
    N, D = x.shape
    _check_path(prob, D)
    if prob.variant == TC:
        raise ValueError("tensor-core block problems run as one call (softmin_ranges_raw), without exposed partials")
    if N != prob.n_rows or y.shape[0] != prob.layout.n_cols:
        raise ValueError("point clouds do not match the ranges problem they are reduced with")
    dev = x.device
    lay = prob.layout
    if part is None:
        part = torch.empty(N, 2, dtype=torch.float32, device=dev)
    cols = ops._scratch(_lib.lib().b200ot_packed_cols_floats(lay.n_slots, D, 1) * 4, dev, "ranges_cols")
    ops._call(dev, "b200ot_softmin_pack_gather", y, h_a, h_b, float(h_scale_b), center, lay.src, lay.n_slots, D,
              int(p), float(eps), cols, launches=1)
    ops._call(dev, "b200ot_softmin_partial_ranges", x, center, cols, prob.seg, prob.n_seg, prob.pieces, part, N, D,
              int(p), float(eps), prob.variant, launches=1)
    return part


def softmin_finalize(parts, n_part, eps, out_old, alpha_old, beta, want_lse2, out=None):
    """Merge the ``n_part`` (m, s) partials ``parts`` (n_part, N, 2) per row, with the fused Sinkhorn epilogue."""
    N = parts.shape[-2]
    dev = parts.device
    if out is None:
        out = torch.empty(N, dtype=torch.float32, device=dev)
    lse2 = torch.empty(N, dtype=torch.float32, device=dev) if want_lse2 else None
    ops._call(dev, "b200ot_softmin_finalize", parts, int(n_part), ops._f32c(out_old, "out_old"), float(alpha_old),
              float(beta), out, lse2, N, float(eps), launches=1)
    return out, lse2


def _blocks_args(prob, x, y):
    """Shared arguments of the b200ot_*_blocks entries: row / column gather and the host descriptors."""
    N, D = x.shape
    if N != prob.n_rows or y.shape[0] != prob.layout.n_cols:
        raise ValueError("point clouds do not match the block problem they are reduced with")
    rl, cl = prob.row_layout, prob.layout
    nbytes = prob._scratch_bytes.get(D)
    if nbytes is None:
        nbytes = ops._query(x.device, "b200ot_blocks_scratch_bytes", N, rl.n_slots, cl.n_slots, ops._ptr(prob.seg),
                            prob.n_seg, ops._ptr(prob.pieces), D)
        if nbytes <= 0:
            raise ValueError("invalid tensor-core block problem")
        prob._scratch_bytes[D] = nbytes
    return (N, rl.src, rl.n_slots, cl.src, cl.n_slots, prob.seg, prob.n_seg, prob.pieces, D), nbytes


def softmin_blocks_raw(eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, out_old=None, alpha_old=0.0,
                       beta=1.0, want_lse2=False, out=None):
    """One block-sparse softmin on the tensor cores (8 < D <= 64): pack + reduction + finalize in one C call."""
    x, y, h_a, h_b, center, out_old = (ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"),
                                                                    (center, "center"), (out_old, "out_old")))
    _check_path(prob, x.shape[1])
    dev = x.device
    (N, *rest), nbytes = _blocks_args(prob, x, y)
    if out is None:
        out = torch.empty(N, dtype=torch.float32, device=dev)
    lse2 = torch.empty(N, dtype=torch.float32, device=dev) if want_lse2 else None
    scratch = ops._scratch(nbytes, dev, "blocks")
    ops._call(dev, "b200ot_softmin_fwd_blocks", x, y, h_a, h_b, float(h_scale_b), center, out_old, float(alpha_old),
              float(beta), out, lse2, N, *rest, int(p), float(eps), scratch, nbytes, launches=4)
    return out, lse2


def softmin_blocks_bwd_x(eps, x, y, h_a, h_b, h_scale_b, prob, lse2, grad_out, *, p=2, center=None):
    x, y, h_a, h_b, center, lse2, grad_out = (
        ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"), (center, "center"),
                                     (lse2, "lse2"), (grad_out, "grad_out")))
    _check_path(prob, x.shape[1])
    dev = x.device
    (N, *rest), nbytes = _blocks_args(prob, x, y)
    gx = torch.empty_like(x)
    scratch = ops._scratch(nbytes, dev, "blocks")
    ops._call(dev, "b200ot_softmin_bwd_x_blocks", x, y, h_a, h_b, float(h_scale_b), center, lse2, grad_out, gx, N,
              *rest, int(p), float(eps), scratch, nbytes, launches=4)
    return gx


def softmin_ranges_raw(eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, out_old=None, alpha_old=0.0,
                       beta=1.0, want_lse2=False, out=None):
    if x.shape[1] > ops.MAX_D:
        return softmin_blocks_raw(eps, x, y, h_a, h_b, h_scale_b, prob, p=p, center=center, out_old=out_old,
                                  alpha_old=alpha_old, beta=beta, want_lse2=want_lse2, out=out)
    part = softmin_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, p=p, center=center)
    return softmin_finalize(part, 1, eps, out_old, alpha_old, beta, want_lse2, out=out)


def softmin_bwd_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, lse2, *, p=2, center=None):
    """(N, D+1) row-gradient sums over this problem's pieces."""
    x, y, h_a, h_b, center, lse2 = (ops._f32c(t, n) for t, n in ((x, "x"), (y, "y"), (h_a, "h_a"), (h_b, "h_b"),
                                                                 (center, "center"), (lse2, "lse2")))
    N, D = x.shape
    _check_path(prob, D)
    if prob.variant == TC:
        raise ValueError("tensor-core block problems run as one call (softmin_blocks_bwd_x), without exposed sums")
    dev = x.device
    lay = prob.layout
    sums = torch.zeros(N, D + 1, dtype=torch.float32, device=dev)
    cols = ops._scratch(_lib.lib().b200ot_packed_cols_floats(lay.n_slots, D, 1) * 4, dev, "ranges_cols")
    ops._call(dev, "b200ot_softmin_pack_gather", y, h_a, h_b, float(h_scale_b), center, lay.src, lay.n_slots, D,
              int(p), float(eps), cols, launches=1)
    ops._call(dev, "b200ot_softmin_bwd_partial_ranges", x, center, cols, lse2, prob.seg, prob.n_seg, prob.pieces, sums,
              N, D, int(p), float(eps), prob.variant, launches=1)
    return sums


def softmin_bwd_finalize(sums, eps, x, center, grad_out, p):
    """grad_x from the (N, D+1) row-gradient sums of all the column pieces (summed over shards)."""
    x, center, grad_out = ops._f32c(x, "x"), ops._f32c(center, "center"), ops._f32c(grad_out, "grad_out")
    N, D = x.shape
    gx = torch.empty_like(x)
    ops._call(x.device, "b200ot_softmin_bwd_finalize", sums, 1, x, center, grad_out, gx, N, D, int(p), float(eps),
              launches=1)
    return gx


def softmin_ranges_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None, prob):
    """grad_x of <grad_out, softmin_ranges_raw(eps, x, y, h, prob)> with y, h constant (the row-gradient operator of
    ``ops._Softmin``, ``prob`` bound by keyword)."""
    if prob.variant == TC:
        return softmin_blocks_bwd_x(eps, x, y, h_a, h_b, h_scale_b, prob, lse2, grad_out, p=p, center=center)
    sums = softmin_bwd_shard_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, lse2, p=p, center=center)
    return softmin_bwd_finalize(sums, eps, x, center, grad_out, p)


def softmin_ranges(eps, x, y, h_a, h_b, h_scale_b, prob, *, p=2, center=None, scale_out=1.0):
    return ops._softmin_apply(partial(softmin_ranges_raw, prob=prob), partial(softmin_ranges_grad_rows, prob=prob),
                              eps, x, y, h_a, h_b, h_scale_b, p, center, scale_out)


# ------------------------------------------------------------------------------------------------------
# kernel convolutions
# ------------------------------------------------------------------------------------------------------
def _conv_width(kind_id, D, backward):
    if not backward:
        return 1
    return D + 1 if (kind_id & 0xFF) == 0 else D


def conv_shard_ranges(kind_id, x, y, w, blur, prob, *, center=None, backward=False):
    """(N,) sums (forward) or (N, width) row-gradient sums over this problem's pieces."""
    x, y, w, center = ops._f32c(x, "x"), ops._f32c(y, "y"), ops._f32c(w, "w"), ops._f32c(center, "center")
    N, D = x.shape
    if N != prob.n_rows or y.shape[0] != prob.layout.n_cols:
        raise ValueError("point clouds do not match the ranges problem they are reduced with")
    dev = x.device
    lay = prob.layout
    part = torch.zeros(N, _conv_width(kind_id, D, backward), dtype=torch.float32, device=dev)
    cols = ops._scratch(_lib.lib().b200ot_packed_cols_floats(lay.n_slots, D, 2) * 4, dev, "ranges_cols")
    ops._call(dev, "b200ot_kernel_conv_pack_gather", y, w, center, lay.src, lay.n_slots, D, int(kind_id), float(blur),
              cols, launches=1)
    ops._call(dev, "b200ot_kernel_conv_partial_ranges", x, center, cols, prob.seg, prob.n_seg, prob.pieces, part, N, D,
              int(kind_id), float(blur), 1 if backward else 0, prob.variant, launches=1)
    return part


def conv_finalize(kind_id, part):
    N = part.shape[0]
    out = torch.empty(N, dtype=torch.float32, device=part.device)
    ops._call(part.device, "b200ot_kernel_conv_finalize", part, 1, out, N, int(kind_id), launches=1)
    return out


def conv_bwd_finalize(kind_id, part, x, center, grad_out, blur):
    x, center, grad_out = ops._f32c(x, "x"), ops._f32c(center, "center"), ops._f32c(grad_out, "grad_out")
    N, D = x.shape
    gx = torch.empty_like(x)
    ops._call(x.device, "b200ot_kernel_conv_bwd_finalize", part, 1, x, center, grad_out, gx, N, D, int(kind_id),
              float(blur), launches=1)
    return gx


def _conv_ops(prob):
    """``ops._ConvOps`` of the ranges problem ``prob`` (None: no operators)."""
    if prob is None:
        return None

    def raw(kind_id, x, y, w, blur, *, center=None):
        return conv_finalize(kind_id, conv_shard_ranges(kind_id, x, y, w, blur, prob, center=center))

    def grad_rows(kind_id, x, y, w, blur, grad_out, *, center=None):
        part = conv_shard_ranges(kind_id, x, y, w, blur, prob, center=center, backward=True)
        return conv_bwd_finalize(kind_id, part, x, center, grad_out, blur)

    return ops._ConvOps(raw, grad_rows)


def kernel_conv_ranges(kind_id, x, y, w, blur, prob, prob_t=None, *, center=None):
    """out = (K(x, y) restricted to prob) @ w, differentiable w.r.t. x, y and w; ``prob_t`` is the transposed problem
    (rows y, columns x) that serves the y- and w-gradients (kernels are symmetric)."""
    return ops._KernelConv.apply(_conv_ops(prob), _conv_ops(prob_t), x, y, w, kind_id, blur, center, False)

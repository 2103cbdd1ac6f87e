"""CPU-only checks of the block-sparse tensor-core softmins (b200ot_*_blocks, 8 < D <= 64; the fine phase of the
labelled two-scale Sinkhorn above D = 8):
  * the descriptors ranges.build_problem(variant=TC) writes list exactly the kept (row cluster, column cluster) blocks,
    each pair once, on whole 128-point tiles;
  * every bad argument is refused before any CUDA call: -1 (EINVAL), -4 (EALIGN), -2 (ESCRATCH).  The device pointers
    are fakes and are never dereferenced; the descriptor arrays are host memory, read by the library.
Every call below has at least one bad argument, so that nothing is ever launched."""
import ctypes

import numpy as np
import pytest
import torch

from geomloss_b200 import _build, _lib

NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
SYMBOLS = ["b200ot_blocks_shape", "b200ot_blocks_scratch_bytes", "b200ot_softmin_fwd_blocks",
           "b200ot_softmin_bwd_x_blocks"]


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _host(a, offset=0):
    """ctypes pointer to a copy of int32 array `a`, 64-byte aligned plus `offset` bytes (kept alive by the caller)."""
    raw = np.zeros(a.size * 4 + 128, dtype=np.uint8)
    start = (-raw.ctypes.data) % 64 + offset
    view = raw[start:start + a.size * 4].view(np.int32)
    view[:] = a.ravel()
    return raw, ctypes.c_void_p(view.ctypes.data)


# two row clusters (1 and 129 rows: three row tiles), two column clusters (128 and 1 columns: two column tiles)
SEG = np.array([[128, 128, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]], dtype=np.int32)
PIECES = np.array([[0, 128], [0, 256]], dtype=np.int32)
N_ROWS, ROW_SLOTS, COL_SLOTS = 130, 384, 256


def _call(L, which, seg=SEG, pieces=PIECES, seg_off=0, pieces_off=0, n_seg=None, N=N_ROWS, row_slots=ROW_SLOTS,
          col_slots=COL_SLOTS, D=16, p=2, eps=0.1, x=FAKE, y=FAKE, h=FAKE, row_src=FAKE, col_src=FAKE, out=FAKE,
          lse2=FAKE, go=FAKE, gx=FAKE, scratch=FAKE, nbytes=BIG, seg_ptr=None, pieces_ptr=None):
    keep_s, sp = _host(seg, seg_off)
    keep_p, pp = _host(pieces, pieces_off)
    sp = sp if seg_ptr is None else seg_ptr
    pp = pp if pieces_ptr is None else pieces_ptr
    n_seg = len(seg) if n_seg is None else n_seg
    if which == "fwd":
        return L.b200ot_softmin_fwd_blocks(x, y, h, NULL, 0.0, NULL, NULL, 0.0, 1.0, out, NULL, N, row_src, row_slots,
                                           col_src, col_slots, sp, n_seg, pp, D, p, eps, scratch, nbytes, NULL)
    return L.b200ot_softmin_bwd_x_blocks(x, y, h, NULL, 0.0, NULL, lse2, go, gx, N, row_src, row_slots, col_src,
                                         col_slots, sp, n_seg, pp, D, p, eps, scratch, nbytes, NULL)


def _need(L, seg=SEG, pieces=PIECES, N=N_ROWS, D=16):
    _ks, sp = _host(seg)
    _kp, pp = _host(pieces)
    return L.b200ot_blocks_scratch_bytes(N, ROW_SLOTS, COL_SLOTS, sp, len(seg), pp, D)


def test_symbols_and_shape(L):
    for name in SYMBOLS:
        assert hasattr(L, name) and name in _lib.exported_symbols(), name
    from geomloss_b200 import ranges

    assert ranges.blocks_shape() == (128, 128)
    # the CUDA-core ranges shapes keep their answers
    assert ranges.shape(ranges.BIG) == (512, 1024, 16) and ranges.shape(ranges.SMALL) == (128, 256, 16)


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_bad_arguments_are_refused(L, which):
    small = dict(nbytes=16)  # every otherwise valid call below fails on the scratch size, never launches
    assert _call(L, which, **small) == -2
    assert _call(L, which, p=2 | 0x100, **small) == -2  # the KeOps convention of the two-scale Sinkhorn is legal
    assert _call(L, which, D=9, **small) == -2 and _call(L, which, D=64, **small) == -2
    ptrs = ["x", "y", "h", "row_src", "col_src", "scratch"] + (["out"] if which == "fwd" else ["lse2", "go", "gx"])
    for ptr in ptrs:
        if which == "fwd" and ptr == "out":
            assert _call(L, which, out=NULL, lse2=NULL) == -1  # neither out nor lse2
            continue
        assert _call(L, which, **{ptr: NULL}) == -1, ptr
    assert _call(L, which, seg_ptr=NULL) == -1 and _call(L, which, pieces_ptr=NULL) == -1
    for kw in (dict(D=8), dict(D=1), dict(D=65), dict(D=0), dict(p=1), dict(p=1 | 0x100), dict(p=3), dict(p=0x202),
               dict(eps=0.0), dict(eps=-1.0), dict(N=0), dict(n_seg=0), dict(n_seg=-1)):
        assert _call(L, which, **kw) == -1, kw
    # descriptors off the tile grid or inconsistent with the slot counts
    bad_pieces = ([[64, 128], [0, 256]], [[0, 100], [0, 256]], [[0, 128], [0, 384]], [[0, 0], [0, 256]],
                  [[-128, 128], [0, 256]])
    for pc in bad_pieces:
        assert _call(L, which, pieces=np.array(pc, dtype=np.int32)) == -1, pc
    bad_segs = ([[64, 128, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]],    # row tile off the grid
                [[128, 128, 1, 2], [128, 1, 1, 2], [0, 1, 0, 1]],   # two segments on one row tile
                [[128, 0, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]],     # no live row
                [[128, 129, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]],   # more rows than a tile
                [[128, 128, 2, 1], [256, 1, 1, 2], [0, 1, 0, 1]],   # piece_end < piece_begin
                [[128, 128, 1, 3], [256, 1, 1, 2], [0, 1, 0, 1]],   # a piece past the list: checked like the others
                [[384, 128, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]])   # row tile past the slots
    for sg in bad_segs:
        arr = np.array(sg, dtype=np.int32)
        pieces = PIECES if sg[0][3] != 3 else np.array([[0, 128], [0, 256], [0, 64]], dtype=np.int32)
        assert _call(L, which, seg=arr, pieces=pieces) == -1, sg
    assert _call(L, which, n_seg=2) == -1          # one segment per row tile
    assert _call(L, which, row_slots=383) == -1    # slots are whole tiles
    assert _call(L, which, col_slots=200) == -1
    assert _call(L, which, col_slots=0) == -1
    # misaligned descriptor arrays and scratch
    assert _call(L, which, seg_off=4) == -4
    assert _call(L, which, seg_off=8) == -4
    assert _call(L, which, pieces_off=4) == -4
    assert _call(L, which, scratch=ctypes.c_void_p(0x1004)) == -4


@pytest.mark.parametrize("which", ["fwd", "bwd"])
def test_small_scratch(L, which):
    for D in (9, 16, 33, 64):
        need = _need(L, D=D)
        assert need > 0
        assert _call(L, which, D=D, nbytes=need - 1) == -2
    # descriptors with no piece at all (every row cluster keeps nothing) are valid
    empty = np.array([[128, 128, 0, 0], [256, 1, 0, 0], [0, 1, 0, 0]], dtype=np.int32)
    need = _need(L, seg=empty)
    assert need > 0 and _call(L, which, seg=empty, nbytes=need - 1) == -2


def test_scratch_query(L, monkeypatch):
    assert _need(L, D=8) == 0 and _need(L, D=65) == 0
    assert _need(L, pieces=np.array([[64, 128], [0, 256]], dtype=np.int32)) == 0
    assert _need(L, N=0) == 0
    # the split count (B200OT_FORCE_SPLITS applies, capped by the longest segment: 2 tiles) sizes the partials
    monkeypatch.setenv("B200OT_FORCE_SPLITS", "1")
    one = _need(L)
    monkeypatch.setenv("B200OT_FORCE_SPLITS", "2")
    two = _need(L)
    monkeypatch.setenv("B200OT_FORCE_SPLITS", "7")
    assert _need(L) == two > one


def _blocks_mask(prob, n_rows, n_cols):
    """(n_rows, n_cols) count of how often the block problem visits each (row, column) pair, in cloud order."""
    seg, pieces = prob.seg.tolist(), prob.pieces.tolist()
    rsrc, csrc = prob.row_layout.src.tolist(), prob.layout.src.tolist()
    mask = torch.zeros(n_rows, n_cols, dtype=torch.int32)
    for r0, rc, pb, pe in seg:
        rows = [r for r in rsrc[r0:r0 + 128] if r >= 0]
        assert len(rows) == rc
        cols = [c for q in range(pb, pe) for c in csrc[pieces[q][0]:pieces[q][0] + pieces[q][1]] if c >= 0]
        if rows and cols:
            mask[torch.tensor(rows)[:, None], torch.tensor(cols)[None, :]] += 1
    return mask


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_blocks_descriptors_list_exactly_the_kept_cluster_pairs(L, seed):
    """segments x pieces == keep[lab_rows][:, lab_cols], each pair exactly once, on whole 128-point tiles; one segment
    per row tile, heaviest first; a problem built for one family of kernels is refused by the other."""
    from geomloss_b200 import ranges

    g = torch.Generator().manual_seed(seed)
    R, C = 19, 14
    row_counts = torch.randint(1, 400, (R,), generator=g)
    col_counts = torch.randint(1, 400, (C,), generator=g)
    row_counts[:4] = torch.tensor([1, 127, 128, 129])
    col_counts[:4] = torch.tensor([129, 128, 1, 127])
    keep = torch.rand(R, C, generator=g) < 0.4
    keep[3] = False  # a row cluster that keeps nothing
    keep[5] = True   # ... and one that keeps everything (one run)
    lay = ranges.ColumnLayout(col_counts, align=128)
    n_rows, n_cols = int(row_counts.sum()), int(col_counts.sum())
    lab_r = torch.repeat_interleave(torch.arange(R), row_counts)
    lab_c = torch.repeat_interleave(torch.arange(C), col_counts)
    want = keep[lab_r][:, lab_c].to(torch.int32)
    prob = ranges.build_problem(keep, row_counts, lay, variant=ranges.TC)
    assert prob.variant == ranges.TC and prob.seg.device.type == "cpu" and prob.pieces.device.type == "cpu"
    assert torch.equal(_blocks_mask(prob, n_rows, n_cols), want)
    seg, pieces = prob.seg, prob.pieces
    assert seg.dtype == torch.int32 and pieces.dtype == torch.int32
    assert bool((seg[:, 0] % 128 == 0).all()) and bool((pieces % 128 == 0).all())
    assert sorted((seg[:, 0] // 128).tolist()) == list(range(prob.row_layout.n_slots // 128))
    assert int(seg[:, 1].min()) >= 1 and int(seg[:, 1].max()) <= 128
    widths = torch.tensor([int(pieces[pb:pe, 1].sum()) for _, _, pb, pe in seg.tolist()])
    assert bool((widths[:-1] >= widths[1:]).all())  # heaviest segments first
    assert abs(prob.density - want.double().mean().item()) < 1e-12
    # padded (computed) pairs: whole 128 x 128 tiles of the kept blocks
    tiles = (row_counts + 127) // 128 * 128
    ctiles = (col_counts + 127) // 128 * 128
    computed = (keep.double() * tiles.double()[:, None] * ctiles.double()[None, :]).sum() / (n_rows * n_cols)
    assert abs(prob.computed - computed.item()) < 1e-9 and prob.computed >= prob.density
    # the library accepts the descriptors as they are
    nb = L.b200ot_blocks_scratch_bytes(n_rows, prob.row_layout.n_slots, lay.n_slots,
                                       ctypes.c_void_p(seg.data_ptr()), prob.n_seg,
                                       ctypes.c_void_p(pieces.data_ptr()), 16)
    assert nb > 0
    # one family per problem
    with pytest.raises(ValueError):
        ranges._check_path(prob, 8)
    with pytest.raises(ValueError):
        ranges._check_path(prob, 65)
    ranges._check_path(prob, 9)
    old = ranges.build_problem(keep, row_counts, ranges.ColumnLayout(col_counts), variant=ranges.SMALL)
    ranges._check_path(old, 8)
    with pytest.raises(ValueError):
        ranges._check_path(old, 16)
    with pytest.raises(ValueError):  # a tensor-core problem needs the 128-slot column layout
        ranges.build_problem(keep, row_counts, ranges.ColumnLayout(col_counts), variant=ranges.TC)

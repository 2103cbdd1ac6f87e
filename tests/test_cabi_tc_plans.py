"""Exact scratch sizes of the tensor-core plans (CPU only): the dense, batched and block-sparse size queries must keep
their answers, since callers allocate from them and the kernels carve the same scratch.  $B200OT_FORCE_SPLITS fixes the
column splits, so that the sizes do not depend on the SM count.  Each table maps the query's arguments to its answer at
1 and at 3 forced splits."""
import ctypes

import numpy as np
import pytest

from geomloss_b200 import _build, _lib

# (N, M, D)
SOFTMIN = {
    (1, 1, 9): (25600, 25600),
    (130, 700, 9): (107008, 117248),
    (1000, 4000, 9): (548352, 628224),
    (5000, 300, 9): (730368, 1130240),
    (1, 1, 16): (25600, 25600),
    (130, 700, 16): (110592, 128256),
    (1000, 4000, 16): (576256, 712192),
    (5000, 300, 16): (870400, 1550336),
    (1, 1, 33): (58368, 58368),
    (130, 700, 33): (250624, 285952),
    (1000, 4000, 33): (1299712, 1571584),
    (5000, 300, 33): (1914880, 3274752),
    (1, 1, 64): (75008, 75008),
    (130, 700, 64): (332288, 399872),
    (1000, 4000, 64): (1751296, 2271232),
    (5000, 300, 64): (2887168, 5487104),
}
CONV = {
    (1, 1, 9): (25600, 25600),
    (130, 700, 9): (107008, 117248),
    (1000, 4000, 9): (548352, 628224),
    (5000, 300, 9): (730368, 1130240),
    (1, 1, 16): (25600, 25600),
    (130, 700, 16): (110592, 128256),
    (1000, 4000, 16): (576256, 712192),
    (5000, 300, 16): (870400, 1550336),
    (1, 1, 33): (58368, 58368),
    (130, 700, 33): (250624, 285952),
    (1000, 4000, 33): (1299712, 1571584),
    (5000, 300, 33): (1914880, 3274752),
    (1, 1, 64): (75008, 75008),
    (130, 700, 64): (332288, 399872),
    (1000, 4000, 64): (1751296, 2271232),
    (5000, 300, 64): (2887168, 5487104),
}
# (B, N, M, D)
BATCHED = {
    (1, 1, 1, 9): (25600, 25600),
    (1, 130, 700, 9): (107008, 117248),
    (1, 1000, 4000, 9): (548352, 628224),
    (3, 1, 1, 9): (75776, 75776),
    (3, 130, 700, 9): (320000, 351232),
    (3, 1000, 4000, 9): (1644032, 1884160),
    (64, 1, 1, 9): (1608704, 1608704),
    (64, 130, 700, 9): (6821376, 7486976),
    (64, 1000, 4000, 9): (35066368, 40186368),
    (1, 1, 1, 16): (25600, 25600),
    (1, 130, 700, 16): (110592, 128256),
    (1, 1000, 4000, 16): (576256, 712192),
    (3, 1, 1, 16): (75776, 75776),
    (3, 130, 700, 16): (331008, 384000),
    (3, 1000, 4000, 16): (1728000, 2136064),
    (64, 1, 1, 16): (1610496, 1610496),
    (64, 130, 700, 16): (7054336, 8185856),
    (64, 1000, 4000, 16): (36858368, 45562368),
    (1, 1, 1, 33): (58368, 58368),
    (1, 130, 700, 33): (250624, 285952),
    (1, 1000, 4000, 33): (1299712, 1571584),
    (3, 1, 1, 33): (174336, 174336),
    (3, 130, 700, 33): (750848, 856832),
    (3, 1000, 4000, 33): (3898112, 4714240),
    (64, 1, 1, 33): (3712000, 3712000),
    (64, 130, 700, 33): (16008704, 18271744),
    (64, 1000, 4000, 33): (83153408, 100561408),
    (1, 1, 1, 64): (75008, 75008),
    (1, 130, 700, 64): (332288, 399872),
    (1, 1000, 4000, 64): (1751296, 2271232),
    (3, 1, 1, 64): (224000, 224000),
    (3, 130, 700, 64): (995840, 1198592),
    (3, 1000, 4000, 64): (5253120, 6813184),
    (64, 1, 1, 64): (4768512, 4768512),
    (64, 130, 700, 64): (21234688, 25561088),
    (64, 1000, 4000, 64): (112060928, 145340928),
}
# descriptor sets: rows, row slots, column slots, segments (row_start, row_count, piece_begin, piece_end), pieces
# (col_start, col_count)
DESCRIPTORS = {
    # two row clusters (1 and 129 rows), two column clusters (128 and 1 columns)
    "two_by_two": (130, 384, 256, [[128, 128, 1, 2], [256, 1, 1, 2], [0, 1, 0, 1]], [[0, 128], [0, 256]]),
    # no segment keeps a piece
    "no_pieces": (130, 384, 256, [[128, 128, 0, 0], [256, 1, 0, 0], [0, 1, 0, 0]], [[0, 128]]),
    # a segment with no piece, and piece 1 shared by segments 0 and 2
    "one_empty": (300, 384, 1280, [[0, 100, 0, 2], [128, 128, 2, 2], [256, 72, 1, 3]],
                  [[0, 512], [512, 640], [1152, 128]]),
    # eight segments over one 32-tile piece
    "long": (1000, 1024, 4096, [[s * 128, 128, 0, 1] for s in range(8)], [[0, 4096]]),
}
# (descriptor set, D)
BLOCKS = {
    ("two_by_two", 9): (68352, 73472),
    ("no_pieces", 9): (68352, 68352),
    ("one_empty", 9): (177408, 201472),
    ("long", 9): (548608, 628480),
    ("two_by_two", 16): (71936, 80896),
    ("no_pieces", 16): (71936, 71936),
    ("one_empty", 16): (185856, 226816),
    ("long", 16): (576512, 712448),
    ("two_by_two", 33): (162816, 180480),
    ("no_pieces", 33): (162816, 162816),
    ("one_empty", 33): (419328, 500992),
    ("long", 33): (1299968, 1571840),
    ("two_by_two", 64): (219904, 253696),
    ("no_pieces", 64): (219904, 219904),
    ("one_empty", 64): (562944, 719104),
    ("long", 64): (1751552, 2271488),
}


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _host(rows, width):
    """ctypes pointer to an int32 (len(rows), width) copy of `rows`, 64-byte aligned (kept alive by the caller)."""
    a = np.asarray(rows, dtype=np.int32).reshape(-1, width)
    raw = np.zeros(a.size * 4 + 64, dtype=np.uint8)
    start = (-raw.ctypes.data) % 64
    view = raw[start:start + a.size * 4].view(np.int32)
    view[:] = a.ravel()
    return raw, ctypes.c_void_p(view.ctypes.data)


@pytest.mark.parametrize("column", [0, 1], ids=["1_split", "3_splits"])
def test_dense_and_batched_plans(L, monkeypatch, column):
    monkeypatch.setenv("B200OT_FORCE_SPLITS", "13"[column])
    for (N, M, D), want in SOFTMIN.items():
        assert L.b200ot_softmin_scratch_bytes(N, M, D) == want[column], (N, M, D)
    for (N, M, D), want in CONV.items():
        assert L.b200ot_kernel_conv_scratch_bytes(N, M, D) == want[column], (N, M, D)
    for (B, N, M, D), want in BATCHED.items():
        assert L.b200ot_batched_scratch_bytes(B, N, M, D) == want[column], (B, N, M, D)


@pytest.mark.parametrize("column", [0, 1], ids=["1_split", "3_splits"])
def test_blocks_plans(L, monkeypatch, column):
    monkeypatch.setenv("B200OT_FORCE_SPLITS", "13"[column])
    for (name, D), want in BLOCKS.items():
        N, row_slots, col_slots, seg, pieces = DESCRIPTORS[name]
        _ks, sp = _host(seg, 4)
        _kp, pp = _host(pieces, 2)
        assert L.b200ot_blocks_scratch_bytes(N, row_slots, col_slots, sp, len(seg), pp, D) == want[column], (name, D)

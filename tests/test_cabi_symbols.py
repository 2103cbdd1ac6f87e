"""CPU-only checks of the C-ABI library: it loads, exports every symbol include/b200ot.h declares, and its
argument validation (which runs before any CUDA call) returns the documented error codes."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from geomloss_b200 import _build, _lib


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _declared():
    text = open(os.path.join(ROOT, "include", "b200ot.h")).read()
    return sorted(set(re.findall(r"B200OT_API\s+[\w\s\*]+?\b(b200ot_\w+)\s*\(", text)))


def test_header_and_binding_agree():
    assert _declared() == _lib.exported_symbols()


def test_every_declared_symbol_is_exported(L):
    for name in _declared():
        assert hasattr(L, name), name


def test_version_and_strerror(L):
    assert L.b200ot_version() == 202
    assert L.b200ot_strerror(0) == b"ok"
    assert b"invalid" in L.b200ot_strerror(-1)
    assert b"scratch" in L.b200ot_strerror(-2)
    assert b"unknown" in L.b200ot_strerror(-99)


def test_size_queries_are_pure(L):
    # pack padding: 1024 columns; D=3 softmin packets are 8 floats per column pair
    assert L.b200ot_packed_cols_floats(1000, 3, 1) == 1024 // 2 * 8
    assert L.b200ot_packed_cols_floats(1025, 3, 1) == 2048 // 2 * 8
    assert L.b200ot_packed_cols_floats(1000, 3, 2) == 1024 // 2 * 12
    assert L.b200ot_packed_cols_floats(1000, 1, 1) == 1024 // 2 * 4
    assert L.b200ot_packed_cols_floats(0, 3, 1) == 0
    n = L.b200ot_softmin_num_splits(10**6, 10**6, 3)
    assert 1 <= n <= 64
    assert L.b200ot_softmin_scratch_bytes(10**6, 10**6, 3) >= L.b200ot_packed_cols_floats(10**6, 3, 1) * 4
    assert L.b200ot_softmin_scratch_bytes(0, 5, 3) == 0


def test_argument_validation_needs_no_gpu(L):
    null = ctypes.c_void_p(None)
    fake = ctypes.c_void_p(0x1000)
    # null pointers / bad sizes / bad p / bad eps -> EINVAL, before any CUDA call
    assert L.b200ot_softmin_fwd(null, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, 2, 0.1,
                                fake, 1 << 30, null) == -1
    assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, 3, 0.1,
                                fake, 1 << 30, null) == -1
    assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, 2, -1.0,
                                fake, 1 << 30, null) == -1
    assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 99, 2, 0.1,
                                fake, 1 << 30, null) == -1
    # scratch too small -> ESCRATCH; misaligned scratch -> EALIGN
    assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, 2, 0.1,
                                fake, 16, null) == -2
    assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, 2, 0.1,
                                ctypes.c_void_p(0x1004), 1 << 30, null) == -4
    assert L.b200ot_kernel_conv_fwd(fake, fake, fake, null, fake, 10, 10, 3, 7, 0.1, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_fwd(fake, fake, fake, null, fake, 10, 10, 3, 0, 0.0, fake, 1 << 30, null) == -1
    assert L.b200ot_softmin_finalize(null, 1, null, 0.0, 1.0, fake, null, 10, 0.1, null) == -1
    assert L.b200ot_softmin_merge(fake, 0, fake, 10, null) == -1


def test_routing_below_nine_dimensions_shows_in_the_scratch_size(L, monkeypatch):
    """D <= 8: large forward problems take the tensor-core path from D = 7 (softmin) / D = 5 (gaussian)
    (csrc/b200ot_tc.cu: tc_routed); the size queries then cover both paths.  $B200OT_TC_MIN_D /
    $B200OT_TC_MIN_PAIRS are read on every call.  (Observed on a small shape with the size threshold lifted: there the
    tensor-core images are the larger of the two needs.)"""
    def sizes():
        return {d: (L.b200ot_softmin_scratch_bytes(1000, 1000, d), L.b200ot_kernel_conv_scratch_bytes(1000, 1000, d))
                for d in range(1, 9)}

    monkeypatch.delenv("B200OT_TC_MIN_D", raising=False)
    monkeypatch.delenv("B200OT_TC_MIN_PAIRS", raising=False)
    default = sizes()  # 1e6 pairs: below the 8e8-pair threshold, never routed
    monkeypatch.setenv("B200OT_TC_MIN_D", "9")
    assert sizes() == default
    monkeypatch.setenv("B200OT_TC_MIN_PAIRS", "0")
    cuda_core = sizes()
    assert cuda_core == default
    monkeypatch.delenv("B200OT_TC_MIN_D")
    routed = sizes()  # default dimension thresholds, any size
    for d in range(1, 5):
        assert routed[d] == cuda_core[d], d  # no operator of these dimensions leaves the CUDA cores
    for d in range(5, 9):
        assert routed[d][0] > cuda_core[d][0] and routed[d][1] > cuda_core[d][1], d  # one size for all operators of a shape
    monkeypatch.setenv("B200OT_TC_MIN_D", "7,9,5,9")  # the defaults, spelled out
    assert sizes() == routed
    monkeypatch.setenv("B200OT_TC_MIN_D", "1")
    assert all(sizes()[d][0] > cuda_core[d][0] for d in range(1, 9))
    monkeypatch.setenv("B200OT_TC_MIN_D", "7,9,9,9")  # only the forward softmin, only D >= 7
    assert sizes()[6] == cuda_core[6] and sizes()[7][0] > cuda_core[7][0]
    # a big problem is never sized below what either path needs; above B200OT_MAX_D nothing is configurable
    monkeypatch.delenv("B200OT_TC_MIN_D")
    monkeypatch.delenv("B200OT_TC_MIN_PAIRS")
    n = 100_000
    big = L.b200ot_softmin_scratch_bytes(n, n, 8)
    monkeypatch.setenv("B200OT_TC_MIN_D", "9")
    assert big >= L.b200ot_softmin_scratch_bytes(n, n, 8)
    assert L.b200ot_softmin_scratch_bytes(n, n, 16) > 0 and L.b200ot_softmin_scratch_bytes(n, n, 65) == 0


def test_forced_column_splits_reach_both_plans(L, monkeypatch):
    """$B200OT_FORCE_SPLITS (csrc/plan.cuh) is read on every call and sets the column splits of the tensor-core plan
    (make_tc_plan) as well as the dense one, so that the streaming tests (test_gpu_tc_streaming.py) really stream
    many column tiles through one CTA.  It shows in the scratch size: the row-gradient partials take
    n_split * N * (D+1) * 4 bytes, the larger need of the shape.  Splits cover ceil(13 / ceil(13 / k)) tiles each."""
    n, m, d = 256, 128 * 13 - 37, 64  # 2 row tiles, 13 column tiles; N (D+1) 4 is a multiple of the 256-byte grain
    per_split = n * (d + 1) * 4
    monkeypatch.delenv("B200OT_FORCE_SPLITS", raising=False)
    default = (L.b200ot_softmin_scratch_bytes(n, m, d), L.b200ot_kernel_conv_scratch_bytes(n, m, d))
    sizes = {}
    for k in (1, 2, 3, 13, 99):
        monkeypatch.setenv("B200OT_FORCE_SPLITS", str(k))
        sizes[k] = (L.b200ot_softmin_scratch_bytes(n, m, d), L.b200ot_kernel_conv_scratch_bytes(n, m, d))
    for k, n_split in ((2, 2), (3, 3), (13, 13), (99, 13)):  # 7+6, 5+5+3, one tile each, never more than the tiles
        assert sizes[k][0] - sizes[1][0] == (n_split - 1) * per_split, (k, sizes)
        assert sizes[k][1] - sizes[1][1] == (n_split - 1) * per_split, (k, sizes)
    # default: ceil(4 SMs / 2 row tiles) splits, capped at one per column tile
    assert default == sizes[13]
    # the dense plan of the CUDA-core kernels follows the same variable, re-read on every call
    ntiles = -(-10**5 // 1024)
    for k in (1, 5, 7):
        monkeypatch.setenv("B200OT_FORCE_SPLITS", str(k))
        assert L.b200ot_softmin_num_splits(10**5, 10**5, 3) == -(-ntiles // -(-ntiles // k))
    monkeypatch.delenv("B200OT_FORCE_SPLITS")
    assert L.b200ot_softmin_scratch_bytes(n, m, d) == default[0]


def test_one_pass_value_and_gradient_entry_validates_its_arguments(L):
    null, fake = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
    args = (10, 10, 3)
    # gaussian only; out and grad_unit are both required
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, fake, *args, 1, 0.1, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, null, fake, *args, 0, 0.1, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, null, *args, 0, 0.1, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, fake, *args, 0, 0.0, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, fake, *args, 0, 0.1, fake, 16, null) == -2
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, fake, 10, 10, 65, 0, 0.1, fake, 1 << 30, null) == -1


def test_product_requires_cuda_tensors():
    """The host wrappers refuse CPU tensors instead of falling back to a CPU implementation."""
    import torch

    from geomloss_b200 import SamplesLoss

    x = torch.rand(10, 3)
    y = torch.rand(12, 3)
    with pytest.raises(_lib.B200OTError):
        SamplesLoss("sinkhorn")(x, y)
    with pytest.raises(_lib.B200OTError):
        SamplesLoss("gaussian")(x, y)


def test_scratch_plans_cover_every_shape(L):
    """Host-side launch plans (no GPU work): scratch sizes are positive, 256-byte granular, monotone in the cloud
    sizes, and large enough for the packed columns plus one set of partials, across the CUDA-core dimensions, the
    tensor-core dimensions (8 < D <= 64: operand images, padded to two row tiles) and extreme shapes."""
    shapes = [(1, 1), (1, 5000), (5000, 1), (129, 65), (10**4, 10**4), (10**6, 10**6), (10**7, 3 * 10**6)]
    for D in (1, 3, 8, 9, 16, 33, 64):
        prev = 0
        for N, M in shapes:
            sb = L.b200ot_softmin_scratch_bytes(N, M, D)
            kb = L.b200ot_kernel_conv_scratch_bytes(N, M, D)
            assert sb > 0 and kb > 0 and sb % 256 == 0 and kb % 256 == 0, (N, M, D, sb, kb)
            if D <= 8:
                assert sb >= L.b200ot_packed_cols_floats(M, D, 1) * 4 + N * 8
                assert kb >= L.b200ot_packed_cols_floats(M, D, 2) * 4 + N * 4
                ns = L.b200ot_softmin_num_splits(N, M, D)
                assert 1 <= ns <= max(1, -(-M // 256)), (N, M, D, ns)
            else:
                # operand images: 2 fp16 terms + a 16-wide rank-one chunk per point, 128-point tiles
                dk = -(-D // 16) * 16
                assert sb >= (N + M) * (2 * dk + 16) * 2, (N, M, D, sb)
        assert L.b200ot_softmin_scratch_bytes(10**6, 10**6, D) >= L.b200ot_softmin_scratch_bytes(10**5, 10**5, D)
    assert L.b200ot_softmin_scratch_bytes(10, 10, 65) == 0 or L.b200ot_softmin_scratch_bytes(10, 10, 65) > 0  # no crash
    for variant, rows, cols in ((0, 512, 1024), (1, 128, 256)):
        r, c, al = ctypes.c_int32(0), ctypes.c_int32(0), ctypes.c_int32(0)
        L.b200ot_ranges_shape(variant, ctypes.byref(r), ctypes.byref(c), ctypes.byref(al))
        assert (r.value, c.value) == (rows, cols) and al.value == 16 and c.value % al.value == 0


def test_ranges_and_flag_validation_needs_no_gpu(L):
    null = ctypes.c_void_p(None)
    fake = ctypes.c_void_p(0x1000)
    # p = 1 | UNCLAMPED and p = 2 | UNCLAMPED are legal, other flag bits are not
    for p, rc in ((0x101, -2), (0x102, -2), (0x201, -1), (0x103, -1)):
        assert L.b200ot_softmin_fwd(fake, fake, fake, null, 0.0, null, null, 0.0, 1.0, fake, null, 10, 10, 3, p, 0.1,
                                    fake, 16, null) == rc
    for kind, rc in ((0x101, -2), (0x102, -2), (0x103, -1), (0x201, -1)):
        assert L.b200ot_kernel_conv_fwd(fake, fake, fake, null, fake, 10, 10, 3, kind, 0.1, fake, 16, null) == rc
    # ranges entry points: null descriptors, bad variant, misaligned segment array
    assert L.b200ot_softmin_partial_ranges(fake, null, fake, null, 1, fake, fake, 10, 3, 2, 0.1, 0, null) == -1
    assert L.b200ot_softmin_partial_ranges(fake, null, fake, fake, 1, fake, fake, 10, 3, 2, 0.1, 2, null) == -1
    assert L.b200ot_softmin_partial_ranges(fake, null, fake, ctypes.c_void_p(0x1008), 1, fake, fake, 10, 3, 2, 0.1, 0,
                                           null) == -4
    assert L.b200ot_softmin_bwd_partial_ranges(fake, null, fake, fake, fake, 0, fake, fake, 10, 3, 2, 0.1, 0,
                                               null) == -1
    assert L.b200ot_kernel_conv_partial_ranges(fake, null, fake, fake, 1, fake, fake, 10, 3, 9, 0.1, 0, 0, null) == -1
    assert L.b200ot_softmin_pack_gather(fake, fake, null, 0.0, null, null, 10, 3, 2, 0.1, fake, null) == -1
    assert L.b200ot_softmin_bwd_sums(fake, fake, fake, null, 0.0, null, fake, null, 10, 10, 3, 2, 0.1, fake, 1 << 30,
                                     null) == -1

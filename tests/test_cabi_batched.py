"""CPU-only argument validation of the batched tensor-core entry points (b200ot_*_batched, 8 < D <= 64): the symbols
exist, every bad argument is refused with -1 before any CUDA call, a too-small scratch with -2, and the batched scratch
query is consistent with the one-problem one.  Nothing here reaches a CUDA call (the fake pointers are never
dereferenced)."""
import ctypes

import pytest

from geomloss_b200 import _build, _lib

BATCHED = ["b200ot_batched_scratch_bytes", "b200ot_softmin_fwd_batched", "b200ot_softmin_bwd_x_batched",
           "b200ot_kernel_conv_fwd_batched", "b200ot_kernel_conv_bwd_x_batched", "b200ot_kernel_conv_fwd_bwd_x_batched"]
NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _softmin_fwd(L, B=3, N=10, M=12, D=16, p=2, eps=0.1, x=FAKE, y=FAKE, h=FAKE, out=FAKE, lse2=NULL, scratch=FAKE,
                 nbytes=BIG):
    return L.b200ot_softmin_fwd_batched(x, y, h, NULL, 0.0, NULL, NULL, 0.0, 1.0, out, lse2, B, N, M, D, p, eps,
                                        scratch, nbytes, NULL)


def _softmin_bwd(L, B=3, N=10, M=12, D=16, p=2, eps=0.1, x=FAKE, y=FAKE, h=FAKE, lse2=FAKE, go=FAKE, gx=FAKE,
                 scratch=FAKE, nbytes=BIG):
    return L.b200ot_softmin_bwd_x_batched(x, y, h, NULL, 0.0, NULL, lse2, go, gx, B, N, M, D, p, eps, scratch, nbytes,
                                          NULL)


def _conv_fwd(L, B=3, N=10, M=12, D=16, kind=0, blur=0.5, x=FAKE, y=FAKE, w=FAKE, out=FAKE, scratch=FAKE, nbytes=BIG):
    return L.b200ot_kernel_conv_fwd_batched(x, y, w, NULL, out, B, N, M, D, kind, blur, scratch, nbytes, NULL)


def _conv_bwd(L, B=3, N=10, M=12, D=16, kind=0, blur=0.5, x=FAKE, y=FAKE, w=FAKE, go=FAKE, gx=FAKE, scratch=FAKE,
              nbytes=BIG):
    return L.b200ot_kernel_conv_bwd_x_batched(x, y, w, NULL, go, gx, B, N, M, D, kind, blur, scratch, nbytes, NULL)


def _conv_fwd_bwd(L, B=3, N=10, M=12, D=16, kind=0, blur=0.5, x=FAKE, y=FAKE, w=FAKE, out=FAKE, gx=FAKE,
                  scratch=FAKE, nbytes=BIG):
    return L.b200ot_kernel_conv_fwd_bwd_x_batched(x, y, w, NULL, out, gx, B, N, M, D, kind, blur, scratch, nbytes, NULL)


CALLS = {"softmin_fwd": _softmin_fwd, "softmin_bwd": _softmin_bwd, "conv_fwd": _conv_fwd, "conv_bwd": _conv_bwd,
         "conv_fwd_bwd": _conv_fwd_bwd}
POINTERS = {"softmin_fwd": ["x", "y", "h", "scratch"], "softmin_bwd": ["x", "y", "h", "lse2", "go", "gx", "scratch"],
            "conv_fwd": ["x", "y", "w", "out", "scratch"], "conv_bwd": ["x", "y", "w", "go", "gx", "scratch"],
            "conv_fwd_bwd": ["x", "y", "w", "out", "gx", "scratch"]}


def test_symbols_exist(L):
    for name in BATCHED:
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()


@pytest.mark.parametrize("call", sorted(CALLS))
def test_bad_arguments_are_refused(L, call):
    f = CALLS[call]
    for ptr in POINTERS[call]:
        assert f(L, **{ptr: NULL}) == -1, f"{call}: null {ptr}"
    for kw in (dict(B=0), dict(B=-2), dict(N=0), dict(M=0), dict(D=8), dict(D=1), dict(D=65), dict(D=0)):
        assert f(L, **kw) == -1, f"{call}: {kw}"
    if call.startswith("softmin"):
        for kw in (dict(p=1), dict(p=1 | 0x100), dict(p=3), dict(eps=0.0), dict(eps=-1.0)):
            assert f(L, **kw) == -1, f"{call}: {kw}"
    else:
        for kw in (dict(kind=3), dict(kind=0x200), dict(blur=0.0), dict(kind=1, blur=-1.0)):
            assert f(L, **kw) == -1, f"{call}: {kw}"
    if call == "softmin_fwd":
        assert f(L, out=NULL) == -1  # neither out nor lse2
    if call == "conv_fwd_bwd":
        for kind in (1, 2, 1 | 0x100):  # the one-pass value + gradient is gaussian-only
            assert f(L, kind=kind) == -1
    # misaligned scratch
    assert f(L, scratch=ctypes.c_void_p(0x1004)) == -4


@pytest.mark.parametrize("call", sorted(CALLS))
def test_small_scratch(L, call):
    f = CALLS[call]
    for B, N, M, D in ((3, 10, 12, 16), (1, 300, 200, 9), (17, 129, 1000, 64)):
        need = L.b200ot_batched_scratch_bytes(B, N, M, D)
        assert need > 0
        assert f(L, B=B, N=N, M=M, D=D, nbytes=need - 1) == -2
        assert f(L, B=B, N=N, M=M, D=D, nbytes=16) == -2
    # the energy distance ignores blur
    if call.startswith("conv") and call != "conv_fwd_bwd":
        assert f(L, kind=2, blur=0.0, nbytes=16) == -2


def test_scratch_query(L):
    for bad in ((0, 10, 10, 16), (2, 0, 10, 16), (2, 10, 0, 16), (2, 10, 10, 8), (2, 10, 10, 65)):
        assert L.b200ot_batched_scratch_bytes(*bad) == 0, bad
    for N, M, D in ((10, 12, 16), (300, 1000, 9), (129, 4097, 64), (100000, 100000, 33)):
        one = L.b200ot_batched_scratch_bytes(1, N, M, D)
        assert one >= L.b200ot_softmin_scratch_bytes(N, M, D)
        assert one >= L.b200ot_kernel_conv_scratch_bytes(N, M, D)
        # every element is padded to whole tiles on its own: B elements need at least B times the tile images
        assert L.b200ot_batched_scratch_bytes(5, N, M, D) >= 5 * (one - (1 << 16))

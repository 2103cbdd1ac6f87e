"""CPU-only argument validation of the p = 1 softmin entry points in the tensor-core dimensions (b200ot_softmin_l1_*,
8 < D <= 64): the symbols exist, every bad argument is refused with -1 before any CUDA call, a misaligned scratch with
-4, a too-small scratch with -2, and the scratch query is consistent.  Nothing here reaches a CUDA call (the fake
pointers are never dereferenced)."""
import ctypes

import pytest

from geomloss_b200 import _build, _lib

L1 = ["b200ot_softmin_l1_scratch_bytes", "b200ot_softmin_l1_fwd", "b200ot_softmin_l1_bwd_x"]
NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
UNCLAMPED = 0x100


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _fwd(L, B=3, N=10, M=12, D=16, p=1, eps=0.1, x=FAKE, y=FAKE, h=FAKE, out=FAKE, lse2=NULL, scratch=FAKE,
         nbytes=BIG):
    return L.b200ot_softmin_l1_fwd(x, y, h, NULL, 0.0, NULL, NULL, 0.0, 1.0, out, lse2, B, N, M, D, p, eps, scratch,
                                   nbytes, NULL)


def _bwd(L, B=3, N=10, M=12, D=16, p=1, eps=0.1, x=FAKE, y=FAKE, h=FAKE, lse2=FAKE, go=FAKE, gx=FAKE, scratch=FAKE,
         nbytes=BIG):
    return L.b200ot_softmin_l1_bwd_x(x, y, h, NULL, 0.0, NULL, lse2, go, gx, B, N, M, D, p, eps, scratch, nbytes, NULL)


CALLS = {"fwd": _fwd, "bwd": _bwd}
POINTERS = {"fwd": ["x", "y", "h", "scratch"], "bwd": ["x", "y", "h", "lse2", "go", "gx", "scratch"]}


def test_symbols_exist(L):
    for name in L1:
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()


@pytest.mark.parametrize("call", sorted(CALLS))
def test_bad_arguments_are_refused(L, call):
    f = CALLS[call]
    for ptr in POINTERS[call]:
        assert f(L, **{ptr: NULL}) == -1, f"{call}: null {ptr}"
    for kw in (dict(B=0), dict(B=-2), dict(N=0), dict(N=-1), dict(M=0), dict(D=0), dict(D=8), dict(D=1),
               dict(D=65)):
        assert f(L, **kw) == -1, f"{call}: {kw}"
    for kw in (dict(p=2), dict(p=2 | UNCLAMPED), dict(p=3), dict(p=0), dict(p=0x201), dict(p=1 | 0x200),
               dict(eps=0.0), dict(eps=-1.0), dict(eps=float("nan"))):
        assert f(L, **kw) == -1, f"{call}: {kw}"
    if call == "fwd":
        assert f(L, out=NULL) == -1  # neither out nor lse2
    for p in (1, 1 | UNCLAMPED):  # both conventions pass validation: a misaligned scratch is the first refusal
        assert f(L, p=p, scratch=ctypes.c_void_p(0x1004)) == -4
        assert f(L, p=p, scratch=ctypes.c_void_p(0x1008)) == -4


@pytest.mark.parametrize("call", sorted(CALLS))
def test_small_scratch(L, call):
    f = CALLS[call]
    for B, N, M, D in ((3, 10, 12, 16), (1, 300, 200, 9), (17, 129, 1000, 64), (2, 5000, 7000, 33)):
        need = L.b200ot_softmin_l1_scratch_bytes(B, N, M, D)
        assert need > 0
        for p in (1, 1 | UNCLAMPED):
            assert f(L, B=B, N=N, M=M, D=D, p=p, nbytes=need - 1) == -2
            assert f(L, B=B, N=N, M=M, D=D, p=p, nbytes=16) == -2


def test_scratch_query(L):
    for bad in ((0, 10, 10, 16), (-1, 10, 10, 16), (2, 0, 10, 16), (2, 10, 0, 16), (2, 10, 10, 8), (2, 10, 10, 0),
                (2, 10, 10, 65)):
        assert L.b200ot_softmin_l1_scratch_bytes(*bad) == 0, bad
    for N, M, D in ((10, 12, 16), (300, 1000, 9), (129, 4097, 64), (100000, 100000, 33), (500, 500, 48)):
        sizes = [L.b200ot_softmin_l1_scratch_bytes(B, N, M, D) for B in (1, 2, 3, 5, 8, 64, 65)]
        assert all(s > 0 for s in sizes)
        assert sizes == sorted(sizes), (N, M, D, sizes)
        # the row gradient keeps one more sum per row than the p = 2 one: never less scratch than the batched entries
        assert sizes[0] >= L.b200ot_batched_scratch_bytes(1, N, M, D)
        assert sizes[-1] >= L.b200ot_batched_scratch_bytes(65, N, M, D)

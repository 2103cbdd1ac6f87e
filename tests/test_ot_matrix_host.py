"""CPU checks of ``ot.solve`` / ``ot.solve_batch`` and of the dense-matrix C entries: argument errors and their
messages (those of the reference, ot/_implementations/matrix.py and _arguments.py), ``TypeError`` for inputs that
are not float32 CUDA tensors once every argument check has passed, -1 from the C entries for null pointers and
non-positive sizes before any CUDA call, and a scratch query that is a pure function of the shape.  The fake
pointers are never dereferenced."""
import ctypes
import os
import re

import pytest
import torch

from geomloss_b200 import _build, _lib, ops, ot

NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ot.h")
NEW = ["b200ot_dense_scratch_bytes", "b200ot_dense_softmin_pair", "b200ot_dense_softmin_pair_bwd"]


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def C23():
    return torch.tensor([[0.0, 1.0, 4.0], [2.0, 1.0, 0.0]])


def test_exports():
    assert {"solve", "solve_batch", "OTResultMatrix"} <= set(ot.__all__)
    assert "barycenter" not in ot.__all__ and not hasattr(ot, "barycenter")


def test_symbols_in_header_and_binding(L):
    header = open(HEADER).read()
    for name in NEW:
        assert re.search(rf"\b{name}\(", header), name
        assert name in _lib.exported_symbols()
        getattr(L, name)
    assert L.b200ot_version() == 202


@pytest.mark.parametrize("shape", [(3,), (2, 3, 4, 5)])
def test_solve_rank(shape):
    with pytest.raises(ValueError, match=re.escape("The 'cost' matrix should be an array with 2 dimensions. "
                                                   "Instead, ot.solve received an array of shape")):
        ot.solve(torch.zeros(shape), reg=0.1, max_iter=5)


@pytest.mark.parametrize("shape", [(3, 4), (1, 2, 3, 4)])
def test_solve_batch_rank(shape):
    with pytest.raises(ValueError, match=re.escape("The 'cost' matrix should be an array with 3 dimensions (batch, "
                                                   "N, M). Instead, ot.solve received an array of shape")):
        ot.solve_batch(torch.zeros(shape), reg=0.1, max_iter=5)


@pytest.mark.parametrize("solver, C", [(ot.solve, C23()), (ot.solve_batch, C23()[None])])
def test_regularization_errors(solver, C):
    with pytest.raises(TypeError):
        solver(C, reg=None, max_iter=5)
    with pytest.raises(NotImplementedError, match="reg > 0"):
        solver(C, reg=0.0, max_iter=5)
    with pytest.raises(ValueError, match="Parameter 'reg' should be >= 0. Received -1"):
        solver(C, reg=-1.0, max_iter=5)
    with pytest.raises(ValueError, match="Parameter 'unbalanced' should be None"):
        solver(C, reg=0.1, unbalanced=-1.0, max_iter=5)
    with pytest.raises(NotImplementedError, match="rigorous stopping criteria"):
        solver(C, reg=0.1, max_iter=5, tol=1e-3)
    with pytest.raises(NotImplementedError, match="single method"):
        solver(C, reg=0.1, max_iter=5, method="sinkhorn")
    with pytest.raises(NotImplementedError, match="'KL' penalty"):
        solver(C, reg=0.1, max_iter=5, unbalanced=1.0, unbalanced_type="TV")
    with pytest.raises(ValueError, match="max_iter"):
        solver(C, reg=0.1)


def test_marginal_errors():
    C = C23()
    with pytest.raises(ValueError, match=re.escape("The marginal 'a' contains negative values. We require that a >= 0.")):
        ot.solve(C, reg=0.1, a=torch.tensor([-1.0, 2.0]), max_iter=5)
    with pytest.raises(ValueError, match=re.escape("The marginal 'b' should be of shape")):
        ot.solve(C, reg=0.1, b=torch.ones(4) / 4, max_iter=5)
    with pytest.raises(ValueError, match="do not sum up to the same value"):
        ot.solve(C, reg=0.1, a=torch.tensor([2.0, 2.0]), b=torch.tensor([1.0, 1.0, 1.0]), max_iter=5)
    with pytest.raises(ValueError, match="have rows that do not sum up to the same values"):
        ot.solve_batch(torch.stack([C, C]), reg=0.1, a=torch.tensor([[2.0, 2.0], [1.0, 1.0]]),
                       b=torch.tensor([[1.0, 1.0, 2.0], [1.0, 1.0, 1.0]]), max_iter=5)


def test_unequal_masses_are_fine_when_unbalanced():
    """Every argument check passes; the CPU tensor is then refused."""
    with pytest.raises(TypeError, match="float32 CUDA"):
        ot.solve(C23(), reg=0.1, a=torch.tensor([2.0, 2.0]), b=torch.tensor([1.0, 1.0, 1.0]), unbalanced=1.0,
                 max_iter=5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cpu_or_fp64_inputs_raise_type_error(dtype):
    with pytest.raises(TypeError):
        ot.solve(C23().to(dtype), reg=0.1, max_iter=5)
    with pytest.raises(TypeError):
        ot.solve_batch(C23()[None].to(dtype), reg=0.1, max_iter=5)
    with pytest.raises(TypeError):
        ot.solve([[0.0, 1.0], [1.0, 0.0]], reg=0.1, max_iter=5)


def test_ops_shape_checks_before_device():
    C = torch.zeros(2, 3)
    with pytest.raises(ValueError, match="one entry per row"):
        ops.dense_softmin_pair_raw(0.1, C, torch.zeros(3), torch.zeros(3), torch.zeros(2), torch.zeros(3))
    with pytest.raises(ValueError, match="one entry per column"):
        ops.dense_softmin_pair_grad(0.1, C, torch.zeros(2), torch.zeros(3), torch.zeros(2), torch.zeros(3),
                                    torch.zeros(2), torch.zeros(3), torch.zeros(2), torch.zeros(4))
    with pytest.raises(ValueError, match="cost matrix"):
        ops.dense_softmin_pair_raw(0.1, torch.zeros(5), torch.zeros(5), torch.zeros(5), torch.zeros(5), torch.zeros(5))
    with pytest.raises(_lib.B200OTError, match="CUDA device"):
        ops.dense_softmin_pair_raw(0.1, C, torch.zeros(2), torch.zeros(3), torch.zeros(2), torch.zeros(3))


def _pair(L, B=2, N=3, M=4, eps=0.1, inv_eps=10.0, C=FAKE, la=FAKE, lb=FAKE, f=FAKE, g=FAKE, fo=FAKE, go=FAKE,
          scratch=FAKE, nbytes=BIG):
    return L.b200ot_dense_softmin_pair(C, la, lb, f, g, inv_eps, 0.5, 0.5, fo, go, NULL, NULL, B, N, M, eps, scratch,
                                       nbytes, NULL)


def _bwd(L, B=2, N=3, M=4, inv_eps=10.0, ptrs=(FAKE,) * 10):
    C, la, lb, f, g, lr, lc, gf, gg, out = ptrs
    return L.b200ot_dense_softmin_pair_bwd(C, la, lb, f, g, inv_eps, lr, lc, gf, gg, out, B, N, M, NULL)


def test_c_entries_refuse_bad_arguments(L):
    for k in ("C", "la", "lb", "f", "g", "fo", "go", "scratch"):
        assert _pair(L, **{k: NULL}) == -1, k
    for k in ("B", "N", "M"):
        assert _pair(L, **{k: 0}) == -1, k
        assert _pair(L, **{k: -3}) == -1, k
    assert _pair(L, eps=0.0) == -1 and _pair(L, inv_eps=-1.0) == -1
    assert _pair(L, scratch=ctypes.c_void_p(0x1004)) == -4
    assert _pair(L, nbytes=L.b200ot_dense_scratch_bytes(2, 3, 4) - 1) == -2
    for k in range(10):
        ptrs = [FAKE] * 10
        ptrs[k] = NULL
        assert _bwd(L, ptrs=tuple(ptrs)) == -1, k
    for k in ("B", "N", "M"):
        assert _bwd(L, **{k: 0}) == -1, k
    assert _bwd(L, inv_eps=0.0) == -1


def test_scratch_query_is_pure(L):
    q = L.b200ot_dense_scratch_bytes
    for B, N, M in ((1, 1, 1), (1, 5, 1001), (3, 129, 128), (64, 512, 512), (1, 16384, 16384), (1, 46341, 46341)):
        n = q(B, N, M)
        assert n == q(B, N, M) > 0
        # column partials: one (m, s) pair per (128-row tile, column); row partials: one per (column range, row)
        assert n >= -(-N // 128) * B * M * 8 + B * N * 8
        assert n % 256 == 0
    assert q(0, 4, 4) == q(1, 0, 4) == q(1, 4, -1) == 0
    # the share of C's bytes the partials take stays small on large problems
    assert q(1, 16384, 16384) < 0.03 * 4 * 16384 * 16384

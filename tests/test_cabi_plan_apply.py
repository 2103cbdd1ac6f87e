"""CPU-only checks of the plan-times-values operator (b200ot_plan_apply): the symbols exist and match the header, every
bad argument is refused with -1 before any CUDA call, a misaligned scratch with -4, a too-small one with -2, the
scratch query is pure and monotone in K, and the host logic of ``ot.OTResultSample`` on top of it (seen through dense
fp64 stand-ins): one operator call per application, no host synchronisation, cached lse2, barycentric maps, gradient
with respect to the values.  The fake pointers are never dereferenced."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from geomloss_b200 import _build, _lib

NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ot.h")


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _apply(L, N=10, M=12, D=3, K=5, p=2, eps=0.1, x=FAKE, y=FAKE, h_a=FAKE, h_b=NULL, center=NULL, lse2=FAKE, v=FAKE,
           row_factor=NULL, out=FAKE, scratch=FAKE, nbytes=BIG):
    return L.b200ot_plan_apply(x, y, h_a, h_b, 0.0, center, lse2, v, row_factor, out, N, M, D, K, p, eps, scratch,
                               nbytes, NULL)


def test_symbols_match_header(L):
    header = open(HEADER).read()
    for name in ("b200ot_plan_apply_scratch_bytes", "b200ot_plan_apply"):
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()
        assert re.search(rf"B200OT_API int(64_t)? {name}\(", header), name


def test_bad_arguments_are_refused(L):
    for ptr in ("x", "y", "h_a", "lse2", "v", "out", "scratch"):
        assert _apply(L, **{ptr: NULL}) == -1, ptr
    for kw in (dict(N=0), dict(N=-3), dict(M=0), dict(M=-1), dict(D=0), dict(D=65), dict(D=1024), dict(K=0),
               dict(K=-2), dict(K=1 << 31), dict(p=1), dict(p=1 | 0x100), dict(p=3), dict(p=0), dict(p=2 | 0x200),
               dict(eps=0.0), dict(eps=-1.0), dict(eps=float("nan"))):
        assert _apply(L, **kw) == -1, kw
    # accepted arguments get as far as the scratch checks: the optional pointers may be null or not, every D and K
    for kw in (dict(), dict(h_b=FAKE, center=FAKE, row_factor=FAKE), dict(D=1), dict(D=8), dict(D=9), dict(D=64),
               dict(K=1), dict(K=130), dict(p=2 | 0x100)):
        assert _apply(L, nbytes=16, **kw) == -2, kw
        assert _apply(L, scratch=ctypes.c_void_p(0x1004), **kw) == -4, kw
    need = L.b200ot_plan_apply_scratch_bytes(10, 12, 3, 5)
    assert _apply(L, nbytes=need - 1) == -2


def test_scratch_query_is_pure_and_monotone_in_k(L):
    assert L.b200ot_plan_apply_scratch_bytes(0, 5, 3, 1) == 0
    assert L.b200ot_plan_apply_scratch_bytes(5, 5, 65, 1) == 0
    assert L.b200ot_plan_apply_scratch_bytes(5, 5, 3, 0) == 0
    for N, M, D in ((1000, 1300, 3), (100_000, 70_000, 8), (5000, 4000, 16), (300_000, 200_000, 64)):
        sizes = [L.b200ot_plan_apply_scratch_bytes(N, M, D, K) for K in (1, 3, 4, 5, 8, 9, 16, 17, 64, 65, 130)]
        assert sizes[0] > 0 and sizes == sorted(sizes), (N, M, D, sizes)
        assert sizes == [L.b200ot_plan_apply_scratch_bytes(N, M, D, K) for K in (1, 3, 4, 5, 8, 9, 16, 17, 64, 65, 130)]
        # slabs re-use one value buffer and one set of partials: below D = 9 nothing grows past the widest slab
        if D <= 8:
            assert L.b200ot_plan_apply_scratch_bytes(N, M, D, 8) == L.b200ot_plan_apply_scratch_bytes(N, M, D, 80)
        assert L.b200ot_plan_apply_scratch_bytes(N, M, D, 1) >= M * 4


# ------------------------------------------------------------------------------------------------
# host logic of the result object, the two operators replaced by dense fp64 stand-ins
# ------------------------------------------------------------------------------------------------
def _h(h_a, h_b, h_scale_b):
    return h_a.double() if h_b is None else h_a.double() + h_scale_b * h_b.double()


def _cost(x, y):
    return 0.5 * torch.cdist(x.double(), y.double()) ** 2


def _dense_softmin_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                       beta=1.0, out=None, want_lse2=False):
    lse = torch.logsumexp(_h(h_a, h_b, h_scale_b)[None, :] - _cost(x, y) / eps, dim=1)
    val = -eps * lse * beta
    if out_old is not None:
        val = val + alpha_old * out_old.double()
    return val.float(), (lse / np.log(2.0)).float() if want_lse2 else None


class _Counter:
    calls = 0
    shapes = []


def _dense_plan_apply_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    _Counter.calls += 1
    _Counter.shapes.append(tuple(v.shape))
    assert lse2 is not None and lse2.shape == (x.shape[0],)
    w = torch.softmax(_h(h_a, h_b, h_scale_b)[None, :] - _cost(x, y) / eps, dim=1)
    out = w @ v.double()
    if row_factor is not None:
        out = row_factor.double()[:, None] * out
    return out.float()


@pytest.fixture
def dense_ops(monkeypatch):
    from geomloss_b200 import ops, ot

    softmins = []

    def softmin(*a, **kw):
        softmins.append(kw.get("want_lse2", False))
        return _dense_softmin_raw(*a, **kw)

    monkeypatch.setattr(ops, "softmin_raw", softmin)
    monkeypatch.setattr(ops, "plan_apply_raw", _dense_plan_apply_raw)
    monkeypatch.setattr(ot, "_fused_operator", lambda s: True)
    _Counter.calls, _Counter.shapes = 0, []
    return softmins


def _forbid_host_reads(monkeypatch):
    def forbidden(*a, **kw):
        raise AssertionError("host synchronisation inside the operator")

    for name in ("item", "any", "all", "tolist", "__bool__"):
        monkeypatch.setattr(torch.Tensor, name, forbidden)


@pytest.mark.parametrize("unbalanced", [None, 0.7])
def test_result_object_runs_on_the_operator(dense_ops, monkeypatch, unbalanced):
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(3)
    n, m, d = 23, 31, 3
    X_a, X_b = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g) + 0.2
    a = torch.rand(n, generator=g) + 0.1
    b = torch.rand(m, generator=g) + 0.1
    b[4] = 0.0  # a zero-weight column: log weight -1e5
    a, b = a / a.sum(), b / b.sum()
    res = ot.solve_sample(X_a, X_b, a=a, b=b, reg=0.05, max_iter=30, unbalanced=unbalanced)
    P = res.plan.double()
    assert _Counter.calls == 0

    V = torch.randn(m, 5, generator=g)
    n_soft = len(dense_ops)
    with monkeypatch.context() as mp:
        _forbid_host_reads(mp)
        out = res.plan_operator @ V
    assert _Counter.calls == 1 and _Counter.shapes == [(m, 5)]  # one call for five signed columns
    assert len(dense_ops) == n_soft + 1 and dense_ops[-1] is True  # one forward softmin for lse2, then cached
    assert out.shape == (n, 5)
    np.testing.assert_allclose(out.double().numpy(), (P @ V.double()).numpy(), atol=2e-6)

    with monkeypatch.context() as mp:
        _forbid_host_reads(mp)
        out2 = res.plan_operator @ torch.randn(m, 2, 4, generator=g)  # trailing dimensions, cached lse2
    assert out2.shape == (n, 2, 4) and _Counter.calls == 2 and len(dense_ops) == n_soft + 1
    # marginal_a is the cached row factor of the same direction: no further pass
    np.testing.assert_allclose(res.marginal_a.double().numpy(), P.sum(1).numpy(), atol=1e-6)
    assert len(dense_ops) == n_soft + 1
    outT = res.plan_operator.T @ torch.ones(n)
    np.testing.assert_allclose(outT.double().numpy(), P.sum(0).numpy(), atol=1e-6)
    np.testing.assert_allclose(res.marginal_b.double().numpy(), P.sum(0).numpy(), atol=1e-6)
    assert len(dense_ops) == n_soft + 2 and res.plan_operator.shape == (n, m)
    dens = res.density.double()
    np.testing.assert_allclose((res.density_operator @ V).double().numpy(), (dens @ V.double()).numpy(),
                               atol=2e-5 * float((dens @ V.double().abs()).max()))
    assert len(dense_ops) == n_soft + 3  # the unweighted direction has a softmin of its own

    # barycentric maps: (n, d) / (m, d) displacements to the conditional means, detached and cached
    ab, ba = res.a_to_b, res.b_to_a
    assert ab.shape == (n, d) and ba.shape == (m, d) and not ab.requires_grad
    ref = (P @ X_b.double()) / P.sum(1, keepdim=True) - X_a.double()
    np.testing.assert_allclose(ab.double().numpy(), ref.numpy(), atol=2e-6)
    live = b > 0  # a point without mass has no row in the transposed plan's conditional mean
    ref = (P.t() @ X_a.double()) / P.sum(0)[:, None] - X_b.double()
    np.testing.assert_allclose(ba.double().numpy()[live], ref.numpy()[live], atol=2e-6)
    assert res.a_to_b is ab and res.lazy_plan is None and res.lazy_density is None

    # cache_clear drops lse2 and the maps
    calls, n_soft = _Counter.calls, len(dense_ops)
    res.cache_clear()
    assert "_apply_cache" not in res.__dict__ and "a_to_b" not in res.__dict__
    res.plan_operator @ V
    assert _Counter.calls == calls + 1 and len(dense_ops) == n_soft + 1


def test_operator_is_differentiable_in_the_values(dense_ops):
    from geomloss_b200 import ot

    g = torch.Generator().manual_seed(5)
    n, m = 17, 12
    X_a, X_b = torch.rand(n, 2, generator=g), torch.rand(m, 2, generator=g)
    res = ot.solve_sample(X_a, X_b, reg=0.1, max_iter=10)
    P, dens = res.plan.double(), res.density.double()
    for op, mat in ((res.plan_operator, P), (res.density_operator, dens), (res.plan_operator.T, P.t())):
        V = torch.randn(mat.shape[1], 3, generator=g, requires_grad=True)
        G = torch.randn(mat.shape[0], 3, generator=g)
        out = op @ V
        assert out.requires_grad
        (gv,) = torch.autograd.grad((out * G).sum(), V)
        ref = mat.t() @ G.double()
        np.testing.assert_allclose(gv.double().numpy(), ref.numpy(), atol=1e-5 * float(ref.abs().max()))
    with torch.no_grad():
        assert not (res.plan_operator @ torch.randn(m, 2, requires_grad=True)).requires_grad

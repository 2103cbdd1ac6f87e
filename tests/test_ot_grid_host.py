"""CPU-only checks of ``ot.solve_grid`` (argument parsing and every refusal, before any kernel runs) and of the two C
entries behind it, ``b200ot_softmin_grid_axes`` and ``b200ot_grid_plan_apply``: every bad argument is refused with
B200OT_EINVAL before any CUDA call.  Every call below breaks exactly one rule, so none reaches a launch (the fake
pointers are never dereferenced; they lie far enough apart that the arrays they stand for do not overlap)."""
import ctypes
import re

import pytest
import torch

from geomloss_b200 import _build, _lib, ot

EINVAL = -1
NULL = ctypes.c_void_p(None)
H_A, H_B, OLD, OUT, V, ELL, S = (ctypes.c_void_p(k << 24) for k in range(1, 8))


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _geometry(sides, pitch, periodic):
    """Host arrays of the per-axis geometry; None stands for a null pointer."""
    return (None if sides is None else (ctypes.c_int32 * len(sides))(*sides),
            None if pitch is None else (ctypes.c_float * len(pitch))(*pitch),
            None if periodic is None else (ctypes.c_int32 * len(periodic))(*periodic))


def _softmin(L, h_a=H_A, h_b=H_B, out_old=OLD, out=OUT, batch=3, dim=2, sides=(16, 9), pitch=(0.1, 0.2),
             periodic=(0, 1), eps=0.1):
    s, p, per = _geometry(sides, pitch, periodic)
    return L.b200ot_softmin_grid_axes(h_a, h_b, 0.5, out_old, 0.5, 1.0, out, batch, dim, s, p, per, eps, NULL)


def _apply(L, h_a=H_A, h_b=H_B, v=V, ell=ELL, s=S, batch=3, K=5, dim=2, sides=(16, 9), pitch=(0.1, 0.2),
           periodic=(0, 1), eps=0.1):
    sd, p, per = _geometry(sides, pitch, periodic)
    return L.b200ot_grid_plan_apply(h_a, h_b, 0.5, v, ell, s, batch, K, dim, sd, p, per, eps, NULL)


GEOMETRY = [
    dict(batch=0), dict(batch=-1),
    dict(dim=0), dict(dim=4), dict(dim=-1),
    dict(sides=(0, 9)), dict(sides=(16, -3)), dict(sides=(1025, 9)), dict(sides=(16, 4096)),
    dict(pitch=(0.0, 0.2)), dict(pitch=(0.1, -1.0)), dict(pitch=(float("nan"), 0.2)), dict(pitch=(0.1, float("inf"))),
    dict(eps=0.0), dict(eps=-0.0), dict(eps=-1.0), dict(eps=float("nan")), dict(eps=float("inf")),
]


def _ids(cases):
    return [",".join(f"{k}={v.value if isinstance(v, ctypes.c_void_p) else v}" for k, v in kw.items()) for kw in cases]


def test_symbols_exist(L):
    for name in ("b200ot_softmin_grid_axes", "b200ot_grid_plan_apply"):
        assert hasattr(L, name) and name in _lib.exported_symbols()


SOFTMIN_CASES = GEOMETRY + [
    dict(h_a=NULL), dict(out=NULL), dict(sides=None), dict(pitch=None),
    # the passes run in place on `out`: it may not overlap an input
    dict(out=H_A), dict(out=H_B), dict(out=OLD), dict(out=ctypes.c_void_p(H_A.value + 64)),
]


@pytest.mark.parametrize("kw", SOFTMIN_CASES, ids=_ids(SOFTMIN_CASES))
def test_softmin_grid_axes_refuses(L, kw):
    assert _softmin(L, **kw) == EINVAL
    if kw.get("out") not in (H_B, OLD):
        assert _softmin(L, **dict(dict(h_b=NULL, out_old=NULL, periodic=None), **kw)) == EINVAL


APPLY_CASES = GEOMETRY + [
    dict(h_a=NULL), dict(v=NULL), dict(ell=NULL), dict(s=NULL), dict(sides=None), dict(pitch=None),
    dict(K=0), dict(K=-4),
    # outputs overlapping an input or each other
    dict(ell=H_A), dict(ell=H_B), dict(ell=V), dict(s=H_A), dict(s=H_B), dict(s=V), dict(s=ELL),
    dict(ell=ctypes.c_void_p(V.value + 4 * 3 * 16 * 9 * 4)),  # inside the last of the 5 value channels
    dict(s=ctypes.c_void_p(ELL.value - 4 * 3 * 16 * 9 * 5 + 4)),  # s ends one float into ell
]


@pytest.mark.parametrize("kw", APPLY_CASES, ids=_ids(APPLY_CASES))
def test_grid_plan_apply_refuses(L, kw):
    assert _apply(L, **kw) == EINVAL
    if kw.get("ell") is not H_B and kw.get("s") is not H_B:
        assert _apply(L, **dict(dict(h_b=NULL, periodic=None), **kw)) == EINVAL


# ---------------------------------------------------------------------------------------------------------------------
# ot.solve_grid argument checks: every one raises before the first kernel, so CPU tensors reach them
# ---------------------------------------------------------------------------------------------------------------------
def _ab(shape=(2, 6, 5)):
    a = torch.full(shape, 1.0 / 30)
    return a, a.clone()


def _raises(exc, match, *args, **kw):
    with pytest.raises(exc, match=match):
        ot.solve_grid(*args, **kw)


def test_exports():
    assert "solve_grid" in ot.__all__ and "OTResultGrid" in ot.__all__
    assert not any(name.startswith("barycenter") for name in ot.__all__)


def test_cost_and_p():
    a, b = _ab()
    _raises(NotImplementedError, "sqeuclidean", a, b, cost="euclidean", reg=0.1, max_iter=5)
    _raises(NotImplementedError, "p = 2", a, b, p=1, reg=0.1, max_iter=5)
    _raises(NotImplementedError, "p = 2", a, b, p=3, reg=0.1, max_iter=5)


def test_redundant_and_regularization():
    a, b = _ab()
    _raises(ValueError, "'reg' and 'blur' are redundant", a, b, reg=0.1, blur=0.1, max_iter=5)
    _raises(ValueError, "'unbalanced' and 'reach' are redundant", a, b, reg=0.1, unbalanced=1.0, reach=1.0,
            max_iter=5)
    _raises(TypeError, "NoneType", a, b, max_iter=5)
    _raises(ValueError, "'reg' should be >= 0", a, b, reg=-1.0, max_iter=5)
    _raises(NotImplementedError, "reg > 0", a, b, reg=0.0, max_iter=5)
    _raises(ValueError, "'unbalanced' should be None", a, b, reg=0.1, unbalanced=-1.0, max_iter=5)
    _raises(NotImplementedError, "'KL' penalty", a, b, reg=0.1, unbalanced=1.0, unbalanced_type="TV", max_iter=5)
    _raises(NotImplementedError, "single method", a, b, reg=0.1, method="lbfgs", max_iter=5)
    _raises(ValueError, "max_iter", a, b, reg=0.1)
    _raises(NotImplementedError, "stopping criteria", a, b, reg=0.1, tol=1e-3, max_iter=5)
    # blur and reach go through the same checks as reg and unbalanced
    _raises(ValueError, "'unbalanced' should be None", a, b, blur=0.1, reach=0.0, max_iter=5)


def test_shapes_sides_and_devices():
    a, b = _ab()
    _raises(TypeError, "torch CUDA tensors", a.numpy(), b, reg=0.1, max_iter=5)
    _raises(ValueError, r"\(B, N1\[, N2\[, N3\]\]\)", a[0, 0], b[0, 0], reg=0.1, max_iter=5)
    _raises(ValueError, r"\(B, N1\[, N2\[, N3\]\]\)", torch.ones(1, 2, 2, 2, 2), torch.ones(1, 2, 2, 2, 2), reg=0.1,
            max_iter=5)
    _raises(ValueError, "should be of shape", a, b[:, :5], reg=0.1, max_iter=5)
    _raises(ValueError, "sides up to 1024", torch.ones(1, 1025), torch.ones(1, 1025), reg=0.1, max_iter=5)
    _raises(ValueError, "'b' contains negative values", a, -b, reg=0.1, max_iter=5)
    _raises(TypeError, "float32 CUDA tensor", a, b, reg=0.1, max_iter=5)  # CPU tensors fail loudly
    _raises(TypeError, "float32 CUDA tensor", a.double(), b.double(), reg=0.1, max_iter=5)


def _geometry_of(shape, **kw):
    return ot._Grid(shape, kw.get("axes"), kw.get("periodic", False))


def test_axes_and_periodic_parsing():
    g = _geometry_of((4, 8))
    assert g.lo == (0.0, 0.0) and g.pitch == (0.25, 0.125) and g.periodic == (False, False)
    g = _geometry_of((4, 8), axes=(-1.0, 1.0), periodic=True)
    assert g.lo == (-1.0, -1.0) and g.pitch == (0.5, 0.25) and g.periodic == (True, True)
    g = _geometry_of((4, 8, 2), axes=((0, 1), (0, 2), (1, 5)), periodic=(True, False, True))
    assert g.pitch == (0.25, 0.25, 2.0) and g.periodic == (True, False, True)
    # diameter: (N - 1) h per plain axis, floor(N / 2) h per periodic one
    assert g.diameter == pytest.approx((0.5**2 + 1.75**2 + 2.0**2) ** 0.5)
    with pytest.raises(NotImplementedError, match="explicit pixel coordinates"):
        _geometry_of((4, 8), axes=(torch.linspace(0, 1, 4), torch.linspace(0, 1, 8)))
    with pytest.raises(NotImplementedError, match="explicit pixel coordinates"):
        _geometry_of((4,), axes=torch.linspace(0, 1, 4))
    for bad in ((0.0, 1.0, 2.0), ((0, 1),), ((0, 1), (0, 1), (0, 1)), "unit", ((0, 1), (0, "a"))):
        with pytest.raises(ValueError, match="'axes' should be"):
            _geometry_of((4, 8), axes=bad)
    for bad in ((1.0, 0.0), (0.0, 0.0), (0.0, float("inf"))):
        with pytest.raises(ValueError, match="lo < hi"):
            _geometry_of((4, 8), axes=bad)
    for bad in ((True,), (True, False, True), 1, "yes", (1, 0)):
        with pytest.raises(ValueError, match="'periodic' should be"):
            _geometry_of((4, 8), periodic=bad)


def test_geometry_errors_reach_the_caller():
    a, b = _ab()
    _raises(ValueError, "'periodic' should be", a, b, periodic=(True,), reg=0.1, max_iter=5)
    _raises(ValueError, "'axes' should be", a, b, axes=((0, 1), (0, 1), (0, 1)), reg=0.1, max_iter=5)
    _raises(NotImplementedError, "explicit pixel coordinates", a, b, axes=(torch.arange(6.0), torch.arange(5.0)),
            reg=0.1, max_iter=5)


def test_masses_per_batch_element():
    """Balanced problems need equal masses in every batch element (checked before the device, as in solve_batch)."""
    a, b = _ab()
    b[1] *= 1.01
    with pytest.raises(ValueError, match=re.escape("have rows that do not sum up to the same values")):
        ot.solve_grid(a, b, reg=0.1, max_iter=5)
    with pytest.raises(ValueError, match=re.escape("do not sum up to the same value.")):
        ot.solve_grid(a[1:], b[1:], reg=0.1, max_iter=5)


def test_exact_cost_at_infinity_is_separable():
    """The eps = +inf start from per-axis marginals equals the dense average of the cost matrix (fp64, CPU)."""
    g = torch.Generator().manual_seed(0)
    for shape, periodic in (((5, 7), (False, True)), ((3, 4, 6), (True, False, False)), ((9,), True)):
        geo = ot._Grid(shape, None, periodic)
        w_rows = torch.rand((2,) + shape, generator=g, dtype=torch.float64)
        w_cols = torch.rand((2,) + shape, generator=g, dtype=torch.float64)
        f = geo.at_infinity(w_rows, w_cols, 0.7).double()
        C = geo.cost("cpu")
        wc = w_cols.reshape(2, -1)
        dense = (C[None] * wc[:, None, :]).sum(-1) / wc.sum(-1, keepdim=True)
        ref = 0.7 * (dense - 0.5 * w_rows.reshape(2, -1) * dense)
        torch.testing.assert_close(f.reshape(2, -1), ref, rtol=1e-6, atol=1e-7)

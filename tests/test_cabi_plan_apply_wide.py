"""CPU-only checks of the plan-times-values operator above D = 64 (b200ot_wide_plan_apply, 64 < D <= 1024): the symbols
exist and match the header, every bad argument is refused with -1 before any CUDA call, a misaligned scratch with -4, a
too-small one with -2, the scratch query is pure, monotone in K and 0 for a refused shape; ``ot.solve_sample`` above
D = 64 reaches the wide operators only (seen through dense fp64 stand-ins) and reproduces the reference's fixtures
(tests/golden/make_golden_ot_wide.py), which the oracle restatement reproduces in fp64.  The fake pointers are never
dereferenced."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from geomloss_b200 import _build, _lib
from oracle import geomloss_oracle as O

NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ot.h")
NEW = ["b200ot_wide_plan_apply_scratch_bytes", "b200ot_wide_plan_apply"]
CASES = golden_names("ot_sample_wide_case")


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _apply(L, N=10, M=12, D=128, K=5, p=2, eps=0.1, x=FAKE, y=FAKE, h_a=FAKE, h_b=NULL, center=NULL, lse2=FAKE,
           v=FAKE, row_factor=NULL, out=FAKE, scratch=FAKE, nbytes=BIG):
    return L.b200ot_wide_plan_apply(x, y, h_a, h_b, 0.0, center, lse2, v, row_factor, out, N, M, D, K, p, eps, scratch,
                                    nbytes, NULL)


def test_symbols_match_header(L):
    header = open(HEADER).read()
    for name in NEW:
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()
        assert re.search(rf"B200OT_API int(64_t)? {name}\(", header), name
    # the same arguments as b200ot_plan_apply
    assert _lib._SIGNATURES["b200ot_wide_plan_apply"] == _lib._SIGNATURES["b200ot_plan_apply"]
    assert _lib._SIGNATURES["b200ot_wide_plan_apply_scratch_bytes"] == _lib._SIGNATURES["b200ot_plan_apply_scratch_bytes"]
    assert L.b200ot_version() == 202


def test_bad_arguments_are_refused(L):
    for ptr in ("x", "y", "h_a", "lse2", "v", "out", "scratch"):
        assert _apply(L, **{ptr: NULL}) == -1, ptr
    for kw in (dict(N=0), dict(N=-3), dict(M=0), dict(M=-1), dict(D=0), dict(D=3), dict(D=64), dict(D=1025),
               dict(D=4096), dict(K=0), dict(K=-2), dict(K=1 << 31), dict(p=1), dict(p=1 | 0x100), dict(p=3),
               dict(p=0), dict(p=2 | 0x200), dict(eps=0.0), dict(eps=-1.0), dict(eps=float("nan"))):
        assert _apply(L, **kw) == -1, kw
    # accepted arguments get as far as the scratch checks: optional pointers null or not, both cost conventions
    for kw in (dict(), dict(h_b=FAKE, center=FAKE, row_factor=FAKE), dict(D=65), dict(D=200), dict(D=1024),
               dict(K=1), dict(K=64), dict(K=65), dict(K=130), dict(p=2 | 0x100)):
        assert _apply(L, nbytes=16, **kw) == -2, kw
        assert _apply(L, scratch=ctypes.c_void_p(0x1004), **kw) == -4, kw
        assert _apply(L, scratch=ctypes.c_void_p(0x1008), **kw) == -4, kw
    need = L.b200ot_wide_plan_apply_scratch_bytes(10, 12, 128, 5)
    assert need > 0 and _apply(L, nbytes=need - 1) == -2


def test_scratch_query_is_pure_monotone_and_zero_when_refused(L):
    for bad in ((0, 5, 128, 1), (5, 0, 128, 1), (5, 5, 64, 1), (5, 5, 1025, 1), (5, 5, 3, 1), (5, 5, 128, 0),
                (5, 5, 128, -1), (5, 5, 128, 1 << 31)):
        assert L.b200ot_wide_plan_apply_scratch_bytes(*bad) == 0, bad
    # the D <= 64 entry keeps refusing the wide shapes
    assert L.b200ot_plan_apply_scratch_bytes(5, 5, 65, 1) == 0
    Ks = (1, 3, 15, 16, 17, 63, 64, 65, 128, 130, 1024)
    for N, M, D in ((10, 12, 65), (1000, 1300, 96), (5000, 4000, 200), (200_000, 200_000, 1024), (129, 4097, 512)):
        sizes = [L.b200ot_wide_plan_apply_scratch_bytes(N, M, D, K) for K in Ks]
        assert sizes[0] > 0 and sizes == sorted(sizes), (N, M, D, sizes)
        assert sizes == [L.b200ot_wide_plan_apply_scratch_bytes(N, M, D, K) for K in Ks]
        # the images of both clouds (two fp16 terms of dk, 16 rank-one halves; fp32 column slot), the value image of
        # one slab of 64 columns and the column maxima of V
        dk = -(-D // 16) * 16
        kp = 2 * dk + 16
        images = (-(-N // 128)) * 128 * kp * 2 + (-(-M // 128)) * 128 * (kp * 2 + 4)
        for K, s in zip(Ks, sizes):
            dkv = -(-min(K, 64) // 16) * 16
            assert s >= images + (-(-M // 128)) * 128 * 4 * dkv + K * 4 + N * (1 + min(K, 64)) * 4, (N, M, D, K)
        # slabs re-use one value image and one set of partials: past 64 columns only the K column maxima grow
        assert sizes[Ks.index(1024)] - sizes[Ks.index(64)] <= round(1024 * 4 / 256 + 1) * 256


# ------------------------------------------------------------------------------------------------
# ot.solve_sample above D = 64: dense fp64 stand-ins for the wide operators (same signatures), CPU tensors
# ------------------------------------------------------------------------------------------------
def _h(h_a, h_b, h_scale_b):
    return h_a.double() if h_b is None else h_a.double() + h_scale_b * h_b.double()


def _cost(x, y):
    return 0.5 * torch.cdist(x.double(), y.double()) ** 2


SEEN: list = []


def _dense_softmin_wide_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                            beta=1.0, out=None, want_lse2=False):
    assert p & 0xFF == 2
    SEEN.append(("softmin", x.shape[1]))
    lse = torch.logsumexp(_h(h_a, h_b, h_scale_b)[None, :] - _cost(x, y) / eps, dim=1)
    val = -eps * lse * beta
    if out_old is not None:
        val = val + alpha_old * out_old.double()
    return val.float(), (lse / np.log(2.0)).float() if want_lse2 else None


def _dense_softmin_wide_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    assert p & 0xFF == 2 and lse2 is not None and lse2.shape == (x.shape[0],)
    SEEN.append(("grad_rows", x.shape[1]))
    w = torch.softmax(_h(h_a, h_b, h_scale_b)[None, :] - _cost(x, y) / eps, dim=1)
    return (grad_out.double()[:, None] * (x.double() - w @ y.double())).float()


def _dense_plan_apply_wide_raw(eps, x, y, h_a, h_b, h_scale_b, lse2, v, *, row_factor=None, center=None):
    assert lse2 is not None and lse2.shape == (x.shape[0],)
    SEEN.append(("apply", x.shape[1]))
    w = torch.softmax(_h(h_a, h_b, h_scale_b)[None, :] - _cost(x, y) / eps, dim=1)
    out = w @ v.double()
    if row_factor is not None:
        out = (row_factor.double()[:, None] if out.dim() == 2 else row_factor.double()) * out
    return out.float()


@pytest.fixture
def wide_ot_stand_ins(monkeypatch):
    from geomloss_b200 import ops, ot

    SEEN.clear()

    def forbidden(*a, **k):
        raise AssertionError("an operator of the D <= 64 family was called above D = 64")

    monkeypatch.setattr(ops, "softmin_wide_raw", _dense_softmin_wide_raw)
    monkeypatch.setattr(ops, "softmin_wide_grad_rows", _dense_softmin_wide_grad_rows)
    monkeypatch.setattr(ops, "plan_apply_wide_raw", _dense_plan_apply_wide_raw)
    for name in ("softmin_raw", "softmin_grad_rows", "plan_apply_raw"):
        monkeypatch.setattr(ops, name, forbidden)
    monkeypatch.setattr(ot, "_fused_operator", lambda s: True)
    return SEEN


def _kw(z):
    kw = {k[3:]: float(z[k]) for k in z if k.startswith("kw_")}
    kw["max_iter"] = int(kw["max_iter"])
    if "debias" in kw:
        kw["debias"] = bool(kw["debias"])
    return kw


def test_wide_fixtures_cover_d_65_to_1024():
    assert len(CASES) == 6
    dims = sorted(load_golden(c)["X_a"].shape[1] for c in CASES)
    assert dims == [65, 96, 128, 200, 512, 1024]
    for c in CASES:  # every case has the weight gradients; the cloud gradients up to D = 200
        z = load_golden(c)
        assert "grad_a_f64" in z and "grad_b_f64" in z
        assert ("grad_X_a_f64" in z) == (z["X_a"].shape[1] <= 200)


@pytest.mark.parametrize("name", CASES)
def test_solve_sample_above_64_reaches_the_wide_operators(wide_ot_stand_ins, name):
    from geomloss_b200 import ot

    z = load_golden(name)
    kw = _kw(z)
    n, m = z["X_a"].shape[0], z["X_b"].shape[0]
    D = z["X_a"].shape[1]
    a0 = torch.from_numpy(z["a"]) if "a" in z else torch.full((n,), 1.0 / n)
    b0 = torch.from_numpy(z["b"]) if "b" in z else torch.full((m,), 1.0 / m)
    leaves = [t.clone().requires_grad_(True) for t in (torch.from_numpy(z["X_a"]), torch.from_numpy(z["X_b"]), a0, b0)]
    res = ot.solve_sample(leaves[0], leaves[1], a=leaves[2], b=leaves[3], **kw)
    ref = float(z["value_f64"])
    assert abs(res.value.item() - ref) <= 2e-5 * abs(ref)
    res.value.backward()
    for leaf, gname in zip(leaves, ("grad_X_a", "grad_X_b", "grad_a", "grad_b")):
        assert leaf.grad is not None and torch.isfinite(leaf.grad).all(), gname
        if gname + "_f64" not in z:  # cloud gradients are stored up to D = 200 (make_golden_ot_wide.py)
            continue
        r = z[gname + "_f64"]
        np.testing.assert_allclose(leaf.grad.numpy(), r, atol=2e-4 * float(np.abs(r).max()), err_msg=gname)
    names = ["potential_a", "potential_b", "marginal_a", "marginal_b", "plan"] + (
        ["potential_aa", "potential_bb"] if kw.get("debias") else [])
    for attr in names:
        r = z[attr + "_f64"]
        tol = 1e-5 * max(1.0, float(np.abs(r).max())) if "potential" in attr else 1e-4 * float(np.abs(r).max())
        np.testing.assert_allclose(getattr(res, attr).detach().numpy(), r, atol=tol, err_msg=attr)
    # the plan as an operator, its transpose, the density, the barycentric maps and the gradient w.r.t. the values
    P = torch.from_numpy(z["plan_f64"])
    g = torch.Generator().manual_seed(D)
    V = torch.randn(m, 3, generator=g, dtype=torch.float64)
    W = torch.randn(n, 2, generator=g, dtype=torch.float64)
    assert ((res.plan_operator @ V.float()).double() - P @ V).abs().max() <= 1e-4 * (P @ V.abs()).max()
    assert ((res.plan_operator.T @ W.float()).double() - P.t() @ W).abs().max() <= 1e-4 * (P.t() @ W.abs()).max()
    dens = P / (torch.from_numpy(z["a"]) if "a" in z else a0.double().detach())[:, None]
    dens = dens / (torch.from_numpy(z["b"]) if "b" in z else b0.double().detach())[None, :]
    assert ((res.density_operator @ V.float()).double() - dens @ V).abs().max() <= 1e-4 * (dens @ V.abs()).max()
    Xa, Xb = torch.from_numpy(z["X_a"]).double(), torch.from_numpy(z["X_b"]).double()
    ab = (P @ Xb) / P.sum(1, keepdim=True) - Xa
    ba = (P.t() @ Xa) / P.sum(0)[:, None] - Xb
    assert (res.a_to_b.double() - ab).abs().max() <= 1e-5 * (1 + Xb.abs().max())
    assert (res.b_to_a.double() - ba).abs().max() <= 1e-5 * (1 + Xa.abs().max())
    G = torch.randn(n, 3, generator=g, dtype=torch.float64)
    Vg = V.float().clone().requires_grad_(True)
    (gv,) = torch.autograd.grad(((res.plan_operator @ Vg) * G.float()).sum(), Vg)
    assert (gv.double() - P.t() @ G).abs().max() <= 1e-4 * (P.t() @ G.abs()).max()
    kinds = {k for k, _ in wide_ot_stand_ins}
    assert kinds == {"softmin", "grad_rows", "apply"} and all(d == D for _, d in wide_ot_stand_ins)


def test_solve_sample_above_1024_raises():
    from geomloss_b200 import ot

    x, y = torch.rand(7, 1025), torch.rand(5, 1025)
    with pytest.raises(NotImplementedError, match="1024"):
        ot.solve_sample(x, y, reg=1.0, max_iter=3)


def test_plan_apply_wide_raw_refuses_dimensions_outside_its_range():
    from geomloss_b200 import ops

    for D in (64, 1025):
        x, y = torch.rand(7, D), torch.rand(5, D)
        with pytest.raises(NotImplementedError, match="64 < D <= 1024"):
            ops.plan_apply_wide_raw(0.1, x, y, torch.zeros(5), None, 0.0, torch.zeros(7), torch.rand(5, 3))


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_wide_fixtures_in_fp64(name):
    z = load_golden(name)
    kw = _kw(z)
    t = lambda k: torch.from_numpy(z[k]).double()  # noqa: E731
    args = dict(X_a=t("X_a"), X_b=t("X_b"), a=t("a") if "a" in z else None, b=t("b") if "b" in z else None)
    out = O.ot_solve_sample(**args, **kw)
    for key, val in out.items():
        ref = z[key + "_f64"]
        np.testing.assert_allclose(val.numpy(), ref, rtol=0, atol=1e-11 * max(1.0, float(np.abs(ref).max())),
                                   err_msg=key)
    n, m = args["X_a"].shape[0], args["X_b"].shape[0]
    if args["a"] is None:
        args["a"], args["b"] = torch.full((n,), 1.0 / n, dtype=torch.float64), torch.full((m,), 1.0 / m, dtype=torch.float64)
    leaves = {k: v.clone().requires_grad_(True) for k, v in args.items()}
    val = O.ot_solve_sample(**leaves, **kw)["value"]
    grads = torch.autograd.grad(val, [leaves[k] for k in ("X_a", "X_b", "a", "b")])
    for g, gname in zip(grads, ("grad_X_a", "grad_X_b", "grad_a", "grad_b")):
        if gname + "_f64" not in z:
            continue
        ref = z[gname + "_f64"]
        np.testing.assert_allclose(g.numpy(), ref, rtol=0, atol=1e-11 * max(1.0, float(np.abs(ref).max())),
                                   err_msg=gname)

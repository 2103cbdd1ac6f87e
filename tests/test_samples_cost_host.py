"""Host side of ``SamplesLoss("sinkhorn", cost=callable)`` without a GPU: the routing rules and their order, the calls
made to the user's cost, the checks on its matrices, the driver (sinkhorn.sinkhorn_cost_matrices) with the two dense
row operators replaced by fp64 torch stand-ins against the reference's fixtures, and the C entries' validation."""
import ctypes
import math

import numpy as np
import pytest
import torch

from geomloss_b200 import SamplesLoss, _build, _lib, ops, samples_loss, sinkhorn
from test_oracle_samples_cost import CASES, G, fixture


# ---- fp64 stand-ins with the operators' contracts ------------------------------------------------------------------
def _h(eps, log_w, pot):
    return log_w if pot is None else log_w + pot / eps


def rows_raw(eps, problems, *, alpha_old=0.0, beta=1.0, want_lse2=False):
    assert 1 <= len(problems) <= 4
    res = []
    for C, log_w, pot, out_old in problems:
        lse = torch.logsumexp(_h(eps, log_w, pot).unsqueeze(-2) - C / eps, dim=-1)
        out = beta * (-eps * lse) + (0 if out_old is None else alpha_old * out_old)
        res.append((out, lse / math.log(2) if want_lse2 else None))
    return res


def rows_grad(eps, C, log_w, pot, lse2, go):
    return go.unsqueeze(-1) * torch.exp(_h(eps, log_w, pot).unsqueeze(-2) - C / eps - (lse2 * math.log(2)).unsqueeze(-1))


@pytest.fixture
def fp64_ops(monkeypatch):
    calls = []

    def raw(*args, **kw):
        calls.append(len(args[1]))
        return rows_raw(*args, **kw)

    monkeypatch.setattr(ops, "dense_softmin_rows_raw", raw)
    monkeypatch.setattr(ops, "dense_softmin_rows_grad", rows_grad)
    return calls


# ---- routing ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def routed(monkeypatch):
    """Pretend the inputs are float32 CUDA tensors and record what reaches the cost-matrix driver."""
    seen = []
    monkeypatch.setattr(samples_loss, "_cuda_f32", lambda *ts: all(t.dtype == torch.float32 for t in ts))
    monkeypatch.setattr(samples_loss, "sinkhorn_cost_matrices",
                        lambda a, x, b, y, cost, **kw: seen.append((tuple(x.shape), kw)) or torch.zeros(()))
    return seen


def _never(u, v):
    raise AssertionError("the cost must not be called on a refused route")


def test_routes_to_the_cost_matrices(routed):
    x, y = torch.rand(5, 3), torch.rand(7, 3)
    SamplesLoss("sinkhorn", cost=_never)(x, y)  # "auto" below 5000^2 pairs
    SamplesLoss("sinkhorn", cost=_never, backend="tensorized", p=3)(x, y)  # any p
    with pytest.warns(UserWarning, match="multiscale"):  # the reference's batched multiscale fallback
        SamplesLoss("sinkhorn", cost=_never, backend="multiscale")(torch.rand(2, 5, 3), torch.rand(2, 7, 3))
    SamplesLoss("sinkhorn", cost=_never)(torch.rand(3, 5, 2000), torch.rand(3, 7, 2000))  # any D
    assert [s for s, _ in routed] == [(5, 3), (5, 3), (2, 5, 3), (3, 5, 2000)]
    assert routed[1][1]["p"] == 3


@pytest.mark.parametrize("make", [
    lambda: (SamplesLoss("sinkhorn", cost="SqDist(X,Y) / IntCst(2)"), "callable"),
    lambda: (SamplesLoss("sinkhorn", cost=_never, backend="online"), "tensorized"),
    lambda: (SamplesLoss("sinkhorn", cost=_never, backend="multiscale"), "tensorized"),
    lambda: (SamplesLoss("gaussian", cost=_never), "loss='sinkhorn'"),
    lambda: (SamplesLoss("energy", cost=_never, backend="tensorized"), "loss='sinkhorn'"),
])
def test_refused_routes_raise_before_calling_the_cost(routed, make):
    loss, words = make()
    with pytest.raises(NotImplementedError, match=words):
        loss(torch.rand(5, 3), torch.rand(7, 3))
    assert routed == []


def test_auto_above_the_tensorized_limit_is_refused(routed):
    x, y = torch.rand(5001, 3), torch.rand(5000, 3)  # N M > 5000^2: "auto" picks "online"
    with pytest.raises(NotImplementedError, match="tensorized"):
        SamplesLoss("sinkhorn", cost=_never)(x, y)
    SamplesLoss("sinkhorn", cost=_never, backend="tensorized")(x, y)
    assert len(routed) == 1


def test_labels_engines_and_dtypes_are_refused(routed):
    x, y = torch.rand(5, 3), torch.rand(7, 3)
    a, b = torch.full((5,), 0.2), torch.full((7,), 1 / 7)
    with pytest.raises(NotImplementedError):
        SamplesLoss("sinkhorn", cost=_never)(torch.zeros(5), a, x, torch.zeros(7), b, y)
    loss = SamplesLoss("sinkhorn", cost=_never)
    loss._engine = {"softmin_raw": None}
    with pytest.raises(NotImplementedError):
        loss(x, y)
    with pytest.raises(NotImplementedError):
        SamplesLoss("sinkhorn", cost=_never)(x.double(), y.double())
    assert routed == []


def test_cpu_inputs_are_refused():
    with pytest.raises(NotImplementedError):
        SamplesLoss("sinkhorn", cost=_never)(torch.rand(5, 3), torch.rand(7, 3))


# ---- the calls to the cost and the checks on its matrices ------------------------------------------------------------
def test_cost_calls_follow_the_reference(fp64_ops):
    x = torch.rand(6, 3, dtype=torch.float64, requires_grad=True)
    y = torch.rand(4, 3, dtype=torch.float64, requires_grad=True)
    a, b = torch.full((6,), 1 / 6, dtype=torch.float64), torch.full((4,), 0.25, dtype=torch.float64)
    log = []

    def cost(u, v):
        log.append((tuple(u.shape), tuple(v.shape), u.requires_grad, v.requires_grad))
        return G.half_sqdist(u, v)

    sinkhorn.sinkhorn_cost_matrices(a, x, b, y, cost)
    assert log == [((1, 6, 3), (1, 4, 3), True, False), ((1, 4, 3), (1, 6, 3), True, False),
                   ((1, 6, 3), (1, 6, 3), True, False), ((1, 4, 3), (1, 4, 3), True, False)]
    log.clear()
    sinkhorn.sinkhorn_cost_matrices(a[None].expand(2, 6), x.detach()[None].expand(2, 6, 3), b[None].expand(2, 4),
                                    y.detach()[None].expand(2, 4, 3), cost, debias=False)
    assert log == [((2, 6, 3), (2, 4, 3), False, False), ((2, 4, 3), (2, 6, 3), False, False)]


def test_every_iteration_is_one_grouped_call(fp64_ops):
    x, y = torch.rand(6, 3, dtype=torch.float64), torch.rand(4, 3, dtype=torch.float64)
    a, b = torch.full((6,), 1 / 6, dtype=torch.float64), torch.full((4,), 0.25, dtype=torch.float64)
    n_eps = len(sinkhorn.scaling_parameters(x, y, 2, 0.05, None, None, 0.5)[2])
    sinkhorn.sinkhorn_cost_matrices(a, x, b, y, G.half_sqdist)
    assert fp64_ops == [4] * (n_eps + 2)  # the init group, one group per eps, the last update
    fp64_ops.clear()
    sinkhorn.sinkhorn_cost_matrices(a, x, b, y, G.half_sqdist, debias=False)
    assert fp64_ops == [2] * (n_eps + 2)


@pytest.mark.parametrize("bad, err, words", [
    (lambda u, v: G.half_sqdist(u, v)[0], ValueError, "C_xy"),
    (lambda u, v: G.half_sqdist(u, v).transpose(1, 2), ValueError, "C_xy"),
    (lambda u, v: G.half_sqdist(u, v)[..., :-1] if u.shape[1] == 4 else G.half_sqdist(u, v), ValueError, "C_yx"),
    (lambda u, v: G.half_sqdist(u, v).float(), TypeError, "C_xy"),
])
def test_cost_results_are_checked(fp64_ops, bad, err, words):
    x, y = torch.rand(6, 3, dtype=torch.float64), torch.rand(4, 3, dtype=torch.float64)
    a, b = torch.full((6,), 1 / 6, dtype=torch.float64), torch.full((4,), 0.25, dtype=torch.float64)
    with pytest.raises(err, match=words):
        sinkhorn.sinkhorn_cost_matrices(a, x, b, y, bad)
    assert fp64_ops == []  # before any launch


# ---- the driver against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_driver_matches_reference_fixtures(fp64_ops, name):
    g, cost, kw = fixture(name)
    a, x, b, y = (torch.from_numpy(g[k]).double().requires_grad_(True) for k in ("a", "x", "b", "y"))
    out = sinkhorn.sinkhorn_cost_matrices(a, x, b, y, cost, **kw)
    if kw.get("potentials"):
        assert out[0].shape == (1, x.shape[0]) and out[1].shape == (1, y.shape[0])
        np.testing.assert_allclose(out[0].detach().numpy(), g["F_f64"], rtol=0, atol=1e-9)
        np.testing.assert_allclose(out[1].detach().numpy(), g["G_f64"], rtol=0, atol=1e-9)
        return
    assert out.shape == g["value_f64"].shape
    np.testing.assert_allclose(out.detach().numpy(), g["value_f64"], rtol=0, atol=1e-9)
    out.sum().backward()
    for k, t in zip(("grad_x", "grad_y", "grad_a", "grad_b"), (x, y, a, b)):
        np.testing.assert_allclose(t.grad.numpy(), g[k + "_f64"], rtol=0, atol=1e-9, err_msg=k)


# ---- the C entries ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _group(*shapes, fake=0x1000):
    descs = (_lib.DenseRows * len(shapes))()
    for d, (B, n, m) in zip(descs, shapes):
        d.C = d.log_w = d.out = fake
        d.B, d.n_rows, d.n_cols = B, n, m
    return descs


def test_scratch_size_is_a_pure_function_of_the_shapes(L):
    def size(*shapes):
        return L.b200ot_dense_rows_scratch_bytes(_group(*shapes), len(shapes))

    # 64-row CTAs, 128-column steps, splits of at least 4 steps while the grid is below 2048 CTAs, 256-byte grain
    assert size((1, 1, 1)) == 256
    assert size((1, 100, 4096)) == -(-(8 * 100 * 8) // 256) * 256  # 2 row blocks: 8 splits of 4 steps
    assert size((1, 16384, 16384)) == 8 * 16384 * 8  # 256 row blocks: 8 splits
    assert size((64, 512, 512)) == 64 * 512 * 8  # 512 CTAs, one split
    one, two = size((1, 5000, 5000)), size((1, 4097, 33))
    assert size((1, 5000, 5000), (1, 4097, 33)) == one + two
    assert size((1, 5000, 5000), (1, 4097, 33)) == size((1, 5000, 5000), (1, 4097, 33))
    assert size((1, 46341, 46341)) > 0
    assert L.b200ot_dense_rows_scratch_bytes(_group((1, 4, 4)), 0) == 0
    assert L.b200ot_dense_rows_scratch_bytes(_group(*[(1, 4, 4)] * 5), 5) == 0
    assert L.b200ot_dense_rows_scratch_bytes(_group((1, 0, 4)), 1) == 0
    assert L.b200ot_dense_rows_scratch_bytes(None, 1) == 0


def test_c_entries_validate_before_any_launch(L):
    null, fake = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
    run = L.b200ot_dense_softmin_rows
    g = _group((1, 10, 10), (2, 5, 7))
    assert run(g, 2, 0.1, 0.0, 1.0, fake, 16, null) == -2  # ESCRATCH
    assert run(g, 2, 0.1, 0.0, 1.0, ctypes.c_void_p(0x1004), 1 << 30, null) == -4  # EALIGN
    assert run(g, 2, 0.0, 0.0, 1.0, fake, 1 << 30, null) == -1  # eps
    assert run(g, 0, 0.1, 0.0, 1.0, fake, 1 << 30, null) == -1
    assert run(_group(*[(1, 4, 4)] * 5), 5, 0.1, 0.0, 1.0, fake, 1 << 30, null) == -1
    assert run(None, 1, 0.1, 0.0, 1.0, fake, 1 << 30, null) == -1
    assert run(g, 2, 0.1, 0.0, 1.0, null, 1 << 30, null) == -1
    for field, value in (("C", None), ("log_w", None), ("out", None), ("B", 0), ("n_rows", 0), ("n_cols", -1)):
        bad = _group((1, 10, 10), (2, 5, 7))
        setattr(bad[1], field, value)
        assert run(bad, 2, 0.1, 0.0, 1.0, fake, 1 << 30, null) == -1, field
    bad = _group((1, 10, 10))
    bad[0].out, bad[0].lse2 = None, 0x2000  # lse2 alone is a result
    assert run(bad, 1, 0.1, 0.0, 1.0, fake, 16, null) == -2
    assert run(_group((1 << 20, 1 << 20, 4)), 1, 0.1, 0.0, 1.0, fake, 1 << 62, null) == -1  # 2^34 CTAs
    bwd = L.b200ot_dense_softmin_rows_bwd
    assert bwd(fake, fake, null, 10.0, fake, fake, null, 1, 4, 4, null) == -1
    assert bwd(fake, null, null, 10.0, fake, fake, fake, 1, 4, 4, null) == -1
    assert bwd(fake, fake, null, 0.0, fake, fake, fake, 1, 4, 4, null) == -1
    assert bwd(fake, fake, null, 10.0, fake, fake, fake, 1, 0, 4, null) == -1


def test_operator_checks_shapes_then_lengths_then_device():
    C = torch.zeros(4, 5)
    with pytest.raises(ValueError, match="1 to 4 problems"):
        ops.dense_softmin_rows_raw(0.1, [])
    with pytest.raises(ValueError, match="1 to 4 problems"):
        ops.dense_softmin_rows_raw(0.1, [(C, torch.zeros(5), None, None)] * 5)
    with pytest.raises(ValueError, match="cost matrix"):
        ops.dense_softmin_rows_raw(0.1, [(torch.zeros(5), torch.zeros(5), None, None)])
    with pytest.raises(ValueError, match="log_w"):
        ops.dense_softmin_rows_raw(0.1, [(C, torch.zeros(4), None, None)])
    with pytest.raises(ValueError, match="out_old"):
        ops.dense_softmin_rows_raw(0.1, [(C, torch.zeros(5), torch.zeros(5), torch.zeros(5))])
    with pytest.raises(_lib.B200OTError):  # lengths right: the device check refuses a CPU tensor
        ops.dense_softmin_rows_raw(0.1, [(C, torch.zeros(5), None, None)])
    with pytest.raises(ValueError, match="lse2"):
        ops.dense_softmin_rows_grad(0.1, C, torch.zeros(5), None, torch.zeros(5), torch.zeros(4))
    with pytest.raises(_lib.B200OTError):
        ops.dense_softmin_rows_grad(0.1, C, torch.zeros(5), None, torch.zeros(4), torch.zeros(4))


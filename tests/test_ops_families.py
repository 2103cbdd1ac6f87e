"""The checks every public operator of ``ops`` makes before it reaches the library, and which operators serve which
clouds.  CPU tensors: a per-point vector of the wrong length is refused before the device check, so nothing here needs
a GPU or the library."""
import pytest
import torch

from geomloss_b200 import ops

B, N, M = 2, 5, 7


def _clouds(D, batched):
    lead = (B,) if batched else ()
    return torch.rand(*lead, N, D), torch.rand(*lead, M, D), lead


def _softmin_fwd_args(D, batched):
    x, y, lead = _clouds(D, batched)
    kw = dict(h_b=torch.zeros(*lead, M), out_old=torch.zeros(*lead, N), out=torch.zeros(*lead, N))
    return (0.1, x, y, torch.zeros(*lead, M)), kw, dict(h_a=3, h_b="h_b", out_old="out_old", out="out")


def _softmin_grad_args(D, batched):
    x, y, lead = _clouds(D, batched)
    args = (0.1, x, y, torch.zeros(*lead, M), torch.zeros(*lead, M), 0.5, torch.zeros(*lead, N), torch.ones(*lead, N))
    return args, {}, dict(h_a=3, h_b=4, lse2=6, grad_out=7)


def _conv_args(D, batched, grad):
    x, y, lead = _clouds(D, batched)
    args = (0, x, y, torch.ones(*lead, M), 0.5) + ((torch.ones(*lead, N),) if grad else ())
    return args, {}, dict(w=3, **({"grad_out": 5} if grad else {}))


def _plan_args(D):
    x, y, _ = _clouds(D, False)
    args = (0.1, x, y, torch.zeros(M), torch.zeros(M), 0.5, torch.zeros(N), torch.rand(M, 3))
    return args, dict(row_factor=torch.ones(N)), dict(h_a=3, h_b=4, lse2=6, v=7, row_factor="row_factor")


# (operator, D, batched clouds, p): every raw, row-gradient and plan-apply operator, in each cloud rank it serves
CASES = [
    ("softmin_raw", 3, False, 2), ("softmin_raw", 40, False, 2), ("softmin_grad_rows", 3, False, 2),
    ("softmin_batched_raw", 16, True, 2), ("softmin_batched_grad_rows", 16, True, 2),
    ("softmin_l1_raw", 16, False, 1), ("softmin_l1_raw", 16, True, 1), ("softmin_l1_grad_rows", 16, True, 1),
    ("softmin_wide_raw", 65, False, 2), ("softmin_wide_raw", 65, True, 1), ("softmin_wide_grad_rows", 65, True, 2),
    ("kernel_conv_raw", 3, False, None), ("kernel_conv_grad_rows", 3, False, None),
    ("kernel_conv_value_and_grad_rows", 16, False, None), ("kernel_conv_batched_raw", 16, True, None),
    ("kernel_conv_batched_grad_rows", 16, True, None), ("kernel_conv_batched_value_and_grad_rows", 16, True, None),
    ("kernel_conv_wide_raw", 65, True, None), ("kernel_conv_wide_grad_rows", 65, False, None),
    ("plan_apply_raw", 3, False, None), ("plan_apply_raw", 16, False, None), ("plan_apply_wide_raw", 65, False, None),
]


def _args(name, D, batched, p):
    """The arguments of a valid call, and where each per-point vector sits in them: a position or a keyword."""
    if name.startswith("softmin"):
        args, kw, where = (_softmin_grad_args if name.endswith("grad_rows") else _softmin_fwd_args)(D, batched)
        kw["p"] = p
    elif name.startswith("kernel_conv"):
        args, kw, where = _conv_args(D, batched, name.endswith("_grad_rows") and "value" not in name)
    else:
        args, kw, where = _plan_args(D)
    return list(args), kw, where


@pytest.mark.parametrize("name, D, batched, p", CASES)
def test_short_per_point_vectors_are_refused(name, D, batched, p):
    fn = getattr(ops, name)
    args, kw, where = _args(name, D, batched, p)
    for vec, at in where.items():
        a, k = list(args), dict(kw)
        t = a[at] if isinstance(at, int) else k[at]
        short = t[:-1] if vec == "v" else t.reshape(-1)[:-1]
        if isinstance(at, int):
            a[at] = short
        else:
            k[at] = short
        with pytest.raises(ValueError, match=f"{vec} must"):
            fn(*a, **k)
    # the same call with every length right gets past these checks to the device check
    with pytest.raises(ops._lib.B200OTError, match="CUDA device"):
        fn(*args, **kw)


def test_wide_checks_the_dimension_before_the_device():
    x, y = torch.rand(N, 1025), torch.rand(M, 1025)
    with pytest.raises(NotImplementedError, match="64 < D <= 1024"):
        ops.softmin_wide_raw(0.1, x, y, torch.zeros(M))
    with pytest.raises(NotImplementedError, match="laplacian and energy"):
        ops.softmin_raw(0.1, x[:, :65], y[:, :65], torch.zeros(M))


def test_the_p_rules_of_the_families():
    x, y, lead = _clouds(16, True)
    h, lse2, go = torch.zeros(B, M), torch.zeros(B, N), torch.ones(B, N)
    for fn in (lambda p: ops.softmin_batched_raw(0.1, x, y, h, p=p),
               lambda p: ops.softmin_batched_grad_rows(0.1, x, y, h, None, 0.0, lse2, go, p=p)):
        with pytest.raises(NotImplementedError, match="p = 2"):
            fn(1)
    for fn in (lambda p: ops.softmin_l1_raw(0.1, x, y, h, p=p),
               lambda p: ops.softmin_l1_grad_rows(0.1, x, y, h, None, 0.0, lse2, go, p=p)):
        with pytest.raises(ValueError, match="p = 1"):
            fn(2)


# ------------------------------------------------------------------------------------------------
# which operators serve which clouds
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D, p, batched, raw", [
    (3, 2, False, "softmin_raw"), (8, 1, False, "softmin_raw"), (9, 2, False, "softmin_raw"),
    (9, 1, False, "softmin_l1_raw"), (64, 1 | ops.P_UNCLAMPED, False, "softmin_l1_raw"),
    (64, 2, True, "softmin_batched_raw"), (9, 1, True, "softmin_l1_raw"), (8, 2, True, None), (3, 1, True, None),
    (65, 2, False, "softmin_wide_raw"), (1024, 1, True, "softmin_wide_raw"), (1025, 2, False, "softmin_wide_raw"),
])
def test_softmin_operators(D, p, batched, raw):
    found = ops.softmin_operators(D, p, batched)
    if raw is None:
        assert found is None
        return
    public = raw[:-len("_raw")] if raw != "softmin_raw" else "softmin"
    assert found == (getattr(ops, raw), getattr(ops, public))


@pytest.mark.parametrize("D, batched, conv", [
    (3, False, "kernel_conv"), (64, False, "kernel_conv"), (8, True, None), (9, True, "kernel_conv_batched"),
    (64, True, "kernel_conv_batched"), (65, False, "kernel_conv_wide"), (1024, True, "kernel_conv_wide"),
])
def test_kernel_conv_operator(D, batched, conv):
    assert ops.kernel_conv_operator(D, batched) is (None if conv is None else getattr(ops, conv))


def test_ot_operators():
    assert ops.ot_operators(64) == (ops.softmin_raw, ops.softmin_grad_rows, ops.plan_apply_raw)
    assert ops.ot_operators(65) == (ops.softmin_wide_raw, ops.softmin_wide_grad_rows, ops.plan_apply_wide_raw)


def test_lookups_return_replaced_operators(monkeypatch):
    stand_in = object()
    monkeypatch.setattr(ops, "softmin_l1_raw", stand_in)
    monkeypatch.setattr(ops, "kernel_conv_batched", stand_in)
    monkeypatch.setattr(ops, "plan_apply_wide_raw", stand_in)
    assert ops.softmin_operators(16, 1)[0] is stand_in
    assert ops.kernel_conv_operator(16, batched=True) is stand_in
    assert ops.ot_operators(100)[2] is stand_in


@pytest.mark.gpu
def test_supplied_out_is_written_in_place_or_refused():
    dev = "cuda"
    x, y, h = torch.rand(N, 3, device=dev), torch.rand(M, 3, device=dev), torch.zeros(M, device=dev)
    out = torch.empty(N, device=dev)
    assert ops.softmin_raw(0.1, x, y, h, out=out)[0] is out
    with pytest.raises(ValueError, match="contiguous"):
        ops.softmin_raw(0.1, x, y, h, out=torch.empty(2 * N, device=dev)[::2])
    with pytest.raises(TypeError):
        ops.softmin_raw(0.1, x, y, h, out=torch.empty(N, device=dev, dtype=torch.float64))

"""CPU-only checks of the operators above D = 64 (b200ot_wide_*, 64 < D <= 1024): the symbols exist and match the
header, every bad argument is refused with -1 before any CUDA call, a misaligned scratch with -4, a too-small scratch
with -2, the scratch query is pure and covers both plans, and SamplesLoss routes D = 65 / 1024 to the wide operators
(seen through dense fp64 stand-ins) and refuses D = 1025.  The fake pointers are never dereferenced."""
import ctypes
import os
import re

import pytest
import torch

from geomloss_b200 import _build, _lib

WIDE = ["b200ot_wide_scratch_bytes", "b200ot_wide_softmin_fwd", "b200ot_wide_softmin_bwd_x",
        "b200ot_wide_kernel_conv_fwd", "b200ot_wide_kernel_conv_bwd_x"]
NULL, FAKE = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
BIG = 1 << 40
UNCLAMPED = 0x100
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "b200ot.h")


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _sfwd(L, B=3, N=10, M=12, D=128, p=2, eps=0.1, x=FAKE, y=FAKE, h=FAKE, out=FAKE, lse2=NULL, scratch=FAKE,
          nbytes=BIG, **_):
    return L.b200ot_wide_softmin_fwd(x, y, h, NULL, 0.0, NULL, NULL, 0.0, 1.0, out, lse2, B, N, M, D, p, eps, scratch,
                                     nbytes, NULL)


def _sbwd(L, B=3, N=10, M=12, D=128, p=2, eps=0.1, x=FAKE, y=FAKE, h=FAKE, lse2=FAKE, go=FAKE, gx=FAKE, scratch=FAKE,
          nbytes=BIG, **_):
    return L.b200ot_wide_softmin_bwd_x(x, y, h, NULL, 0.0, NULL, lse2, go, gx, B, N, M, D, p, eps, scratch, nbytes,
                                       NULL)


def _cfwd(L, B=3, N=10, M=12, D=128, kind=0, blur=0.5, x=FAKE, y=FAKE, w=FAKE, out=FAKE, scratch=FAKE, nbytes=BIG,
          **_):
    return L.b200ot_wide_kernel_conv_fwd(x, y, w, NULL, out, B, N, M, D, kind, blur, scratch, nbytes, NULL)


def _cbwd(L, B=3, N=10, M=12, D=128, kind=0, blur=0.5, x=FAKE, y=FAKE, w=FAKE, go=FAKE, gx=FAKE, scratch=FAKE,
          nbytes=BIG, **_):
    return L.b200ot_wide_kernel_conv_bwd_x(x, y, w, NULL, go, gx, B, N, M, D, kind, blur, scratch, nbytes, NULL)


CALLS = {"softmin_fwd": _sfwd, "softmin_bwd": _sbwd, "conv_fwd": _cfwd, "conv_bwd": _cbwd}
POINTERS = {"softmin_fwd": ["x", "y", "h", "scratch"], "softmin_bwd": ["x", "y", "h", "lse2", "go", "gx", "scratch"],
            "conv_fwd": ["x", "y", "w", "out", "scratch"], "conv_bwd": ["x", "y", "w", "go", "gx", "scratch"]}


def test_symbols_match_header(L):
    header = open(HEADER).read()
    assert re.search(r"#define B200OT_MAX_D_WIDE 1024\b", header)
    for name in WIDE:
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()
        assert re.search(rf"B200OT_API int(64_t)? {name}\(", header), name
    assert L.b200ot_version() == 202


@pytest.mark.parametrize("call", sorted(CALLS))
def test_bad_arguments_are_refused(L, call):
    f = CALLS[call]
    for ptr in POINTERS[call]:
        assert f(L, **{ptr: NULL}) == -1, f"{call}: null {ptr}"
    for kw in (dict(B=0), dict(B=-2), dict(N=0), dict(N=-1), dict(M=0), dict(D=0), dict(D=8), dict(D=64),
               dict(D=1025), dict(D=4096)):
        assert f(L, **kw) == -1, f"{call}: {kw}"
    if call.startswith("softmin"):
        for kw in (dict(p=3), dict(p=0), dict(p=0x201), dict(p=2 | 0x200), dict(eps=0.0), dict(eps=-1.0),
                   dict(eps=float("nan"))):
            assert f(L, **kw) == -1, f"{call}: {kw}"
        if call == "softmin_fwd":
            assert f(L, out=NULL) == -1  # neither out nor lse2
        good = [dict(p=p) for p in (1, 2, 1 | UNCLAMPED, 2 | UNCLAMPED)]
    else:
        for kw in (dict(kind=3), dict(kind=-1), dict(kind=0x200), dict(kind=0, blur=0.0), dict(kind=1, blur=-1.0),
                   dict(kind=0, blur=float("nan"))):
            assert f(L, **kw) == -1, f"{call}: {kw}"
        good = [dict(kind=k) for k in (0, 1, 2, 1 | UNCLAMPED, 2 | UNCLAMPED)] + [dict(kind=2, blur=0.0)]
    for kw in good:  # these pass validation: a misaligned scratch is the first refusal
        for D in (65, 1024):
            assert f(L, D=D, scratch=ctypes.c_void_p(0x1004), **kw) == -4, (call, kw, D)
            assert f(L, D=D, scratch=ctypes.c_void_p(0x1008), **kw) == -4, (call, kw, D)


@pytest.mark.parametrize("call", sorted(CALLS))
def test_small_scratch(L, call):
    f = CALLS[call]
    for B, N, M, D in ((3, 10, 12, 65), (1, 300, 200, 128), (17, 129, 1000, 1024), (2, 5000, 7000, 200)):
        need = L.b200ot_wide_scratch_bytes(B, N, M, D)
        assert need > 0
        assert f(L, B=B, N=N, M=M, D=D, nbytes=need - 1) == -2
        assert f(L, B=B, N=N, M=M, D=D, nbytes=16) == -2


def test_scratch_query(L):
    for bad in ((0, 10, 10, 128), (-1, 10, 10, 128), (2, 0, 10, 128), (2, 10, 0, 128), (2, 10, 10, 64),
                (2, 10, 10, 1025), (2, 10, 10, 0)):
        assert L.b200ot_wide_scratch_bytes(*bad) == 0, bad
    for N, M, D in ((10, 12, 65), (300, 1000, 127), (129, 4097, 256), (100000, 100000, 1024), (500, 500, 1000)):
        sizes = [L.b200ot_wide_scratch_bytes(B, N, M, D) for B in (1, 2, 3, 5, 8, 64, 65)]
        assert all(s > 0 for s in sizes)
        assert sizes == sorted(sizes), (N, M, D, sizes)
        # pure: the same answer every time
        assert sizes == [L.b200ot_wide_scratch_bytes(B, N, M, D) for B in (1, 2, 3, 5, 8, 64, 65)]
        # both plans fit: the images, and the row-gradient sums (D + 2 floats per row for the p = 1 softmin)
        for B in (1, 65):
            s = L.b200ot_wide_scratch_bytes(B, N, M, D)
            dk = -(-D // 16) * 16
            kp = 2 * dk + 16
            images = B * (-(-N // 128)) * 128 * kp * 2 + B * (-(-M // 128)) * 128 * (kp * 2 + 4)
            assert s >= images + B * N * (D + 2) * 4, (B, N, M, D)
    # the existing families keep refusing D > 64
    assert L.b200ot_softmin_scratch_bytes(100, 100, 65) == 0
    assert L.b200ot_batched_scratch_bytes(2, 100, 100, 65) == 0
    assert L.b200ot_softmin_l1_scratch_bytes(2, 100, 100, 65) == 0


# ------------------------------------------------------------------------------------------------
# routing: dense fp64 stand-ins for the wide operators (same signatures), CPU tensors
# ------------------------------------------------------------------------------------------------
def _cost(x, y, p):
    d2 = ((x[..., :, None, :] - y[..., None, :, :]) ** 2).sum(-1)
    return d2 / 2 if p == 2 else d2.clamp_min(1e-8).sqrt()


def _dense_softmin_raw(eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, out_old=None, alpha_old=0.0,
                       beta=1.0, out=None, want_lse2=False):
    CALLS_SEEN.append(("softmin", tuple(x.shape)))
    h = h_a.double() if h_b is None else h_a.double() + h_scale_b * h_b.double()
    h = h.view(*y.shape[:-1])
    val = -eps * torch.logsumexp(h[..., None, :] - _cost(x.double(), y.double(), p & 0xFF) / eps, dim=-1) * beta
    if out_old is not None:
        val = val + alpha_old * out_old.double().view_as(val)
    return val.float(), (torch.zeros_like(val).float() if want_lse2 else None)


def _dense_softmin_grad_rows(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
    h = h_a.double() if h_b is None else h_a.double() + h_scale_b * h_b.double()
    h = h.view(*y.shape[:-1])
    w = torch.softmax(h[..., None, :] - _cost(x.double(), y.double(), p & 0xFF) / eps, dim=-1)
    return (grad_out.double().view(*x.shape[:-1])[..., None] * (x.double() - w @ y.double())).float()


def _dense_conv(kind, x, y, w, blur, *, center=None):
    CALLS_SEEN.append(("conv", tuple(x.shape)))
    d2 = ((x.double()[..., :, None, :] - y.double()[..., None, :, :]) ** 2).sum(-1)
    k = (kind if isinstance(kind, int) else {"gaussian": 0, "laplacian": 1, "energy": 2}[kind]) & 0xFF
    K = (-d2 / (2 * blur ** 2)).exp() if k == 0 else ((-d2.clamp_min(1e-8).sqrt() / blur).exp() if k == 1
                                                       else -d2.clamp_min(1e-8).sqrt())
    return (K @ w.double().view(*y.shape[:-1])[..., None]).squeeze(-1).float()


CALLS_SEEN: list = []


@pytest.fixture
def wide_stand_ins(monkeypatch):
    from geomloss_b200 import ops

    CALLS_SEEN.clear()

    def forbidden(*a, **k):
        raise AssertionError("an operator of the D <= 64 families was called above D = 64")

    monkeypatch.setattr(ops, "softmin_wide_raw", _dense_softmin_raw)
    monkeypatch.setattr(ops, "softmin_wide_grad_rows", _dense_softmin_grad_rows)
    monkeypatch.setattr(ops, "kernel_conv_wide_raw", _dense_conv)
    for name in ("softmin_raw", "softmin_batched_raw", "softmin_l1_raw", "kernel_conv_raw", "kernel_conv_batched_raw"):
        monkeypatch.setattr(ops, name, forbidden)
    return CALLS_SEEN


@pytest.mark.parametrize("D", [65, 1024])
@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("batch", [0, 3])
def test_sinkhorn_routes_to_wide(wide_stand_ins, D, p, batch):
    from geomloss_b200 import SamplesLoss

    g = torch.Generator().manual_seed(D + p)
    shape = (batch,) if batch else ()
    x = torch.randn(*shape, 7, D, generator=g)
    y = torch.randn(*shape, 5, D, generator=g)
    val = SamplesLoss("sinkhorn", p=p, blur=0.5)(x, y)
    assert torch.isfinite(val).all()
    assert wide_stand_ins and all(kind == "softmin" for kind, _ in wide_stand_ins)
    if batch:  # one launch group per softmin for the whole batch
        assert all(len(shape) == 3 and shape[0] == batch for _, shape in wide_stand_ins)


@pytest.mark.parametrize("D", [65, 1024])
@pytest.mark.parametrize("loss", ["gaussian", "laplacian", "energy"])
@pytest.mark.parametrize("batch", [0, 3])
def test_kernel_losses_route_to_wide(wide_stand_ins, D, loss, batch):
    from geomloss_b200 import SamplesLoss

    g = torch.Generator().manual_seed(D)
    shape = (batch,) if batch else ()
    x = torch.randn(*shape, 7, D, generator=g)
    y = torch.randn(*shape, 5, D, generator=g)
    val = SamplesLoss(loss, blur=2.0)(x, y)
    assert torch.isfinite(val).all()
    assert wide_stand_ins and all(kind == "conv" for kind, _ in wide_stand_ins)


@pytest.mark.parametrize("loss", ["sinkhorn", "gaussian", "energy"])
@pytest.mark.parametrize("batch", [0, 3])
def test_above_max_d_wide_raises(loss, batch):
    """D = 1025: the library's own wide operators refuse the shape before anything reaches the device."""
    from geomloss_b200 import SamplesLoss

    shape = (batch,) if batch else ()
    x, y = torch.randn(*shape, 7, 1025), torch.randn(*shape, 5, 1025)
    with pytest.raises(NotImplementedError, match="1024"):
        SamplesLoss(loss, blur=0.5)(x, y)


def test_labelled_multiscale_above_64_raises():
    from geomloss_b200 import SamplesLoss

    x, y = torch.randn(7, 65), torch.randn(5, 65)
    lx, ly = torch.zeros(7, dtype=torch.long), torch.zeros(5, dtype=torch.long)
    a, b = torch.full((7,), 1 / 7), torch.full((5,), 1 / 5)
    with pytest.raises(NotImplementedError, match="two-scale"):
        SamplesLoss("sinkhorn", blur=0.5, backend="multiscale")(lx, a, x, ly, b, y)

"""CPU tests of the two autograd contracts of ``ops``, driven with fp64 dense stand-ins of their operators:

* ``ops._Softmin``: ``scale_out * softmin(eps, (x, y), h_a + h_scale_b*h_b)``, the gradient to the row cloud x only;
* ``ops._KernelConv``: ``K(x, y) @ w``, gradients to x, y and w, the y- and w-gradients from the transposed problem.

The public operators (``ops.softmin*``, ``ops.kernel_conv*``, ``ranges.*_ranges``) are checked to bind their own
operators, looked up by name at call time, so that replacing those names by the stand-ins runs them on the CPU."""
import pytest
import torch

from geomloss_b200 import ops, ranges

LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
F64 = dict(dtype=torch.float64)


def _rand(g, *shape):
    return torch.rand(*shape, generator=g, **F64)


def _diff(x, y):
    return x.unsqueeze(-2) - y.unsqueeze(-3)  # (..., N, M, D)


class DenseSoftmin:
    """fp64 softmin operators with the signatures of ``ops.softmin_raw`` / ``ops.softmin_grad_rows`` (cost
    |x - y|^2 / 2 for p = 2, |x - y| for p = 1; one problem or a batch), lse2 in the kernels' log2 units.  Every call
    records the centre it was given, the forward whether it was asked for lse2."""

    def __init__(self):
        self.centers, self.want_lse2 = [], []

    @staticmethod
    def _t(eps, x, y, h_a, h_b, h_scale_b, p):
        h = h_a if h_b is None else h_a + h_scale_b * h_b
        d = _diff(x, y).norm(dim=-1)
        return LOG2E * (h.unsqueeze(-2) - (d * d / 2 if p == 2 else d) / eps)

    def fwd(self, eps, x, y, h_a, h_b=None, h_scale_b=0.0, *, p=2, center=None, beta=1.0, want_lse2=False):
        self.centers.append(center)
        self.want_lse2.append(want_lse2)
        lse2 = torch.logsumexp(LN2 * self._t(eps, x, y, h_a, h_b, h_scale_b, p), -1) * LOG2E
        return -eps * LN2 * lse2 * beta, (lse2 if want_lse2 else None)

    def bwd(self, eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, p=2, center=None):
        self.centers.append(center)
        w = torch.exp2(self._t(eps, x, y, h_a, h_b, h_scale_b, p) - lse2.unsqueeze(-1))
        diff = _diff(x, y)
        dc = diff if p == 2 else diff / diff.norm(dim=-1, keepdim=True)
        return grad_out.unsqueeze(-1) * (w.unsqueeze(-1) * dc).sum(-2)


def _softmin_ref(eps, x, y, h, p):
    d = _diff(x, y).norm(dim=-1)
    return -eps * torch.logsumexp(h.unsqueeze(-2) - (d * d / 2 if p == 2 else d) / eps, -1)


def _softmin_inputs(batched, extras, seed=0):
    g = torch.Generator().manual_seed(seed)
    lead = (3,) if batched else ()
    x = _rand(g, *lead, 5, 4).requires_grad_(True)
    y = _rand(g, *lead, 7, 4) + 0.5
    h_a, h_b = _rand(g, *lead, 7), (_rand(g, *lead, 7) if extras else None)
    center = _rand(g, 4) if extras else None
    return x, y, h_a, h_b, center


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("extras", [True, False], ids=["h_b+center", "no-h_b-no-center"])
def test_softmin_value_and_row_gradient(p, batched, extras):
    x, y, h_a, h_b, center = _softmin_inputs(batched, extras)
    eps, h_scale_b, scale_out = 0.2, 0.3, 0.7
    op = DenseSoftmin()

    def f(x):
        return ops._Softmin.apply(op.fwd, op.bwd, x, y, h_a, h_b, h_scale_b, eps, p, center, scale_out)

    h = h_a if h_b is None else h_a + h_scale_b * h_b
    torch.testing.assert_close(f(x), scale_out * _softmin_ref(eps, x, y, h, p))
    assert torch.autograd.gradcheck(f, (x,))
    # the row-gradient operator receives the forward's centre, None included
    assert all((c is None) == (center is None) for c in op.centers)
    assert all(c is None or torch.equal(c, center) for c in op.centers)


def test_softmin_columns_and_potentials_get_no_gradient():
    x, y, h_a, h_b, center = _softmin_inputs(False, True)
    y, h_a, h_b = (t.requires_grad_(True) for t in (y, h_a, h_b))
    op = DenseSoftmin()
    out = ops._Softmin.apply(op.fwd, op.bwd, x, y, h_a, h_b, 0.3, 0.2, 2, center, 0.7)
    gx, gy, ga, gb = torch.autograd.grad(out.sum(), [x, y, h_a, h_b], allow_unused=True)
    assert gx is not None and gy is None and ga is None and gb is None
    # lse2 is asked for only when the row cloud needs a gradient
    ops._Softmin.apply(op.fwd, op.bwd, x.detach(), y, h_a, h_b, 0.3, 0.2, 2, center, 0.7)
    assert op.want_lse2 == [True, False]


@pytest.mark.parametrize("public, raw, grad_rows, p, batched", [
    ("softmin", "softmin_raw", "softmin_grad_rows", 2, False),
    ("softmin_batched", "softmin_batched_raw", "softmin_batched_grad_rows", 2, True),
    ("softmin_l1", "softmin_l1_raw", "softmin_l1_grad_rows", 1, False),
    ("softmin_l1", "softmin_l1_raw", "softmin_l1_grad_rows", 1, True),
])
def test_public_softmins_bind_their_operators(monkeypatch, public, raw, grad_rows, p, batched):
    op = DenseSoftmin()
    monkeypatch.setattr(ops, raw, op.fwd)
    monkeypatch.setattr(ops, grad_rows, op.bwd)
    x, y, h_a, h_b, center = _softmin_inputs(batched, True, seed=1)
    y, h_a, h_b = (t.requires_grad_(True) for t in (y, h_a, h_b))
    out = getattr(ops, public)(0.2, x, y, h_a, h_b, 0.3, p=p, center=center, scale_out=0.7)
    torch.testing.assert_close(out, 0.7 * _softmin_ref(0.2, x, y, h_a + 0.3 * h_b, p))
    gx, gy, ga, gb = torch.autograd.grad(out.sum(), [x, y, h_a, h_b], allow_unused=True)
    assert gy is None and ga is None and gb is None
    assert torch.autograd.gradcheck(
        lambda x: getattr(ops, public)(0.2, x, y, h_a, h_b, 0.3, p=p, center=center, scale_out=0.7), (x,))


def test_softmin_ranges_binds_its_problem(monkeypatch):
    op, the_prob = DenseSoftmin(), object()

    def fwd(eps, x, y, h_a, h_b, h_scale_b, prob, **kw):
        assert prob is the_prob
        return op.fwd(eps, x, y, h_a, h_b, h_scale_b, **kw)

    def bwd(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, *, prob, **kw):
        assert prob is the_prob
        return op.bwd(eps, x, y, h_a, h_b, h_scale_b, lse2, grad_out, **kw)

    monkeypatch.setattr(ranges, "softmin_ranges_raw", fwd)
    monkeypatch.setattr(ranges, "softmin_ranges_grad_rows", bwd)
    x, y, h_a, h_b, center = _softmin_inputs(False, True, seed=2)
    assert torch.autograd.gradcheck(
        lambda x: ranges.softmin_ranges(0.2, x, y, h_a, h_b, 0.3, the_prob, center=center, scale_out=0.7), (x,))


class DenseConv:
    """fp64 gaussian-kernel matvec operators with the signatures of ``ops.kernel_conv_raw`` / ``_grad_rows`` /
    ``_value_and_grad_rows`` (one problem or a batch).  Every call records its name and the centre it was given."""

    def __init__(self):
        self.calls = []

    @staticmethod
    def _conv(x, y, w, blur):
        k = torch.exp(-(_diff(x, y) ** 2).sum(-1) / (2 * blur ** 2))
        return (k @ w.unsqueeze(-1)).squeeze(-1)

    def _grad(self, x, y, w, blur, grad_out):
        with torch.enable_grad():  # called from inside an autograd backward
            xr = x.detach().requires_grad_(True)
            (g,) = torch.autograd.grad(self._conv(xr, y.detach(), w.detach(), blur), xr, grad_out.detach())
        return g

    def raw(self, kind, x, y, w, blur, *, center=None):
        self.calls.append(("raw", center))
        return self._conv(x, y, w, blur)

    def grad_rows(self, kind, x, y, w, blur, grad_out, *, center=None):
        self.calls.append(("grad_rows", center))
        return self._grad(x, y, w, blur, grad_out)

    def value_and_grad_rows(self, kind, x, y, w, blur, *, center=None):
        self.calls.append(("value_and_grad_rows", center))
        return self._conv(x, y, w, blur), self._grad(x, y, w, blur, torch.ones(x.shape[:-1], **F64))

    def ops(self):
        return ops._ConvOps(self.raw, self.grad_rows, self.value_and_grad_rows)


def _conv_inputs(batched, seed=0):
    g = torch.Generator().manual_seed(seed)
    lead = (3,) if batched else ()
    return (_rand(g, *lead, 5, 4).requires_grad_(True), _rand(g, *lead, 6, 4).requires_grad_(True),
            _rand(g, *lead, 6).requires_grad_(True))


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("fused", [True, False], ids=["one-pass", "two-pass"])
def test_kernel_conv_gradients(batched, fused):
    x, y, w = _conv_inputs(batched)
    center = torch.rand(4, **F64)
    rows, cols = DenseConv(), DenseConv()

    def f(x, y, w):
        return ops._KernelConv.apply(rows.ops(), cols.ops(), x, y, w, "gaussian", 0.8, center, fused)

    torch.testing.assert_close(f(x, y, w), DenseConv._conv(x, y, w, 0.8))
    assert torch.autograd.gradcheck(f, (x, y, w))
    # the rows' operators serve the value and the x-gradient, the transposed problem's the y- and w-gradients
    rows.calls, cols.calls = [], []
    torch.autograd.grad(f(x, y, w).sum(), [x, y, w])
    assert [n for n, _ in rows.calls] == (["value_and_grad_rows"] if fused else ["raw", "grad_rows"])
    assert [n for n, _ in cols.calls] == ["grad_rows", "raw"]
    assert all(torch.equal(c, center) for _, c in rows.calls + cols.calls)


def test_kernel_conv_without_transposed_problem():
    x, y, w = _conv_inputs(False)
    rows = DenseConv().ops()
    for wants in ([y], [w]):
        out = ops._KernelConv.apply(rows, None, x, y, w, "gaussian", 0.8, None, False)
        with pytest.raises(RuntimeError, match="transposed"):
            torch.autograd.grad(out.sum(), wants)
    # the row gradient alone does not need it
    out = ops._KernelConv.apply(rows, None, x, y.detach(), w.detach(), "gaussian", 0.8, None, False)
    (gx,) = torch.autograd.grad(out.sum(), [x])
    assert gx.shape == x.shape


@pytest.mark.parametrize("public, batched", [("kernel_conv", False), ("kernel_conv_batched", True)])
@pytest.mark.parametrize("fused", [True, False], ids=["one-pass", "two-pass"])
def test_public_kernel_convs_bind_their_operators(monkeypatch, public, batched, fused):
    conv = DenseConv()
    suffix = "_batched" if batched else ""
    for name in ("raw", "grad_rows", "value_and_grad_rows"):
        monkeypatch.setattr(ops, f"kernel_conv{suffix}_{name}", getattr(conv, name))
    monkeypatch.setattr(ops, "FUSED_CONV_GRAD", fused)
    x, y, w = _conv_inputs(batched, seed=1)
    assert torch.autograd.gradcheck(lambda x, y, w: getattr(ops, public)("gaussian", x, y, w, 0.8), (x, y, w))
    # the one-pass evaluation serves a gaussian kernel whose row cloud needs a gradient; no laplacian or energy kernel
    for kind, one_pass in (("gaussian", fused), ("energy", False)):
        conv.calls = []
        getattr(ops, public)(kind, x, y, w, 0.8)
        assert conv.calls[0][0] == ("value_and_grad_rows" if one_pass else "raw")


def test_kernel_conv_ranges_binds_its_problems(monkeypatch):
    conv, prob, prob_t = DenseConv(), object(), object()
    seen = []

    def shard(kind_id, x, y, w, blur, prob_, *, center=None, backward=False):
        seen.append((prob_, backward))
        return conv.grad_rows(kind_id, x, y, w, blur, torch.ones(x.shape[0], **F64)) if backward else conv.raw(
            kind_id, x, y, w, blur)

    monkeypatch.setattr(ranges, "conv_shard_ranges", shard)
    monkeypatch.setattr(ranges, "conv_finalize", lambda kind_id, part: part)
    monkeypatch.setattr(ranges, "conv_bwd_finalize",
                        lambda kind_id, part, x, center, grad_out, blur: grad_out.unsqueeze(-1) * part)
    x, y, w = _conv_inputs(False, seed=2)
    assert torch.autograd.gradcheck(lambda x, y, w: ranges.kernel_conv_ranges(0, x, y, w, 0.8, prob, prob_t),
                                    (x, y, w))
    assert {s for s in seen if s[0] is prob} == {(prob, False), (prob, True)}
    assert {s for s in seen if s[0] is prob_t} == {(prob_t, False), (prob_t, True)}
    out = ranges.kernel_conv_ranges(0, x, y, w, 0.8, prob)
    with pytest.raises(RuntimeError, match="transposed"):
        torch.autograd.grad(out.sum(), [x, y, w])

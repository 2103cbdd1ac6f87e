"""The separable grid softmin (csrc/b200ot_grid.cu, grid_pass_kernel) against an fp64 reference of the same operator.

b200ot_softmin_grid is the only operator of sinkhorn_divergence on images and volumes and of ImagesBarycenter, forward
and backward.  One launch per axis, the last axis first; a CTA holds TW lines of the axis (32, or 16 when two 32-line
tiles of N x 33 floats exceed 227 KB of shared memory, i.e. N > 880: two half-warps then share a line), every thread
owns 8 consecutive outputs of a line and sweeps the inputs 8 at a time, the last chunk padded with -inf, on a lazy
running max that starts at the output's own term and rebases when a chunk sums past 2^64.

  A. 2-D at sides 1 ... 1024 around every chunk, tile and tile-width edge, both p, five temperatures down to a quarter
     pixel; dim = 1 through the C ABI at the same sides; lines per pass not a multiple of the tile width;
  B. 3-D: full outputs at small sides, sampled outputs on the 16-line tile at N = 881 and 1024;
  C. the h_b / h_scale_b fold, the out_old / alpha_old / beta epilogue, pixels at the -10000 floor, -inf pixels and a
     translated input;
  D. the lazy max: a plateau 60 log2 units up, then a spike 66, 140 or 300 units up at each position of a chunk, along
     every axis in turn, on both tile widths; the rebase must carry the plateau's sum;
  E. checks without a reference on full volumes: batch independence (bitwise), reflections and transpositions;
  F. the closed-form backward of barycenter_images._GridSoftmin against fp64 autograd;
  G. sinkhorn_divergence and ImagesBarycenter at sides the golden fixtures do not cover.

The reference (fp64_refs.grid_softmin64) runs in fp64 on the GPU, cross-checked against oracle.softmin_grid_dense on
the CPU (test_oracle_golden.py) and here.  Value bar: 3e-6 max(1, |ref|) per batch element, that of
test_gpu_parity.py::test_grid_softmin_vs_oracle.  The largest error-to-bar ratio per section, and the module's peak
device memory, are printed when the module ends.
"""
import math

import pytest
import torch

from fp64_refs import check, grid_softmin64, grid_softmin_grad64
from oracle import geomloss_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
VALUE_BAR = 3e-6
LN2 = math.log(2.0)

# 1, 2, 3, 5, 7: a single partial chunk; 8 .. 1024: one more or one less than a whole chunk, a power of two, or a
# tile-width edge: 880 is the largest side of the 32-line tile, 881 the smallest of the 16-line one
SIDES = [1, 2, 3, 5, 7, 8, 9, 15, 17, 31, 33, 63, 100, 127, 129, 255, 257, 513, 879, 880, 881, 1000, 1023, 1024]
LINES = 3  # batch x channel: 3 N lines in the last-axis pass, a multiple of 16 only when N is

RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    torch.cuda.init()
    torch.cuda.reset_peak_memory_stats(DEV)
    yield
    for sec in sorted(RATIOS):
        what, r = RATIOS[sec]
        print(f"\n[grid] section {sec}: largest error / bar = {r:.3g} ({what})")
    print(f"\n[grid] peak device memory {torch.cuda.max_memory_allocated(DEV) / 2**30:.2f} GiB "
          f"({torch.cuda.get_device_name(DEV)})")


def _temps(n, p):
    return (10.0, 1.0, (2.0 / n) ** p, (1.0 / n) ** p, (0.25 / n) ** p)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _elements(t, batch_dims):
    return t.reshape(math.prod(t.shape[:batch_dims]), -1)


def _check(sec, what, got, ref, batch_dims=2, factor=1.0):
    """|got - ref| <= factor VALUE_BAR max(1, |ref|) per batch element; infinite results must be equal, and no result
    may be NaN."""
    got, ref = _elements(got.double(), batch_dims), _elements(ref.double(), batch_dims).to(got.device)
    assert not bool(got.isnan().any()), what
    fin = torch.isfinite(ref)
    assert torch.equal(got[~fin], ref[~fin]), what
    got, ref = torch.where(fin, got, 0.0), torch.where(fin, ref, 0.0)
    bar = factor * VALUE_BAR * ref.abs().amax(dim=1).clamp_min(1.0)
    check(RATIOS, sec, what, got, ref, bar)
    return bar


def _softmin(eps, p, h, h_b=None, h_scale_b=0.0, **kw):
    """sinkhorn_images.softmin_grid, which must enqueue one launch per axis."""
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn_images import softmin_grid

    before = ops.launches()
    out = softmin_grid(eps, p, h, h_b, h_scale_b, **kw)
    assert ops.launches() - before == h.dim() - 2
    return out


def _softmin_1d(eps, p, h):
    """b200ot_softmin_grid at dim = 1 (the Python wrapper serves 2 and 3 only): h (batch, N)."""
    from geomloss_b200 import ops

    out = torch.empty_like(h)
    before = ops.launches()
    ops._call(h.device, "b200ot_softmin_grid", h, None, 0.0, None, 0.0, 1.0, out, h.shape[0], h.shape[1], 1, int(p),
              float(eps), launches=1)
    assert ops.launches() - before == 1
    return out


def _ref(eps, p, h, dim=None, rows=None):
    dim = h.dim() - 2 if dim is None else dim
    return grid_softmin64(eps, p, h, dim, rows=rows, device=DEV)


def _sample(t, rows):
    for axis, r in enumerate(rows):
        t = t.index_select(t.dim() - len(rows) + axis, torch.as_tensor(r, device=t.device))
    return t


def test_gpu_reference_matches_the_cpu_oracle():
    from test_oracle_golden import grid64_vs_oracle

    assert grid64_vs_oracle(DEV) <= 1e-11


# ------------------------------------------------------------------------------------------------------
# A. side lengths and tile widths
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("n", SIDES)
def test_sides_2d_and_1d(n, p):
    g = _gen(10 * n + p)
    h = torch.randn(LINES, 1, n, n, device=DEV, generator=g) * 2.0
    h1 = torch.randn(37, n, device=DEV, generator=g) * 2.0  # 37 lines: a partial tile of 5 on both tile widths
    for eps in _temps(n, p):
        _check("A", f"2-D N={n} p={p} eps={eps:.3g}", _softmin(eps, p, h), _ref(eps, p, h))
        _check("A", f"1-D N={n} p={p} eps={eps:.3g}", _softmin_1d(eps, p, h1), _ref(eps, p, h1, 1), 1)


# ------------------------------------------------------------------------------------------------------
# B. 3-D
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("n", [5, 17, 33, 64])
def test_volumes_full(n, p):
    h = torch.randn(LINES, 1, n, n, n, device=DEV, generator=_gen(20 * n + p)) * 2.0
    for eps in (1.0, (2.0 / n) ** p, (0.25 / n) ** p):
        _check("B", f"3-D N={n} p={p} eps={eps:.3g}", _softmin(eps, p, h), _ref(eps, p, h))


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("n", [881, 1024])
def test_volumes_16_line_tile_sampled(n, p):
    """One volume (2.7 GB at 881^3, 4.3 GB at 1024^3) on 8 sampled indices per axis, the first and last included."""
    g = _gen(30 * n + p)
    h = torch.randn(1, 1, n, n, n, device=DEV, generator=g) * 2.0
    rows = []
    for _ in range(3):
        r = torch.randint(1, n - 1, (8,), device=DEV, generator=g)
        r[0], r[-1] = 0, n - 1
        rows.append(r)
    for eps in (1.0, (2.0 / n) ** p, (0.5 / n) ** p):
        out = _softmin(eps, p, h)
        _check("B", f"3-D N={n} p={p} eps={eps:.3g}", _sample(out, rows), _ref(eps, p, h, rows=rows))
        del out


# ------------------------------------------------------------------------------------------------------
# C. epilogue and inputs
# ------------------------------------------------------------------------------------------------------
C_SHAPES = [(LINES, 1, 33, 33), (2, 1, 881, 881), (LINES, 1, 17, 17, 17)]


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("shape", C_SHAPES, ids=["x".join(map(str, s)) for s in C_SHAPES])
def test_epilogue_and_inputs(shape, p):
    n, dim = shape[-1], len(shape) - 2
    g = _gen(sum(shape) + p)
    h = torch.randn(*shape, device=DEV, generator=g) * 2.0
    h_b = torch.randn(*shape, device=DEV, generator=g)
    old = torch.randn(*shape, device=DEV, generator=g)
    for eps in (1.0, (2.0 / n) ** p):
        tag = f"{shape} p={p} eps={eps:.3g}"
        # the fold h_a + h_scale_b h_b, with h_scale_b other than 1 / eps
        ref = _ref(eps, p, h.double() + 0.37 * h_b.double())
        _check("C", f"{tag} h_b fold", _softmin(eps, p, h, h_b, 0.37), ref)
        # alpha_old out_old + beta softmin, with and without out_old (alpha_old is then ignored)
        out = _softmin(eps, p, h, h_b, 0.37, out_old=old, alpha_old=0.5, beta=0.4)
        _check("C", f"{tag} out_old, alpha_old, beta", out, 0.5 * old.double() + 0.4 * ref)
        out = _softmin(eps, p, h, h_b, 0.37, alpha_old=0.7, beta=-1.3)
        _check("C", f"{tag} beta, no out_old", out, -1.3 * ref)

        # the -10000 floor of log_dens: a line along the first and along the last axis, a line empty but for one
        # pixel, and in 3-D a slab at each end; an element empty but for one pixel; an element all at the floor
        hf = h.clone()
        hf[0, 0, 1] = -10000.0
        hf[0, 0, ..., 2] = -10000.0
        hf[0, 0, ..., 4, :] = -10000.0
        hf[0, 0, ..., 4, n // 2] = 0.5
        if dim == 3:
            hf[0, 0, :, 0] = -10000.0
            hf[0, 0, :, :, n - 1] = -10000.0
        hf[1] = -10000.0
        hf[1].view(-1)[(n ** dim) // 3] = 1.0
        if shape[0] > 2:
            hf[2] = -10000.0
        _check("C", f"{tag} floor pixels", _softmin(eps, p, hf), _ref(eps, p, hf))

        # -inf pixels: one in five, a whole last-axis line, an element all -inf (its output is +inf)
        hi = h.clone()
        hi[torch.rand(*shape, device=DEV, generator=g) < 0.2] = -math.inf
        hi[0, 0, ..., 3, :] = -math.inf
        hi[1] = -math.inf
        out = _softmin(eps, p, hi)
        ref = _ref(eps, p, hi)
        assert bool(torch.isinf(ref[1]).all()) and bool(torch.isfinite(ref[0]).all())
        _check("C", f"{tag} -inf pixels", out, ref)

        # a translated input: the output shifts by -eps c
        out = _softmin(eps, p, h)
        for c in (50.0, -3000.0):
            out_c = _softmin(eps, p, h + c)
            _check("C", f"{tag} translated by {c}", out_c, _ref(eps, p, h + c))
            _check("C", f"{tag} shifted by {-eps * c:.3g}", out_c, out.double() - eps * c, factor=2.0)


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("n", [1, 7, 9, 881])
def test_inf_lines_1d(n, p):
    """dim = 1: an all -inf line gives +inf, as -eps LSE does; a line of -inf but for one pixel; scattered -inf."""
    g = _gen(40 * n + p)
    h = torch.randn(5, n, device=DEV, generator=g) * 2.0
    h[0] = -math.inf
    h[1] = -math.inf
    h[1, n // 2] = 0.25
    h[2, torch.rand(n, device=DEV, generator=g) < 0.5] = -math.inf
    h[3] = -10000.0
    for eps in (1.0, (1.0 / n) ** p):
        out = _softmin_1d(eps, p, h)
        ref = _ref(eps, p, h, 1)
        assert bool((ref[0] == math.inf).all())
        _check("C", f"1-D N={n} p={p} eps={eps:.3g} -inf lines", out, ref, 1)


# ------------------------------------------------------------------------------------------------------
# D. lazy max
# ------------------------------------------------------------------------------------------------------
PLATEAU = 60.0  # log2 units: a chunk of 8 plateau terms sums to 2^63, below the 2^64 guard
SPIKES = (66.0, 140.0, 300.0)  # a rebase that must carry K 2^-6 ~ 1 spike; ex2 overflows to +inf; the carry underflows
EPS_D = {2: 4.0, 1: 8.0}  # the cost along a line stays below 0.2 log2 units
BASE_RUN, SPIKE_CHUNK = 16, 80  # base pixels [0, 16), plateau [16, 80 + q), the spike at 80 + q, base pixels after


def _lazy_levels(n, spikes, plateau=PLATEAU):
    """(len(spikes) x 8, n) log2 levels: line (s, q) holds spikes[s] at position q of the chunk [80, 88), after
    64 + q plateau pixels.  The base pixels, level 0, are the probes: their lazy max starts 60 units below the plateau
    and 66 or more below the spike."""
    lv = torch.zeros(len(spikes), 8, n, dtype=torch.float64)
    for q in range(8):
        lv[:, q, BASE_RUN:SPIKE_CHUNK + q] = plateau
        lv[:, q, SPIKE_CHUNK + q] = torch.tensor(spikes, dtype=torch.float64)
    return lv.reshape(-1, n)


def _along(levels, axis, dim):
    """(E, 1, N, .., N) natural-log input: each element's levels along ``axis``, constant along the other axes, so
    that the passes before the one along ``axis`` shift the pattern by a constant and it reaches its pass intact."""
    E, n = levels.shape
    view = [E, 1] + [n if a == axis else 1 for a in range(dim)]
    return (levels.reshape(view) * LN2).expand([E, 1] + [n] * dim).to(DEV, torch.float32).contiguous()


D_CASES = [(2, 256), (3, 256), (2, 1024)]  # 256: the 32-line tile; 1024: the 16-line tile


@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("dim,n", D_CASES, ids=[f"{d}d-{n}" for d, n in D_CASES])
def test_lazy_max_rebase(dim, n, p):
    eps = EPS_D[p]
    probe_rows = list(range(0, BASE_RUN)) + list(range(SPIKE_CHUNK, SPIKE_CHUNK + 16)) + list(range(n - 16, n))
    other_rows = [0, n // 2 + 1, n - 1]
    spiked = _lazy_levels(n, SPIKES)
    no_spike = _lazy_levels(n, (0.0,) * len(SPIKES))
    no_plateau = _lazy_levels(n, SPIKES, plateau=0.0)
    for axis in range(dim):
        rows = [probe_rows if a == axis else other_rows for a in range(dim)]
        h = _along(spiked, axis, dim)
        out = _sample(_softmin(eps, p, h), rows)
        ref = _ref(eps, p, h, rows=rows)
        what = f"{dim}-D N={n} p={p} pattern along axis {axis}"
        bar = _check("D", what, out, ref)
        # negative controls: without the spike every element misses; at S = 66 so does every element without the
        # plateau, whose sum the rebase carries
        miss = (_elements(out.double(), 2) - _elements(_ref(eps, p, _along(no_spike, axis, dim), rows=rows), 2))
        assert bool((miss.abs().amax(1) >= 10 * bar).all()), what
        miss = (_elements(out.double(), 2) - _elements(_ref(eps, p, _along(no_plateau, axis, dim), rows=rows), 2))
        assert bool((miss.abs().amax(1)[:8] >= 10 * bar[:8]).all()), what


# ------------------------------------------------------------------------------------------------------
# E. checks without a reference, on full volumes
# ------------------------------------------------------------------------------------------------------
E_BATCH = [(2, 100), (2, 881), (2, 1024), (3, 33)]


@pytest.mark.parametrize("dim,n", E_BATCH, ids=[f"{d}d-{n}" for d, n in E_BATCH])
def test_batch_independence(dim, n):
    """Each of 37 batch x channel elements run alone equals, bit for bit, its slice of the batched call: no line leaks
    into another through a partial tile."""
    h = torch.randn(37, 1, *([n] * dim), device=DEV, generator=_gen(50 * n + dim)) * 2.0
    for p, eps in ((2, (2.0 / n) ** 2), (1, 1.0 / n)):
        out = _softmin(eps, p, h)
        for e in range(37):
            assert torch.equal(_softmin(eps, p, h[e:e + 1]), out[e:e + 1]), (dim, n, p, e)


def _max_diff_by_slab(out, moved, flip_axis=None):
    """max |moved' - out|, moved' = moved flipped along ``flip_axis`` (None: moved itself), one slab of the first grid
    axis at a time: neither the flip of a 2.7 GB volume nor the difference is formed whole."""
    n, worst = out.shape[2], 0.0
    for s in range(n):
        if flip_axis == 2:
            m = moved[:, :, n - 1 - s]
        elif flip_axis is None:
            m = moved[:, :, s]
        else:
            m = moved[:, :, s].flip(flip_axis - 1)
        worst = max(worst, (m - out[:, :, s]).abs().max().item())
    return worst


E_SYM = [(2, 881), (2, 1024), (3, 100), (3, 881)]


@pytest.mark.parametrize("dim,n", E_SYM, ids=[f"{d}d-{n}" for d, n in E_SYM])
def test_reflections_and_transpositions(dim, n):
    """The cost is symmetric under x -> 1 - 1/N - x and under exchanging two axes, so the softmin commutes with
    flips and transpositions, within twice the value bar (a flip moves the chunk boundaries: not bitwise)."""
    B = 1 if n > 500 and dim == 3 else 2
    h = torch.randn(B, 1, *([n] * dim), device=DEV, generator=_gen(60 * n + dim)) * 2.0
    for p, eps in ((2, (2.0 / n) ** 2), (1, 1.0 / n)):
        out = _softmin(eps, p, h)
        bar = 2 * VALUE_BAR * max(1.0, out.abs().max().item())
        for axis in range(2, 2 + dim):
            moved = _softmin(eps, p, h.flip(axis))
            err = _max_diff_by_slab(out, moved, flip_axis=axis)
            del moved
            check(RATIOS, "E", f"{dim}-D N={n} p={p} flip axis {axis - 2}", torch.tensor(err), torch.tensor(0.0), bar)
        for a, b in ((2, 3), (2, 4), (3, 4))[:1 if dim == 2 else 3]:
            moved = _softmin(eps, p, h.transpose(a, b).contiguous())
            err = _max_diff_by_slab(out, moved.transpose(a, b))
            del moved
            check(RATIOS, "E", f"{dim}-D N={n} p={p} transpose {a - 2},{b - 2}", torch.tensor(err),
                  torch.tensor(0.0), bar)
        del out


# ------------------------------------------------------------------------------------------------------
# F. the closed-form backward
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1, 2])
@pytest.mark.parametrize("n", [16, 33, 64])
def test_closed_form_backward(n, p):
    """barycenter_images._GridSoftmin's gradient against fp64 autograd through oracle.softmin_grid_dense, within the
    allowance the value bar implies (fp64_refs.grid_softmin_grad64).  The upstream gradient is signed with exact
    zeros; h has a floor region and scattered floor pixels.  Negative control: the reference without the negative
    part of the upstream gradient misses by 10x."""
    from geomloss_b200.barycenter_images import _GridSoftmin

    g = _gen(70 * n + p)
    h = torch.randn(LINES, 1, n, n, device=DEV, generator=g)
    h[0, 0, : n // 4] = -10000.0
    h[1][torch.rand(1, n, n, device=DEV, generator=g) < 0.1] = -10000.0
    go = torch.randn(LINES, 1, n, n, device=DEV, generator=g)
    go[torch.rand(LINES, 1, n, n, device=DEV, generator=g) < 0.3] = 0.0
    for eps in (1.0, (2.0 / n) ** p, (1.0 / n) ** p):
        hr = h.clone().requires_grad_(True)
        (got,) = torch.autograd.grad(_GridSoftmin.apply(hr, eps, p), hr, go)
        ref, allow = grid_softmin_grad64(eps, p, h, go, VALUE_BAR, device=DEV)
        bar = allow.reshape(-1) + torch.finfo(torch.float32).tiny  # fp32 resolves nothing below its smallest normal
        what = f"N={n} p={p} eps={eps:.3g}"
        check(RATIOS, "F", what, got.reshape(-1), ref.reshape(-1), bar)
        bad, _ = grid_softmin_grad64(eps, p, h, go.clamp_min(0.0), VALUE_BAR, device=DEV)
        assert ((got.double() - bad).abs().reshape(-1) / bar).max().item() >= 10, what


# ------------------------------------------------------------------------------------------------------
# G. drivers
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 1, 128, 128), (1, 1, 64, 64, 64)], ids=["2d-128", "3d-64"])
def test_image_divergence_at_new_sides(shape):
    """sinkhorn_divergence against oracle.sinkhorn_images (fp64, on the GPU): values and potentials, bars of
    test_gpu_parity.py::test_image_sinkhorn_vs_oracle."""
    from geomloss_b200 import sinkhorn_divergence

    g = _gen(len(shape) + shape[-1])
    a = torch.rand(*shape, device=DEV, generator=g) ** 3
    b = torch.rand(*shape, device=DEV, generator=g) ** 3
    a[..., :3] = 0.0
    a, b = a / a.sum(), b / b.sum()
    for kw in (dict(p=2), dict(p=2, reach=0.3, scaling=0.7), dict(p=1)):
        ref = O.sinkhorn_images(a.double(), b.double(), **kw)
        val = sinkhorn_divergence(a, b, **kw)
        assert val.shape == (shape[0],)
        assert ((val.double() - ref).abs() <= 2e-4 * ref.abs() + 1e-9).all(), (kw, val.tolist(), ref.tolist())
        Fr, Gr = O.sinkhorn_images(a.double(), b.double(), potentials=True, **kw)
        F, G = sinkhorn_divergence(a, b, potentials=True, **kw)
        for got, r in ((F, Fr), (G, Gr)):
            check(RATIOS, "G", f"{shape} {kw} potential", got.reshape(-1), r.reshape(-1),
                  1e-5 * max(1.0, r.abs().max().item()))


@pytest.mark.parametrize("p", [1, 2])
def test_images_barycenter_at_128(p):
    from geomloss_b200 import ImagesBarycenter
    from test_gpu_parity import _bary_inputs

    imgs, w = _bary_inputs(128, 3, 2, seed=128 + p)
    ref = O.images_barycenter(imgs.to(DEV).double(), w.to(DEV).double(), p=p, scaling_N=4)
    out = ImagesBarycenter(imgs.to(DEV), w.to(DEV), p=p, scaling_N=4)
    assert out.shape == (2, 1, 128, 128)
    check(RATIOS, "G", f"barycenter 128 p={p}", out.reshape(-1), ref.reshape(-1), 2e-4 * ref.max().item())

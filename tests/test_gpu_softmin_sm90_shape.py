"""The dense D = 3, 4 softmin shapes (csrc/b200ot_softmin.cu, `Variants`) against the fp64 oracle where they are
easiest to get wrong: a term that jumps far above a row's lazy running max at every column-pair position of a
32-pair chunk, with the last CTA's 128-thread x 4-row layout partly empty, and ragged last tiles at D = 4."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CHUNK_PAIRS = 32  # the longest dense chunk; every pair position of one is planted once
PRE_PAIRS = 256   # column pairs of a split that the max pre-pass reads (softmin.cuh)


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()  # fails loudly if libb200ot.so is missing: there is no fallback to test
    yield


@pytest.mark.parametrize("d", [3, 4])
@pytest.mark.parametrize("n", [4100, 4608, 5000])
@pytest.mark.parametrize("jump", [70.0, 140.0])
def test_stale_max_every_chunk_position(d, n, jump, monkeypatch):
    """One column whose log2-domain exponent exceeds every row's running max by more than `jump` (> 64: the chunk-sum
    guard must see it; > 127: beyond the exponent range of a float) is planted past the pre-pass, once per column-pair
    position of a chunk (alternating the column within the pair).  One column split, so the plant is never absorbed
    by the pre-pass of another split."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    monkeypatch.setenv("B200OT_FORCE_SPLITS", "1")
    m, eps = 4096, 0.5
    g = torch.Generator().manual_seed(n + 10 * d + int(jump))
    x = torch.rand(n, d, generator=g)
    y = torch.rand(m, d, generator=g)
    h = torch.rand(m, generator=g) - 0.5
    base = O.softmin_points(eps, x.double(), y.double(), h.double(), p=2, row_block=1024)
    # every cost is below d/2 / eps in natural units, every other term below max(h): this clears the running max by `jump`
    h_plant = float(h.max()) + d / (2 * eps) + (jump + 1.0) * math.log(2.0)
    xd, yd = x.to(DEV), y.to(DEV)
    center = ops.default_center(xd, yd)
    bad = []
    for pos in range(CHUNK_PAIRS):
        j = 2 * (2 * PRE_PAIRS + 3 * CHUNK_PAIRS + pos) + (pos & 1)
        hp = h.clone()
        hp[j] = h_plant
        # fp64 oracle: the base sum with column j replaced by the planted term
        col = O.softmin_points(eps, x.double(), y[j:j + 1].double(), torch.tensor([h_plant], dtype=torch.float64), p=2)
        old = O.softmin_points(eps, x.double(), y[j:j + 1].double(), h[j:j + 1].double(), p=2)
        lse = torch.logsumexp(torch.stack([-base / eps, -col / eps]), dim=0)
        lse = lse + torch.log1p(-torch.exp(-old / eps - lse))
        ref = (-eps * lse).numpy()
        out, _ = ops.softmin_raw(eps, xd, yd, hp.to(DEV), p=2, center=center)
        got = out.cpu().numpy()
        err = np.abs(got - ref).max() if np.isfinite(got).all() else float("inf")
        if not err <= 3e-6 * max(1.0, np.abs(ref).max()):
            bad.append((pos, err))
    assert not bad, f"positions with a wrong softmin (pair position, max abs error): {bad}"


@pytest.mark.parametrize("shape", [(4100, 4097, 4), (4100, 4128, 4), (4100, 4129, 4), (4100, 5120, 4), (5000, 8191, 4)])
def test_softmin_d4_big_shape_tile_edges(shape):
    """D = 4 with the last tile of the big shape cut to 1 / 1 / 2 / 32 chunks of 32 columns (and a whole tile), as the
    D = 3 cases of test_softmin_vs_oracle_shapes."""
    from geomloss_b200 import ops
    from oracle import geomloss_oracle as O

    n, m, d = shape
    g = torch.Generator().manual_seed(n * 7 + m)
    x = torch.rand(n, d, generator=g)
    y = torch.rand(m, d, generator=g) * 1.1 - 0.05
    h = torch.randn(m, generator=g) * 2.0 - np.log(m)
    for eps in (0.5, 0.01, 5e-4):
        ref = O.softmin_points(eps, x.double(), y.double(), h.double(), p=2, row_block=512).numpy()
        out, lse2 = ops.softmin_raw(eps, x.to(DEV), y.to(DEV), h.to(DEV), p=2,
                                    center=ops.default_center(x.to(DEV), y.to(DEV)), want_lse2=True)
        got = out.cpu().numpy()
        np.testing.assert_allclose(got, ref, atol=3e-6 * max(1.0, np.abs(ref).max()), err_msg=f"eps={eps}")
        np.testing.assert_allclose(-eps * np.log(2.0) * lse2.cpu().numpy(), got, rtol=1e-6, atol=1e-7)

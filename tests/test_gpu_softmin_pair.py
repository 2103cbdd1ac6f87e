"""The paired softmins (csrc/softmin_pair.cuh): the xy / yx updates of a Jacobi Sinkhorn iteration from one pass over
the pairs (ops.softmin_raw_many -> b200ot_softmin_fwd_pair) and the xx / yy updates over the unordered pairs (the
symmetric route of b200ot_softmin_fwd), against the unpaired path ($B200OT_PAIR=0) and the fp64 oracle; the range
check and its bit-identical recomputation; reproducibility."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    yield


def _ref(eps, x, y, h, out_old=None, alpha=0.0, beta=1.0):
    """alpha * out_old + beta * softmin_eps(x, y, h) in fp64, p = 2: -eps log sum_j exp(h_j - |x_i - y_j|^2 / 2eps)."""
    x, y, h = x.double(), y.double(), h.double()
    out = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
    for i in range(0, x.shape[0], 2048):
        c = ((x[i:i + 2048, None, :] - y[None]) ** 2).sum(-1) / 2
        out[i:i + 2048] = -eps * torch.logsumexp(h[None] - c / eps, dim=1)
    out = beta * out
    return out if out_old is None else out + alpha * out_old.double()


def _state(n, m, eps, seed, iters=3):
    """Clouds, log-weights and potentials after a few averaged Jacobi iterations (unpaired path)."""
    from geomloss_b200 import ops

    g = torch.Generator().manual_seed(seed)
    x, y = torch.rand(n, 3, generator=g).to(DEV), torch.rand(m, 3, generator=g).to(DEV)
    a_log = torch.full((n,), -math.log(n), device=DEV)
    b_log = torch.full((m,), -math.log(m), device=DEV)
    c = ops.default_center(x, y)
    f = ops.softmin_raw(eps, x, y, b_log, p=2, center=c)[0]
    gg = ops.softmin_raw(eps, y, x, a_log, p=2, center=c)[0]
    fa = ops.softmin_raw(eps, x, x, a_log, p=2, center=c)[0]
    for _ in range(iters):
        kw = dict(p=2, center=c, alpha_old=0.5, beta=0.5)
        f, gg = (ops.softmin_raw(eps, x, y, b_log, gg, 1 / eps, out_old=f, **kw)[0],
                 ops.softmin_raw(eps, y, x, a_log, f, 1 / eps, out_old=gg, **kw)[0])
        fa = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, out_old=fa, **kw)[0]
    return x, y, a_log, b_log, c, f, gg, fa


def _mirror_calls(eps, x, y, a_log, b_log, c, f, g, avg, want_lse2):
    kw = dict(p=2, center=c, alpha_old=0.5 if avg else 0.0, beta=0.5 if avg else 0.9, want_lse2=want_lse2)
    return [((eps, x, y, b_log, g, 1 / eps), dict(out_old=f, **kw)),
            ((eps, y, x, a_log, f, 1 / eps), dict(out_old=g, **kw))]


def _flags():
    """The recomputation flags of the last paired call: the first two int32 of its scratch."""
    from geomloss_b200 import ops

    buf = ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream, "softmin_pair")]
    return buf[:8].view(torch.int32).tolist()


def _run_many(calls, paired, monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR", "1" if paired else "0")
    res = ops.softmin_raw_many(calls)
    torch.cuda.synchronize()
    return res


@pytest.mark.parametrize("n,m", [(5000, 7300), (9000, 4500), (4096, 4096)])
@pytest.mark.parametrize("tiles", ["1", "64"])  # one tile per block (many blocks) / one block per axis
@pytest.mark.parametrize("avg,want_lse2", [(True, False), (False, True)])
def test_pair_matches_unpaired_and_fp64(n, m, tiles, avg, want_lse2, monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", tiles)
    eps = 0.01
    x, y, a_log, b_log, c, f, g, _ = _state(n, m, eps, seed=n + m)
    calls = _mirror_calls(eps, x, y, a_log, b_log, c, f, g, avg, want_lse2)
    assert ops.pair_plan(calls) == [(0, 1)]
    got = _run_many(calls, True, monkeypatch)
    assert _flags() == [0, 0]
    ref = _run_many(calls, False, monkeypatch)
    for (o, l), (ro, rl), (args, kw) in zip(got, ref, calls):
        assert torch.allclose(o, ro, rtol=0, atol=1e-6), (o - ro).abs().max()
        exact = _ref(eps, args[1], args[2], args[3] + args[4] / eps, kw["out_old"], kw["alpha_old"], kw["beta"])
        assert (o.double() - exact).abs().max() < 2e-6
        if want_lse2:
            assert torch.allclose(l, rl, rtol=0, atol=2e-4), (l - rl).abs().max()
        else:
            assert l is None


@pytest.mark.parametrize("n", [4096, 6000, 11000])
@pytest.mark.parametrize("tiles", ["1", "2", "64"])  # diagonal + off-diagonal blocks, uneven blocks, one block
def test_symmetric_matches_unpaired_and_fp64(n, tiles, monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", tiles)
    eps = 0.01
    x, _, a_log, _, c, _, _, fa = _state(n, 4096, eps, seed=n)
    kw = dict(p=2, center=c, out_old=fa, alpha_old=0.5, beta=0.5, want_lse2=True)
    monkeypatch.setenv("B200OT_PAIR", "1")
    got, lse2 = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, **kw)
    flag = ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream, "softmin")]
    assert flag[:4].view(torch.int32).item() == 0
    monkeypatch.setenv("B200OT_PAIR", "0")
    ref, rlse2 = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, **kw)
    assert torch.allclose(got, ref, rtol=0, atol=1e-6), (got - ref).abs().max()
    assert torch.allclose(lse2, rlse2, rtol=0, atol=2e-4)
    exact = _ref(eps, x, x, a_log + fa / eps, fa, 0.5, 0.5)
    assert (got.double() - exact).abs().max() < 2e-6


def test_symmetric_writes_every_slot_once(monkeypatch):
    """With the partial slots poisoned with NaN before the call, a slot the symmetric kernel misses shows up in the
    result (and a slot written twice by two blocks would differ from the fp64 sums)."""
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", "1")
    monkeypatch.setenv("B200OT_PAIR", "1")
    eps, n = 0.01, 7000
    x, _, a_log, _, c, _, _, fa = _state(n, 4096, eps, seed=3)
    ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, p=2, center=c)  # sizes the scratch
    ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream, "softmin")].fill_(0xFF)
    got = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, p=2, center=c)[0]
    assert torch.isfinite(got).all()
    assert (got.double() - _ref(eps, x, x, a_log + fa / eps)).abs().max() < 2e-6


@pytest.mark.parametrize("plant", ["zero_weight", "overflow", "moved"])
def test_fallback_is_bit_identical(plant, monkeypatch):
    from geomloss_b200 import ops

    eps, n, m = 0.01, 6000, 5000
    x, y, a_log, b_log, c, f, g, fa = _state(n, m, eps, seed=11)
    if plant == "zero_weight":  # log 0 of the engine: every term of that row underflows
        a_log = a_log.clone()
        a_log[17] = -100000.0
    elif plant == "overflow":  # one column whose h overflows 2^T
        g = g.clone()
        g[123] += 200.0 * eps
    else:  # potentials moved by about 100 nats in one step
        f = f + 100.0 * eps
        fa = fa + 100.0 * eps
    calls = _mirror_calls(eps, x, y, a_log, b_log, c, f, g, True, True)
    got = _run_many(calls, True, monkeypatch)
    flags = _flags()
    assert flags[0] == 1  # the planted row or potential reaches the rows' softmin in every case
    ref = _run_many(calls, False, monkeypatch)
    for (o, l), (ro, rl), flag in zip(got, ref, flags):
        if flag:  # recomputed on the unpaired path
            assert torch.equal(o, ro) and torch.equal(l, rl)
        else:
            assert torch.allclose(o, ro, rtol=0, atol=1e-6)
    if plant != "overflow":
        kw = dict(p=2, center=c, out_old=fa, alpha_old=0.5, beta=0.5)
        monkeypatch.setenv("B200OT_PAIR", "1")
        s = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, **kw)[0]
        assert ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream,
                                   "softmin")][:4].view(torch.int32).item() == 1
        monkeypatch.setenv("B200OT_PAIR", "0")
        assert torch.equal(s, ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, **kw)[0])


def test_reproducible(monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", "1")
    eps = 0.01
    x, y, a_log, b_log, c, f, g, fa = _state(8000, 6000, eps, seed=5)
    calls = _mirror_calls(eps, x, y, a_log, b_log, c, f, g, True, True)
    one, two = _run_many(calls, True, monkeypatch), _run_many(calls, True, monkeypatch)
    for (o1, l1), (o2, l2) in zip(one, two):
        assert torch.equal(o1, o2) and torch.equal(l1, l2)
    s1 = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, p=2, center=c)[0]
    s2 = ops.softmin_raw(eps, x, x, a_log, fa, 1 / eps, p=2, center=c)[0]
    assert torch.equal(s1, s2)


def test_pair_refuses_aliased_outputs():
    """The entry refuses an out that overlaps an input the recomputation would read."""
    from geomloss_b200 import _lib, ops

    L = _lib.lib()
    eps, n = 0.01, 5000
    x, y, a_log, b_log, c, f, g, _ = _state(n, n, eps, seed=2, iters=0)
    nbytes = L.b200ot_softmin_pair_scratch_bytes(n, n, 3)
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    out_b = torch.empty(n, device=DEV)
    args = lambda out_a: (p(x), p(y), p(b_log), p(g), 1 / eps, p(f), 0.5, 0.5, p(out_a), None, p(a_log), p(f),  # noqa
                          1 / eps, p(g), 0.5, 0.5, p(out_b), None, p(c), n, n, 3, 2, eps, p(scratch), nbytes, None)
    assert L.b200ot_softmin_fwd_pair(*args(f)) == -1
    assert L.b200ot_softmin_fwd_pair(*args(g)) == -1
    assert L.b200ot_softmin_fwd_pair(*args(out_b)) == -1
    assert L.b200ot_softmin_pair_scratch_bytes(100, 100, 3) == 0  # the small-problem shapes are not paired
    assert L.b200ot_softmin_pair_scratch_bytes(5000, 5000, 4) == 0
    del ops


def test_full_size_sampled_rows(monkeypatch):
    """N = M = 1e6 at the benchmark's inputs (uniform cube, blur = .01) after warm-up iterations: 64 sampled rows of
    each of the four paired updates against fp64, no worse than the unpaired path's error plus 1e-8, and the range
    check never fires."""
    from geomloss_b200 import ops
    from geomloss_b200.sinkhorn import softmin_many

    n, eps = 1_000_000, 1e-4
    g = torch.Generator().manual_seed(0)
    x, y = torch.rand(n, 3, generator=g).to(DEV), torch.rand(n, 3, generator=g).to(DEV)
    a_log = torch.full((n,), -math.log(n), device=DEV)
    b_log = a_log.clone()
    c = ops.default_center(x, y)
    monkeypatch.setenv("B200OT_PAIR", "0")
    pots = [ops.softmin_raw(eps, r, col, lw, p=2, center=c)[0] for r, col, lw in
            ((x, y, b_log), (y, x, a_log), (x, x, a_log), (y, y, b_log))]
    kw = dict(p=2, center=c, alpha_old=0.5, beta=0.5)

    def calls(pt):
        f, gg, fa, gb = pt
        return [((eps, x, y, b_log, gg, 1 / eps), dict(out_old=f, **kw)),
                ((eps, y, x, a_log, f, 1 / eps), dict(out_old=gg, **kw)),
                ((eps, x, x, a_log, fa, 1 / eps), dict(out_old=fa, **kw)),
                ((eps, y, y, b_log, gb, 1 / eps), dict(out_old=gb, **kw))]

    for _ in range(3):
        pots = [o for o, _ in softmin_many(ops.softmin_raw, calls(pots))]
    cl = calls(pots)
    monkeypatch.setenv("B200OT_PAIR", "1")
    got = [o for o, _ in softmin_many(ops.softmin_raw, cl)]
    assert _flags() == [0, 0]
    monkeypatch.setenv("B200OT_PAIR", "0")
    ref = [o for o, _ in softmin_many(ops.softmin_raw, cl)]
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:64].to(DEV)
    for o, r, (args, k) in zip(got, ref, cl):
        exact = _ref(eps, args[1][rows], args[2], args[3] + args[4] / eps, k["out_old"][rows], 0.5, 0.5)
        e_pair = (o[rows].double() - exact).abs().max().item()
        e_ref = (r[rows].double() - exact).abs().max().item()
        assert e_pair <= e_ref + 1e-8, (e_pair, e_ref)
        assert (o - r).abs().max().item() <= 1e-7

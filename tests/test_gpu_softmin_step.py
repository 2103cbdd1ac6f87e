"""The step group (ops.softmin_raw_many -> b200ot_softmin_fwd_step): the four softmins of a symmetric Jacobi Sinkhorn
iteration, the xy / yx pair and the xx, yy symmetric softmins, from one launch of the paired kernel.  Bit for
bit what one pair call and two symmetric calls compute; every partial slot written once; a softmin that fails the
range check recomputed alone; aliased outputs refused; reproducible."""
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


def _state(n, m, eps, seed):
    """Clouds, log-weights, center and the four potentials after two averaged Jacobi iterations, one call at a time."""
    from geomloss_b200 import ops

    g = torch.Generator().manual_seed(seed)
    x, y = torch.rand(n, 3, generator=g).to(DEV), torch.rand(m, 3, generator=g).to(DEV)
    a_log = torch.full((n,), -math.log(n), device=DEV)
    b_log = torch.full((m,), -math.log(m), device=DEV)
    c = ops.default_center(x, y)
    pots = [ops.softmin_raw(eps, r, col, lw, p=2, center=c)[0] for r, col, lw in
            ((x, y, b_log), (y, x, a_log), (x, x, a_log), (y, y, b_log))]
    for _ in range(2):
        pots = [o for o, _ in _calls_run(_calls(eps, x, y, a_log, b_log, c, pots, False), lambda cs: [
            ops.softmin_raw(*a, **k) for a, k in cs])]
    return x, y, a_log, b_log, c, pots


def _calls(eps, x, y, a_log, b_log, c, pots, want_lse2):
    f, g, fa, gb = pots
    kw = dict(p=2, center=c, alpha_old=0.5, beta=0.5, want_lse2=want_lse2)
    return [((eps, x, y, b_log, g, 1 / eps), dict(out_old=f, **kw)),
            ((eps, y, x, a_log, f, 1 / eps), dict(out_old=g, **kw)),
            ((eps, x, x, a_log, fa, 1 / eps), dict(out_old=fa, **kw)),
            ((eps, y, y, b_log, gb, 1 / eps), dict(out_old=gb, **kw))]


def _calls_run(calls, run):
    res = run(calls)
    torch.cuda.synchronize()
    return res


def _step(calls, monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR", "1")
    assert ops.step_plan(calls) == [(0, 1, 2, 3)]
    return _calls_run(calls, ops.softmin_raw_many)


def _separate(calls, monkeypatch):
    """The same four softmins as one pair call and two symmetric calls."""
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR", "1")
    return _calls_run(calls, lambda cs: ops.softmin_raw_many(cs[:2]) + [ops.softmin_raw(*a, **k) for a, k in cs[2:]])


def _flags():
    """The recomputation flags of the last step call: the first four int32 of its scratch."""
    from geomloss_b200 import ops

    buf = ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream, "softmin_pair")]
    return buf[:16].view(torch.int32).tolist()


def _fp64_rows(eps, x, y, h, out_old, rows):
    """0.5 out_old + 0.5 softmin_eps(x, y, h) in fp64 at the sampled rows."""
    xr, y, h = x[rows].double(), y.double(), h.double()
    c = ((xr[:, None, :] - y[None]) ** 2).sum(-1) / 2
    return 0.5 * out_old[rows].double() - 0.5 * eps * torch.logsumexp(h[None] - c / eps, dim=1)


@pytest.mark.parametrize("n,m", [(5000, 7300), (9000, 4500), (6000, 6000)])
@pytest.mark.parametrize("tiles", ["1", "2", "64"])  # many blocks / uneven blocks / one block per axis
def test_step_matches_pair_and_symmetric_calls(n, m, tiles, monkeypatch):
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", tiles)
    eps = 0.01
    x, y, a_log, b_log, c, pots = _state(n, m, eps, seed=n + 7 * m)
    calls = _calls(eps, x, y, a_log, b_log, c, pots, True)
    l0 = ops.launches()
    got = _step(calls, monkeypatch)
    assert ops.launches() - l0 == 21
    assert _flags() == [0, 0, 0, 0]
    ref = _separate(calls, monkeypatch)
    for (o, l), (ro, rl) in zip(got, ref):
        assert torch.equal(o, ro) and torch.equal(l, rl)
    rows = torch.randperm(min(n, m), generator=torch.Generator().manual_seed(1))[:32].to(DEV)
    for (o, _), (args, kw) in zip(got, calls):
        exact = _fp64_rows(eps, args[1], args[2], args[3] + args[4] / eps, kw["out_old"], rows)
        assert (o[rows].double() - exact).abs().max() < 2e-6


def test_many_items_per_cta_write_every_slot_once(monkeypatch):
    """N = M = 65000 at one tile per block: 64 blocks per axis, 4096 + 2 x 2080 = 8256 items of three problems in one
    launch, many waves of CTAs.  With the partial slots poisoned with NaN before the call, a slot no item writes shows
    up in the result, and one written by two items differs from the separate calls."""
    from geomloss_b200 import ops

    monkeypatch.setenv("B200OT_PAIR_TILES", "1")
    eps, n = 0.01, 65000
    x, y, a_log, b_log, c, pots = _state(n, n, eps, seed=4)
    calls = _calls(eps, x, y, a_log, b_log, c, pots, False)
    _step(calls, monkeypatch)  # sizes the scratch
    ops._scratch_cache[(torch.device(DEV), torch.cuda.current_stream(DEV).cuda_stream, "softmin_pair")].fill_(0xFF)
    got = _step(calls, monkeypatch)
    assert _flags() == [0, 0, 0, 0]
    ref = _separate(calls, monkeypatch)
    for (o, _), (ro, _) in zip(got, ref):
        assert torch.isfinite(o).all()
        assert torch.equal(o, ro)


def test_only_the_failing_softmin_is_recomputed(monkeypatch):
    """f_aa, which only the xx softmin reads (its potential and its old value), moved by 100 nats: the xx sums leave
    the paired range, xx alone is recomputed on the unpaired path, bit for bit; the other three keep their paired
    results."""
    from geomloss_b200 import ops

    eps = 0.01
    x, y, a_log, b_log, c, pots = _state(6000, 5000, eps, seed=11)
    pots[2] = pots[2] + 100.0 * eps
    calls = _calls(eps, x, y, a_log, b_log, c, pots, True)
    got = _step(calls, monkeypatch)
    assert _flags() == [0, 0, 1, 0]
    paired = _separate(calls, monkeypatch)
    monkeypatch.setenv("B200OT_PAIR", "0")
    unpaired = _calls_run(calls, ops.softmin_raw_many)
    for k, ((o, l), (po, pl), (uo, ul)) in enumerate(zip(got, paired, unpaired)):
        if k == 2:
            assert torch.equal(o, uo) and torch.equal(l, ul)
        else:
            assert torch.equal(o, po) and torch.equal(l, pl)


def test_step_refuses_aliased_outputs():
    """The entry refuses an output that overlaps an input of any of the four softmins or another output."""
    from geomloss_b200 import _lib

    L = _lib.lib()
    eps, n, m = 0.01, 5000, 4500
    x, y, a_log, b_log, c, (f, g, fa, gb) = _state(n, m, eps, seed=2)
    nbytes = L.b200ot_softmin_step_scratch_bytes(n, m, 3)
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    outs = [torch.empty(k, device=DEV) for k in (n, m, n, m)]

    def run(out):
        slots = (_lib.SoftminSlot * 4)()
        for s, h_a, h_b, old, o in zip(slots, (b_log, a_log, a_log, b_log), (g, f, fa, gb), (f, g, fa, gb), out):
            s.h_a, s.h_b, s.h_scale_b, s.out_old, s.alpha_old, s.beta = h_a.data_ptr(), h_b.data_ptr(), 1 / eps, \
                old.data_ptr(), 0.5, 0.5
            s.out, s.lse2 = o.data_ptr(), None
        rc = L.b200ot_softmin_fwd_step(x.data_ptr(), y.data_ptr(), slots, c.data_ptr(), n, m, 3, 2, eps,
                                       scratch.data_ptr(), nbytes, None)
        torch.cuda.synchronize()
        return rc

    assert run(outs) == 0
    assert run([outs[0], outs[1], f, outs[3]]) == -1  # xx writes the xy softmin's old value
    assert run([outs[0], outs[1], outs[2], g]) == -1  # yy writes the potential the xy softmin reads
    assert run([outs[0], outs[1], outs[2], outs[1]]) == -1  # two softmins write one output
    assert run([outs[0], outs[1], x.view(-1)[:n], outs[3]]) == -1  # xx overwrites its own cloud
    assert L.b200ot_softmin_step_scratch_bytes(100, 100, 3) == 0  # the small-problem shapes are not paired
    assert L.b200ot_softmin_step_scratch_bytes(5000, 100, 3) == 0
    assert L.b200ot_softmin_step_scratch_bytes(5000, 5000, 4) == 0


def test_step_reproducible(monkeypatch):
    monkeypatch.setenv("B200OT_PAIR_TILES", "1")
    eps = 0.01
    x, y, a_log, b_log, c, pots = _state(8000, 6000, eps, seed=5)
    calls = _calls(eps, x, y, a_log, b_log, c, pots, True)
    one, two = _step(calls, monkeypatch), _step(calls, monkeypatch)
    for (o1, l1), (o2, l2) in zip(one, two):
        assert torch.equal(o1, o2) and torch.equal(l1, l2)

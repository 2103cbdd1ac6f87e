"""Which softmin calls of one Jacobi iteration ops.softmin_raw_many runs as one paired launch group (CPU only: the plan
looks at the arguments alone)."""
import torch

from geomloss_b200 import ops


def _calls(n=50, m=40, d=3):
    g = torch.Generator().manual_seed(0)
    x, y = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g)
    a_log, b_log = torch.zeros(n), torch.zeros(m)
    f, gg, fa, gb = torch.zeros(n), torch.zeros(m), torch.zeros(n), torch.zeros(m)
    c = torch.zeros(d)
    kw = dict(p=2, center=c, alpha_old=0.5, beta=0.5)
    return [((0.1, x, y, b_log, gg, 10.0), dict(out_old=f, **kw)),
            ((0.1, y, x, a_log, f, 10.0), dict(out_old=gg, **kw)),
            ((0.1, x, x, a_log, fa, 10.0), dict(out_old=fa, **kw)),
            ((0.1, y, y, b_log, gb, 10.0), dict(out_old=gb, **kw))]


def test_mirror_pair_and_self_calls():
    # the xy / yx updates pair; the self updates run alone (the library evaluates their unordered pairs once)
    assert ops.pair_plan(_calls()) == [(0, 1), (2,), (3,)]
    c = _calls()
    assert ops.pair_plan([c[2], c[1], c[3], c[0]]) == [(0,), (1, 3), (2,)]


def test_detached_views_pair():
    # the Sinkhorn loop hands over clouds detached per slot: new tensor objects on the same data
    c = _calls()
    x, y = c[0][0][1], c[0][0][2]
    c[0] = ((0.1, x.detach(), y.detach()) + c[0][0][3:], c[0][1])
    c[1] = ((0.1, y.detach(), x.detach()) + c[1][0][3:], c[1][1])
    assert ops.pair_plan(c) == [(0, 1), (2,), (3,)]
    c[1] = ((0.1, y.detach(), x[:, :2].detach()) + c[1][0][3:], c[1][1])  # another view of x is another cloud
    assert ops.pair_plan(c) == [(0,), (1,), (2,), (3,)]


def test_not_paired():
    def plan(edit):
        c = _calls()
        edit(c)
        return ops.pair_plan(c)

    def kw1(**k):
        return lambda c: c[1][1].update(k)

    alone = [(0,), (1,), (2,), (3,)]
    assert plan(lambda c: c.__setitem__(1, ((0.2,) + c[1][0][1:], c[1][1]))) == alone  # another eps
    assert plan(kw1(center=torch.zeros(3))) == alone  # another center
    assert plan(kw1(p=1)) == alone
    assert plan(lambda c: [kw.update(p=2 | ops.P_UNCLAMPED) for _, kw in c]) == alone
    assert ops.pair_plan(_calls(d=2)) == alone
    assert ops.pair_plan(_calls(d=4)) == alone
    # an output that overlaps an input the recomputation would read, or the other output
    assert plan(lambda c: c[0][1].update(out=c[0][1]["out_old"])) == alone
    assert plan(lambda c: c[0][1].update(out=c[1][0][4])) == alone
    assert plan(lambda c: c[0][1].update(out=c[1][1]["out_old"])) == alone
    shared = torch.zeros(50)
    assert plan(lambda c: (c[0][1].update(out=shared), c[1][1].update(out=shared))) == alone
    # distinct fresh outputs are fine
    assert plan(lambda c: (c[0][1].update(out=torch.zeros(50)), c[1][1].update(out=torch.zeros(40)))) == \
        [(0, 1), (2,), (3,)]

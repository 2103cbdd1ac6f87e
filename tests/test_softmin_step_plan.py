"""Which softmin calls of one Jacobi iteration ops.softmin_raw_many runs as one step group: the mirrored pair and the
symmetric softmins of its two clouds (CPU only: the plan looks at the arguments alone)."""
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


def test_step_group():
    c = _calls()
    assert ops.step_plan(c) == [(0, 1, 2, 3)]
    assert ops.pair_plan(c) == [(0, 1), (2,), (3,)]  # the pair plan underneath is unchanged
    # any call order: the group's first call is the pair's first, then its mirror, the self call on the first call's
    # rows and the one on its columns, at the place of the pair
    assert ops.step_plan([c[3], c[2], c[1], c[0]]) == [(2, 3, 0, 1)]
    assert ops.step_plan([c[2], c[1], c[3], c[0]]) == [(1, 3, 2, 0)]


def test_detached_views_group():
    # the Sinkhorn loop hands over clouds detached per slot: new tensor objects on the same data
    c = _calls()
    x, y = c[0][0][1], c[0][0][2]
    for k, (r, col) in enumerate(((x, y), (y, x), (x, x), (y, y))):
        c[k] = ((0.1, r.detach(), col.detach()) + c[k][0][3:], c[k][1])
    assert ops.step_plan(c) == [(0, 1, 2, 3)]


def test_not_a_step_group():
    def plan(edit):
        c = _calls()
        edit(c)
        return ops.step_plan(c)

    def kw(k, **upd):
        return lambda c: c[k][1].update(upd)

    pair = [(0, 1), (2,), (3,)]
    assert ops.step_plan(_calls()[:3]) == [(0, 1), (2,)]  # one self call missing
    assert plan(lambda c: c.__setitem__(2, ((0.2,) + c[2][0][1:], c[2][1]))) == pair  # another eps
    assert plan(kw(3, center=torch.zeros(3))) == pair  # another center
    assert plan(kw(2, p=1)) == pair
    assert plan(lambda c: c.__setitem__(2, ((0.1, c[2][0][1], c[2][0][1][:, :2].contiguous()) + c[2][0][3:],
                                            c[2][1]))) == pair  # not the symmetric softmin of x
    x2 = _calls()[0][0][1].clone()
    assert plan(lambda c: c.__setitem__(2, ((0.1, x2, x2) + c[2][0][3:], c[2][1]))) == pair  # a copy of x is another cloud
    # an output of the four that overlaps an input of any of them, or another output
    assert plan(lambda c: c[2][1].update(out=c[0][0][1])) == pair  # overwrites a cloud
    assert plan(lambda c: c[2][1].update(out=c[0][1]["out_old"])) == pair
    assert plan(lambda c: c[3][1].update(out=c[0][0][4])) == pair
    shared = torch.zeros(50)
    assert plan(lambda c: (c[0][1].update(out=shared), c[2][1].update(out=shared))) == pair
    assert ops.step_plan(_calls(d=2)) == [(0,), (1,), (2,), (3,)]
    # distinct fresh outputs are fine
    assert plan(lambda c: [kw_.update(out=torch.zeros(len(args[1]))) for args, kw_ in c]) == [(0, 1, 2, 3)]


def test_two_iterations_in_one_list():
    c = _calls() + _calls()
    assert ops.step_plan(c) == [(0, 1, 2, 3), (4, 5, 6, 7)]

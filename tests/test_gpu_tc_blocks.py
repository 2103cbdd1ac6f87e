"""Block-sparse softmins on the tensor cores (8 < D <= 64; ranges.build_problem(variant=TC), b200ot_*_blocks) and the
labelled two-scale Sinkhorn they serve above D = 8.

  * operator values and row gradients against an fp64 softmin restricted to the kept blocks: random masks, a row cluster
    that keeps nothing, cluster sizes 1 / 127 / 128 / 129 / a few hundred, default, 1 and 3 forced column splits;
  * keep = everything: the dense tensor-core softmin, to 2e-6 relative;
  * D = 8 clouds zero-padded to D = 16 (every distance unchanged): the CUDA-core ranges path at D = 8 on the same
    problem, empty rows included, and zero gradients in the padded columns;
  * whole labelled losses against the reference fixtures tests/golden/labels_hd_*.npz (bars of the ms_sinkhorn_*
    fixtures in test_gpu_reference_goldens.py);
  * one fine-phase softmin is the same few launches whatever the number of clusters.
"""
import numpy as np
import pytest
import torch

from conftest import golden_kwargs, golden_names, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module", autouse=True)
def _lib_loaded():
    from geomloss_b200 import _lib

    _lib.lib()
    yield


def _clusters(seed, D, row_sizes, col_sizes, density=0.5, empty_row=True):
    """Clouds whose clusters are contiguous (label-sorted order), their cluster sizes and a random keep matrix."""
    g = torch.Generator().manual_seed(seed)
    rc, cc = torch.tensor(row_sizes), torch.tensor(col_sizes)
    R, C = len(row_sizes), len(col_sizes)
    cen = torch.rand(max(R, C), D, generator=g) * 0.8
    x = cen[torch.repeat_interleave(torch.arange(R), rc)] + 0.3 * torch.rand(int(rc.sum()), D, generator=g)
    y = cen[torch.repeat_interleave(torch.arange(C), cc)] + 0.3 * torch.rand(int(cc.sum()), D, generator=g)
    keep = torch.rand(R, C, generator=g) < density
    if empty_row:
        keep[1] = False
    keep[0] = True
    return x, y, rc, cc, keep


def _masked_softmin64(eps, x, y, h, keep_pairs):
    """fp64: out_i = -eps log sum_{j kept} exp(h_j - |x_i - y_j|^2 / (2 eps)), and the softmax weights."""
    x, y, h = x.double().cpu(), y.double().cpu(), h.double().cpu()
    t = h[None, :] - torch.cdist(x, y) ** 2 / (2 * eps)
    t = torch.where(keep_pairs, t, torch.full_like(t, -float("inf")))
    lse = torch.logsumexp(t, dim=1)
    w = torch.softmax(t, dim=1).nan_to_num(0.0)
    return -eps * lse, w


def _pairs(keep, rc, cc):
    return keep[torch.repeat_interleave(torch.arange(len(rc)), rc)][:, torch.repeat_interleave(torch.arange(len(cc)), cc)]


@pytest.mark.parametrize("D", [9, 16, 33, 64])
@pytest.mark.parametrize("splits", ["default", "1", "3"])
def test_operator_against_fp64(D, splits, monkeypatch):
    from geomloss_b200 import ops, ranges

    if splits != "default":
        monkeypatch.setenv("B200OT_FORCE_SPLITS", splits)
    row_sizes = [1, 300, 127, 128, 129, 40, 257]
    col_sizes = [129, 1, 128, 300, 127, 70, 400, 5, 260]
    x, y, rc, cc, keep = _clusters(D, D, row_sizes, col_sizes)
    eps = 0.1
    g = torch.Generator().manual_seed(100 + D)
    b_log = (torch.rand(len(y), generator=g) - 0.5)
    pot = torch.rand(len(y), generator=g) * 0.2
    prob = ranges.build_problem(keep.to(DEV), rc.to(DEV), ranges.ColumnLayout(cc.to(DEV), align=128),
                                variant=ranges.TC)
    xd, yd, hd, pd = x.to(DEV), y.to(DEV), b_log.to(DEV), pot.to(DEV)
    center = ops.default_center(xd, yd)
    old = torch.rand(len(x), generator=g).to(DEV)
    out, lse2 = ranges.softmin_ranges_raw(eps, xd, yd, hd, pd, 1.0 / eps, prob, p=2 | ops.P_UNCLAMPED, center=center,
                                          out_old=old, alpha_old=0.5, beta=0.7, want_lse2=True)
    pairs = _pairs(keep, rc, cc)
    ref, w = _masked_softmin64(eps, x, y, b_log + pot / eps, pairs)
    live = pairs.any(1)
    assert not bool(live.all())  # a row cluster keeps nothing
    want = 0.5 * old.double().cpu() + 0.7 * ref
    got = out.double().cpu()
    err = (got[live] - want[live]).abs().max().item()
    assert err <= 1e-5 * (1 + want[live].abs().max().item()), err
    assert bool(torch.isinf(got[~live]).all())  # no column at all: -eps log 0, as the CUDA-core ranges path gives
    # row gradient through the autograd wrapper (scale_out folded into the upstream gradient)
    xg = xd.clone().requires_grad_(True)
    val = ranges.softmin_ranges(eps, xg, yd, hd, pd, 1.0 / eps, prob, p=2, center=center, scale_out=0.7)
    go = torch.rand(len(x), generator=g).to(DEV)
    (gx,) = torch.autograd.grad(val, xg, go)
    gref = 0.7 * go.double().cpu()[:, None] * (x.double() - w @ y.double())
    gerr = (gx.double().cpu()[live] - gref[live]).abs().max().item()
    assert gerr <= 5e-5 * max(1.0, gref[live].abs().max().item()), gerr


@pytest.mark.parametrize("D", [16, 64])
def test_keep_all_matches_the_dense_tensor_core_softmin(D):
    from geomloss_b200 import ops, ranges

    x, y, rc, cc, keep = _clusters(7, D, [300, 1, 129, 128, 400], [127, 260, 1, 500, 90], empty_row=False)
    keep[:] = True
    prob = ranges.build_problem(keep.to(DEV), rc.to(DEV), ranges.ColumnLayout(cc.to(DEV), align=128),
                                variant=ranges.TC)
    xd, yd = x.to(DEV), y.to(DEV)
    h = (torch.rand(len(y)) - 0.5).to(DEV)
    center = ops.default_center(xd, yd)
    for eps in (0.05, 0.5):
        blk, _ = ranges.softmin_ranges_raw(eps, xd, yd, h, None, 0.0, prob, p=2, center=center)
        dense, _ = ops.softmin_raw(eps, xd, yd, h, p=2, center=center)
        # relative to the largest value: single rows near zero would turn rounding into large ratios
        rel = ((blk - dense).abs().max() / dense.abs().max()).item()
        assert rel <= 2e-6, (eps, rel)


def test_matches_the_cuda_core_ranges_path_at_d8_padded_to_16():
    """Zero-padding D = 8 clouds to D = 16 leaves every distance unchanged: the tensor-core block path at D = 16 and
    the CUDA-core ranges path at D = 8 compute the same softmin on the same blocks, empty rows included."""
    from geomloss_b200 import ops, ranges

    x, y, rc, cc, keep = _clusters(11, 8, [1, 300, 127, 129, 60], [128, 1, 200, 129, 33, 90], density=0.5)
    xd, yd = x.to(DEV), y.to(DEV)
    xp = torch.cat([xd, torch.zeros(len(x), 8, device=DEV)], 1).contiguous()
    yp = torch.cat([yd, torch.zeros(len(y), 8, device=DEV)], 1).contiguous()
    h = (torch.rand(len(y)) - 0.5).to(DEV)
    ke, rcd, ccd = keep.to(DEV), rc.to(DEV), cc.to(DEV)
    simt = ranges.build_problem(ke, rcd, ranges.ColumnLayout(ccd))
    tc = ranges.build_problem(ke, rcd, ranges.ColumnLayout(ccd, align=128), variant=ranges.TC)
    c8 = ops.default_center(xd, yd)
    c16 = torch.cat([c8, torch.zeros(8, device=DEV)])
    eps = 0.1
    a, _ = ranges.softmin_ranges_raw(eps, xd, yd, h, None, 0.0, simt, p=2, center=c8)
    b, _ = ranges.softmin_ranges_raw(eps, xp, yp, h, None, 0.0, tc, p=2, center=c16)
    fin = torch.isfinite(a)
    assert not bool(fin.all()) and torch.equal(fin, torch.isfinite(b))
    assert torch.equal(a[~fin], b[~fin])
    assert (a[fin] - b[fin]).abs().max().item() <= 1e-5 * (1 + a[fin].abs().max().item())
    go = torch.rand(len(x)).to(DEV)
    x8, x16 = xd.clone().requires_grad_(True), xp.clone().requires_grad_(True)
    (g8,) = torch.autograd.grad(ranges.softmin_ranges(eps, x8, yd, h, None, 0.0, simt, p=2, center=c8), x8, go)
    (g16,) = torch.autograd.grad(ranges.softmin_ranges(eps, x16, yp, h, None, 0.0, tc, p=2, center=c16), x16, go)
    assert bool((g16[:, 8:] == 0).all())
    assert (g16[:, :8] - g8).abs().max().item() <= 5e-5 * max(1.0, g8.abs().max().item())
    # each problem is refused by the other family of kernels
    with pytest.raises(ValueError):
        ranges.softmin_ranges_raw(eps, xp, yp, h, None, 0.0, simt, p=2, center=c16)
    with pytest.raises(ValueError):
        ranges.softmin_ranges_raw(eps, xd, yd, h, None, 0.0, tc, p=2, center=c8)


def _count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
               and "Memset" not in e.name)


def test_launches_do_not_grow_with_the_number_of_clusters():
    from geomloss_b200 import ops, ranges

    counts = []
    for n_cl in (3, 40):
        sizes = [90] * n_cl
        x, y, rc, cc, keep = _clusters(n_cl, 16, sizes, sizes, density=0.3)
        prob = ranges.build_problem(keep.to(DEV), rc.to(DEV), ranges.ColumnLayout(cc.to(DEV), align=128),
                                    variant=ranges.TC)
        xd, yd, h = x.to(DEV), y.to(DEV), torch.zeros(len(y), device=DEV)
        c = ops.default_center(xd, yd)
        ranges.softmin_ranges_raw(0.1, xd, yd, h, None, 0.0, prob, p=2, center=c)  # warm-up (scratch, attributes)
        counts.append(_count_kernels(lambda: ranges.softmin_ranges_raw(0.1, xd, yd, h, None, 0.0, prob, p=2,
                                                                       center=c)))
    assert counts[0] == counts[1] == 4, counts  # pack rows, pack columns, reduction, finalize


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("name", golden_names("labels_hd_"))
def test_labelled_losses_against_the_reference(name):
    from geomloss_b200 import SamplesLoss

    g = load_golden(name)
    kw = golden_kwargs(g)
    pot = bool(g["potentials"])
    a, x, b, y = (cu(g[k + "_f64"]).float() for k in "axby")
    lx, ly = cu(g["labels_x"]), cu(g["labels_y"])
    L = SamplesLoss(potentials=pot, **kw)
    if kw["p"] == 1 and x.shape[1] > 8:
        pytest.skip("no p = 1 fixture above D = 8")
    if pot:
        F, G = L(lx, a, x, ly, b, y)
        assert tuple(F.shape) == g["pot_f_f64"].shape and tuple(G.shape) == g["pot_g_f64"].shape
        assert np.abs(F.cpu().double().numpy() - g["pot_f_f64"]).max() < 1e-5
        assert np.abs(G.cpu().double().numpy() - g["pot_g_f64"]).max() < 1e-5
        return
    leaves = [t.clone().requires_grad_(True) for t in (a, x, b, y)]
    val = L(lx, leaves[0], leaves[1], ly, leaves[2], leaves[3])
    ref = g["value_f64"]
    assert tuple(val.shape) == ref.shape
    assert np.abs(val.detach().cpu().double().numpy() - ref).max() <= 1e-4 * np.abs(ref).max(), (val, ref)
    grads = torch.autograd.grad(val.sum(), leaves)
    for got, key in zip(grads, ("grad_a", "grad_x", "grad_b", "grad_y")):
        r = g[key + "_f64"]
        err = np.abs(got.detach().cpu().double().numpy().reshape(r.shape) - r).max()
        assert err <= 5e-4 * np.abs(r).max() + 1e-12, (key, err, np.abs(r).max())


def test_routing_of_labelled_and_unlabelled_calls():
    """Labels for both clouds above D = 3 take the two-scale solver; without them, backend="multiscale" keeps the
    single-scale route; p = 1 above D = 8 has no kernel."""
    from geomloss_b200 import SamplesLoss
    from geomloss_b200.multiscale import sinkhorn_multiscale

    g = load_golden("labels_hd_d16_trunc1")
    kw = golden_kwargs(g)
    a, x, b, y = (cu(g[k + "_f64"]).float() for k in "axby")
    lx, ly = cu(g["labels_x"]), cu(g["labels_y"])
    two = SamplesLoss(**kw)(lx, a, x, ly, b, y).item()
    kw.pop("loss"), kw.pop("backend")
    direct = sinkhorn_multiscale(a, x, b, y, labels_x=lx, labels_y=ly, **kw).item()
    assert abs(two - direct) <= 1e-6 * abs(direct)  # the centroids come from atomics (index_add): last-bit noise
    single = SamplesLoss("sinkhorn", backend="multiscale", **kw)(a, x, b, y).item()
    online = SamplesLoss("sinkhorn", backend="online", **{k: v for k, v in kw.items() if k not in ("truncate",
                                                                                                  "cluster_scale")})
    assert single == online(a, x, b, y).item() and abs(single - two) > 1e-3 * abs(two)
    with pytest.raises(NotImplementedError):
        SamplesLoss("sinkhorn", backend="multiscale", p=1, blur=0.1)(lx, a, x, ly, b, y)
    with pytest.raises(NotImplementedError):
        sinkhorn_multiscale(a, x, b, y, labels_x=lx, **kw)

"""One small launch of every kernel family of libb200ot.so, for compute-sanitizer (memcheck / racecheck / synccheck):

    compute-sanitizer --tool memcheck  python tools/sanitize_smoke.py
    compute-sanitizer --tool racecheck python tools/sanitize_smoke.py
    B200OT_FORCE_SPLITS=1 compute-sanitizer --tool racecheck python tools/sanitize_smoke.py ring tc

Shapes are the smallest that select each code path (big / small tile shapes, ranges mode, tensor-core kernels, 2-D grid
passes with both tile widths, 3-D grid passes with the 32-line tile); results are checked against torch so a silent
corruption also fails."""
import sys

import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
from geomloss_b200 import SamplesLoss, ops, ranges  # noqa: E402
from geomloss_b200.sinkhorn_images import softmin_grid  # noqa: E402

DEV = "cuda:0"
g = torch.Generator().manual_seed(0)


def ref_softmin(eps, x, y, h, p):
    d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
    C = d2 / 2 if p == 2 else d2.clamp_min(1e-8).sqrt()
    return (-eps * torch.logsumexp(h.double()[None, :] - C / eps, dim=1)).float()


def check(name, got, ref, tol=2e-5):
    err = (got.double().cpu() - ref.double().cpu()).abs().max().item() / max(1.0, ref.abs().max().item())
    print(f"{name}: max err {err:.2e}")
    assert err < tol, name


which = set(sys.argv[1:]) or {"softmin", "pair", "ranges", "conv", "tc", "batched", "l1", "wide", "blocks", "grid", "loss",
                              "small", "apply", "apply_wide", "dense"}
if "ring" in which:
    # the dense kernels with MANY tiles per CTA (B200OT_FORCE_SPLITS=1 in the environment): every stage of the TMA ring
    # is refilled a dozen times — the pattern the N = 1e6 runs live in
    assert __import__("os").environ.get("B200OT_FORCE_SPLITS") == "1", "run with B200OT_FORCE_SPLITS=1"
    x, y, h = torch.rand(4200, 3, generator=g), torch.rand(40000, 3, generator=g), torch.randn(40000, generator=g)
    xg = x.to(DEV).requires_grad_(True)
    out = ops.softmin(0.05, xg, y.to(DEV), h.to(DEV), p=2)
    check("ring_softmin", out, ref_softmin(0.05, x, y, h, 2))
    (gx,) = torch.autograd.grad(out.sum(), xg)
    assert torch.isfinite(gx).all()
    w = torch.rand(40000, generator=g)
    conv = ops.kernel_conv("laplacian", xg, y.to(DEV), w.to(DEV), 0.3)
    assert torch.isfinite(conv).all()
    # the four tensor-core kernels with one split: 32 column tiles of 128 pass through the 4-slot ring of every CTA
    # (tc_reduce_kernel<1>, tc_bwd_kernel<3>, tc_reduce_kernel<0>, tc_bwd_kernel<2>)
    for d in (16, 64):
        x, y = torch.rand(700, d, generator=g), torch.rand(4000, d, generator=g)
        h, w = torch.randn(4000, generator=g), torch.rand(4000, generator=g)
        xd, yd, hd, wd = x.to(DEV), y.to(DEV), h.to(DEV), w.to(DEV)
        center, ones = ops.default_center(xd, yd), torch.ones(700, device=DEV)
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
        out, lse2 = ops.softmin_raw(1.0, xd, yd, hd, p=2, center=center, want_lse2=True)
        check(f"ring_tc_softmin_d{d}", out, ref_softmin(1.0, x, y, h, 2), 1e-4)
        gx = ops.softmin_grad_rows(1.0, xd, yd, hd, None, 0.0, lse2, ones, p=2, center=center)
        prob = torch.softmax(h.double()[None, :] - d2 / 2.0, dim=1)
        check(f"ring_tc_softmin_grad_d{d}", gx, x.double() - prob @ y.double(), 1e-4)
        K = (-d2 / 8.0).exp()  # blur = 2
        conv = ops.kernel_conv_raw("gaussian", xd, yd, wd, 2.0, center=center)
        check(f"ring_tc_conv_d{d}", conv, K @ w.double(), 1e-4)
        gc = ops.kernel_conv_grad_rows("gaussian", xd, yd, wd, 2.0, ones, center=center)
        Kw = K * w.double()[None, :]
        check(f"ring_tc_conv_grad_d{d}", gc, (Kw @ y.double() - Kw.sum(1, keepdim=True) * x.double()) / 4.0, 1e-4)
if "softmin" in which:
    for tag, n, m, d, p in (("big", 4200, 4300, 3, 2), ("small", 300, 500, 2, 1), ("big_p1", 4100, 4100, 1, 1),
                            ("d8", 600, 700, 8, 2)):
        x, y, h = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g), torch.randn(m, generator=g)
        xg = x.to(DEV).requires_grad_(True)
        out = ops.softmin(0.05, xg, y.to(DEV), h.to(DEV), p=p)
        check("softmin_" + tag, out, ref_softmin(0.05, x, y, h, p))
        (gx,) = torch.autograd.grad(out.sum(), xg)
        assert torch.isfinite(gx).all()
if "pair" in which:
    # the paired kernels (softmin_pair.cuh): the xy / yx pair and the symmetric xx softmin, many blocks, ragged sizes
    import os

    os.environ["B200OT_PAIR_TILES"] = "1"
    x, y = torch.rand(5000, 3, generator=g), torch.rand(6100, 3, generator=g)
    hx, hy = torch.randn(5000, generator=g) * 0.1, torch.randn(6100, generator=g) * 0.1
    xd, yd, hxd, hyd = x.to(DEV), y.to(DEV), hx.to(DEV), hy.to(DEV)
    c = ops.default_center(xd, yd)
    (fa, _), (fb, _) = ops.softmin_raw_many([((0.05, xd, yd, hyd), dict(p=2, center=c)),
                                             ((0.05, yd, xd, hxd), dict(p=2, center=c))])
    check("pair_xy", fa, ref_softmin(0.05, x, y, hy, 2))
    check("pair_yx", fb, ref_softmin(0.05, y, x, hx, 2))
    check("pair_xx", ops.softmin_raw(0.05, xd, xd, hxd, p=2, center=c)[0], ref_softmin(0.05, x, x, hx, 2))
    # the step entry: the pair and both symmetric softmins in one launch
    got = ops.softmin_raw_many([((0.05, xd, yd, hyd), dict(p=2, center=c)), ((0.05, yd, xd, hxd), dict(p=2, center=c)),
                                ((0.05, xd, xd, hxd), dict(p=2, center=c)), ((0.05, yd, yd, hyd), dict(p=2, center=c))])
    for name, (o, _), (r, col, h) in zip(("xy", "yx", "xx", "yy"), got, ((x, y, hy), (y, x, hx), (x, x, hx), (y, y, hy))):
        check(f"step_{name}", o, ref_softmin(0.05, r, col, h, 2))
    del os.environ["B200OT_PAIR_TILES"]
if "ranges" in which:
    for variant, n, m in ((ranges.SMALL, 900, 700), (ranges.BIG, 2500, 3000)):
        R = 5
        rc = torch.tensor([n // R] * (R - 1) + [n - (R - 1) * (n // R)])
        cc = torch.tensor([m // R] * (R - 1) + [m - (R - 1) * (m // R)])
        keep = torch.rand(R, R, generator=g) < 0.6
        keep[torch.arange(R), torch.arange(R)] = True
        lay = ranges.ColumnLayout(cc.to(DEV))
        prob = ranges.build_problem(keep.to(DEV), rc.to(DEV), lay, variant=variant)
        x, y, h = torch.rand(n, 3, generator=g), torch.rand(m, 3, generator=g), torch.randn(m, generator=g)
        xg = x.to(DEV).requires_grad_(True)
        out = ranges.softmin_ranges(0.05, xg, y.to(DEV), h.to(DEV), None, 0.0, prob)
        mask = keep[torch.repeat_interleave(torch.arange(R), rc)][:, torch.repeat_interleave(torch.arange(R), cc)]
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1) / 2
        ref = -0.05 * torch.logsumexp((h.double()[None, :] - d2 / 0.05).masked_fill(~mask, -float("inf")), dim=1)
        check(f"ranges_softmin_v{variant}", out, ref.float())
        (gx,) = torch.autograd.grad(out.sum(), xg)
        assert torch.isfinite(gx).all()
        w = torch.rand(m, generator=g)
        conv = ranges.kernel_conv_ranges(0, xg, y.to(DEV), w.to(DEV), 0.2, prob, None)
        refc = ((-d2 / 0.04).exp() * mask) @ w.double()
        check(f"ranges_conv_v{variant}", conv, refc.float())
        (gx,) = torch.autograd.grad(conv.sum(), xg)
        assert torch.isfinite(gx).all()
if "conv" in which:
    for kind in ("gaussian", "laplacian", "energy"):
        x, y, w = torch.rand(4200, 3, generator=g), torch.rand(4100, 3, generator=g), torch.rand(4100, generator=g)
        xg = x.to(DEV).requires_grad_(True)
        out = ops.kernel_conv(kind, xg, y.to(DEV), w.to(DEV), 0.3)
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
        K = {"gaussian": (-d2 / 0.18).exp(), "laplacian": (-(d2 / 0.09).clamp_min(1e-8).sqrt()).exp(),
             "energy": -d2.clamp_min(1e-8).sqrt()}[kind]
        check("conv_" + kind, out, (K @ w.double()).float(), 5e-5)
        (gx,) = torch.autograd.grad(out.sum(), xg)
        assert torch.isfinite(gx).all()
if "tc" in which:
    for d in (16, 64):
        x, y, w = torch.rand(700, d, generator=g), torch.rand(900, d, generator=g), torch.rand(900, generator=g)
        xg = x.to(DEV).requires_grad_(True)
        out = ops.kernel_conv("gaussian", xg, y.to(DEV), w.to(DEV), 2.0)
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
        check(f"tc_conv_d{d}", out, ((-d2 / 8.0).exp() @ w.double()).float(), 1e-4)
        (gx,) = torch.autograd.grad(out.sum(), xg)
        assert torch.isfinite(gx).all()
        h = torch.randn(900, generator=g)
        sm = ops.softmin(1.0, xg, y.to(DEV), h.to(DEV), p=2)
        check(f"tc_softmin_d{d}", sm, ref_softmin(1.0, x, y, h, 2), 1e-4)
        (gx,) = torch.autograd.grad(sm.sum(), xg)
        assert torch.isfinite(gx).all()
        # laplacian / energy kernels (tc_reduce_kernel<4/5>, tc_bwd_kernel<4/5>), both conventions; the self term
        d2 = ((x[:, None, :].double() - x[None, :, :].double()) ** 2).sum(-1)
        for kind, name in ((1, "laplacian"), (2, "energy"), (0x101, "laplacian_unclamped"), (0x102, "energy_unclamped")):
            ka = d2.clamp_min(1e-8 if kind < 0x100 else 0.0).sqrt()
            K = (-ka / 2.0).exp() if (kind & 0xFF) == 1 else -ka
            out = ops.kernel_conv(kind, xg, x.to(DEV), w[:700].to(DEV), 2.0)
            check(f"tc_{name}_d{d}", out, (K @ w[:700].double()).float(), 1e-3)
            (gx,) = torch.autograd.grad(out.sum(), xg)
            assert torch.isfinite(gx).all()
if "batched" in which:
    # the batched tensor-core kernels (tc_reduce_kernel<0/1/4/5, BATCH>, tc_bwd_kernel<2/3/4/5, dk, BATCH>), each
    # element checked against its own columns
    B, n = 3, 300
    for d in (16, 64):
        x, y = torch.rand(B, n, d, generator=g), torch.rand(B, n, d, generator=g)
        h, w = torch.randn(B, n, generator=g), torch.rand(B, n, generator=g)
        xd, yd, hd, wd, ones = x.to(DEV), y.to(DEV), h.to(DEV), w.to(DEV), torch.ones(B, n, device=DEV)
        center = ops.default_center(xd.view(-1, d), yd.view(-1, d))
        d2 = ((x[:, :, None, :].double() - y[:, None, :, :].double()) ** 2).sum(-1)
        out, lse2 = ops.softmin_batched_raw(1.0, xd, yd, hd, p=2, center=center, want_lse2=True)
        check(f"batched_softmin_d{d}", out, (-torch.logsumexp(h.double()[:, None, :] - d2 / 2.0, dim=2)).float(), 1e-4)
        gx = ops.softmin_batched_grad_rows(1.0, xd, yd, hd, None, 0.0, lse2, ones, p=2, center=center)
        prob = torch.softmax(h.double()[:, None, :] - d2 / 2.0, dim=2)
        check(f"batched_softmin_grad_d{d}", gx, x.double() - prob @ y.double(), 1e-4)
        for kind, K in ((0, (-d2 / 8.0).exp()), (1, (-d2.clamp_min(1e-8).sqrt() / 2.0).exp()),
                        (2, -d2.clamp_min(1e-8).sqrt())):
            conv = ops.kernel_conv_batched_raw(kind, xd, yd, wd, 2.0, center=center)
            check(f"batched_conv{kind}_d{d}", conv, (K @ w.double()[:, :, None])[..., 0], 1e-3)
            gc = ops.kernel_conv_batched_grad_rows(kind, xd, yd, wd, 2.0, ones, center=center)
            assert torch.isfinite(gc).all()
        val, gu = ops.kernel_conv_batched_value_and_grad_rows(0, xd, yd, wd, 2.0, center=center)
        check(f"batched_conv_value_d{d}", val, ((-d2 / 8.0).exp() @ w.double()[:, :, None])[..., 0], 1e-4)
        assert torch.isfinite(gu).all()
if "l1" in which:
    # the p = 1 softmin (tc_reduce_kernel<6, BATCH>, tc_bwd_kernel<7, dk, BATCH> at every dk)
    B, n = 2, 300
    for d in (16, 32, 48, 64):
        x, y, h = torch.rand(B, n, d, generator=g), torch.rand(B, n, d, generator=g), torch.randn(B, n, generator=g)
        xd, yd, hd, ones = x.to(DEV), y.to(DEV), h.to(DEV), torch.ones(B, n, device=DEV)
        center = ops.default_center(xd.view(-1, d), yd.view(-1, d))
        dist = ((x[:, :, None, :].double() - y[:, None, :, :].double()) ** 2).sum(-1).clamp_min(1e-8).sqrt()
        out, lse2 = ops.softmin_l1_raw(0.5, xd, yd, hd, p=1, center=center, want_lse2=True)
        check(f"l1_softmin_d{d}", out, (-0.5 * torch.logsumexp(h.double()[:, None, :] - dist / 0.5, dim=2)).float(),
              1e-4)
        gx = ops.softmin_l1_grad_rows(0.5, xd, yd, hd, None, 0.0, lse2, ones, p=1, center=center)
        prob = torch.softmax(h.double()[:, None, :] - dist / 0.5, dim=2)
        unit = (x.double()[:, :, None, :] - y.double()[:, None, :, :]) / dist[..., None]
        check(f"l1_softmin_grad_d{d}", gx, (prob[..., None] * unit).sum(2), 1e-4)
if "wide" in which:
    # above D = 64 (tc_wide_reduce_kernel / tc_wide_bwd_kernel, csrc/tcwide.cuh): one launch of every b200ot_wide_*
    # entry, a batch of 2 at a partial last slab (D = 72) and at two slabs (D = 128)
    B, n = 2, 300
    for d in (72, 128):
        x, y, h = torch.rand(B, n, d, generator=g), torch.rand(B, n, d, generator=g), torch.randn(B, n, generator=g)
        w = torch.rand(B, n, generator=g)
        xd, yd, hd, wd, ones = x.to(DEV), y.to(DEV), h.to(DEV), w.to(DEV), torch.ones(B, n, device=DEV)
        center = ops.default_center(xd.view(-1, d), yd.view(-1, d))
        d2 = ((x[:, :, None, :].double() - y[:, None, :, :].double()) ** 2).sum(-1)
        for p in (1, 2):
            C = d2 / 2 if p == 2 else d2.clamp_min(1e-8).sqrt()
            out, lse2 = ops.softmin_wide_raw(0.5, xd, yd, hd, p=p, center=center, want_lse2=True)
            ref = -0.5 * torch.logsumexp(h.double()[:, None, :] - C / 0.5, dim=2)
            check(f"wide_softmin_p{p}_d{d}", out, ref.float(), 1e-4)
            gx = ops.softmin_wide_grad_rows(0.5, xd, yd, hd, None, 0.0, lse2, ones, p=p, center=center)
            assert torch.isfinite(gx).all()
        for kind in ("gaussian", "energy"):
            val = ops.kernel_conv_wide_raw(kind, xd, yd, wd, 2.0, center=center)
            K = (-d2 / 8.0).exp() if kind == "gaussian" else -d2.clamp_min(1e-8).sqrt()
            check(f"wide_conv_{kind}_d{d}", val, (K @ w.double()[:, :, None])[..., 0], 1e-4)
            gx = ops.kernel_conv_wide_grad_rows(kind, xd, yd, wd, 2.0, ones, center=center)
            assert torch.isfinite(gx).all()
if "blocks" in which:
    # the block-sparse tensor-core softmins (tc_reduce_kernel<1, false, BLOCKS>, tc_bwd_kernel<3, dk, false, BLOCKS>):
    # clusters of 1, 127, 128, 129 and 300 points, a row cluster that keeps nothing, a self problem
    for d in (16, 64):
        rc, cc = torch.tensor([1, 129, 300, 128]), torch.tensor([127, 1, 300, 129, 128])
        keep = torch.rand(4, 5, generator=g) < 0.6
        keep[0], keep[1] = True, False
        prob = ranges.build_problem(keep.to(DEV), rc.to(DEV), ranges.ColumnLayout(cc.to(DEV), align=128),
                                    variant=ranges.TC)
        x, y, h = torch.rand(int(rc.sum()), d, generator=g), torch.rand(int(cc.sum()), d, generator=g), torch.randn(
            int(cc.sum()), generator=g)
        xg = x.to(DEV).requires_grad_(True)
        out = ranges.softmin_ranges(1.0, xg, y.to(DEV), h.to(DEV), None, 0.0, prob)
        mask = keep[torch.repeat_interleave(torch.arange(4), rc)][:, torch.repeat_interleave(torch.arange(5), cc)]
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1) / 2
        ref = -torch.logsumexp((h.double()[None, :] - d2).masked_fill(~mask, -float("inf")), dim=1)
        live = mask.any(1)
        check(f"blocks_softmin_d{d}", out[live.to(DEV)], ref[live].float(), 1e-4)
        (gx,) = torch.autograd.grad(out[live.to(DEV)].sum(), xg)
        assert torch.isfinite(gx).all()
        kxx = torch.rand(4, 4, generator=g) < 0.5
        kxx[torch.arange(4), torch.arange(4)] = True
        pxx = ranges.build_problem(kxx.to(DEV), rc.to(DEV), ranges.ColumnLayout(rc.to(DEV), align=128),
                                   variant=ranges.TC)
        hx = torch.randn(int(rc.sum()), generator=g).to(DEV)
        sxx = ranges.softmin_ranges(1.0, xg, xg.detach(), hx, None, 0.0, pxx)
        (gx,) = torch.autograd.grad(sxx.sum(), xg)
        assert torch.isfinite(sxx).all() and torch.isfinite(gx).all()
        print(f"blocks_self_d{d} ok")
if "grid" in which:
    for shape in ((1, 2, 32, 32), (1, 1, 16, 16, 16), (1, 1, 1024, 1024)):
        h = torch.randn(*shape, generator=g)
        out = softmin_grid(0.01, 2, h.to(DEV))
        assert torch.isfinite(out).all()
        print("grid", shape, "ok")
    # per-axis geometry and the plan applied to K channels: unequal sides, a periodic axis, the 32-, 16- and 8-line
    # tiles of the apply kernel and a partial second slab of channels
    for shape, K in (((2, 33, 7), 5), ((1, 1024), 1), ((1, 1024), 4), ((1, 9, 16, 5), 2)):
        h = torch.randn(*shape, generator=g).to(DEV)
        geo = dict(pitch=[1.0 / n for n in shape[1:]], periodic=[d == 0 for d in range(len(shape) - 1)])
        out = ops.softmin_grid_axes_raw(0.01, h, **geo)
        ell, s = ops.grid_plan_apply_raw(0.01, h, None, 0.0, torch.randn((K,) + shape, generator=g).to(DEV), **geo)
        assert torch.isfinite(out).all() and torch.isfinite(ell).all() and torch.isfinite(s).all()
        print("grid axes / plan apply", shape, K, "ok")
if "loss" in which:
    x, y = torch.rand(3, 300, 3, generator=g).to(DEV), torch.rand(3, 200, 3, generator=g).to(DEV)
    v = SamplesLoss("sinkhorn", blur=0.1)(x.requires_grad_(True), y)
    v.sum().backward()
    print("batched sinkhorn", v.tolist())
    v = SamplesLoss("sinkhorn", blur=0.1, reach=0.5, debias=False)(x.detach().requires_grad_(True), y)
    v.sum().backward()
    print("batched unbalanced sinkhorn (small-problem kernels: iteration, cost, backward)", v.tolist())
    v = SamplesLoss("gaussian", blur=0.1)(x.detach().requires_grad_(True), y)
    v.sum().backward()
    print("batched gaussian (fused MMD + value kernel)", v.tolist())
    big = torch.rand(100000, 3, generator=g).to(DEV)
    for _ in range(2):  # many CTAs: partial boxes + last-block fold, ticket counter re-used
        lh = ops.cloud_extent(big, big[:777])
    assert torch.equal(lh[0], big.min(0).values) and torch.equal(lh[1], big.max(0).values)
    print("cloud_extent ok")
    v = SamplesLoss("sinkhorn", blur=0.05, backend="multiscale", cluster_scale=0.2, truncate=2)(x[0], y[0])
    print("multiscale sinkhorn", v.item())
    v = SamplesLoss("gaussian", blur=0.1, backend="multiscale", truncate=2)(x[0], y[0])
    print("multiscale gaussian", v.item())
if "small" in which:
    # the small-cloud kernels at D = 8 (csrc/b200ot_small.cu): the iteration kernel with 8 warps (one problem: 10 row
    # tiles x 4 problems = 40 CTAs) and with 4 (40 elements: 1600 CTAs), the final backward, both MMD kernels
    d, n, m = 8, 300, 260
    for B in (1, 40):
        x, y = torch.rand(B, n, d, generator=g), torch.rand(B, m, d, generator=g)
        xg = x.to(DEV).requires_grad_(True)
        v = SamplesLoss("sinkhorn", blur=0.3)(xg, y.to(DEV))
        (gx,) = torch.autograd.grad(v.sum(), xg)
        assert torch.isfinite(v).all() and torch.isfinite(gx).all()
        print(f"small sinkhorn B={B} d={d}", v[:2].tolist())
        xg = x.to(DEV).requires_grad_(True)
        v = SamplesLoss("gaussian", blur=0.5)(xg, y.to(DEV))
        (gx,) = torch.autograd.grad(v.sum(), xg)
        assert torch.isfinite(gx).all()
        K = lambda u, w: (-((u[:, :, None].double() - w[:, None].double()) ** 2).sum(-1) / 0.5).exp()  # noqa: E731
        ref = 0.5 * K(x, x).mean((1, 2)) + 0.5 * K(y, y).mean((1, 2)) - K(x, y).mean((1, 2))
        check(f"small_gaussian_B{B}_d{d}", v, ref, 1e-4)
if "apply" in which:
    # the plan applied to a value matrix: both CUDA-core tile shapes with both slab widths (K = 11: slabs of 8 and 4),
    # and the tensor-core kernel with a value image of 16 and of 64 columns plus a second slab (K = 70)
    for tag, n, m, d, k in (("small", 300, 500, 2, 11), ("big", 4200, 4300, 3, 11), ("big_d8", 4100, 4100, 8, 3),
                            ("tc_d16", 700, 900, 16, 5), ("tc_d64", 300, 1000, 64, 70)):
        x, y, h = torch.rand(n, d, generator=g), torch.rand(m, d, generator=g), torch.randn(m, generator=g)
        v = torch.randn(m, k, generator=g)
        xd, yd, hd = x.to(DEV), y.to(DEV), h.to(DEV)
        eps = 0.02 * d
        center = ops.default_center(xd, yd)
        _, lse2 = ops.softmin_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
        out = ops.plan_apply_raw(eps, xd, yd, hd, None, 0.0, lse2, v.to(DEV), center=center)
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
        check("apply_" + tag, out, torch.softmax(h.double()[None, :] - d2 / (2 * eps), dim=1) @ v.double(), 2e-4)
if "apply_wide" in which:
    # above D = 64 (tc_wide_apply_kernel): a partial last K slab (D = 200), a value image of 16 columns and one of 64
    # plus a second slab (K = 70)
    for d, k in ((200, 5), (96, 70)):
        x, y, h = torch.rand(300, d, generator=g), torch.rand(700, d, generator=g), torch.randn(700, generator=g)
        v = torch.randn(700, k, generator=g)
        xd, yd, hd = x.to(DEV), y.to(DEV), h.to(DEV)
        eps = 0.02 * d
        center = ops.default_center(xd, yd)
        _, lse2 = ops.softmin_wide_raw(eps, xd, yd, hd, p=2, center=center, want_lse2=True)
        out = ops.plan_apply_wide_raw(eps, xd, yd, hd, None, 0.0, lse2, v.to(DEV), center=center)
        d2 = ((x[:, None, :].double() - y[None, :, :].double()) ** 2).sum(-1)
        check(f"apply_wide_d{d}_k{k}", out, torch.softmax(h.double()[None, :] - d2 / (2 * eps), dim=1) @ v.double(),
              2e-4)
if "dense" in which:
    # explicit cost matrices: the pair kernel (ring and scalar paths) and its backward, then a group of row softmins
    # (one aligned, one odd n_cols, one batch view off the 16-byte grid) and the row backward
    import math

    def rows_ref(eps, C, lw, pot):
        return -eps * torch.logsumexp((lw.double() + pot.double() / eps)[..., None, :] - C.double() / eps, dim=-1)

    eps = 0.1
    for n, m in ((130, 260), (70, 67)):
        C = torch.rand(2, n, m, generator=g).to(DEV)
        la, lb = torch.full((2, n), -math.log(n), device=DEV), torch.full((2, m), -math.log(m), device=DEV)
        f, gg = torch.randn(2, n, generator=g).to(DEV), torch.randn(2, m, generator=g).to(DEV)
        fo, go, l2r, l2c = ops.dense_softmin_pair_raw(eps, C, la, lb, f, gg, want_lse2=True)
        check(f"dense_pair_{n}x{m}", fo, rows_ref(eps, C, lb, gg))
        check(f"dense_pair_cols_{n}x{m}", go, rows_ref(eps, C.transpose(1, 2), la, f))
        assert torch.isfinite(ops.dense_softmin_pair_grad(eps, C, la, lb, f, gg, l2r, l2c, torch.ones_like(f),
                                                          torch.ones_like(gg))).all()
    buf = torch.rand(3 * 40 * 132 + 1, generator=g).to(DEV)
    probs = []
    for C in (torch.rand(300, 520, generator=g).to(DEV), torch.rand(2, 90, 77, generator=g).to(DEV),
              buf[1:].view(3, 40, 132)):
        m = C.shape[-1]
        probs.append((C, torch.full(C.shape[:-2] + (m,), -math.log(m), device=DEV),
                      torch.randn(C.shape[:-2] + (m,), generator=g).to(DEV), None))
    for k, ((C, lw, pot, _), (out, lse2)) in enumerate(zip(probs, ops.dense_softmin_rows_raw(eps, probs,
                                                                                              want_lse2=True))):
        check(f"dense_rows_{k}", out, rows_ref(eps, C, lw, pot))
        assert torch.isfinite(ops.dense_softmin_rows_grad(eps, C, lw, pot, lse2, torch.ones_like(out))).all()
torch.cuda.synchronize()
print("sanitize_smoke: all launches completed")

"""fp64 references of the CUDA-core reduction operators (softmin values and row gradients, kernel products and their x,
y, w gradients), with the fp32 rounding allowances of the explicit-difference row gradients, and the error-to-bar check
the GPU test modules share.

Each reference runs on ``device`` (the CPU by default; "cuda:0" for the large clouds, where the CPU needs minutes) in
row blocks of ``block`` rows, and returns its results on that device.
"""
import math

import torch

from oracle import geomloss_oracle as O


def check(ratios, sec, what, got, ref, bar):
    """|got - ref| <= bar row by row (``bar``: a number, or one per row), the largest ratio recorded in
    ``ratios[sec]`` as (what, ratio)."""
    err = (got.detach().double() - ref.detach().double().to(got.device)).abs()
    if err.dim() > 1:
        err = err.amax(dim=1)
    if err.numel() == 0:
        return
    if torch.is_tensor(bar):
        bar = bar.to(err.device)
    ratio = err / bar
    r = ratio.max().item()
    if r > ratios.get(sec, ("", -1.0))[1]:
        ratios[sec] = (what, r)
    assert r <= 1.0, f"{what}: error / bar = {r:.3g} (largest error {err.max().item():.3g})"


def cost64(x, y, conv):
    """The cost of convention ``conv``: "p2" |x - y|^2 / 2, "p1" |x - y| with the 1e-8 clamp on |x - y|^2 of the
    tensorized cost, "p1u" pykeops' unclamped |x - y| (p = 1 | P_UNCLAMPED)."""
    if conv == "p2":
        return O.cost_matrix(x, y, 2)
    if conv == "p1":
        return O.cost_matrix(x, y, 1)
    return O.keops_cost(x, y, 1)


def mid(x, y):
    """ops.default_center in fp64: the middle of the joint bounding box."""
    both = torch.cat([x, y]).double()
    return 0.5 * (both.min(0).values + both.max(0).values)


def direction_slack(xb, y, center, clamped):
    """Per pair, a bound on the error of the unit vector (x_i - y_j) / |x_i - y_j| that the p = 1, laplacian and
    energy row gradients (rowsum.cuh, explicit differences) compute in fp32.

    The kernels difference PRE-SCALED coordinates, X = s (x - c) and -Y = -s (y - c), each rounded twice (2^-24
    relative per rounding), so the computed difference is off by up to 2^-23 (|x - c| + |y - c|) in x units, plus
    2^-24 of itself: below 2^-22 (|x - c| + |y - c|) =: e.  The unit vector of a pair at distance d is then off by
    up to min(2, 2 e / d).  This is no concern where the cost is smooth or the gradient vanishes — p = 2, the
    gaussian, and the clamped conventions inside the 1e-8 clamp on |x - y|^2 — but pykeops' unclamped |x - y| keeps a
    full-weight unit vector at any distance, and a pair a few ulps apart (D = 1: 2209 x 3889 random points in
    clusters 0.2 wide come within 1e-7 of each other) gets a direction that rounding alone decides.  The same holds,
    weighted by e / d, for pairs just outside the clamp.  Exactly coincident points (d = 0) give X + (-Y) = 0 exactly
    in the kernel and a zero gradient on both sides: no slack."""
    d = O.keops_norm2(xb, y)
    e = 2.0 ** -22 * ((xb - center).norm(dim=1)[:, None] + (y - center).norm(dim=1)[None, :])
    slack = torch.clamp(2.0 * e / d, max=2.0)
    return torch.where(d > (0.999e-4 if clamped else 0.0), slack, torch.zeros_like(slack))


def softmin64(eps, x, y, h, pairs, conv, go=None, center=None, block=256, device="cpu"):
    """fp64 -eps log sum_{j: pairs[i, j]} exp(h_j - C_ij / eps) per row (``pairs`` None: every pair); with ``go`` also
    the row gradient of <go, softmin> by autograd and, for p = 1, its rounding allowance sum_j |go_i| w_ij slack_ij
    (direction_slack; ``center``: the kernel's, None for none).  Rows without a kept pair: +inf and NaN, never
    compared."""
    x, y, h = (t.detach().to(device, torch.float64) for t in (x, y, h))
    pairs = None if pairs is None else pairs.to(device)
    N = x.shape[0]
    c = torch.zeros(x.shape[1], dtype=torch.float64, device=device) if center is None else center.to(device).double()
    out = torch.empty(N, dtype=torch.float64, device=device)
    gx = torch.empty_like(x) if go is not None else None
    allow = torch.zeros(N, dtype=torch.float64, device=device)
    for s in range(0, N, block):
        xb = x[s:s + block].clone().requires_grad_(go is not None)
        with torch.set_grad_enabled(go is not None):
            t = h[None, :] - cost64(xb, y, conv) / eps
            if pairs is not None:
                t = t.masked_fill(~pairs[s:s + block], -math.inf)
            f = -eps * torch.logsumexp(t, dim=1)
        out[s:s + block] = f.detach()
        if go is not None:
            gb = go[s:s + block].to(device, torch.float64)
            (gx[s:s + block],) = torch.autograd.grad((f * gb).sum(), xb)
            if conv != "p2":
                wgt = torch.softmax(t.detach(), dim=1).nan_to_num(0.0)
                slack = direction_slack(xb.detach(), y, c, clamped=conv == "p1")
                allow[s:s + block] = gb.abs() * (wgt * slack).sum(1)
    return out, gx, allow


def kmat64(kind, unclamped, x, y, blur):
    return (O.keops_kernel_matrix if unclamped else O.kernel_matrix)(kind, x, y, blur)


# Roundings of 2^-24 that a dominant term of the gaussian row-gradient sums goes through (expansion_slack in conv64):
# the product w e, its FMA into the tile sum, the running sum, the merge of the two lanes, up to five column splits,
# X a0, the difference, and the two products of the finalize.
GAUSS_ROUNDINGS = 16


def conv64(kind, unclamped, x, y, w, blur, pairs, go, center, block=256, device="cpu", expansion_slack=False):
    """fp64 out = (K(x, y) masked by ``pairs``) @ w, the x, y, w gradients of <go, out> by autograd, and the rounding
    allowances of the x and y gradients of the laplacian and energy kernels: the sums over i, j of
    |go_i w_j dk/d|x - y|| slack_ij (direction_slack).

    ``expansion_slack``: the same allowances for the gaussian kernel.  Its row gradient (rowsum.cuh, kGaussBwd, and
    conv_bwd_finalize_kernel) forms sum_j w_j k_ij (Y_j - X_i) as a - X_i a0 from a = sum_j w_j e_ij Y_j and
    a0 = sum_j w_j e_ij, over centred coordinates scaled by s = sqrt(log2 e) / blur, then scales it by
    go_i / (s blur^2).  Every rounding on the way is relative to |X_i| a0 or |a|, not to the difference: where a pair
    at (nearly) zero distance dominates a row, as in a self problem at small blur, the difference cancels and those
    roundings are what remains.  Per pair GAUSS_ROUNDINGS 2^-24 |go_i w_j| k_ij (|x_i - c|_inf + |y_j - c|_inf) / blur^2
    bounds them; summed over j for the x gradient, over i for the y gradient (the same reduction on the transpose)."""
    xr, yr, wr = (t.detach().to(device, torch.float64).clone().requires_grad_(True) for t in (x, y, w))
    pairs = None if pairs is None else pairs.to(device)
    c = center.to(device).double()
    out = torch.empty(x.shape[0], dtype=torch.float64, device=device)
    ax = torch.zeros(x.shape[0], dtype=torch.float64, device=device)
    ay = torch.zeros(y.shape[0], dtype=torch.float64, device=device)
    for s in range(0, x.shape[0], block):
        K = kmat64(kind, unclamped, xr[s:s + block], yr, blur)
        if pairs is not None:
            K = K * pairs[s:s + block].double()
        ob = K @ wr
        out[s:s + block] = ob.detach()
        gb = go[s:s + block].to(device, torch.float64)
        (ob * gb).sum().backward()
        if kind != "gaussian":
            dk = K.detach().abs() / blur if kind == "laplacian" else K.detach().ne(0).double()  # |dk / d|x - y||
            pair = gb.abs()[:, None] * dk * wr.detach().abs()[None, :]
            pair = pair * direction_slack(xr[s:s + block].detach(), yr.detach(), c, clamped=not unclamped)
            ax[s:s + block] = pair.sum(1)
            ay += pair.sum(0)
        elif expansion_slack:
            xc = (xr[s:s + block].detach() - c).abs().amax(1)
            yc = (yr.detach() - c).abs().amax(1)
            pair = gb.abs()[:, None] * K.detach() * wr.detach().abs()[None, :] * (xc[:, None] + yc[None, :])
            pair = pair * (GAUSS_ROUNDINGS * 2.0 ** -24 / blur ** 2)
            ax[s:s + block] = pair.sum(1)
            ay += pair.sum(0)
    return out, xr.grad, yr.grad, wr.grad, ax, ay

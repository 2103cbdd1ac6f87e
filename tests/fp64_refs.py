"""fp64 references of the CUDA-core reduction operators (softmin values and row gradients, kernel products and their x,
y, w gradients, the separable grid softmin and its closed-form backward), with the fp32 rounding allowances of the
explicit-difference row gradients and of the grid backward, and the error-to-bar check the GPU test modules share.

Each reference runs on ``device`` (the CPU by default; "cuda:0" for the large clouds and grids, where the CPU needs
minutes) in blocks of rows or lines, and returns its results on that device.
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


def grid_cost64(N, eps, p, device="cpu"):
    """(N, N) fp64 -|x_i - x_j|^p / (p eps) on the pixel grid x = arange(N) / N: one axis of the grid softmin."""
    x = torch.arange(N, dtype=torch.float64, device=device) / N
    d = x[:, None] - x[None, :]
    return -d.abs() / eps if p == 1 else -(d * d) / (2 * eps)


def grid_softmin64(eps, p, h, dim, rows=None, device="cpu", budget=2**25):
    """fp64 -eps * (one log-sum-exp per grid axis) of h (..., N, .., N), whose last ``dim`` axes are the grid, on the
    pixel grid x = arange(N) / N: the last axis first, then the others, as b200ot_softmin_grid and
    oracle.softmin_grid_dense order them.

    ``rows``: per grid axis, the output indices to compute along it (None: all).  The axes are reduced in that order,
    each for its own sampled indices only, so 8 indices per axis of an N^3 volume cost about 8 N^3 terms.  Each axis is
    reduced in blocks of lines of about ``budget`` terms, and h is converted to fp64 one block at a time: neither an
    (N, N, N) temporary of a 1024^2 image nor an fp64 copy of a 1024^3 volume is formed.  Returns on ``device``."""
    N = h.shape[-1]
    k = grid_cost64(N, eps, p, device)
    t = h.detach().to(device)
    for axis in reversed(range(dim)):
        ax = t.dim() - dim + axis
        kr = k if rows is None or rows[axis] is None else k[torch.as_tensor(rows[axis], device=device)]
        src = t.movedim(ax, -1)
        lines = src.reshape(-1, N)
        out = torch.empty(lines.shape[0], kr.shape[0], dtype=torch.float64, device=device)
        step = max(1, budget // (kr.shape[0] * N))
        for s in range(0, lines.shape[0], step):
            out[s:s + step] = torch.logsumexp(lines[s:s + step, None, :].double() + kr[None], dim=-1)
        t = out.reshape(src.shape[:-1] + (kr.shape[0],)).movedim(-1, ax)
    return -eps * t


# Roundings of 2^-24 in a part eps exp(h - conv / eps) of the closed-form grid backward beyond its exponent: the
# exponential, the product by eps and the accumulation into the gradient.
GRID_BWD_ROUNDINGS = 4


def grid_softmin_grad64(eps, p, h, go, value_bar, device="cpu"):
    """fp64 gradient of <go, softmin_grid(eps, p, h)> w.r.t. h (h: (B, C, N, N[, N])) by autograd through
    oracle.softmin_grid_dense, and the allowance of the closed-form backward of barycenter_images._GridSoftmin.

    That backward forms the gradient as  sum over s = +1, -1 of  -s eps exp(h - conv_s / eps), with
    conv_s = softmin_grid(eps, p, log((s go)^+) + out / eps), from two more fp32 grid softmins.  If every grid softmin
    meets the value bar, |error| <= value_bar max(1, |value|) over its batch element: conv_s is off by up to its own
    bar delta_s, plus the bar delta_out of ``out``, which enters its input divided by eps and so moves it by at most
    delta_out.  The part is then off by a factor exp(+-(delta_s + delta_out) / eps), and by the fp32 rounding of its
    exponent, 2^-23 (|h| + |conv_s| / eps) in absolute terms, and GRID_BWD_ROUNDINGS more roundings of 2^-24.  Summed
    over the two parts, per pixel.  Returns (gradient, allowance) on ``device``."""
    from oracle import geomloss_oracle as O

    hr = h.detach().to(device, torch.float64).requires_grad_(True)
    go = go.detach().to(device, torch.float64)
    out = O.softmin_grid_dense(eps, p, hr)
    (grad,) = torch.autograd.grad(out, hr, go)
    out, hr = out.detach(), hr.detach()

    def element_bar(t):
        fin = torch.where(torch.isfinite(t), t.abs(), torch.zeros_like(t))
        return value_bar * fin.flatten(2).amax(dim=2).clamp_min(1.0).reshape(t.shape[:2] + (1,) * (t.dim() - 2))

    dim = h.dim() - 2
    d_out = element_bar(out)
    allow = torch.zeros_like(hr)
    for s in (1.0, -1.0):
        part = (s * go).clamp_min(0.0)
        lw = torch.where(part > 0, part.log(), torch.full_like(part, -math.inf))
        conv = grid_softmin64(eps, p, lw + out / eps, dim, device=device)
        expo = hr - conv / eps
        rel = torch.expm1((element_bar(conv) + d_out) / eps + 2.0**-23 * (hr.abs() + conv.abs() / eps))
        allow += torch.where(torch.isfinite(expo), eps * expo.exp() * (rel + GRID_BWD_ROUNDINGS * 2.0**-24), 0.0)
    return grad, allow

"""A/B timing of the routing knobs of the tensor-core kernels, inside ONE process and ONE build of the library
(the knobs are environment variables the C entry points read on every call):

  part A  CUDA-core vs tensor-core path for D <= 8 (B200OT_TC_MIN_D / B200OT_TC_MIN_PAIRS), per operator and size —
          the cross-over that csrc/b200ot_tc.cu::kTcMinDimDefault encodes;
  part C  value + unit gradient in one pass (b200ot_kernel_conv_fwd_bwd_x) against the two separate reductions;
  part D  BASELINE configs[2] (gaussian MMD, N = M = 1e6, D = 64, forward + gradient), two-pass and one-pass.

Every variant's result is compared with the default path's result on the same inputs (and, for part C, with an fp64
brute force on sampled rows).  One JSON line per measurement.

    python tools/ab_tc_route.py [--quick] > ab_tc_route.jsonl
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import ops  # noqa: E402


def best_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


class env:
    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        for k, v in self.kv.items():
            os.environ[k] = str(v)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


SIMT = dict(B200OT_TC_MIN_D="9", B200OT_TC_MIN_PAIRS="0")
TC = dict(B200OT_TC_MIN_D="1", B200OT_TC_MIN_PAIRS="0")


def emit(**kw):
    print(json.dumps(kw), flush=True)


def relmax(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def part_a(dev, sizes, dims, reps):
    g = torch.Generator().manual_seed(0)
    for N in sizes:
        M = N
        for D in dims:
            x = torch.rand(N, D, generator=g).to(dev)
            y = torch.rand(M, D, generator=g).to(dev)
            h = (torch.rand(M, generator=g) * 0.1).to(dev)
            w = (torch.rand(M, generator=g) / M).to(dev)
            go = torch.rand(N, generator=g).to(dev)
            eps, blur = 1e-4, 0.05
            center = ops.default_center(x, y)
            with env(**SIMT):
                _, lse2 = ops.softmin_raw(eps, x, y, h, p=2, want_lse2=True, center=center)
            table = [
                ("softmin_fwd", lambda: ops.softmin_raw(eps, x, y, h, p=2, center=center)[0]),
                ("softmin_bwd", lambda: ops.softmin_grad_rows(eps, x, y, h, None, 0.0, lse2, go, p=2, center=center)),
                ("conv_fwd", lambda: ops.kernel_conv_raw("gaussian", x, y, w, blur, center=center)),
                ("conv_bwd", lambda: ops.kernel_conv_grad_rows("gaussian", x, y, w, blur, go, center=center)),
            ]
            for name, fn in table:
                res = {}
                for route, e in (("simt", SIMT), ("tc", TC)):
                    with env(**e):
                        ms = best_ms(fn, reps)
                        res[route] = (ms, fn())
                diff = relmax(res["tc"][1], res["simt"][1])
                emit(part="A", op=name, D=D, N=N, simt_ms=round(res["simt"][0], 3), tc_ms=round(res["tc"][0], 3),
                     simt_Tpairs_s=round(N * M / res["simt"][0] * 1e-9, 3),
                     tc_Tpairs_s=round(N * M / res["tc"][0] * 1e-9, 3),
                     tc_speedup=round(res["simt"][0] / res["tc"][0], 3), tc_vs_simt_relmax=diff)


def brute_rows(x, y, w, blur, rows):
    """fp64 value and unit row gradient of the gaussian matvec on sampled rows."""
    xr, yd = x[rows].double(), y.double()
    d2 = (xr * xr).sum(1)[:, None] - 2 * xr @ yd.t() + (yd * yd).sum(1)[None, :]
    k = torch.exp(-d2.clamp_min(0) / (2 * blur * blur)) * w.double()[None, :]
    val = k.sum(1)
    grad = (k @ yd - val[:, None] * xr) / (blur * blur)
    return val, grad


def part_c(dev, N, dims, reps):
    g = torch.Generator().manual_seed(2)
    M = N
    for D in dims:
        x = torch.rand(N, D, generator=g).to(dev)
        y = torch.rand(M, D, generator=g).to(dev)
        w = (torch.rand(M, generator=g) / M).to(dev)
        ones = torch.ones(N, device=dev)
        blur = 0.25 * (D / 3.0) ** 0.5
        center = ops.default_center(x, y)
        rows = torch.randint(0, N, (64,), generator=g).to(dev)
        for self_term in (False, True):
            yy, ww = (x, (torch.rand(N, generator=g) / N).to(dev)) if self_term else (y, w)
            vref, gref = brute_rows(x, yy, ww, blur, rows)
            t_two = best_ms(lambda: (ops.kernel_conv_raw("gaussian", x, yy, ww, blur, center=center),
                                     ops.kernel_conv_grad_rows("gaussian", x, yy, ww, blur, ones, center=center)), reps)
            t_one = best_ms(lambda: ops.kernel_conv_value_and_grad_rows("gaussian", x, yy, ww, blur, center=center),
                            reps)
            v2 = ops.kernel_conv_raw("gaussian", x, yy, ww, blur, center=center)
            g2 = ops.kernel_conv_grad_rows("gaussian", x, yy, ww, blur, ones, center=center)
            v1, g1 = ops.kernel_conv_value_and_grad_rows("gaussian", x, yy, ww, blur, center=center)
            emit(part="C", D=D, N=N, self_term=self_term, two_pass_ms=round(t_two, 3),
                 one_pass_ms=round(t_one, 3), value_vs_fwd_relmax=relmax(v1, v2), grad_vs_bwd_relmax=relmax(g1, g2),
                 value_vs_fp64_relmax_64rows=relmax(v1[rows].double(), vref),
                 fwd_value_vs_fp64_relmax_64rows=relmax(v2[rows].double(), vref),
                 grad_vs_fp64_relmax_64rows=relmax(g1[rows].double(), gref))
        # the configs[2] regime (blur = .05 at D = 64: the loss IS the diagonal of K_xx): value from the one-pass kernel
        if D == 64:
            a = torch.full((N,), 1.0 / N, device=dev)
            v2 = ops.kernel_conv_raw("gaussian", x, x, a, 0.05, center=center)
            v1, _ = ops.kernel_conv_value_and_grad_rows("gaussian", x, x, a, 0.05, center=center)
            emit(part="C", D=D, N=N, regime="configs[2] blur=.05 self term", value_vs_fwd_relmax=relmax(v1, v2),
                 value_vs_exact_diag_relmax=relmax(v1, a))


def part_d(dev, N, reps):
    """BASELINE configs[2] itself: SamplesLoss("gaussian", blur=.05) on N = M = 1e6, D = 64, forward + gradient w.r.t. x,
    with the two-pass and the one-pass evaluation."""
    from geomloss_b200 import SamplesLoss

    g = torch.Generator().manual_seed(0)
    x = torch.rand(N, 64, generator=g).to(dev)
    y = torch.rand(N, 64, generator=g).to(dev)
    L = SamplesLoss("gaussian", blur=0.05, backend="online")
    xg = x.clone().requires_grad_(True)

    def fwd_bwd():
        v = L(xg, y)
        torch.autograd.grad(v, xg)
        return v

    t_fwd = best_ms(lambda: L(x, y), reps)
    emit(part="D", what="forward only (3 reductions)", N=N, ms=round(t_fwd, 2), Tpairs_s=round(3.0 * N * N / t_fwd * 1e-9, 3))
    for label, fused in (("two-pass", False), ("one-pass", True)):
        ops.FUSED_CONV_GRAD = fused
        ms = best_ms(fwd_bwd, reps)
        v = fwd_bwd().item()
        emit(part="D", what=label, N=N, fwd_bwd_ms=round(ms, 2), value=v)
    ops.FUSED_CONV_GRAD = False


def part_e(dev, N, dims, reps):
    """Forward kernels side by side: the softmin epilogue (no column weights: MUFU + FADD) against the gaussian one
    (weights from shared memory: LDS.128 + MUFU + FFMA) — bounds what folding log2 w_j into the exponent could buy."""
    g = torch.Generator().manual_seed(3)
    M = N
    for D in dims:
        x = torch.rand(N, D, generator=g).to(dev)
        y = torch.rand(M, D, generator=g).to(dev)
        h = (torch.rand(M, generator=g) * 0.1).to(dev)
        w = (torch.rand(M, generator=g) / M).to(dev)
        blur = 0.25 * (D / 3.0) ** 0.5
        center = ops.default_center(x, y)
        t_s = best_ms(lambda: ops.softmin_raw(blur * blur, x, y, h, p=2, center=center), reps)
        t_c = best_ms(lambda: ops.kernel_conv_raw("gaussian", x, y, w, blur, center=center), reps)
        emit(part="E", D=D, N=N, softmin_fwd_ms=round(t_s, 3), conv_fwd_ms=round(t_c, 3),
             softmin_Tpairs_s=round(N * M / t_s * 1e-9, 3), conv_Tpairs_s=round(N * M / t_c * 1e-9, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes (functional check of the script)")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--parts", default="CDEA")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    big = 20000 if args.quick else 400000
    if "C" in args.parts:
        part_c(dev, big, (3, 64), args.reps)
    if "D" in args.parts:
        part_d(dev, 50000 if args.quick else 1000000, 1)
    if "E" in args.parts:
        part_e(dev, big, (16, 32, 64), args.reps)
    if "A" in args.parts:
        part_a(dev, [3000] if args.quick else [30000, 100000, 400000], (4, 5, 6, 7, 8), args.reps)


if __name__ == "__main__":
    main()

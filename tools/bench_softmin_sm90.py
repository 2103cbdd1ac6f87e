"""Clock-normalised A/B timing of the dense softmin partial-reduction kernel (the headline hot loop) between builds.

    python -c "from geomloss_b200 import _build; _build.build(extra_flags=['-DB200OT_BIG_CH=16', '-DB200OT_BIG_R=4'], \
               out='build/libR4.so')"
    python tools/bench_softmin_sm90.py build/libA.so build/libR4.so [--dims 3 4] [--reps 5] [--json out.jsonl]

`b200ot_softmin_partial` is timed alone, as bench.py's `kernel_pass` does it: N = M = 1e6 (--n), blur = .01, the
bench's uniform-in-cube clouds (seed 0) and its initial potential as the column weights, the L2 flushed before every
launch, CUDA events around the launch.  The libraries are alternated launch by launch (A B A B ...) in one process,
and the MUFU.EX2 micro-benchmark (`b200ot_ubench`) runs in the same rotation, so every arm sees the same card state.

An NVML thread samples the SM clock every 20 ms and files each sample under the arm that is running.  Each arm reports
pairs/s, pairs per SM-cycle at its median sampled clock, and that figure over the MUFU.EX2 rate per SM-cycle measured
in the same window: the last one is code efficiency alone, whatever clock a power cap holds the card at.
"""
import argparse
import ctypes
import json
import math
import os
import statistics
import sys
import threading

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from geomloss_b200 import _lib, ops  # noqa: E402


def load(path):
    h = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in _lib._SIGNATURES.items():
        fn = getattr(h, name)
        fn.restype, fn.argtypes = res, args
    return h


class Clock:
    """SM clock samples (MHz) filed under the arm named in `self.arm`."""

    def __init__(self, index):
        import pynvml

        pynvml.nvmlInit()
        self.nv, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(index)
        self.arm, self.samples, self.power = None, {}, {}
        self._stop = threading.Event()
        self._thr = threading.Thread(target=self._run, daemon=True)

    def card(self):
        nv, h = self.nv, self.h
        name = nv.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                "sm_max_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)}

    def _run(self):
        while not self._stop.is_set():
            arm = self.arm
            if arm is not None:
                try:
                    self.samples.setdefault(arm, []).append(self.nv.nvmlDeviceGetClockInfo(self.h, self.nv.NVML_CLOCK_SM))
                    self.power.setdefault(arm, []).append(self.nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0)
                except Exception:
                    pass
            self._stop.wait(0.02)

    def __enter__(self):
        self._thr.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._thr.join()


def timed(fn, flush):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+", help="library builds to compare (paths to libb200ot.so variants)")
    ap.add_argument("--dims", type=int, nargs="+", default=[3, 4])
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--blur", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=5, help="timed launches per arm and dimension (after one warm-up)")
    ap.add_argument("--json", default=None, help="also append the result lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_softmin_sm90.py times a CUDA kernel: it needs a GPU")

    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    libs = [(os.path.basename(p), load(p)) for p in args.libs]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sink = torch.zeros(256, dtype=torch.float32, device=dev)
    st = ops._stream(dev)
    N = M = args.n
    eps = args.blur ** 2
    p = 2
    clock = Clock(0)
    card = clock.card()
    out = []

    def ubench(L):
        ops_per = ctypes.c_int32(0)
        iters, blocks = 65536, sms * 8
        _lib.check(L.b200ot_ubench(0, iters, blocks, ops._ptr(sink), ctypes.byref(ops_per), st), "ubench")
        return float(blocks) * 256 * iters * ops_per.value

    with clock:
        for D in args.dims:
            g = torch.Generator().manual_seed(0)
            x = torch.rand(N, D, generator=g).to(dev)
            y = torch.rand(M, D, generator=g).to(dev)
            a_log = torch.full((N,), -math.log(N), device=dev)
            b_log = torch.full((M,), -math.log(M), device=dev)
            center = ops.default_center(x, y)
            # bench.py's column weights: h = log b + g_ab / eps with its initial potential g_ab
            g_ab = ops.softmin_raw(eps, y, x, a_log, p=p, center=center)[0]
            arms = []
            for tag, L in libs:
                nsplit = L.b200ot_softmin_num_splits(N, M, D)
                cols = torch.empty(L.b200ot_packed_cols_floats(M, D, 1), dtype=torch.float32, device=dev)
                part = torch.empty(nsplit * N * 2, dtype=torch.float32, device=dev)
                _lib.check(L.b200ot_softmin_pack(ops._ptr(y), ops._ptr(b_log), ops._ptr(g_ab), float(1.0 / eps),
                                                 ops._ptr(center), M, D, p, float(eps), ops._ptr(cols), st), "pack")

                def run(L=L, cols=cols, part=part, nsplit=nsplit):
                    _lib.check(L.b200ot_softmin_partial(ops._ptr(x), ops._ptr(center), ops._ptr(cols), ops._ptr(part),
                                                        nsplit, N, M, D, p, float(eps), st), "partial")

                arms.append((f"{tag}", run, []))
            mufu = ("mufu_ex2", lambda: None, [])
            work = ubench(libs[0][1])
            for r in range(args.reps + 1):
                for name, run, ts in arms:
                    clock.arm = (D, name) if r > 0 else None
                    t = timed(run, flush)
                    if r > 0:
                        ts.append(t)
                clock.arm = (D, "mufu_ex2") if r > 0 else None
                t = timed(lambda: ubench(libs[0][1]), flush)
                if r > 0:
                    mufu[2].append(t)
                clock.arm = None
            mhz_mufu = statistics.median(clock.samples.get((D, "mufu_ex2"), [float("nan")]))
            mufu_rate = work / statistics.median(mufu[2])
            mufu_per_clk = mufu_rate / (sms * mhz_mufu * 1e6)
            for name, _, ts in arms:
                mhz = statistics.median(clock.samples.get((D, name), [float("nan")]))
                rate = float(N) * M / statistics.median(ts)
                per_clk = rate / (sms * mhz * 1e6)
                line = {"lib": name, "D": D, "N": N, "M": M, "blur": args.blur, "reps": len(ts),
                        "ms_median": round(statistics.median(ts) * 1e3, 3),
                        "ms_min": round(min(ts) * 1e3, 3), "ms_max": round(max(ts) * 1e3, 3),
                        "pairs_per_s": rate, "sm_mhz_median": mhz,
                        "power_w_median": statistics.median(clock.power.get((D, name), [float("nan")])),
                        "pairs_per_sm_cycle": round(per_clk, 3), "mufu_ex2_per_sm_cycle": round(mufu_per_clk, 3),
                        "frac_of_mufu_at_clock": round(per_clk / mufu_per_clk, 4),
                        "mufu_ex2_per_s": mufu_rate, "mufu_sm_mhz_median": mhz_mufu, "card": card}
                out.append(line)
                print(json.dumps(line), flush=True)
            del x, y, g_ab, arms
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "a") as f:
            for line in out:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

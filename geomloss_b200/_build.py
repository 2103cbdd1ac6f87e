"""In-tree build of libb200ot.so (the C-ABI CUDA library) with nvcc for sm_90a (H100).

No torch types cross the boundary, so this is a plain ``nvcc -shared``: it cross-compiles on a machine
without a GPU, and the library is loaded from the package directory.
"""
from __future__ import annotations

import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB_PATH = os.path.join(PKG, "libb200ot.so")
SOURCES = ["b200ot_core.cu", "b200ot_softmin.cu", "b200ot_softmin_bwd.cu", "b200ot_kernel_conv.cu", "b200ot_tc.cu",
           "b200ot_grid.cu", "b200ot_small.cu", "b200ot_wide.cu", "b200ot_plan_apply.cu", "b200ot_dense.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libb200ot.so cannot be built (set $NVCC)")


def _stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "b200ot.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def _compile_one(src: str, obj: str, verbose: bool, extra=()):
    cmd = [_nvcc(), "-c", *NVCC_FLAGS, *extra, "-I", os.path.join(ROOT, "include"), "-I", CSRC, src, "-o", obj]
    if verbose:
        cmd[1:1] = ["-Xptxas", "-v"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    return src, res.returncode, res.stdout + res.stderr


def build(force: bool = False, verbose: bool = False, extra_flags=(), out: str | None = None) -> str:
    """Compile every CUDA translation unit (in parallel) and link geomloss_b200/libb200ot.so; returns its path.

    ``extra_flags`` / ``out`` build a variant library next to the shipped one (``-DB200OT_BIG_CH=8`` ...): the A/B
    timing harness tools/ab_ops.py loads it through $B200OT_LIB."""
    variant = out is not None
    out = out or LIB_PATH
    if not variant and not force and not _stale():
        return LIB_PATH
    from concurrent.futures import ThreadPoolExecutor

    objdir = os.path.join(ROOT, "build", "obj_" + os.path.basename(out) if variant else "obj")
    os.makedirs(objdir, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    objs = [os.path.join(objdir, os.path.basename(s)[:-3] + ".o") for s in srcs]
    with ThreadPoolExecutor(max_workers=len(srcs)) as pool:
        results = list(pool.map(lambda so: _compile_one(so[0], so[1], verbose, tuple(extra_flags)), zip(srcs, objs)))
    for src, rc, log in results:
        if verbose:
            print(log)
        if rc != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{log}")
    cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", *objs, "-o", out + ".tmp"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout + res.stderr)
    os.replace(out + ".tmp", out)
    return out


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

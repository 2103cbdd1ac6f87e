"""CPU-only argument validation of the grid softmin entry point (csrc/b200ot_grid.cu): every bad argument of
``b200ot_softmin_grid`` is refused with B200OT_EINVAL before any CUDA call.  Every call below breaks exactly one rule,
so none reaches a launch (the fake pointers are never dereferenced)."""
import ctypes

import pytest

from geomloss_b200 import _build, _lib

EINVAL = -1  # B200OT_EINVAL
NULL, H_A, H_B, OLD, OUT = (ctypes.c_void_p(v) for v in (None, 0x1000, 0x2000, 0x3000, 0x4000))
MAX_N = 1024


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _grid(L, h_a=H_A, h_b=H_B, h_scale_b=0.5, out_old=OLD, alpha_old=0.5, beta=1.0, out=OUT, batch=3, N=16, dim=2,
          p=2, eps=0.1):
    return L.b200ot_softmin_grid(h_a, h_b, h_scale_b, out_old, alpha_old, beta, out, batch, N, dim, p, eps, NULL)


CASES = [
    dict(h_a=NULL), dict(out=NULL),
    dict(batch=0), dict(batch=-1), dict(batch=-(2**40)),
    dict(N=0), dict(N=-16), dict(N=MAX_N + 1),
    dict(dim=0), dict(dim=4), dict(dim=-1),
    dict(p=0), dict(p=3), dict(p=-2),
    dict(eps=0.0), dict(eps=-0.0), dict(eps=-1.0), dict(eps=float("nan")),
    # the passes run in place on `out`: it may not alias an input
    dict(out=H_A), dict(out=H_B), dict(out=OLD),
]


def test_symbol_exists(L):
    assert hasattr(L, "b200ot_softmin_grid") and "b200ot_softmin_grid" in _lib.exported_symbols()


@pytest.mark.parametrize("kw", CASES, ids=[",".join(f"{k}={v.value if isinstance(v, ctypes.c_void_p) else v}"
                                                    for k, v in kw.items()) for kw in CASES])
def test_softmin_grid_refuses(L, kw):
    assert _grid(L, **kw) == EINVAL
    # the same refusal with the optional inputs absent, where the rule does not involve them
    if kw.get("out") not in (H_B, OLD):
        assert _grid(L, **dict(dict(h_b=NULL, out_old=NULL, alpha_old=0.0), **kw)) == EINVAL

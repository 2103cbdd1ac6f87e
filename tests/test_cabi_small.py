"""CPU-only argument validation of the small-cloud entry points (csrc/b200ot_small.cu): the symbols exist and every bad
argument is refused with -1 before any CUDA call.  Every call below breaks at least one rule, so none reaches a launch
(the fake pointers are never dereferenced); a large batch is valid and therefore has no place here."""
import ctypes

import pytest

from geomloss_b200 import _build, _lib

SMALL = ["b200ot_sinkhorn_iteration_small", "b200ot_sinkhorn_loop_small", "b200ot_sinkhorn_final_bwd_small",
         "b200ot_sinkhorn_cost_small", "b200ot_kernel_mmd_small", "b200ot_kernel_mmd_bwd_small",
         "b200ot_kernel_mmd_value_small"]
NULL, FAKE, FAKE2 = ctypes.c_void_p(None), ctypes.c_void_p(0x1000), ctypes.c_void_p(0x2000)
MAXP = 65536  # B200OT_SMALL_MAX_POINTS
UNCLAMPED = 0x100

# batch, sizes, dimension (all but one valid in every call)
SIZES = [dict(B=0), dict(B=-3), dict(N=0), dict(N=-1), dict(M=0), dict(M=-1), dict(N=MAXP + 1), dict(M=MAXP + 1),
         dict(D=0), dict(D=9), dict(D=-1)]
BAD_P = [dict(p=3), dict(p=0), dict(p=-1), dict(p=2 | 0x200), dict(p=1 | 0x1000), dict(p=1 | UNCLAMPED | 0x10000)]
BAD_EPS = [dict(eps=0.0), dict(eps=-1.0), dict(eps=float("nan"))]


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


def _iteration(L, x=FAKE, y=FAKE, a_log=FAKE, b_log=FAKE, f_ba=NULL, g_ab=NULL, f_aa=NULL, g_bb=NULL, f_ba_out=FAKE,
               g_ab_out=FAKE, f_aa_out=FAKE, g_bb_out=FAKE, lse2=NULL, B=2, N=10, M=12, D=3, p=2, eps=0.1, alpha_old=0.0,
               beta=1.0):
    return L.b200ot_sinkhorn_iteration_small(x, y, a_log, b_log, f_ba, g_ab, f_aa, g_bb, f_ba_out, g_ab_out, f_aa_out,
                                             g_bb_out, lse2, B, N, M, D, p, eps, alpha_old, beta, 1, FAKE, NULL)


def _final_bwd(L, x=FAKE, y=FAKE, a_log=FAKE, b_log=FAKE, lse2=FAKE, grad_x=FAKE, grad_y=FAKE, B=2, N=10, M=12, D=3,
               p=2, eps=0.1):
    return L.b200ot_sinkhorn_final_bwd_small(x, y, a_log, b_log, FAKE, FAKE, FAKE, FAKE, lse2, FAKE, FAKE, FAKE, FAKE,
                                             grad_x, grad_y, B, N, M, D, p, eps, 1.0, NULL, 1, FAKE, NULL)


def _loop(L, x=FAKE, y=FAKE, a=FAKE, b=FAKE, eps_list=(1.0, 0.5), n_eps=None, pots_a=FAKE, pots_b=FAKE2,
          result=True, B=2, N=10, M=12, D=3, p=2, debias=1):
    arr = None if eps_list is None else (ctypes.c_double * len(eps_list))(*eps_list)
    n_eps = (1 if eps_list is None else len(eps_list)) if n_eps is None else n_eps
    which = ctypes.c_int32(-7)
    rc = L.b200ot_sinkhorn_loop_small(x, y, a, b, 1, arr, n_eps, -1.0, debias, pots_a, pots_b,
                                      ctypes.byref(which) if result else None, B, N, M, D, p, FAKE, NULL)
    assert which.value == -7  # nothing reported on a refusal
    return rc


def _cost(L, a=FAKE, b=FAKE, f_ba=FAKE, g_ab=FAKE, f_aa=FAKE, g_bb=FAKE, value=FAKE, B=2, N=10, M=12):
    return L.b200ot_sinkhorn_cost_small(a, b, f_ba, g_ab, f_aa, g_bb, B, N, M, -1.0, 0.1, value, NULL, NULL, NULL, NULL,
                                        NULL, NULL, NULL)


def _mmd(L, x=FAKE, y=FAKE, a=FAKE, b=FAKE, a_x=FAKE, b_y=FAKE, b_x=FAKE, B=2, N=10, M=12, D=3, kind=0, blur=0.5):
    return L.b200ot_kernel_mmd_small(x, y, a, b, a_x, b_y, b_x, FAKE, B, N, M, D, kind, blur, NULL)


def _mmd_bwd(L, x=FAKE, y=FAKE, a=FAKE, b=FAKE, grad_value=FAKE, grad_x=FAKE, grad_y=FAKE, B=2, N=10, M=12, D=3,
             kind=0, blur=0.5):
    return L.b200ot_kernel_mmd_bwd_small(x, y, a, b, grad_value, grad_x, grad_y, B, N, M, D, kind, blur, NULL)


def _mmd_value(L, a=FAKE, b=FAKE, a_x=FAKE, b_y=FAKE, b_x=FAKE, value=FAKE, B=2, N=10, M=12):
    return L.b200ot_kernel_mmd_value_small(a, b, a_x, b_y, b_x, B, N, M, value, NULL)


def test_symbols_exist(L):
    for name in SMALL:
        assert hasattr(L, name), name
        assert name in _lib.exported_symbols()


def _refused(f, L, cases, what):
    for kw in cases:
        assert f(L, **kw) == -1, f"{what}: {kw}"


def test_iteration_small_refuses(L):
    _refused(_iteration, L, [{k: NULL} for k in ("x", "y", "a_log", "b_log", "f_ba_out", "g_ab_out")], "null")
    _refused(_iteration, L, SIZES + BAD_P + BAD_EPS, "argument")
    # the debiasing outputs come as a pair
    _refused(_iteration, L, [dict(f_aa_out=NULL), dict(g_bb_out=NULL)], "one of f_aa_out / g_bb_out")
    # old potentials: all or none; alpha_old != 0 needs them
    partial = [dict(f_ba=FAKE), dict(g_ab=FAKE), dict(f_aa=FAKE), dict(g_bb=FAKE), dict(f_aa=FAKE, g_bb=FAKE),
               dict(f_ba=FAKE, g_ab=FAKE, f_aa=FAKE), dict(f_ba=FAKE, g_ab=FAKE, g_bb=FAKE),
               dict(f_ba=FAKE, g_ab=FAKE, f_aa=NULL, g_bb=NULL, alpha_old=0.5)]
    _refused(_iteration, L, partial, "old potentials")
    _refused(_iteration, L, [dict(alpha_old=0.5), dict(alpha_old=-1.0)], "alpha_old without old potentials")


def test_final_bwd_small_refuses(L):
    _refused(_final_bwd, L, [{k: NULL} for k in ("x", "y", "a_log", "b_log", "lse2", "grad_x", "grad_y")], "null")
    _refused(_final_bwd, L, SIZES + BAD_P + BAD_EPS, "argument")


def test_loop_small_refuses(L):
    _refused(_loop, L, [dict(eps_list=None), dict(n_eps=0), dict(n_eps=-2), dict(pots_a=NULL), dict(pots_b=NULL),
                        dict(result=False), dict(pots_b=FAKE)], "loop argument")
    # everything the first (initialisation) iteration validates, including its temperature
    _refused(_loop, L, [{k: NULL} for k in ("x", "y", "a", "b")], "null")
    _refused(_loop, L, SIZES + BAD_P + [dict(eps_list=(0.0, 0.5)), dict(eps_list=(-1.0,))], "argument")
    _refused(_loop, L, [dict(debias=0, B=0), dict(debias=0, D=9)], "no debias")


def test_cost_small_refuses(L):
    _refused(_cost, L, [{k: NULL} for k in ("a", "b", "f_ba", "g_ab", "value")], "null")
    _refused(_cost, L, [kw for kw in SIZES if "D" not in kw], "size")
    _refused(_cost, L, [dict(f_aa=NULL), dict(g_bb=NULL)], "one of f_aa / g_bb")


@pytest.mark.parametrize("call", ["mmd", "mmd_bwd"])
def test_kernel_mmd_small_refuses(L, call):
    f = {"mmd": _mmd, "mmd_bwd": _mmd_bwd}[call]
    ptrs = ("x", "y", "a", "b", "a_x", "b_y", "b_x") if call == "mmd" else ("x", "y", "a", "b", "grad_value", "grad_x",
                                                                           "grad_y")
    _refused(f, L, [{k: NULL} for k in ptrs], "null")
    _refused(f, L, SIZES, "size")
    _refused(f, L, [dict(kind=3), dict(kind=-1), dict(kind=0x200), dict(kind=1 | 0x400), dict(kind=2 | 0x10000)], "kind")
    # blur <= 0 for the gaussian and the laplacian, in both conventions (the energy distance has no blur)
    for kind in (0, 1, UNCLAMPED, 1 | UNCLAMPED):
        _refused(f, L, [dict(kind=kind, blur=0.0), dict(kind=kind, blur=-0.5), dict(kind=kind, blur=float("nan"))],
                 "blur")


def test_kernel_mmd_value_small_refuses(L):
    _refused(_mmd_value, L, [{k: NULL} for k in ("a", "b", "a_x", "b_y", "b_x", "value")], "null")
    _refused(_mmd_value, L, [kw for kw in SIZES if "D" not in kw], "size")

"""ctypes binding of libb200ot.so — the only way the Python host side reaches the CUDA kernels.

There is deliberately no fallback: if the library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int32, c_int64, c_void_p

_PKG = os.path.dirname(os.path.abspath(__file__))
# $B200OT_LIB: load a variant build instead (A/B kernel timing, tools/ab_ops.py) — never set in tests or the bench
LIB_PATH = os.environ.get("B200OT_LIB") or os.path.join(_PKG, "libb200ot.so")

_lib = None

_P = c_void_p  # device pointers and streams travel as void*
_I32P, _F32P = ctypes.POINTER(c_int32), ctypes.POINTER(c_float)  # small host arrays (per-axis grid geometry)


class B200OTError(RuntimeError):
    pass


_SIGNATURES = {
    "b200ot_version": (c_int32, []),
    "b200ot_strerror": (c_char_p, [c_int32]),
    "b200ot_last_cuda_error": (c_char_p, []),
    "b200ot_softmin_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32]),
    "b200ot_softmin_fwd": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, c_float, c_float, _P, _P, c_int64, c_int64,
                                     c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_softmin_pair_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32]),
    "b200ot_softmin_fwd_pair": (c_int32, [_P, _P, _P, _P, c_float, _P, c_float, c_float, _P, _P, _P, _P, c_float, _P,
                                          c_float, c_float, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_float,
                                          _P, c_int64, _P]),
    "b200ot_softmin_step_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32]),
    "b200ot_softmin_fwd_step": (c_int32, [_P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_float, _P, c_int64,
                                          _P]),
    "b200ot_softmin_bwd_x": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32,
                                       c_float, _P, c_int64, _P]),
    "b200ot_plan_apply_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32, c_int64]),
    "b200ot_plan_apply": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int64,
                                    c_int32, c_float, _P, c_int64, _P]),
    "b200ot_packed_cols_floats": (c_int64, [c_int64, c_int32, c_int32]),
    "b200ot_softmin_pack": (c_int32, [_P, _P, _P, c_float, _P, c_int64, c_int32, c_int32, c_float, _P, _P]),
    "b200ot_softmin_num_splits": (c_int32, [c_int64, c_int64, c_int32]),
    "b200ot_softmin_partial": (c_int32, [_P, _P, _P, _P, c_int32, c_int64, c_int64, c_int32, c_int32, c_float, _P]),
    "b200ot_softmin_finalize": (c_int32, [_P, c_int32, _P, c_float, c_float, _P, _P, c_int64, c_float, _P]),
    "b200ot_ranges_shape": (None, [c_int32, ctypes.POINTER(c_int32), ctypes.POINTER(c_int32),
                                   ctypes.POINTER(c_int32)]),
    "b200ot_softmin_pack_gather": (c_int32, [_P, _P, _P, c_float, _P, _P, c_int64, c_int32, c_int32, c_float, _P, _P]),
    "b200ot_softmin_partial_ranges": (c_int32, [_P, _P, _P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32, c_float,
                                                c_int32, _P]),
    "b200ot_softmin_merge": (c_int32, [_P, c_int32, _P, c_int64, _P]),
    "b200ot_softmin_bwd_partial": (c_int32, [_P, _P, _P, _P, _P, c_int32, c_int64, c_int64, c_int32, c_int32,
                                             c_float, _P]),
    "b200ot_softmin_bwd_partial_ranges": (c_int32, [_P, _P, _P, _P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32,
                                                    c_float, c_int32, _P]),
    "b200ot_softmin_bwd_sums": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, c_int64, c_int64, c_int32, c_int32,
                                          c_float, _P, c_int64, _P]),
    "b200ot_rowsum_merge": (c_int32, [_P, c_int32, c_int32, _P, c_int64, _P]),
    "b200ot_softmin_bwd_finalize": (c_int32, [_P, c_int32, _P, _P, _P, _P, c_int64, c_int32, c_int32, c_float, _P]),
    "b200ot_kernel_conv_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32]),
    "b200ot_kernel_conv_fwd": (c_int32, [_P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_float, _P,
                                         c_int64, _P]),
    "b200ot_kernel_conv_bwd_x": (c_int32, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_float, _P,
                                           c_int64, _P]),
    "b200ot_kernel_conv_fwd_bwd_x": (c_int32, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_float,
                                               _P, c_int64, _P]),
    "b200ot_kernel_conv_pack_gather": (c_int32, [_P, _P, _P, _P, c_int64, c_int32, c_int32, c_float, _P, _P]),
    "b200ot_kernel_conv_partial_ranges": (c_int32, [_P, _P, _P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32,
                                                    c_float, c_int32, c_int32, _P]),
    "b200ot_kernel_conv_finalize": (c_int32, [_P, c_int32, _P, c_int64, c_int32, _P]),
    "b200ot_kernel_conv_bwd_finalize": (c_int32, [_P, c_int32, _P, _P, _P, _P, c_int64, c_int32, c_int32, c_float,
                                                  _P]),
    "b200ot_batched_scratch_bytes": (c_int64, [c_int64, c_int64, c_int64, c_int32]),
    "b200ot_softmin_fwd_batched": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, c_float, c_float, _P, _P, c_int64,
                                             c_int64, c_int64, c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_softmin_bwd_x_batched": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, c_int64, c_int64, c_int64,
                                               c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_kernel_conv_fwd_batched": (c_int32, [_P, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32, c_int32,
                                                 c_float, _P, c_int64, _P]),
    "b200ot_kernel_conv_bwd_x_batched": (c_int32, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32, c_int32,
                                                   c_float, _P, c_int64, _P]),
    "b200ot_kernel_conv_fwd_bwd_x_batched": (c_int32, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32,
                                                       c_int32, c_float, _P, c_int64, _P]),
    "b200ot_softmin_l1_scratch_bytes": (c_int64, [c_int64, c_int64, c_int64, c_int32]),
    "b200ot_softmin_l1_fwd": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, c_float, c_float, _P, _P, c_int64, c_int64,
                                        c_int64, c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_softmin_l1_bwd_x": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32,
                                          c_int32, c_float, _P, c_int64, _P]),
    "b200ot_wide_scratch_bytes": (c_int64, [c_int64, c_int64, c_int64, c_int32]),
    "b200ot_wide_softmin_fwd": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, c_float, c_float, _P, _P, c_int64, c_int64,
                                          c_int64, c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_wide_softmin_bwd_x": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, c_int64, c_int64, c_int64,
                                            c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_wide_kernel_conv_fwd": (c_int32, [_P, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32, c_int32, c_float,
                                              _P, c_int64, _P]),
    "b200ot_wide_kernel_conv_bwd_x": (c_int32, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int32, c_int32,
                                                c_float, _P, c_int64, _P]),
    "b200ot_wide_plan_apply_scratch_bytes": (c_int64, [c_int64, c_int64, c_int32, c_int64]),
    "b200ot_wide_plan_apply": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32,
                                         c_int64, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_dense_scratch_bytes": (c_int64, [c_int64, c_int64, c_int64]),
    "b200ot_dense_softmin_pair": (c_int32, [_P, _P, _P, _P, _P, c_float, c_float, c_float, _P, _P, _P, _P, c_int64,
                                            c_int64, c_int64, c_float, _P, c_int64, _P]),
    "b200ot_dense_softmin_pair_bwd": (c_int32, [_P, _P, _P, _P, _P, c_float, _P, _P, _P, _P, _P, c_int64, c_int64,
                                                c_int64, _P]),
    "b200ot_dense_rows_scratch_bytes": (c_int64, [_P, c_int32]),
    "b200ot_dense_softmin_rows": (c_int32, [_P, c_int32, c_float, c_float, c_float, _P, c_int64, _P]),
    "b200ot_dense_softmin_rows_bwd": (c_int32, [_P, _P, _P, c_float, _P, _P, _P, c_int64, c_int64, c_int64, _P]),
    "b200ot_blocks_shape": (None, [ctypes.POINTER(c_int32), ctypes.POINTER(c_int32)]),
    "b200ot_blocks_scratch_bytes": (c_int64, [c_int64, c_int64, c_int64, _P, c_int64, _P, c_int32]),
    "b200ot_softmin_fwd_blocks": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, c_float, c_float, _P, _P, c_int64, _P,
                                            c_int64, _P, c_int64, _P, c_int64, _P, c_int32, c_int32, c_float, _P,
                                            c_int64, _P]),
    "b200ot_softmin_bwd_x_blocks": (c_int32, [_P, _P, _P, _P, c_float, _P, _P, _P, _P, c_int64, _P, c_int64, _P,
                                              c_int64, _P, c_int64, _P, c_int32, c_int32, c_float, _P, c_int64, _P]),
    "b200ot_sinkhorn_iteration_small": (c_int32, [_P] * 13 + [c_int64, c_int64, c_int64, c_int32, c_int32, c_float,
                                                  c_float, c_float, c_int32, _P, _P]),
    "b200ot_sinkhorn_loop_small": (c_int32, [_P, _P, _P, _P, c_int32, ctypes.POINTER(ctypes.c_double), c_int32,
                                             ctypes.c_double, c_int32, _P, _P, ctypes.POINTER(c_int32), c_int64,
                                             c_int64, c_int64, c_int32, c_int32, _P, _P]),
    "b200ot_sinkhorn_final_bwd_small": (c_int32, [_P] * 15 + [c_int64, c_int64, c_int64, c_int32, c_int32, c_float,
                                                  c_float, _P, c_int32, _P, _P]),
    "b200ot_sinkhorn_cost_small": (c_int32, [_P] * 6 + [c_int64, c_int64, c_int64, c_float, c_float] + [_P] * 8),
    "b200ot_kernel_mmd_value_small": (c_int32, [_P] * 5 + [c_int64, c_int64, c_int64, _P, _P]),
    "b200ot_cloud_extent_scratch_bytes": (c_int64, []),
    "b200ot_cloud_extent": (c_int32, [_P, c_int64, _P, c_int64, c_int32, _P, _P, c_int64, _P]),
    "b200ot_kernel_mmd_small": (c_int32, [_P] * 8 + [c_int64, c_int64, c_int64, c_int32, c_int32, c_float, _P]),
    "b200ot_kernel_mmd_bwd_small": (c_int32, [_P] * 7 + [c_int64, c_int64, c_int64, c_int32, c_int32, c_float, _P]),
    "b200ot_softmin_grid": (c_int32, [_P, _P, c_float, _P, c_float, c_float, _P, c_int64, c_int32, c_int32, c_int32,
                                      c_float, _P]),
    "b200ot_softmin_grid_axes": (c_int32, [_P, _P, c_float, _P, c_float, c_float, _P, c_int64, c_int32, _I32P, _F32P,
                                           _I32P, c_float, _P]),
    "b200ot_grid_plan_apply": (c_int32, [_P, _P, c_float, _P, _P, _P, c_int64, c_int32, c_int32, _I32P, _F32P, _I32P,
                                         c_float, _P]),
    "b200ot_ubench": (c_int32, [c_int32, c_int32, c_int32, _P, ctypes.POINTER(c_int32), _P]),
}


class SoftminSlot(ctypes.Structure):
    """``b200ot_softmin_slot`` of include/b200ot.h: one softmin of a b200ot_softmin_fwd_step group."""
    _fields_ = [("h_a", _P), ("h_b", _P), ("h_scale_b", c_float), ("out_old", _P), ("alpha_old", c_float),
                ("beta", c_float), ("out", _P), ("lse2", _P)]


class DenseRows(ctypes.Structure):
    """``b200ot_dense_rows`` of include/b200ot.h: one problem of a b200ot_dense_softmin_rows group."""
    _fields_ = [("C", _P), ("log_w", _P), ("pot", _P), ("out_old", _P), ("out", _P), ("lse2", _P), ("B", c_int64),
                ("n_rows", c_int64), ("n_cols", c_int64)]


def exported_symbols():
    """Names every build of the library must export (mirrors include/b200ot.h)."""
    return sorted(_SIGNATURES)


def lib():
    """Load (once) and return the C-ABI library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200OTError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  geomloss_b200 has no CPU or eager fallback.")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(code: int, what: str):
    if code != 0:
        L = lib()
        msg = L.b200ot_strerror(code).decode()
        if code == -3:
            msg += ": " + L.b200ot_last_cuda_error().decode()
        raise B200OTError(f"{what} failed: {msg}")

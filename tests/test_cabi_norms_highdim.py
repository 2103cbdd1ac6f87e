"""CPU-only argument validation of the laplacian and energy kernel convolutions in the tensor-core dimensions
(8 < D <= 64): the entry points accept them (a too-small scratch is the first thing refused, -2) and still refuse
D = 65 (-1).  Nothing here reaches a CUDA call."""
import ctypes

import pytest

from geomloss_b200 import _build, _lib, ops


@pytest.fixture(scope="module")
def L():
    _build.build()
    return _lib.lib()


@pytest.mark.parametrize("kind", [1, 2, 1 | 0x100, 2 | 0x100])
def test_norm_kinds_accept_tensor_core_dimensions(L, kind):
    null, fake = ctypes.c_void_p(None), ctypes.c_void_p(0x1000)
    for d in (9, 16, 33, 64):
        assert L.b200ot_kernel_conv_fwd(fake, fake, fake, null, fake, 10, 10, d, kind, 0.1, fake, 16, null) == -2
        assert L.b200ot_kernel_conv_bwd_x(fake, fake, fake, null, fake, fake, 10, 10, d, kind, 0.1, fake, 16,
                                          null) == -2
    assert L.b200ot_kernel_conv_fwd(fake, fake, fake, null, fake, 10, 10, 65, kind, 0.1, fake, 1 << 30, null) == -1
    assert L.b200ot_kernel_conv_bwd_x(fake, fake, fake, null, fake, fake, 10, 10, 65, kind, 0.1, fake, 1 << 30,
                                      null) == -1
    # the one-pass value + gradient stays gaussian-only, the ranges stages stay at D <= 8
    assert L.b200ot_kernel_conv_fwd_bwd_x(fake, fake, fake, null, fake, fake, 10, 10, 16, kind, 0.1, fake, 1 << 30,
                                          null) == -1
    assert L.b200ot_kernel_conv_partial_ranges(fake, null, fake, fake, 1, fake, fake, 10, 16, kind, 0.1, 0, 0,
                                               null) == -1


def test_dimension_error_says_what_is_served_where():
    import torch

    ops._check_clouds(torch.rand(5, 64), torch.rand(6, 64), ops.MAX_D_TC)
    with pytest.raises(NotImplementedError, match="laplacian and energy"):
        ops._check_clouds(torch.rand(5, 65), torch.rand(6, 65), ops.MAX_D_TC)

"""CPU: the host-side tile / split-K plan of the weight-gradient convolution (etb_conv_wgrad_workspace_bytes) for every
small output map, square or not.  The plan runs on the host only, so no GPU is needed: for each geometry the call must
return, and the workspace must be a whole number (1..512) of fp32 [Cout, k*k*Cin] split-K slices.  Output maps of at most
3 pixels (a 3x3 s2 conv on a 2x2 map, the stride-32 level of a 32-pixel image) once left the K tile unset and divided
by zero on the host."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from efficientteacher_b200 import _lib
    return _lib


def _params(lib, N, Cin, H, W, Cout, k, s, p):
    cp = lib.EtbConvParams()
    cp.N, cp.H, cp.W, cp.Cin, cp.Cout = N, H, W, Cin, Cout
    cp.kh = cp.kw = k
    cp.stride, cp.pad = s, p
    cp.x_cstride, cp.y_cstride = Cin, (Cout + 7) // 8 * 8
    return cp


def _splits(lib, case):
    N, Cin, H, W, Cout, k, s, p = case
    nbytes = int(lib.lib().etb_conv_wgrad_workspace_bytes(C.byref(_params(lib, *case))))
    slice_bytes = Cout * k * k * Cin * 4
    assert nbytes > 0 and nbytes % slice_bytes == 0, (case, nbytes, slice_bytes)
    sk = nbytes // slice_bytes
    assert 1 <= sk <= 512, (case, sk)
    return sk


def _geometries():
    """(k, s, p, H, W) for every output map Ho x Wo in 1..12 x 1..12: 3x3 s1, 3x3 s2 from both the odd (2n-1) and the even
    (2n) input extent, 1x1 s1 (the flat pointwise tiling) and 1x1 s2 (tiled)."""
    out = []
    for ho in range(1, 13):
        for wo in range(1, 13):
            out.append((3, 1, 1, ho, wo))
            out.append((1, 1, 0, ho, wo))
            for dh in (1, 0):
                for dw in (1, 0):
                    out.append((3, 2, 1, 2 * ho - dh, 2 * wo - dw))
                    out.append((1, 2, 0, 2 * ho - dh, 2 * wo - dw))
    return out


@pytest.mark.parametrize("N,Cin,Cout", [(1, 32, 64), (2, 128, 256), (32, 512, 512)])
def test_wgrad_plan_small_maps(lib, N, Cin, Cout):
    n = 0
    for k, s, p, H, W in _geometries():
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        assert 1 <= Ho <= 12 and 1 <= Wo <= 12
        _splits(lib, (N, Cin, H, W, Cout, k, s, p))
        n += 1
    assert n == 144 * 10


# (Wo, Ho) in {(1,1), (1,2), (1,3), (2,1), (3,1)}: no 16-row K box fits within twice the map, so the plan needs its fallback
PLAN_HOLES = [
    (2, 512, 2, 2, 1024, 3, 2, 1),     # 3x3 s2 on a 2x2 map -> 1x1
    (1, 64, 1, 1, 64, 3, 1, 1),        # 1x1 map, 3x3 s1
    (4, 256, 4, 2, 512, 3, 2, 1),      # 1x2 (Wo x Ho) from a 2x4 (W x H) input
    (2, 32, 5, 1, 64, 3, 2, 1),        # 1x3
    (2, 128, 1, 3, 128, 3, 1, 1),      # 3x1 (Wo = 3, Ho = 1)
    (3, 64, 2, 4, 64, 3, 2, 1),        # 2x1
    (2, 512, 2, 6, 512, 3, 2, 1),      # 3x1: the stride-2 conv into the stride-32 level of a 32x96 (H x W) image
]

REAL = [
    (32, 64, 160, 160, 64, 3, 1, 1),
    (32, 128, 160, 160, 256, 3, 2, 1),
    (32, 256, 40, 40, 256, 3, 1, 1),
    (32, 2048, 20, 20, 1024, 1, 1, 0),
    (2, 512, 11, 20, 512, 3, 1, 1),    # stride-32 level of a 352x640 letterboxed batch
    (2, 256, 22, 40, 512, 3, 2, 1),
]


@pytest.mark.parametrize("case", PLAN_HOLES + REAL)
def test_wgrad_plan_named_shapes(lib, case):
    _splits(lib, case)


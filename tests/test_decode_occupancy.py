"""b2q_debug_decode_occupancy: resident CTAs per SM of the decode tier's launch plans (tools/decode_launch_cost.py)."""
import ctypes

import pytest

from gptqmodel_b200 import _lib as g


def test_occupancy_query_rejects_bad_arguments_without_gpu():
    blocks = ctypes.c_int(0)
    for args in ((3, 1, 4096, 4096), (1, 9, 4096, 4096), (2, 1, 4000, 4096), (1, 1, 4096, 48)):
        assert g.lib.b2q_debug_decode_occupancy(*args, 0, 0, ctypes.byref(blocks)) == -2, args
    assert g.lib.b2q_debug_decode_occupancy(1, 1, 4096, 4096, 0, 0, None) == -2


@pytest.mark.gpu
@pytest.mark.parametrize("version,K,N,ks,warps", [(1, 4096, 4096, 0, 0), (1, 14336, 4096, 0, 0),
                                                  (2, 4096, 6144, 1, 16), (2, 4096, 28672, 1, 16)])
def test_occupancy_of_bench_launch_plans(version, K, N, ks, warps):
    # every plan the planner returns must be launchable: at least one CTA of it fits on an SM
    plan = (ctypes.c_int * 8)()
    assert g.lib.b2q_debug_decode_plan(version, 1, K, N, ks, warps, plan) == 0
    blocks = ctypes.c_int(0)
    assert g.lib.b2q_debug_decode_occupancy(version, 1, K, N, ks, warps, ctypes.byref(blocks)) == 0, g.lib.b2q_last_error()
    assert blocks.value >= 1

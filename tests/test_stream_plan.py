"""The streamed scan's planner through the C ABI (no GPU needed): how a device budget is split between
the fixed part, the two chunk buffers and the resident candidate / S lists (DESIGN.md §4c)."""
import ctypes as C

import pytest

from smudgeplot_b200 import _lib


def _plan(n, k, ibyte, budget):
    lay = _lib.StreamLayout()
    rc = _lib.lib().hm_stream_plan(n, k, ibyte, budget, C.byref(lay))
    return rc, lay


@pytest.mark.parametrize("n,k,ibyte", [(200_000_000, 31, 3), (4_400_000_000, 31, 3), (20_000_000, 40, 3),
                                       (9674, 21, 2), (112_316, 11, 1), (1_000_000, 64, 2)])
def test_stream_plan_fits_the_budget_and_is_monotone(built, n, k, ibyte):
    prev = 0
    feasible = 0
    for budget in [int(x) for x in (2e5, 1e6, 4.6e6, 6e6, 2e7, 1.7e8, 3e8, 1e9, 4e9, 2e10, 8e10)]:
        rc, lay = _plan(n, k, ibyte, budget)
        if rc != 0:
            assert rc == -3 and prev == 0                      # HM_ENOMEM, and only below every feasible budget
            assert b"cannot hold one chunk" in _lib.lib().hm_last_error()
            continue
        feasible += 1
        assert lay.budget == budget
        assert lay.fixed_bytes + lay.chunk_bytes + lay.list_bytes <= budget      # lists + two chunk buffers fit
        assert lay.list_bytes >= lay.chunk_list_bytes >= 0                       # room for the first chunk at least
        assert 1 <= lay.chunk <= n
        assert lay.chunk >= prev                                                 # monotone in the budget
        prev = lay.chunk
    assert feasible >= 3


def test_stream_plan_refuses_a_budget_without_room_for_one_chunk(built):
    rc, lay = _plan(200_000_000, 31, 3, 100 << 20)         # the 128 MB stub index alone does not fit
    assert rc == -3
    msg = _lib.lib().hm_last_error()
    assert b"cannot hold one chunk" in msg and b"104857600" in msg
    assert _plan(10, 31, 3, -1)[0] == -1                    # bad arguments
    assert _plan(10, 65, 3, 1 << 30)[0] == -1
    assert _plan(10, 31, 4, 1 << 30)[0] == -1


def test_stream_plan_takes_the_whole_table_when_the_budget_allows(built):
    rc, lay = _plan(50_000, 31, 2, 1 << 34)
    assert rc == 0 and lay.chunk == 50_000


def test_stream_symbols_are_exported_and_bound(built):
    L = _lib.lib()
    for sym in ("hm_set_device_budget", "hm_stream_plan", "hm_scan_residency"):
        assert sym in _lib.ABI_SYMBOLS
        assert hasattr(L, sym)
    assert L.hm_abi_version() == 1                          # new functions only: the ABI version stays
    L.hm_set_device_budget(0)                               # 0 = free device memory minus the reserve

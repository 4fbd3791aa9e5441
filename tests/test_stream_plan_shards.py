"""The sharded streamed scan's planner through the C ABI (no GPU needed): each of G shards plans for the
whole-table Bloom filter plus the lists and chunks of its 1/G share (DESIGN.md §4c)."""
import ctypes as C

import pytest

from smudgeplot_b200 import _lib


def _plan(n, k, ibyte, budget, shards=None):
    lay = _lib.StreamLayout()
    if shards is None:
        rc = _lib.lib().hm_stream_plan(n, k, ibyte, budget, C.byref(lay))
    else:
        rc = _lib.lib().hm_stream_plan_shards(n, k, ibyte, budget, shards, C.byref(lay))
    return rc, lay


def _fields(lay):
    return {f: getattr(lay, f) for f, _ in _lib.StreamLayout._fields_}


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("n,k,ibyte", [(200_000_000, 31, 3), (20_000_000_000, 31, 3), (20_000_000, 40, 3),
                                       (9674, 21, 2), (1_000_000, 64, 2)])
def test_shard_plan_fits_the_budget_and_its_chunk_grows_with_it(built, n, k, ibyte, G):
    prev = 0
    feasible = 0
    for budget in [int(x) for x in (2e5, 1e6, 6e6, 2e7, 1.7e8, 3e8, 1e9, 4e9, 2e10, 8e10)]:
        rc, lay = _plan(n, k, ibyte, budget, G)
        if rc != 0:
            assert rc == -3 and prev == 0                      # HM_ENOMEM, and only below every feasible budget
            assert b"cannot hold one chunk" in _lib.lib().hm_last_error()
            continue
        feasible += 1
        assert lay.budget == budget
        assert lay.fixed_bytes + lay.chunk_bytes + lay.list_bytes <= budget
        assert lay.list_bytes >= lay.chunk_list_bytes >= 0
        assert 1 <= lay.chunk <= -(-n // G)                    # no longer than a share
        assert lay.chunk >= prev
        prev = lay.chunk
    assert feasible >= 3


@pytest.mark.parametrize("n,k,ibyte", [(200_000_000, 31, 3), (4_400_000_000, 31, 3), (20_000_000, 40, 3),
                                       (9674, 21, 2), (112_316, 11, 1), (1_000_000, 64, 2), (0, 31, 2)])
def test_one_shard_is_hm_stream_plan(built, n, k, ibyte):
    for budget in [int(x) for x in (1e6, 2e7, 3e8, 4e9, 8e10)]:
        rc1, a = _plan(n, k, ibyte, budget)
        rc2, b = _plan(n, k, ibyte, budget, 1)
        assert rc1 == rc2
        if rc1 == 0:
            assert _fields(a) == _fields(b)


def test_list_room_per_shard_grows_with_the_shard_count(built):
    n, k, ibyte, budget = 50_000_000, 31, 3, 2 * 10 ** 10     # chunks as long as a share
    bloom = n // 8                                             # 1 bit per table entry
    prev = None
    for G in (1, 2, 4, 8, 16):
        rc, lay = _plan(n, k, ibyte, budget, G)
        assert rc == 0
        assert lay.fixed_bytes >= 8 * (1 << 24) + 8 * _lib.PLOT_CELLS + bloom      # stub index, plot, whole filter
        assert lay.fixed_bytes < 8 * (1 << 24) + 8 * _lib.PLOT_CELLS + bloom + (1 << 20)
        if prev is not None:
            assert lay.chunk <= prev.chunk
            assert lay.list_bytes > prev.list_bytes                  # smaller share: smaller chunks, more list room
            assert lay.list_bytes * G > prev.list_bytes * (G // 2)   # room per entry of the share: more than doubles
        prev = lay


def test_shard_plan_refuses_bad_arguments(built):
    assert _plan(10, 31, 3, 1 << 30, 0)[0] == -1
    assert _plan(10, 31, 3, 1 << 30, 17)[0] == -1
    assert _plan(10, 31, 3, -1, 2)[0] == -1
    rc, _ = _plan(200_000_000, 31, 3, 100 << 20, 4)              # the 128 MB stub index alone does not fit
    assert rc == -3 and b"cannot hold one chunk" in _lib.lib().hm_last_error()


def test_shard_plan_symbol_is_exported_and_bound(built):
    L = _lib.lib()
    assert "hm_stream_plan_shards" in _lib.ABI_SYMBOLS
    assert hasattr(L, "hm_stream_plan_shards")
    assert L.hm_stream_plan_shards.argtypes is not None and len(L.hm_stream_plan_shards.argtypes) == 6
    assert L.hm_abi_version() == 1

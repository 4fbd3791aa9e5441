"""CPU tests of the planning of conditioning across the ranks into new table files (dist.condition_ktab, DESIGN.md
§4f): the rank cuts on stub-bucket boundaries, every rank's sub-ranges under its budget (hm_rank_condition_cut), the
per-pass counts the histograms give, and the working-set function (hm_rank_condition_bytes)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from smudgeplot_b200 import _lib  # noqa: E402
from smudgeplot_b200 import dist as hd  # noqa: E402

MAX_RANGE = 1 << 31                                           # HM_COND_MAX_RANGE


@pytest.fixture(scope="module")
def L(built):
    return _lib.lib()


def _starts(cuts):
    return list(zip(cuts, cuts[1:]))


@pytest.mark.parametrize("k,ibyte", [(12, 1), (12, 2), (12, 3), (21, 1), (21, 2), (31, 3), (40, 2), (64, 1), (4, 1)])
def test_rank_cuts_lie_on_buckets_and_cover_every_prefix(k, ibyte):
    hb = min(_lib.COND_HIST_BITS, 2 * k)
    rng = np.random.default_rng(k * 10 + ibyte)
    for world in (1, 2, 3, 5, 8):
        for shape in ("random", "one", "empty"):
            h = rng.integers(0, 9, size=1 << hb).astype(np.int64) * (rng.random(1 << hb) < 0.5)
            if shape == "one":
                h[:] = 0
                h[(1 << hb) // 3] = 1000
                h[7] = 1
            elif shape == "empty":
                h[:] = 0
            cuts = hd.bucket_condition_cuts(h, world, hb, ibyte)
            assert len(cuts) == world + 1 and cuts[0] == 0 and cuts[-1] == 1 << hb
            assert all(a <= b for a, b in zip(cuts, cuts[1:]))
            step = 1 << max(hb - 8 * ibyte, 0)                # prefixes per bucket where buckets are coarser
            assert all(c % step == 0 for c in cuts), (cuts, step)
            if 8 * ibyte >= hb:                               # buckets as fine as prefixes: the plain cut
                assert cuts == hd.condition_cuts(h, world)
            spans = [hd.prefix_buckets(a, b, hb, ibyte) for a, b in _starts(cuts) if a < b]
            assert spans[0][0] == 0 and spans[-1][1] == 1 << (8 * ibyte)          # the spans tile the buckets
            assert all(x[1] == y[0] for x, y in zip(spans, spans[1:]))


def test_prefix_buckets():
    assert hd.prefix_buckets(0, 1 << 20, 20, 3) == (0, 1 << 24)
    assert hd.prefix_buckets(5, 6, 20, 3) == (80, 96)
    assert hd.prefix_buckets(5, 6, 20, 1) == (0, 1)
    assert hd.prefix_buckets(4096, 8193, 20, 1) == (1, 3)
    assert hd.prefix_buckets(3, 4, 8, 1) == (3, 4)


def _cut(L, k, ibyte, world, share, symm, budget, h):
    h = np.ascontiguousarray(h, dtype=np.int64)
    cuts = np.zeros(h.size + 1, dtype=np.int64)
    n = C.c_int64()
    rc = L.hm_rank_condition_cut(k, ibyte, world, share, symm, budget, h.ctypes.data, h.size, cuts.ctypes.data,
                                 C.byref(n))
    return rc, cuts[:n.value + 1].tolist()


def _fits(L, k, ibyte, world, share, symm, budget, t):
    return L.hm_rank_condition_bytes(k, ibyte, world, share, t, t, t if symm else 0, symm) <= budget


@pytest.mark.parametrize("k,symm", [(21, 1), (31, 0), (40, 1), (64, 0)])
def test_sub_ranges_stay_within_the_budget_and_are_greedy(L, k, symm):
    ibyte, world, share = 2, 3, 5_000_000
    rng = np.random.default_rng(k)
    h = rng.integers(0, 3000, size=1 << 14).astype(np.int64)
    base = L.hm_rank_condition_bytes(k, ibyte, world, share, 0, 0, 0, symm)
    for extra in (64 << 20, 256 << 20, 1 << 30):
        budget = base + extra
        rc, cuts = _cut(L, k, ibyte, world, share, symm, budget, h)
        assert rc == 0 and cuts[0] == 0 and cuts[-1] == h.size and len(cuts) >= 2
        for a, b in _starts(cuts):
            t = int(h[a:b].sum())
            assert a < b and t <= MAX_RANGE and _fits(L, k, ibyte, world, share, symm, budget, t)
            if b < h.size:                                    # greedy: the next prefix would not have fitted
                assert not _fits(L, k, ibyte, world, share, symm, budget, t + int(h[b]))
    rc, cuts = _cut(L, k, ibyte, world, share, symm, base + (1 << 30), np.zeros(100, dtype=np.int64))
    assert rc == 0 and cuts == [0, 100]
    rc, cuts = _cut(L, k, ibyte, world, share, symm, base + (1 << 30), np.zeros(0, dtype=np.int64))
    assert rc == 0 and cuts == [0]                        # an empty range: no sub-range


def test_sub_ranges_are_capped_at_the_largest_range(L):
    h = np.full(64, 1 << 28, dtype=np.int64)                  # 2^34 entries; a budget far beyond any GPU
    rc, cuts = _cut(L, 31, 3, 2, 1000, 1, 1 << 50, h)
    assert rc == 0 and len(cuts) - 1 == 8
    assert all(int(h[a:b].sum()) <= MAX_RANGE for a, b in _starts(cuts))


def test_a_prefix_larger_than_the_room_is_refused_with_the_sizes(L):
    k, ibyte, world, share = 31, 3, 2, 1_000_000
    h = np.zeros(1 << 10, dtype=np.int64)
    h[100] = 50_000_000
    budget = L.hm_rank_condition_bytes(k, ibyte, world, share, 0, 0, 0, 1) + (64 << 20)
    rc, _ = _cut(L, k, ibyte, world, share, 1, budget, h)
    msg = L.hm_last_error().decode()
    assert rc == -3 and str(budget) in msg and "50000000" in msg and str(share) in msg, msg
    with pytest.raises(_lib.HetmersError) as e:             # rank_sub_cuts names the rank
        hd.rank_sub_cuts(k, ibyte, [share, share], 1, [1 << 40, budget], np.concatenate([h, h]), [0, 1024, 2048])
    assert e.value.code == -3 and str(e.value).count("rank 1:") == 1 and str(budget) in str(e.value)
    rc, _ = _cut(L, k, ibyte, world, share, 1, 1 << 20, np.zeros(4, dtype=np.int64))   # not even the load fits
    assert rc == -3


def test_bytes_are_monotone_in_every_count(L):
    rng = np.random.default_rng(5)
    for k in (16, 31, 33, 64):
        for symm in (0, 1):
            for _ in range(200):
                args = [int(x) for x in rng.integers(0, 1 << 30, size=4)]
                share, sent, recv = args[:3]
                rc = min(args[3], recv) if symm else 0
                b = L.hm_rank_condition_bytes(k, 2, 3, share, sent, recv, rc, symm)
                assert b > 0
                d = int(rng.integers(1, 1 << 24))
                assert L.hm_rank_condition_bytes(k, 2, 3, share + d, sent, recv, rc, symm) >= b
                assert L.hm_rank_condition_bytes(k, 2, 3, share, sent + d, recv, rc, symm) >= b
                assert L.hm_rank_condition_bytes(k, 2, 3, share, sent, recv + d, rc, symm) >= b
                if symm:
                    assert L.hm_rank_condition_bytes(k, 2, 3, share, sent, recv + d, rc + d, symm) >= b
                assert L.hm_rank_condition_bytes(k, 2, 4, share, sent, recv, rc, symm) >= b
    assert L.hm_rank_condition_bytes(31, 2, 3, 10, 10, 5, 6, 1) == -1          # more reverse complements than entries
    assert L.hm_rank_condition_bytes(31, 4, 3, 10, 10, 5, 5, 1) == -1


def test_pass_counts_match_a_brute_force_restatement():
    rng = np.random.default_rng(9)
    world, np_ = 3, 256
    locs = [rng.integers(0, 20, size=(2, np_)) for _ in range(world)]
    for h in locs:
        h[1] += h[0]                                          # kept originals + reverse complements
    h_all = sum(locs)
    cuts = hd.condition_cuts(h_all[1], world)
    subs = []
    for d in range(world):                                    # 1, 2 and 4 sub-ranges
        a, b = cuts[d], cuts[d + 1]
        n = [1, 2, 4][d]
        subs.append(sorted({a + (b - a) * i // n for i in range(n)} | {b}))
    for rank in range(world):
        plan = hd.rank_pass_counts(locs[rank], h_all, subs, rank)
        assert len(plan) == max(len(s) - 1 for s in subs)
        for p, (sent, recv, rc, orig, rcs) in enumerate(plan):
            owner = np.full(np_, -1)
            for d in range(world):
                if p < len(subs[d]) - 1:
                    owner[subs[d][p]:subs[d][p + 1]] = d
            inwin = owner >= 0
            assert sent == int(locs[rank][1][inwin].sum())
            assert orig == int(h_all[0][inwin].sum()) and rcs == int((h_all[1] - h_all[0])[inwin].sum())
            mine = owner == rank
            assert recv == int(h_all[1][mine].sum()) and rc == int((h_all[1] - h_all[0])[mine].sum())
        assert sum(c[1] for c in plan) == int(h_all[1][cuts[rank]:cuts[rank + 1]].sum())

"""CPU pins of the streamed scan's lists in host memory (DESIGN.md §4c, *Lists in host memory*).

hm_spill_plan is restated in Python: the same slice and partition sizes for the same sizes and room, both sides
within the room, and the floor refused.  The parked rule of pass 2 is restated with the helpers of
test_stream_route_rule.py: every candidate with a Bloom hit is parked, its keys that hit become queries, the sorted
S list is cut into key-range partitions, a query is looked up only in the partition whose range holds it, and a
parked candidate none of whose queries is found is counted.  The plot must be the oracle's, also when the filter
answers yes to every key (every candidate is parked) and when partitions start at queried keys."""
import ctypes as C

import numpy as np
import pytest

from smudgeplot_b200 import _lib
from test_stream_route_rule import Rank, _oracle, host_cuts
from test_symm_identity import _symmetric_table


def slice_bytes(c, kw):
    return c * (8 * kw + 8) + 8 * c + 2 * c * (2 * (8 * kw + 8) + 1) + 2 * c * _lib.SPILL_SORT_Q + _lib.SPILL_SORT_FIXED


def part_bytes(p, kw):
    return p * 8 * kw + 4 * ((1 << _lib.lib().hm_pick_bucket_bits(p)) + 1)


def largest(most, room, kw, f):
    lo, hi = 0, most
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        if f(mid, kw) <= room:
            lo = mid
        else:
            hi = mid - 1
    return lo


def plan(n_cand, n_s, k, room):
    """-> (slice, part), or None where hm_spill_plan refuses"""
    kw = 2 if k > 32 else 1
    nc, np_ = min(max(n_cand, 1), _lib.SPILL_MAX_SLICE), min(max(n_s, 1), _lib.SPILL_MAX_PART)
    if slice_bytes(nc, kw) + part_bytes(np_, kw) <= room:
        sl, pt = nc, np_
    else:
        sl = largest(nc, room // 2, kw, slice_bytes)
        pt = largest(np_, room - slice_bytes(sl, kw), kw, part_bytes)
        sl = largest(nc, room - part_bytes(pt, kw), kw, slice_bytes)
    if sl < min(nc, _lib.SPILL_MIN) or pt < min(np_, _lib.SPILL_MIN):
        return None
    return sl, pt


@pytest.mark.parametrize("k", [21, 31, 40, 64])
@pytest.mark.parametrize("n_cand,n_s", [(0, 0), (10, 30), (5000, 9000), (10**6, 2 * 10**6), (3 * 10**9, 5 * 10**9)])
def test_spill_plan_equals_its_restatement(n_cand, n_s, k):
    kw = 2 if k > 32 else 1
    lay = _lib.SpillLayout()
    for room in [0, 1 << 16, 300_000, 500_000, 1 << 20, 7_777_777, 1 << 26, 1 << 30, 80 << 30]:
        rc = _lib.lib().hm_spill_plan(n_cand, n_s, k, room, C.byref(lay))
        want = plan(n_cand, n_s, k, room)
        if want is None:
            assert rc == -3, (room, lay.slice, lay.part)
            assert "device room" in _lib.lib().hm_last_error().decode()
            continue
        assert rc == 0 and (lay.slice, lay.part) == want, room
        assert lay.queries == 2 * lay.slice and lay.part_bits == _lib.lib().hm_pick_bucket_bits(lay.part)
        assert lay.slice_bytes == slice_bytes(lay.slice, kw) and lay.part_bytes == part_bytes(lay.part, kw)
        assert lay.slice_bytes + lay.part_bytes <= room                  # every round and partition fits
        assert lay.slice <= max(n_cand, 1) and lay.part <= max(n_s, 1)
        assert lay.slice <= _lib.SPILL_MAX_SLICE and lay.part <= _lib.SPILL_MAX_PART


@pytest.mark.parametrize("k", [31, 40])
@pytest.mark.parametrize("n", [2.5e10, 5e10, 1e11])
def test_spill_plan_indexes_fit_32_bits_at_h100_sizes(n, k):
    """an 80 GB H100 at the default budget, tables of 2.5e10..1e11 entries (10 % candidates, 17.5 % S keys):
    partitions stay below what a 32-bit bucket index holds, and a round's queries below 2^31"""
    lay = _lib.SpillLayout()
    n = int(n)
    for room in (int(78e9), 80 << 30, 1 << 40):
        assert _lib.lib().hm_spill_plan(n // 10, n * 175 // 1000, k, room, C.byref(lay)) == 0
        assert (lay.slice, lay.part) == plan(n // 10, n * 175 // 1000, k, room)
        assert lay.part <= _lib.SPILL_MAX_PART < 0xFFFFFFFF and lay.part_bits <= 30
        assert lay.queries <= 2 * _lib.SPILL_MAX_SLICE < 1 << 31
        assert lay.slice_bytes + lay.part_bytes <= room


def test_spill_plan_floor():
    """the smallest room the plan takes holds slices and partitions of HM_SPILL_MIN; one byte less is refused"""
    lay = _lib.SpillLayout()
    lo, hi = 1, 1 << 30
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.lib().hm_spill_plan(10**6, 10**6, 31, mid, C.byref(lay)) == 0:
            hi = mid
        else:
            lo = mid + 1
    assert _lib.lib().hm_spill_plan(10**6, 10**6, 31, lo, C.byref(lay)) == 0
    assert lay.slice >= _lib.SPILL_MIN and lay.part >= _lib.SPILL_MIN
    assert _lib.lib().hm_spill_plan(10**6, 10**6, 31, lo - 1, C.byref(lay)) == -3
    assert _lib.lib().hm_spill_plan(-1, 0, 31, 1 << 30, C.byref(lay)) == -1


# ------------------------------------------------------------------ the parked rule ------------------------------

def parked_plot(keys, cnt, k, seg_bits, slice_, cuts, all_hit=False):
    """one GPU's parked pass 2 over host lists: -> (plot, rounds, queries equal to a partition's first key,
    queries found)"""
    rk = Rank(keys, cnt, k, [0, len(keys)], 0, seg_bits)
    seg = np.ones_like(rk.seg) if all_hit else rk.seg
    S = np.array(sorted(rk.S), dtype=object)
    parts = [set(S[a:b].tolist()) for a, b in zip(cuts[:-1], cuts[1:])]
    first = [int(S[a]) for a in cuts[:-1] if a < len(S)]
    rounds, edge, nfound = 0, 0, 0
    for c0 in range(0, len(rk.cand), slice_):
        rounds += 1
        pend, queries = [], []
        for x, cx, cy, p, yb in rk.cand[c0:c0 + slice_]:
            rx = _rc(x, k)
            sh = 62 - 2 * (k - 1 - p)
            ry = (rx & ~(3 << sh)) | ((3 - yb) << sh)
            hit = [q for q in (rx, ry) if seg[q % len(seg)]]
            if not hit:
                rk.count(cx, cy, p)
                continue
            queries += [(q, len(pend)) for q in hit]
            pend.append((cx, cy, p))
        found = set()
        for q, slot in sorted(queries):
            i = max(0, int(np.searchsorted(np.array(first, dtype=object), q, side="right")) - 1) if first else 0
            edge += bool(first) and q == first[i]
            if parts and q in parts[i]:
                found.add(slot)
                nfound += 1
        rk.settle(pend, found)
    return rk.plot, rounds, edge, nfound


def _rc(x, k):
    import oracle_util as ou
    return ou._rc(x, k)


CASES = [(21, 1500, 40, 1), (31, 1500, 40, 2), (12, 1200, 40, 3), (32, 1000, 700, 4), (17, 1500, 520, 8)]   # one-word keys


@pytest.mark.parametrize("k,n0,cmax,seed", CASES)
def test_parked_rule_equals_the_oracle(k, n0, cmax, seed):
    keys, cnt = _symmetric_table(k, n0, cmax, seed)
    want = _oracle(keys, cnt, k)
    ns = len(Rank(keys, cnt, k, [0, len(keys)], 0, 1 << 20).S)
    rng = np.random.default_rng(seed)
    for part in (1, 7, max(ns // 3, 1), max(ns, 1)):               # one key per partition ... one partition
        cuts = list(range(0, ns, part)) + [ns]
        for seg_bits, all_hit in ((1 << 20, False), (61, False), (61, True)):
            got, rounds, edge, nfound = parked_plot(keys, cnt, k, seg_bits, 64, cuts, all_hit)
            assert np.array_equal(got, want), (part, seg_bits, all_hit)
            assert rounds >= 2
            if part == 1:
                assert edge == nfound                                # every query found in S is a first key
    cuts = sorted({0, ns, *rng.integers(0, ns + 1, size=5).tolist()})   # uneven partitions
    assert np.array_equal(parked_plot(keys, cnt, k, 61, 50, cuts)[0], want)


def test_parked_rule_with_runs_longer_than_a_chunk():
    from test_gpu_symm import _symmetric_closure
    k = 3
    rng = np.random.default_rng(5150)
    vals = np.arange(4 ** k, dtype=np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    assert host_cuts(keys, k, 5)[4] == len(keys)
    want = _oracle(keys, cnt, k)
    ns = len(Rank(keys, cnt, k, [0, len(keys)], 0, 1 << 12).S)
    for part in (1, 5, max(ns, 1)):
        cuts = list(range(0, ns, part)) + [ns]
        for all_hit in (False, True):
            assert np.array_equal(parked_plot(keys, cnt, k, 1 << 12, 8, cuts, all_hit)[0], want), (part, all_hit)

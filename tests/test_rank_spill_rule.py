"""CPU pin of the parked routed pass 2 of ranks whose lists are in host memory (hm_rank_scan_* with a list host
budget, DESIGN.md §4c, *Lists in host memory*, *ranks*), against the oracle, next to test_stream_route_rule.py.
Each rank holds what pass 1 and the Bloom all-gather leave (test_stream_route_rule.Rank), but its S list is not
resident: in rounds over slices, a Bloom miss is counted (or listed) at once and every candidate with a hit is
parked, each hit key a query to its owner -- this rank included.  Each owner sorts the keys it receives, answers
them against its S list cut into partitions of a few keys (a key is answered by the partition whose key range
holds it, only partitions some key falls in are looked at), and returns the answers in receive order; the
parked candidates none of whose keys was found are counted (or listed).

The plot must be the oracle's, and the merged list the oracle's extract_kmer_pairs lines, for world 1, 2 and 3,
several slice sizes and partition sizes; queries on a partition's first key must occur."""
import bisect

import numpy as np
import pytest

import oracle_util as ou
from test_route_extract_rule import ListingRank, _lines, _oracle_lines
from test_stream_route_rule import _oracle, host_cuts
from test_symm_extract_rule import _symmetric_table_any_k
from test_symm_identity import _symmetric_table


class ParkedRank(ListingRank):
    """a rank whose candidates and S list are in host memory; S is cut into partitions of `part` keys"""

    def __init__(self, keys, cnt, k, cuts, r, seg_bits, pix, part, listing):
        super().__init__(keys, cnt, k, cuts, r, seg_bits, pix)
        s = sorted(self.S)
        self.parts = [s[i:i + part] for i in range(0, len(s), part)]
        self.firsts = [p[0] for p in self.parts]
        self.listing = listing
        self.first_key_queries = 0
        self.uploaded = 0

    def settle_one(self, c):
        if self.listing:
            self.list_pair(c)
        else:
            _, cx, cy, p, _ = c
            self.count(cx, cy, p)

    def park_round(self, c0, c1, segs):
        """one slice: -> (parked candidates, queries[owner] = [(key, slot)]), the owner possibly this rank"""
        pend, queries = [], {}
        for c in self.cand[c0:c1]:
            x, cx, cy, p, yb = c
            rx = ou._rc(x, self.k)
            sh = 62 - 2 * (self.k - 1 - p)
            ry = (rx & ~(3 << sh)) | ((3 - yb) << sh)
            hit = [(q, self.owner(q)) for q in (rx, ry) if segs[self.owner(q)][q % len(segs[0])]]
            if not hit:                                       # Bloom miss: settled at once
                self.settle_one(c)
                continue
            for q, o in hit:                                  # every hit parked, no look-up here
                queries.setdefault(o, []).append((q, len(pend)))
            pend.append(c)
        return pend, queries

    def answer_parked(self, keys_in):
        """the keys received, sorted, answered partition by partition, the answers back in receive order"""
        order = sorted(range(len(keys_in)), key=lambda i: keys_in[i])      # stable, as the radix sort
        srt = [keys_in[i] for i in order]
        ans_sorted = [0] * len(srt)
        lo = 0
        for p, part in enumerate(self.parts):
            if lo >= len(srt):
                break
            hi = bisect.bisect_left(srt, self.firsts[p + 1], lo) if p + 1 < len(self.parts) else len(srt)
            if hi == lo:
                continue                                      # no key here: the partition is not uploaded
            self.uploaded += 1
            self.first_key_queries += srt[lo] == part[0]
            members = set(part)
            for i in range(lo, hi):
                ans_sorted[i] = int(srt[i] in members)
            lo = hi
        ans = [0] * len(keys_in)
        for i, a in zip(order, ans_sorted):                   # scattered back to receive order
            ans[i] = a
        return ans

    def settle_parked(self, pend, found):
        for i, c in enumerate(pend):
            if i not in found:
                self.settle_one(c)


def parked(keys, cnt, k, world, seg_bits, slice_, part, listing, pix=None):
    """-> (summed plot or merged sorted records, rounds, queries[(from, to)], first-key queries)"""
    cuts = host_cuts(keys, k, world)
    if pix is None:
        pix = np.zeros((ou.SMAX + 1, ou.PLOT_W), dtype=np.uint16)
    ranks = [ParkedRank(keys, cnt, k, cuts, r, seg_bits, pix, part, listing) for r in range(world)]
    segs = [rk.seg for rk in ranks]
    rounds = max((len(rk.cand) + slice_ - 1) // slice_ for rk in ranks)
    sent = {}
    for rd in range(rounds):
        work = [rk.park_round(min(rd * slice_, len(rk.cand)), min((rd + 1) * slice_, len(rk.cand)), segs)
                for rk in ranks]
        # every rank receives the keys of every sender (itself included), in sender order, as all_to_all_single
        recv = [[(src, slot, q) for src, (_, queries) in enumerate(work) for q, slot in queries.get(dst, [])]
                for dst in range(world)]
        found = [set() for _ in ranks]
        for dst, got in enumerate(recv):
            for (src, slot, _), a in zip(got, ranks[dst].answer_parked([q for _, _, q in got])):
                sent[(src, dst)] = sent.get((src, dst), 0) + 1
                if a:
                    found[src].add(slot)
        for rk, (pend, _), f in zip(ranks, work, found):
            rk.settle_parked(pend, f)
    fkq = sum(rk.first_key_queries for rk in ranks)
    if listing:
        return sorted((lab, key, pos, alt) for rk in ranks for key, lab, pos, alt in rk.recs), rounds, sent, fkq
    return sum(rk.plot for rk in ranks), rounds, sent, fkq


CASES = [(21, 1500, 40, 1), (31, 1500, 40, 2), (12, 1200, 40, 3), (32, 1000, 700, 4)]


@pytest.mark.parametrize("k,n0,cmax,seed", CASES)
@pytest.mark.parametrize("world", [1, 2, 3])
def test_parked_plot_equals_the_oracle(k, n0, cmax, seed, world):
    keys, cnt = _symmetric_table(k, n0, cmax, seed)
    want = _oracle(keys, cnt, k)
    for seg_bits in (1 << 20, 61):                            # a roomy filter and one full of false hits
        for slice_, part in ((7, 1), (7, 3), (64, 5), (100000, 1 << 20)):
            got, rounds, sent, _ = parked(keys, cnt, k, world, seg_bits, slice_, part, False)
            assert np.array_equal(got, want), (seg_bits, slice_, part)
            if slice_ == 7:
                assert rounds >= 3
            if seg_bits == 61:                                # every rank asks every rank, itself included
                assert all(sent.get((a, b), 0) > 0 for a in range(world) for b in range(world)), sent


@pytest.mark.parametrize("k", [8, 10])
def test_parked_plot_with_keys_found_at_partition_starts(k):
    """a twentieth of every k-mer and its closure (palindromes among them): many Bloom hits are in S, and with
    partitions of 1 to 3 keys queried keys fall on partition first keys"""
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(177 + k)
    vals = rng.choice(4 ** k, size=min(4 ** k // 20, 3000), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    want = _oracle(keys, cnt, k)
    for world in (1, 2, 3):
        for slice_, part in ((5, 1), (16, 2), (40, 3)):
            got, rounds, sent, fkq = parked(keys, cnt, k, world, 61, slice_, part, False)
            assert np.array_equal(got, want), (world, slice_, part)
            assert rounds >= 3 and fkq > 0, (rounds, fkq)
            assert all(sent.get((a, b), 0) > 0 for a in range(world) for b in range(world)), sent


@pytest.mark.parametrize("k,n0,counts,seed", [(11, 1500, "smax", 24), (21, 1500, "wide", 26), (31, 1500, "smax", 27),
                                              (32, 1000, "ties", 28)])
def test_parked_listing_equals_the_oracle_extract(k, n0, counts, seed, tmp_path):
    keys, cnt = _symmetric_table_any_k(k, n0, counts, seed)
    _check_listing(np.array(keys, dtype=np.uint64), cnt, k, tmp_path)


@pytest.mark.parametrize("k", [8, 10])
def test_parked_listing_with_keys_found_at_partition_starts(k, tmp_path):
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(177 + k)
    vals = rng.choice(4 ** k, size=min(4 ** k // 20, 3000), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    assert _check_listing(keys, cnt, k, tmp_path) > 0


def _check_listing(keys, cnt, k, tmp_path):
    """the merged lists equal the oracle's lines for world 1, 2, 3, both filters, two slice / partition sizes
    -> the queries on partition first keys, over all runs"""
    pix, order, want = _oracle_lines(keys, cnt, k, tmp_path)
    assert sum(len(v) for v in want.values()) > 0
    fkq = 0
    for world in (1, 2, 3):
        for seg_bits in (1 << 20, 61):
            for slice_, part in ((7, 1), (64, 5)):
                got, rounds, sent, f = parked(keys, cnt, k, world, seg_bits, slice_, part, True, pix)
                assert _lines(got, k, order) == want, ou.first_pair_difference(_lines(got, k, order), want)
                assert rounds >= 2
                fkq += f
                if seg_bits == 61:
                    assert all(sent.get((a, b), 0) > 0 for a in range(world) for b in range(world)), sent
    return fkq

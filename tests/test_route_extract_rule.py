"""CPU pin of the routed pair listing of a rank that streams its own share (hm_rank_scan_extract_*, DESIGN.md §4c,
*Ranks*), against the oracle's extract_kmer_pairs.  Each rank holds what pass 1 and the Bloom all-gather leave
(test_stream_route_rule.Rank) and lists its candidates in rounds over slices: a Bloom miss is listed at once, a
hit on a key the rank owns is checked in its own S list, and a candidate left with a hit on a key owned elsewhere
is parked with its key while that key goes to its owner as a query; after the answers come back, the parked
candidates none of whose keys was found are listed.  Listing is test_symm_extract_rule.partial_extract's rule.

The ranks' lists, merged and sorted, must be exactly the oracle's lines for a .sma that labels every pixel, for
world 1, 2 and 3."""
import numpy as np
import pytest

import oracle_util as ou
from smudgeplot_b200 import fastk
from test_stream_route_rule import Rank, host_cuts
from test_symm_extract_rule import _label_every_pixel, _symmetric_table_any_k, pair_line


class ListingRank(Rank):
    """Rank with the listing in place of the count: records (key, label, pos, alt) as partial_extract gives them"""

    def __init__(self, keys, cnt, k, cuts, r, seg_bits, pix):
        super().__init__(keys, cnt, k, cuts, r, seg_bits)
        self.pix, self.recs = pix, []

    def list_round(self, c0, c1, segs):
        """one round over candidates [c0, c1): -> (parked candidates, queries[owner] = [(key, slot)])"""
        pend, queries = [], {}
        for c in self.cand[c0:c1]:
            x, cx, cy, p, yb = c
            rx = ou._rc(x, self.k)
            sh = 62 - 2 * (self.k - 1 - p)
            ry = (rx & ~(3 << sh)) | ((3 - yb) << sh)
            hit = [(q, self.owner(q)) for q in (rx, ry) if segs[self.owner(q)][q % len(segs[0])]]
            if not hit:                                                   # Bloom miss: listed at once
                self.list_pair(c)
                continue
            if any(o == self.r and q in self.S for q, o in hit):         # settled in the rank's own S list
                continue
            foreign = [(q, o) for q, o in hit if o != self.r]
            if not foreign:
                self.list_pair(c)
                continue
            for q, o in foreign:                                          # parked with its key
                queries.setdefault(o, []).append((q, len(pend)))
            pend.append(c)
        return pend, queries

    def settle_list(self, pend, found):
        for i, c in enumerate(pend):
            if i not in found:
                self.list_pair(c)

    def list_pair(self, c):
        x, cx, cy, p, by = c
        k = self.k
        lab = int(self.pix[cx + cy][min(cx, cy)])
        if lab == 0:
            return
        sh = 62 - 2 * p
        bx = (x >> sh) & 3
        y = (x & ~(3 << sh)) | (by << sh)
        self.recs.append((y, lab, p, bx) if cx < cy else (x, lab, p, by))
        if 2 * p != k - 1:
            q = k - 1 - p
            sq = 62 - 2 * q
            rx = ou._rc(x, k)
            ry = (rx & ~(3 << sq)) | ((3 - by) << sq)
            self.recs.append((rx, lab, q, 3 - by) if cy < cx else (ry, lab, q, 3 - bx))


def routed_list(keys, cnt, k, world, seg_bits, slice_, pix):
    """-> (merged records sorted as hm_sort_pair_records sorts them, rounds, queries[(from, to)])"""
    cuts = host_cuts(keys, k, world)
    ranks = [ListingRank(keys, cnt, k, cuts, r, seg_bits, pix) for r in range(world)]
    segs = [rk.seg for rk in ranks]
    rounds = max((len(rk.cand) + slice_ - 1) // slice_ for rk in ranks)
    sent = {}
    for rd in range(rounds):
        work = [rk.list_round(min(rd * slice_, len(rk.cand)), min((rd + 1) * slice_, len(rk.cand)), segs)
                for rk in ranks]
        found = [set() for _ in ranks]
        for src, (_, queries) in enumerate(work):
            for dst, qs in queries.items():
                sent[(src, dst)] = sent.get((src, dst), 0) + len(qs)
                for (_, slot), a in zip(qs, ranks[dst].answer([q for q, _ in qs])):
                    if a:
                        found[src].add(slot)
        for rk, (pend, _), f in zip(ranks, work, found):
            rk.settle_list(pend, f)
    merged = sorted((lab, key, pos, alt) for rk in ranks for key, lab, pos, alt in rk.recs)
    return merged, rounds, sent


def _oracle_lines(keys, cnt, k, tmp_path):
    kb = (k + 3) // 4
    kbytes = np.array([list(int(x).to_bytes(8, "big")[:kb]) for x in keys], dtype=np.uint8)
    name = str(tmp_path / "t")
    fastk.write_ktab(name, k, kbytes, cnt, ibyte=1, nparts=2)
    pix, order = _label_every_pixel(str(tmp_path / "all.sma"))
    assert ou.oracle_extract(name, 1, str(tmp_path / "all.sma"), str(tmp_path / "ora")) == 0
    want = {lab: v for lab, v in ou.sorted_pair_files(str(tmp_path / "ora")).items() if v}
    return pix, order, want


def _lines(recs, k, order):
    got = {}
    for lab, key, pos, alt in recs:
        got.setdefault(order[lab - 1], []).append(pair_line(key, k, pos, alt))
    return {lab: sorted(v) for lab, v in got.items()}


def _check_worlds(keys, cnt, k, tmp_path, slice_=64, ask_all=True):
    pix, order, want = _oracle_lines(keys, cnt, k, tmp_path)
    assert sum(len(v) for v in want.values()) > 0
    for world in (1, 2, 3):
        for seg_bits in (1 << 20, 61):                   # a roomy filter and one full of false hits
            got, rounds, sent = routed_list(keys, cnt, k, world, seg_bits, slice_, pix)
            assert _lines(got, k, order) == want, ou.first_pair_difference(_lines(got, k, order), want)
            assert rounds >= 2
            if ask_all and world > 1 and seg_bits == 61:   # every rank asks every other
                assert all(sent.get((a, b), 0) > 0 for a in range(world) for b in range(world) if a != b), sent
    return got


@pytest.mark.parametrize("k,n0,counts,seed", [(11, 1500, "smax", 24), (16, 1200, "ties", 25), (21, 1500, "wide", 26),
                                              (31, 1500, "smax", 27), (32, 1000, "ties", 28)])
def test_routed_listing_equals_the_oracle_extract(k, n0, counts, seed, tmp_path):
    """odd and even k, count ties and counts whose pair sums straddle SMAX"""
    keys, cnt = _symmetric_table_any_k(k, n0, counts, seed)
    got = _check_worlds(np.array(keys, dtype=np.uint64), cnt, k, tmp_path)
    if k % 2 == 1:                                       # middle-base pairs are listed once
        assert any(pos == k // 2 for _, _, pos, _ in got)


@pytest.mark.parametrize("k", [8, 10])
def test_routed_listing_even_k_with_palindromes(k, tmp_path):
    """a twentieth of every k-mer and its closure: k-mers equal to their own reverse complement among them"""
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(177 + k)
    vals = rng.choice(4 ** k, size=min(4 ** k // 20, 3000), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    assert sum(ou._rc(int(x), k) == int(x) for x in keys) > 0
    _check_worlds(keys, cnt, k, tmp_path, 32)


def test_routed_listing_with_runs_longer_than_a_share(tmp_path):
    """k = 12, half the entries in one run (one 6-base prefix, 300 suffixes) and the other half their reverse
    complements: the run is longer than a share of 2 or 3 ranks, and every candidate is in it"""
    from test_gpu_symm import _symmetric_closure
    k = 12
    rng = np.random.default_rng(5151)
    suffix = rng.choice(4 ** 6, size=300, replace=False).astype(np.uint64)
    keys, cnt = _symmetric_closure(((np.uint64(0x16c) << np.uint64(12)) | suffix) << np.uint64(64 - 2 * k), k, rng, 300)
    pfx = (keys >> np.uint64(64 - k)).tolist()
    assert max(pfx.count(v) for v in set(pfx)) > len(keys) / 3
    _check_worlds(keys, cnt, k, tmp_path, 4, ask_all=False)

"""CPU pin of the routed pass 2 of a rank that streams its own share (hm_rank_scan_*, DESIGN.md §4c, *Ranks*),
against the oracle.  Rank r scans [c_r, c_r+1) (the in-process shards' cuts), keeps its candidates, the S keys of
its share and Bloom segment r; after the segments are all-gathered it settles its candidates in rounds over
slices: a Bloom miss counts at once, a hit on a key it owns is looked up in its own S list, and a candidate left
with a hit on a key owned elsewhere is parked while that key goes to its owner as a query; the owner answers one
byte per key and the parked candidates none of whose keys was found are counted with count_pair's weight.

`routed_plot` restates that rule with the ranks' exchanges done in one process; the plot must be the oracle's for
world 1, 2 and 3.  The cuts computed from the table files alone must equal dist.run_aligned_cuts."""
import numpy as np
import pytest
import torch

import oracle_util as ou
from smudgeplot_b200 import dist as hd
from smudgeplot_b200 import fastk
from test_symm_identity import _symmetric_table


def host_cuts(keys, k, world):
    n = len(keys)
    pfx = keys >> np.uint64(64 - 2 * (k // 2))
    starts = np.concatenate([[0], np.nonzero(pfx[1:] != pfx[:-1])[0] + 1, [n]])
    return [0] + [int(starts[np.searchsorted(starts, n * r // world)]) for r in range(1, world)] + [n]


def s_list(keys, cnt, k, lo, hi):
    """the S keys of [lo, hi): entries with a partner at a position >= k - k/2 (count sum <= SMAX)"""
    pos_of = {int(x): i for i, x in enumerate(keys.tolist())}
    pup, out = k - k // 2, set()
    for i in range(lo, hi):
        x = int(keys[i])
        for p in range(pup, k):
            sh = 62 - 2 * p
            b = (x >> sh) & 3
            if any(alt != b and (j := pos_of.get((x & ~(3 << sh)) | (alt << sh))) is not None and
                   int(cnt[i]) + int(cnt[j]) <= ou.SMAX for alt in range(4)):
                out.add(x)
                break
    return out


class Rank:
    """what one rank holds after pass 1 and the Bloom all-gather"""

    def __init__(self, keys, cnt, k, cuts, r, seg_bits):
        n = len(keys)
        self.k, self.r = k, r
        self.seg, self.cand = ou.partial_runscan(keys, cnt, k, cuts[r], cuts[r + 1], seg_bits)
        self.S = s_list(keys, cnt, k, cuts[r], cuts[r + 1])
        live = max([q + 1 for q in range(len(cuts) - 1) if cuts[q] < n] + [1])
        self.first = [int(keys[cuts[q]]) if cuts[q] < n else (1 << 64) - 1 for q in range(live)]
        self.plot = np.zeros((ou.SMAX + 1, ou.PLOT_W), dtype=np.int64)

    def owner(self, q):
        return sum(1 for f in self.first[1:] if q >= f)

    def resolve(self, c0, c1, segs):
        """one round over candidates [c0, c1): -> (pending metas, queries[owner] = [(key, slot)])"""
        k = self.k
        pend, queries = [], {}
        for x, cx, cy, p, yb in self.cand[c0:c1]:
            rx = ou._rc(x, k)
            sh = 62 - 2 * (k - 1 - p)
            ry = (rx & ~(3 << sh)) | ((3 - yb) << sh)
            hit = [(q, self.owner(q)) for q in (rx, ry) if segs[self.owner(q)][q % len(segs[0])]]
            if not hit:
                self.count(cx, cy, p)
                continue
            if any(o == self.r and q in self.S for q, o in hit):
                continue
            foreign = [(q, o) for q, o in hit if o != self.r]
            if not foreign:
                self.count(cx, cy, p)
                continue
            for q, o in foreign:
                queries.setdefault(o, []).append((q, len(pend)))
            pend.append((cx, cy, p))
        return pend, queries

    def answer(self, keys_in):
        return [int(q in self.S) for q in keys_in]

    def settle(self, pend, found):
        for i, (cx, cy, p) in enumerate(pend):
            if i not in found:
                self.count(cx, cy, p)

    def count(self, cx, cy, p):
        self.plot[cx + cy, min(cx, cy)] += 1 if 2 * p == self.k - 1 else 2


def routed_plot(keys, cnt, k, world, seg_bits, slice_):
    """-> (summed plot, rounds, queries[(from, to)])"""
    cuts = host_cuts(keys, k, world)
    ranks = [Rank(keys, cnt, k, cuts, r, seg_bits) for r in range(world)]
    segs = [rk.seg for rk in ranks]
    rounds = max((len(rk.cand) + slice_ - 1) // slice_ for rk in ranks)
    sent = {}
    for rd in range(rounds):
        work = [rk.resolve(min(rd * slice_, len(rk.cand)), min((rd + 1) * slice_, len(rk.cand)), segs) for rk in ranks]
        found = [set() for _ in ranks]
        for src, (_, queries) in enumerate(work):
            for dst, qs in queries.items():
                sent[(src, dst)] = sent.get((src, dst), 0) + len(qs)
                for (_, slot), a in zip(qs, ranks[dst].answer([q for q, _ in qs])):
                    if a:
                        found[src].add(slot)
        for rk, (pend, _), f in zip(ranks, work, found):
            rk.settle(pend, f)
    return sum(rk.plot for rk in ranks), rounds, sent


def _oracle(keys, cnt, k):
    plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    return plot


CASES = [(21, 1500, 40, 1), (31, 1500, 40, 2), (12, 1200, 40, 3), (32, 1000, 700, 4), (17, 1500, 520, 8)]


@pytest.mark.parametrize("k,n0,cmax,seed", CASES)
@pytest.mark.parametrize("world", [1, 2, 3])
def test_routed_pass2_equals_the_oracle(k, n0, cmax, seed, world):
    keys, cnt = _symmetric_table(k, n0, cmax, seed)
    want = _oracle(keys, cnt, k)
    for seg_bits in (1 << 20, 61):                         # a roomy filter and one full of false hits
        got, rounds, sent = routed_plot(keys, cnt, k, world, seg_bits, 64)
        assert np.array_equal(got, want), (seg_bits, world)
        assert rounds >= 2
        if world > 1 and seg_bits == 61:                   # false hits everywhere: every rank asks every other
            assert all(sent.get((a, b), 0) > 0 for a in range(world) for b in range(world) if a != b), sent


@pytest.mark.parametrize("world", [1, 2, 3])
def test_routed_pass2_with_runs_longer_than_a_share(world):
    """k = 3, every k-mer: 4 runs of 16 entries; with three ranks a share is shorter than a run, so shards are empty"""
    from test_gpu_symm import _symmetric_closure
    k = 3
    rng = np.random.default_rng(5150)
    vals = np.arange(4 ** k, dtype=np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    cuts = host_cuts(keys, k, 5)
    assert cuts[4] == cuts[5]
    want = _oracle(keys, cnt, k)
    for w in (world, 5):
        for seg_bits in (1 << 12, 61):
            got, _, _ = routed_plot(keys, cnt, k, w, seg_bits, 8)
            assert np.array_equal(got, want), (w, seg_bits)


@pytest.mark.parametrize("k", [8, 10])
def test_routed_pass2_even_k_with_palindromes(k):
    from test_gpu_symm import _symmetric_closure
    rng = np.random.default_rng(177 + k)
    vals = rng.choice(4 ** k, size=min(4 ** k // 20, 3000), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    want = _oracle(keys, cnt, k)
    for world in (1, 2, 3):
        got, _, _ = routed_plot(keys, cnt, k, world, 61, 32)
        assert np.array_equal(got, want), world


@pytest.mark.parametrize("k,ibyte,nparts", [(21, 3, 2), (31, 2, 3), (12, 1, 1), (3, 1, 1)])
def test_cuts_from_the_files_equal_run_aligned_cuts(k, ibyte, nparts, tmp_path):
    if k == 3:
        from test_gpu_symm import _symmetric_closure
        keys, cnt = _symmetric_closure(np.arange(64, dtype=np.uint64) << np.uint64(58), 3,
                                       np.random.default_rng(1), 300)
    else:
        keys, cnt = _symmetric_table(k, 1500, 40, k)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=ibyte, nparts=nparts)
    replica = torch.from_numpy(keys.view(np.int64).copy())
    for world in (1, 2, 3, 5, 16):
        want = hd.run_aligned_cuts(replica, k, world)
        assert hd.file_run_aligned_cuts(fastk.read_ktab(str(tmp_path / "t")), world, window=7) == want
        assert hd.file_run_aligned_cuts(kt, world) == want == host_cuts(keys, k, world)

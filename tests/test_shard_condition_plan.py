"""CPU tests of the host logic of conditioning across the ranks of a one-process-per-GPU job
(dist.ShardedScan.from_ktab(L=...), DESIGN.md §4e): the cut of the key prefixes into one range per rank, the window
whose counts decide "trimmed?", and the job-wide examine verdicts reduced over 2-3 gloo ranks on CPU tensors,
against single-process restatements of hm_scan_examine's rules."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from smudgeplot_b200 import dist as hd  # noqa: E402


# ---------------------------------------------------------------- the range cut ---------------------------------

def _cuts_numpy(h, world):
    """restatement: cut r is the prefix boundary whose count of entries below it is nearest to total*r//world, the
    lower boundary on a tie (the last boundary not above the target, else the first one above it)"""
    before = np.concatenate([[0], np.cumsum(h)])
    total = int(before[-1])
    cuts = [0]
    for r in range(1, world):
        want = total * r // world
        below = [p for p in range(len(before)) if before[p] <= want]
        above = [p for p in range(len(before)) if before[p] > want]
        p = below[-1]
        if above and before[above[0]] - want < want - before[p]:
            p = above[0]
        cuts.append(max(p, cuts[-1]))
    return cuts + [len(h)]


def _check_cuts(h, world):
    cuts = hd.condition_cuts(h, world)
    assert cuts == _cuts_numpy(h, world), (cuts, world)
    assert len(cuts) == world + 1 and cuts[0] == 0 and cuts[-1] == len(h)          # covering
    assert all(a <= b for a, b in zip(cuts, cuts[1:]))                              # contiguous, monotone
    before = np.concatenate([[0], np.cumsum(h)])
    total, big = int(before[-1]), int(max(h)) if len(h) else 0
    for r in range(1, world):                                                       # near-equal: off by at most
        assert abs(int(before[cuts[r]]) - total * r // world) * 2 <= big            #   half of one prefix
    sizes = [int(before[b] - before[a]) for a, b in zip(cuts, cuts[1:])]
    assert sum(sizes) == total
    return cuts, sizes


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8, 16])
def test_range_cut_matches_restatement(world):
    rng = np.random.default_rng(world)
    for np_ in (4, 64, 1 << 10):
        for _ in range(5):
            h = rng.integers(0, 50, size=np_) * (rng.random(np_) < 0.7)
            _, sizes = _check_cuts(h, world)
            if world > 1:                               # each end off by half a prefix at most
                assert max(sizes) - min(sizes) <= 2 * h.max() + 2, sizes


def test_range_cut_one_dominant_prefix_and_empty_ranges():
    h = np.zeros(1 << 12, dtype=np.int64)
    h[777] = 10_000                                         # one prefix holds the table
    h[5] = h[3000] = 1
    for world in (2, 3, 5):
        cuts, sizes = _check_cuts(h, world)
        assert max(sizes) >= 10_000 and sizes.count(0) >= world - 3
        owner = next(d for d in range(world) if cuts[d] <= 777 < cuts[d + 1])
        assert sizes[owner] >= 10_000
    cuts, sizes = _check_cuts(np.zeros(256, dtype=np.int64), 4)                     # empty table
    assert sizes == [0, 0, 0, 0]
    cuts, sizes = _check_cuts(np.array([3, 0, 0, 0]), 8)                            # more ranks than entries
    assert sum(sizes) == 3 and sizes.count(0) == 7
    assert hd.condition_cuts(np.full(1 << 20, 3, dtype=np.int64), 4) == [0, 1 << 18, 1 << 19, 3 << 18, 1 << 20]


# ---------------------------------------------------------------- the examine window ----------------------------

def test_examine_window_below_at_and_above_1e8():
    assert hd.examine_window(0) == (0, 0)
    assert hd.examine_window(99_999_996) == (0, 99_999_996)                   # n + 3 < 1e8: every entry
    for n in (99_999_997, 99_999_999, 100_000_000, 100_000_001, 250_000_001, 6_000_000_000):
        f, l_ = hd.examine_window(n)                                          # the 1e8 around the middle,
        assert (f, l_) == (max(n // 2 - 50_000_000, 0), min(n // 2 + 50_000_000, n))   # inside the table
        assert (n < 100_000_000) == (l_ - f < 100_000_000)
    for n in (99_999_996, 100_000_001, 250_000_001):                          # the ranks' parts tile the window
        f, l_ = hd.examine_window(n)
        for world in (1, 2, 3, 7):
            parts = [(max(a, f), min(b, l_)) for a, b in (hd.share_range(n, world, r) for r in range(world))]
            parts = [p for p in parts if p[0] < p[1]]
            assert parts[0][0] == f and parts[-1][1] == l_ and all(a[1] == b[0] for a, b in zip(parts, parts[1:]))


# ---------------------------------------------------------------- the verdicts over gloo ranks ------------------

def _rc_str(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def _pack(s, k):
    v = 0
    for ch in s:
        v = (v << 2) | "ACGT".index(ch)
    v <<= (128 if k > 32 else 64) - 2 * k
    return (v >> 64, v & ((1 << 64) - 1)) if k > 32 else (v, 0)


def _unpack(words, k):
    bits = 128 if k > 32 else 64
    v = (words[0] << 64 | words[1]) if k > 32 else words[0]
    return "".join("ACGT"[(v >> (bits - 2 * (j + 1))) & 3] for j in range(k))


def _table(kmers, counts, k):
    """(sorted unique k-mer strings, counts) -> (words uint64[n, 2], counts uint16[n])"""
    order = sorted(range(len(kmers)), key=lambda i: kmers[i])
    w = np.array([_pack(kmers[i], k) for i in order], dtype=np.uint64).reshape(-1, 2)
    return w, np.array([counts[i] for i in order], dtype=np.uint16)


def _examine_numpy(words, cnt, k, L):
    """restatement of hm_scan_examine on the whole table"""
    n = len(cnt)
    f, l_ = hd.examine_window(n)
    v = cnt[f:l_].view(np.int16).astype(np.int64)
    v = v[v >= 1]
    trim = (int(v.min()) if v.size else 0x8000) >= L
    keys = [tuple(int(x) for x in row) for row in words]
    where = {key: i for i, key in enumerate(keys)}
    for sidx in range(1, n):
        pos = where.get(_pack(_rc_str(_unpack(keys[sidx], k)), k), -1)
        if pos < 0:
            return trim, False
        if pos != sidx:
            return trim, True
    return trim, True


def _verdict_worker(rank, world, port, cases, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        out = []
        for words, cnt, k, L in cases:
            n = len(cnt)
            lo, hi = hd.share_range(n, world, rank)
            keys = torch.from_numpy(words[lo:hi, 0].copy().view(np.int64))
            klo = torch.from_numpy(words[lo:hi, 1].copy().view(np.int64)) if k > 32 else None
            share = cnt[lo:hi].view(np.int16)

            def min_count(a, b):                        # min_count_kernel's rule on this rank's counts
                v = share[a:b].astype(np.int64)
                v = v[v >= 1]
                return int(v.min()) if v.size else 0x8000
            out.append(hd.job_examine(L, k, n, keys, klo, min_count))
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _verdict_cases():
    rng = np.random.default_rng(7)
    cases = []

    def rand_kmers(k, m):
        return ["".join(rng.choice(list("ACGT"), size=k)) for _ in range(m)]
    for k in (8, 12, 21, 32, 33, 40, 64):
        base = sorted(set(rand_kmers(k, 300)))
        canon = sorted({min(s, _rc_str(s)) for s in base})
        cnt = rng.integers(1, 40, size=len(canon)).tolist()
        both = {}
        for s, c in zip(canon, cnt):
            both[s] = c
            both[_rc_str(s)] = c
        sym = sorted(both)
        for kmers, counts in ((canon, cnt), (sym, [both[s] for s in sym])):
            w, c = _table(kmers, counts, k)
            for L in (1, 5, 40):
                cases.append((w, c, k, L))
    # entry 1 is a palindrome (even k): the probe moves on to entry 2, which decides
    for k in (8, 32, 40):
        half = "A" * (k // 2 - 1) + "C"
        pal = half + _rc_str(half)
        assert _rc_str(pal) == pal
        for tail in (["C" * k], ["G" * k, "C" * k]):                  # CCC..: its reverse complement is absent
            w, c = _table(["A" * k] + [pal] + tail, [3] * (2 + len(tail)), k)
            cases.append((w, c, k, 2))
    # top-bit keys (G/T first) only, counts read as int16 (a count >= 0x8000 is negative there)
    w, c = _table(["G" * 21, "T" * 21, "GA" + "C" * 19], [0x8001, 7, 9], 21)
    cases.append((w, c, 21, 8))
    for k in (21, 40):                                                # 0 and 1 entries
        w, c = _table([], [], k)
        cases.append((w.reshape(0, 2), c, k, 4))
        w, c = _table(["C" * k], [2], k)
        cases.append((w, c, k, 4))
    return cases


@pytest.mark.parametrize("world", [2, 3])
def test_job_examine_verdicts_over_gloo_ranks(world):
    cases = _verdict_cases()
    want = [_examine_numpy(w, c, k, L) for w, c, k, L in cases]
    assert {v for v in want} >= {(True, True), (False, False), (True, False), (False, True)}
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000) + world
    procs = [ctx.Process(target=_verdict_worker, args=(r, world, port, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank in range(world):
        for i, (w, c, k, L) in enumerate(cases):
            assert res[rank][i] == want[i], (rank, i, k, L, len(c), res[rank][i], want[i])


def test_share_find_handles_the_top_bit():
    """keys at or above 2^63 (first base G or T) come last in unsigned order but first would come in torch's signed
    order: every key of a table spanning both halves is found where it is, absent keys are not"""
    rng = np.random.default_rng(3)
    ku = np.unique(rng.integers(0, 1 << 63, size=500, dtype=np.uint64) * np.uint64(2) + np.uint64(1))
    keys = torch.from_numpy(ku.view(np.int64))
    assert (ku >= (1 << 63)).any() and (ku < (1 << 63)).any()
    for i in range(0, len(ku), 7):
        assert hd._share_find(keys, None, int(ku[i]), 0) == i
        assert hd._share_find(keys, None, int(ku[i]) - 1, 0) == -1
    two = np.stack([np.repeat(ku[:20], 3), np.tile(ku[-3:], 20)], axis=1)        # equal first words: second decides
    kt, kl = torch.from_numpy(two[:, 0].copy().view(np.int64)), torch.from_numpy(two[:, 1].copy().view(np.int64))
    for i in range(len(two)):
        assert hd._share_find(kt, kl, int(two[i, 0]), int(two[i, 1])) == i
    assert hd._share_find(kt, kl, int(two[0, 0]), int(ku[0])) == -1
    assert hd._share_find(torch.empty(0, dtype=torch.int64), None, 5, 0) == -1

"""The cut rule of StreamedShardedScan.from_ktab(L=...) (dist.run_condition_cuts, DESIGN.md §4f) against a numpy
restatement: every rank's range of key prefixes starts on a run boundary (the first k//2 bases) and on a stub
bucket, each cut is the allowed boundary nearest to r/world of the output (the lower one on a tie), and where runs
are no finer than buckets the rule is condition_ktab's (bucket_condition_cuts)."""
import numpy as np
import pytest

from smudgeplot_b200 import dist as hd


def restated(hist, world, hb, ibyte, k):
    """numpy: the boundaries of min(hb, 8*ibyte, 2*(k//2))-bit prefixes, as hb-bit prefixes; cut r the last of them
    with at most total*r//world entries below it, or the next one if that is strictly nearer; never below cut r-1"""
    bits = min(hb, 8 * ibyte, 2 * (k >> 1))
    step = 1 << (hb - bits)
    bounds = np.arange(0, (1 << hb) + 1, step)
    below = np.concatenate([[0], np.cumsum(hist)])[bounds]
    total = int(below[-1])
    cuts = [0]
    for r in range(1, world):
        want = total * r // world
        lo = int(np.flatnonzero(below <= want)[-1])
        if lo + 1 < len(bounds) and below[lo + 1] - want < want - below[lo]:
            lo += 1
        cuts.append(max(int(bounds[lo]), cuts[-1]))
    return cuts + [1 << hb]


@pytest.mark.parametrize("k", [4, 9, 12, 15, 17, 19, 20, 21, 31, 40])
@pytest.mark.parametrize("ibyte", [1, 2, 3])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_run_cuts_match_the_restatement(k, ibyte, world):
    if ibyte > (k + 3) >> 2:
        pytest.skip("ibyte above the k-mer's bytes")
    hb = min(20, 2 * k)
    rng = np.random.default_rng(k * 100 + ibyte * 10 + world)
    for shape in ("uniform", "skewed", "one", "empty_tail"):
        h = rng.integers(0, 50, 1 << hb).astype(np.int64)
        if shape == "skewed":
            h[: 1 << max(hb - 3, 0)] *= 40
        elif shape == "one":
            h[:] = 0
            h[rng.integers(0, 1 << hb)] = 1000
        elif shape == "empty_tail":
            h[(1 << hb) // 7:] = 0
        got = hd.run_condition_cuts(h, world, hb, ibyte, k)
        assert got == restated(h, world, hb, ibyte, k), (shape, got)
        step = 1 << max(hb - min(8 * ibyte, 2 * (k >> 1)), 0)
        assert all(c % step == 0 for c in got) and got == sorted(got)
        if 2 * (k >> 1) >= min(hb, 8 * ibyte):
            assert got == hd.bucket_condition_cuts(h, world, hb, ibyte)


def test_small_k_cuts_are_coarser_than_buckets():
    """at ibyte 3 and k < 20 bucket cuts can split a run; the rule moves them to a run boundary"""
    k, ibyte, hb, world = 12, 3, 20, 3
    h = np.ones(1 << hb, dtype=np.int64)
    buckets = hd.bucket_condition_cuts(h, world, hb, ibyte)
    runs = hd.run_condition_cuts(h, world, hb, ibyte, k)
    step = 1 << (hb - 2 * (k >> 1))
    assert any(c % step for c in buckets) and all(c % step == 0 for c in runs)

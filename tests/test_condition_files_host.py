"""CPU tests of the pieces of hm_scan_condition_files that need no GPU: the incremental FastK table writer
(hm_table_write_*) and the range planner (hm_condition_plan), through the C ABI."""
import ctypes as C
import filecmp
import os

import numpy as np
import pytest

from smudgeplot_b200 import _lib, fastk
from tools import synth

import oracle_util as ou


def random_table(k, n, seed, one_bucket=False):
    """n distinct sorted k-mers as uint8[n, kbyte] (pad bits zero) + counts"""
    rng = np.random.default_rng(seed)
    kb = (k + 3) >> 2
    keys = rng.integers(0, 256, size=(n, kb), dtype=np.uint8)
    if k % 4:
        keys[:, -1] &= np.uint8((0xFF << (2 * (4 - k % 4))) & 0xFF)
    if one_bucket:
        keys[:, :3] = 7 if kb >= 3 else keys[:, :3]
        keys[:, 0] = 7
    keys = np.unique(keys, axis=0)
    cnt = rng.integers(1, 3000, size=len(keys), dtype=np.uint16)
    return keys, cnt


def c_write(name, kt, nparts, pieces, hint=None):
    """write kt's records with the C writer, appended in `pieces` slices of ordinals (buckets split across them)"""
    L = _lib.lib()
    n, pb = kt.nels, kt.pbyte
    rec = kt.all_records()
    ends = kt.index.astype(np.int64)
    starts = np.concatenate([[0], ends[:-1]])
    w = C.c_void_p()
    _lib.check(L.hm_table_write_open(name.encode(), kt.kmer, kt.ibyte, kt.minval, nparts, n if hint is None else hint,
                                     C.byref(w)))
    bounds = sorted(set([0, n] + [int(x) for x in pieces]))
    for a, b in zip(bounds[:-1], bounds[1:]):
        ba = int(np.searchsorted(ends, a, side="right"))
        bb = int(np.searchsorted(ends, b - 1, side="right"))
        cnt = (np.minimum(ends[ba:bb + 1], b) - np.maximum(starts[ba:bb + 1], a)).clip(0).astype(np.int64)
        _lib.check(L.hm_table_write_buckets(w, ba, bb - ba + 1, cnt.ctypes.data))
        chunk = np.ascontiguousarray(rec[a * pb:b * pb])
        _lib.check(L.hm_table_write_append(w, chunk.ctypes.data, b - a))
    _lib.check(L.hm_table_write_close(w))


def same_files(a, b, nparts):
    assert filecmp.cmp(fastk.stub_path(a), fastk.stub_path(b), shallow=False)
    for p in range(1, nparts + 1):
        assert filecmp.cmp(fastk.part_path(a, p), fastk.part_path(b, p), shallow=False), f"part {p}"


CASES = [(4, 1), (12, 1), (12, 2), (12, 3), (21, 2), (21, 3), (31, 1), (31, 3), (32, 2), (40, 3), (64, 1), (64, 3)]


@pytest.mark.parametrize("k,ibyte", CASES)
@pytest.mark.parametrize("nparts", [1, 2, 3, 4])
def test_writer_matches_write_ktab(built, tmp_path, k, ibyte, nparts):
    keys, cnt = random_table(k, 5000 if k > 4 else 200, seed=k * 10 + ibyte)
    want = str(tmp_path / "want")
    kt = fastk.write_ktab(want, k, keys, cnt, ibyte=ibyte, nparts=nparts, minval=3)
    got = str(tmp_path / "got")
    n = kt.nels
    c_write(got, kt, nparts, [n // 7, n // 3, n // 3 + 1, (2 * n) // 3])     # appends that split buckets
    same_files(got, want, nparts)
    assert fastk.read_ktab(got).nels == n


@pytest.mark.parametrize("nparts", [1, 2, 4])
def test_writer_empty_parts_and_empty_table(built, tmp_path, nparts):
    keys, cnt = random_table(31, 3000, seed=5, one_bucket=True)     # one bucket: every cut on its start
    for tag, (kk, cc) in {"one": (keys, cnt), "zero": (keys[:0], cnt[:0])}.items():
        want, got = str(tmp_path / f"w{tag}"), str(tmp_path / f"g{tag}")
        kt = fastk.write_ktab(want, 31, kk, cc, ibyte=3, nparts=nparts)
        assert tag == "zero" or nparts == 1 or 0 in kt.part_nels
        c_write(got, kt, nparts, [kt.nels // 2])
        same_files(got, want, nparts)


def test_writer_cuts_on_buckets_for_any_hint(built, tmp_path):
    """with an upper bound instead of the exact count, parts still end on stub buckets and hold everything"""
    keys, cnt = random_table(21, 8000, seed=9)
    kt = fastk.write_ktab(str(tmp_path / "src"), 21, keys, cnt, ibyte=2, nparts=3)
    got = str(tmp_path / "got")
    c_write(got, kt, 3, [1000, 4000], hint=kt.nels + 2500)
    back = fastk.read_ktab(got)
    assert back.nels == kt.nels and np.array_equal(back.index, kt.index)
    assert np.array_equal(back.all_records(), kt.all_records())
    starts = set(np.concatenate([[0], kt.index]).tolist())
    assert all(c in starts for c in np.cumsum(back.part_nels).tolist())


def test_writer_failure_leaves_nothing(built, tmp_path):
    L = _lib.lib()
    name = str(tmp_path / "bad")
    w = C.c_void_p()
    _lib.check(L.hm_table_write_open(name.encode(), 21, 2, 1, 2, 10, C.byref(w)))
    rec = np.zeros(7 * 10, dtype=np.uint8)
    cnt = np.array([4], dtype=np.int64)
    _lib.check(L.hm_table_write_buckets(w, 3, 1, cnt.ctypes.data))
    assert L.hm_table_write_append(w, rec.ctypes.data, 10) == -1           # beyond the announced buckets
    assert L.hm_table_write_close(w) == -1
    assert os.listdir(tmp_path) == []
    w = C.c_void_p()
    _lib.check(L.hm_table_write_open(name.encode(), 21, 2, 1, 2, 10, C.byref(w)))
    L.hm_table_write_abort(w)
    assert os.listdir(tmp_path) == []


def test_reference_reads_a_c_written_table(built, tmp_path):
    if not ou.have_ref():
        pytest.skip("the reference binary was not built")
    keys, cnt = synth.synth_table(31, 20000, ploidy=2, het=0.02, cov=40, L=8, seed=12)
    src = str(tmp_path / "src")
    kt = synth.write_table(src, 31, keys, cnt, ibyte=3, nparts=3)
    got = str(tmp_path / "got")
    c_write(got, kt, 3, [kt.nels // 2])
    r = ou.run_ref(got, str(tmp_path / "ref"), 8)
    assert r.returncode == 0, r.stderr
    kb, cn = fastk.unpack_host(kt)
    want, _ = ou.oracle_scan(kb, cn, 31)
    assert open(str(tmp_path / "ref.smu")).read() == ou.smu_text(want)


# ------------------------------------------------------------------------------------------- plan --

def plan(n, k, ibyte, budget, hist, symm=1):
    L = _lib.lib()
    hist = np.ascontiguousarray(hist, dtype=np.int64)
    hb = int(np.log2(len(hist)))
    cuts = np.zeros(len(hist) + 1, dtype=np.int64)
    lay = _lib.ConditionLayout()
    rc = L.hm_condition_plan(n, k, ibyte, budget, symm, hist.ctypes.data, hb, cuts.ctypes.data, C.byref(lay))
    return rc, lay, cuts[:lay.n_ranges + 1].copy() if rc == 0 else None


def range_cap(room, k, ibyte, symm):
    """the most entries a range may hold: restated by bisection over hm_condition_range_bytes"""
    L = _lib.lib()
    lo, hi = 0, 1 << 31
    while lo < hi:
        mid = lo + (hi - lo + 1) // 2
        if L.hm_condition_range_bytes(mid, symm, k, ibyte) <= room:
            lo = mid
        else:
            hi = mid - 1
    return lo


def plan_numpy(hist, cap):
    """greedy cuts in key order: a prefix starts a new range when it would overfill the current one"""
    cuts, t = [0], 0
    for p, h in enumerate(hist.tolist()):
        if t + h > cap:
            cuts.append(p)
            t = 0
        t += h
    cuts.append(len(hist))
    return np.array(cuts, dtype=np.int64)


def random_hist(seed, bits=12, big=None):
    rng = np.random.default_rng(seed)
    h = rng.poisson(rng.uniform(0, 40000), size=1 << bits).astype(np.int64)
    if big is not None:
        h[rng.integers(0, len(h))] = big
    return h


@pytest.mark.parametrize("seed,k,ibyte,big", [(1, 31, 3, None), (2, 21, 2, None), (3, 40, 3, None),
                                              (4, 31, 2, 30_000_000), (5, 64, 3, 12_000_000), (6, 12, 1, None)])
def test_plan_agrees_with_numpy_and_fits(built, seed, k, ibyte, big):
    hist = random_hist(seed, big=big)
    n = int(hist.sum()) // 2
    L = _lib.lib()
    prev_ranges, feasible = None, 0
    for budget in [int(x) for x in (3e8, 6e8, 1e9, 1.6e9, 3e9, 8e9, 3e10, 8e10)]:
        rc, lay, cuts = plan(n, k, ibyte, budget, hist)
        if rc != 0:
            assert rc == -3 and feasible == 0                  # HM_ENOMEM only below every feasible budget
            assert b"cannot hold one range" in L.hm_last_error()
            continue
        feasible += 1
        cap = range_cap(lay.range_room, k, ibyte, 1)
        assert np.array_equal(cuts, plan_numpy(hist, cap))
        sizes = np.add.reduceat(hist, cuts[:-1])
        assert cuts[0] == 0 and cuts[-1] == len(hist) and np.all(np.diff(cuts) > 0)   # cover the keys in order
        assert sizes.max() == lay.range_cap <= cap
        assert lay.range_bytes == L.hm_condition_range_bytes(lay.range_cap, 1, k, ibyte)
        assert lay.fixed_bytes + lay.range_bytes <= budget                         # no range exceeds the budget
        assert prev_ranges is None or lay.n_ranges <= prev_ranges                  # monotone in the budget
        prev_ranges = lay.n_ranges
    assert feasible >= 3


def test_plan_enomem_names_the_sizes(built):
    hist = random_hist(7)
    hist[100] = 3_000_000_000                                   # one prefix larger than any range can be
    rc, lay, _ = plan(int(hist.sum()), 31, 3, int(8e10), hist)
    assert rc == -3
    msg = _lib.lib().hm_last_error().decode()
    assert "80000000000" in msg and "3000000000" in msg
    rc, _, _ = plan(1000, 31, 3, 100 << 20, np.zeros(1 << 12, dtype=np.int64))   # the stub index pair alone
    assert rc == -3


def test_plan_takes_one_range_when_it_fits(built):
    hist = random_hist(8, bits=20) // 1000
    rc, lay, cuts = plan(int(hist.sum()), 31, 3, 8 << 30, hist)
    assert rc == 0 and lay.n_ranges == 1 and list(cuts) == [0, 1 << 20]
    assert plan(10, 31, 3, -1, hist)[0] == -1                   # bad arguments
    assert plan(10, 65, 3, 1 << 30, hist)[0] == -1
    rc, lay, cuts = plan(int(hist.sum()), 31, 3, 8 << 30, hist, symm=0)
    assert rc == 0 and lay.range_bytes < _lib.lib().hm_condition_range_bytes(lay.range_cap, 1, 31, 3)

"""CPU tests of the table writer's positional mode (hm_table_write_place / _at / _seal), which the conditioning on
several GPUs writes through: ranges placed in table order and written at their offsets from several threads in any
order give the files of the append path, byte for byte, and a failure or an abort leaves nothing."""
import ctypes as C
import os
import random
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from smudgeplot_b200 import _lib, fastk

from test_condition_files_host import random_table, same_files


def bucket_counts(kt, a, b):
    """(b0, counts) of the stub buckets holding ordinals [a, b): what the conditioning's pack step reports"""
    ends = kt.index.astype(np.int64)
    starts = np.concatenate([[0], ends[:-1]])
    if b <= a:
        return 0, np.zeros(0, dtype=np.int64)
    ba = int(np.searchsorted(ends, a, side="right"))
    bb = int(np.searchsorted(ends, b - 1, side="right"))
    cnt = (np.minimum(ends[ba:bb + 1], b) - np.maximum(starts[ba:bb + 1], a)).clip(0).astype(np.int64)
    return ba, cnt


def open_writer(name, kt, nparts, hint=None):
    w = C.c_void_p()
    _lib.check(_lib.lib().hm_table_write_open(name.encode(), kt.kmer, kt.ibyte, kt.minval, nparts,
                                              kt.nels if hint is None else hint, C.byref(w)))
    return w


def place(w, kt, a, b):
    b0, cnt = bucket_counts(kt, a, b)
    first = C.c_int64(-1)
    _lib.check(_lib.lib().hm_table_write_place(w, b0, len(cnt), cnt.ctypes.data if len(cnt) else None,
                                               C.byref(first)))
    assert first.value == a
    return first.value


def write_at(w, rec, pb, a, b):
    chunk = np.ascontiguousarray(rec[a * pb:b * pb])
    return _lib.lib().hm_table_write_at(w, a, chunk.ctypes.data if b > a else None, b - a)


def pieces(a, b, rng):
    """[a, b) cut into one to three slices"""
    cuts = sorted(set([a, b] + [int(x) for x in rng.integers(a, b + 1, size=rng.integers(0, 3))]))
    return list(zip(cuts[:-1], cuts[1:])) or [(a, a)]


def range_bounds(n, rng, n_ranges):
    """n_ranges contiguous ordinal ranges over [0, n), some of them empty"""
    inner = sorted(int(x) for x in rng.integers(0, n + 1, size=n_ranges - 1))
    bounds = [0] + inner + [n]
    return list(zip(bounds[:-1], bounds[1:]))


def positional_write(name, kt, nparts, ranges, rng, interleave, hint=None):
    """place `ranges` in order; write their slices on 4 threads, shuffled: while the later ranges are still being
    placed (interleave) or after every range is placed"""
    L = _lib.lib()
    rec, pb = kt.all_records(), kt.pbyte
    w = open_writer(name, kt, nparts, hint)
    jobs = []
    with ThreadPoolExecutor(4) as pool:
        futures = []
        for a, b in ranges:
            place(w, kt, a, b)
            sl = pieces(a, b, rng)
            if interleave:
                rng.shuffle(sl)
                futures += [pool.submit(write_at, w, rec, pb, x, y) for x, y in sl]
            else:
                jobs += sl
        random.Random(int(rng.integers(1 << 30))).shuffle(jobs)
        futures += [pool.submit(write_at, w, rec, pb, x, y) for x, y in jobs]
        time.sleep(0.01)
        L.hm_table_write_seal(w)
        for f in futures:
            assert f.result() == 0
    _lib.check(L.hm_table_write_close(w))


CASES = [(12, 1), (21, 2), (31, 3), (40, 3), (64, 2)]


@pytest.mark.parametrize("k,ibyte", CASES)
@pytest.mark.parametrize("nparts", [1, 2, 3, 4])
@pytest.mark.parametrize("interleave", [False, True])
def test_positional_matches_append_path(built, tmp_path, k, ibyte, nparts, interleave):
    keys, cnt = random_table(k, 6000, seed=k * 10 + ibyte + nparts)
    want = str(tmp_path / "want")
    kt = fastk.write_ktab(want, k, keys, cnt, ibyte=ibyte, nparts=nparts, minval=3)
    rng = np.random.default_rng(k + 100 * nparts + 7 * interleave)
    n = kt.nels
    astride = sorted({0, n} | {min(max(c + d, 0), n) for c in np.cumsum(kt.part_nels)[:-1].tolist() for d in (-3, 3)})
    for trial, ranges in enumerate([range_bounds(n, rng, 9),                      # random ranges, some empty
                                    [(0, 0), (0, n), (n, n)],                     # one range over every cut
                                    list(zip(astride[:-1], astride[1:]))]):       # short ranges astride the cuts
        got = str(tmp_path / f"got{trial}")
        positional_write(got, kt, nparts, ranges, rng, interleave)
        same_files(got, want, nparts)
    assert fastk.read_ktab(got).nels == n


@pytest.mark.parametrize("nparts", [1, 2, 4])
def test_positional_upper_bound_hint_and_empty_table(built, tmp_path, nparts):
    """a hint above the count (the conditioning's histogram total) cuts as the append path cuts; an empty table and
    a table in one bucket (every cut at its start) too"""
    from test_condition_files_host import c_write
    rng = np.random.default_rng(nparts)
    keys, cnt = random_table(21, 8000, seed=9)
    one, one_cnt = random_table(31, 3000, seed=5, one_bucket=True)
    for tag, (k, kk, cc, ibyte, hint) in {"hint": (21, keys, cnt, 2, 2500), "zero": (21, keys[:0], cnt[:0], 2, 0),
                                          "one": (31, one, one_cnt, 3, 0)}.items():
        kt = fastk.write_ktab(str(tmp_path / f"src{tag}"), k, kk, cc, ibyte=ibyte, nparts=nparts)
        want, got = str(tmp_path / f"w{tag}"), str(tmp_path / f"g{tag}")
        c_write(want, kt, nparts, [kt.nels // 2], hint=kt.nels + hint)
        positional_write(got, kt, nparts, range_bounds(kt.nels, rng, 5), rng, True, hint=kt.nels + hint)
        same_files(got, want, nparts)


def test_last_bucket_is_held_until_the_next_place(built, tmp_path):
    """records of the last bucket announced may still fall on either side of a cut: hm_table_write_at returns at
    once and the next place writes them"""
    L = _lib.lib()
    keys, cnt = random_table(31, 4000, seed=3)
    kt = fastk.write_ktab(str(tmp_path / "want"), 31, keys, cnt, ibyte=3, nparts=2)
    rec, pb, n = kt.all_records(), kt.pbyte, kt.nels
    w = open_writer(str(tmp_path / "got"), kt, 2)
    a = n // 4
    place(w, kt, 0, a)
    assert write_at(w, rec, pb, 0, a) == 0                          # its last bucket's records are held
    last = int(np.searchsorted(kt.index, a - 1, side="right"))      # the bucket holding ordinal a - 1
    start = int(kt.index[last - 1]) if last > 0 else 0
    part1 = open(fastk.part_path(str(tmp_path / "got"), 1) + f".tmp{os.getpid()}", "rb").read()
    assert 0 < start < a and len(part1) == 12 + start * pb          # written up to that bucket's start
    place(w, kt, a, n)
    assert write_at(w, rec, pb, a, n) == 0
    _lib.check(L.hm_table_write_close(w))
    same_files(str(tmp_path / "got"), str(tmp_path / "want"), 2)


def skewed_table(k, ibyte, sizes, seed):
    """sorted distinct k-mers whose first ibyte bytes are the keys of `sizes` ({prefix: entries}): a few large
    stub buckets"""
    rng = np.random.default_rng(seed)
    kb = (k + 3) >> 2
    parts = []
    for pre, m in sorted(sizes.items()):
        x = rng.integers(0, 256, size=(m * 2, kb), dtype=np.uint8)
        for j in range(ibyte):
            x[:, j] = (pre >> (8 * (ibyte - 1 - j))) & 0xFF
        if k % 4:
            x[:, -1] &= np.uint8((0xFF << (2 * (4 - k % 4))) & 0xFF)
        parts.append(np.unique(x, axis=0)[:m])
    keys = np.concatenate(parts)
    return keys, rng.integers(1, 3000, size=len(keys), dtype=np.uint16)


def driver_order(w, kt, ranges, gpus, pieces_of):
    """what hm_scan_condition_files does on `gpus` GPUs: GPU g takes ranges g, g + G, ...; before placing a range
    it joins the writer of its previous one, places the ranges in order, then starts the range's writer thread.
    -> False if the threads did not finish (they would wait for each other forever)"""
    rec, pb = kt.all_records(), kt.pbyte
    cv = threading.Condition()
    state = {"next": 0, "rc": []}

    def writer(a, b):
        for x, y in pieces_of(a, b):
            state["rc"].append(write_at(w, rec, pb, x, y))

    def gpu(g):
        prev = None
        for r in range(g, len(ranges), gpus):
            if prev is not None:
                prev.join()
            with cv:
                cv.wait_for(lambda: state["next"] == r)
                place(w, kt, *ranges[r])
                state["next"] = r + 1
                cv.notify_all()
            prev = threading.Thread(target=writer, args=ranges[r])
            prev.start()
        if prev is not None:
            prev.join()
    threads = [threading.Thread(target=gpu, args=(g,), daemon=True) for g in range(gpus)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(30)
    done = not any(t.is_alive() for t in threads)
    assert not done or all(rc == 0 for rc in state["rc"])
    return done


def test_driver_order_with_ranges_inside_one_bucket(built, tmp_path):
    """ibyte 1, two parts, hint 1000: ranges 0 and 1 each hold 100 records of bucket 5, range 2 finishes it and
    holds bucket 200, where the cut's ordinal lies.  Range 0's last records stay in doubt until range 2 is placed,
    and GPU 0 joins range 0's writer before it places range 2: the writer must not wait for that place."""
    keys, cnt = skewed_table(21, 1, {5: 300, 200: 700}, seed=1)
    want = str(tmp_path / "want")
    kt = fastk.write_ktab(want, 21, keys, cnt, ibyte=1, nparts=2)
    got = str(tmp_path / "got")
    w = open_writer(got, kt, 2, 1000)
    assert driver_order(w, kt, [(0, 100), (100, 200), (200, 1000)], 2, lambda a, b: [(a, b)])
    _lib.check(_lib.lib().hm_table_write_close(w))
    same_files(got, want, 2)


@pytest.mark.parametrize("ibyte", [1, 2])
@pytest.mark.parametrize("nparts", [3, 4])
@pytest.mark.parametrize("gpus", [2, 3])
def test_driver_order_with_ranges_smaller_than_a_bucket(built, tmp_path, ibyte, nparts, gpus):
    """a few stub buckets, each cut into many ranges (as a large ibyte 1 or 2 table under a small budget is): the
    driver's order finishes and writes the files of the append path"""
    rng = np.random.default_rng(ibyte * 100 + nparts * 10 + gpus)
    keys, cnt = skewed_table(21, ibyte, {3: 1500, 77: 4000, 78: 20, 250: 2500}, seed=ibyte + nparts)
    want = str(tmp_path / "want")
    kt = fastk.write_ktab(want, 21, keys, cnt, ibyte=ibyte, nparts=nparts)
    for trial in range(2):
        got = str(tmp_path / f"got{trial}")
        w = open_writer(got, kt, nparts)
        assert driver_order(w, kt, range_bounds(kt.nels, rng, 40), gpus, lambda a, b: pieces(a, b, rng))
        _lib.check(_lib.lib().hm_table_write_close(w))
        same_files(got, want, nparts)


def test_positional_failures_and_abort_leave_nothing(built, tmp_path):
    L = _lib.lib()
    keys, cnt = random_table(21, 3000, seed=4)
    kt = fastk.write_ktab(str(tmp_path / "src"), 21, keys, cnt, ibyte=2, nparts=3)
    rec, pb, n = kt.all_records(), kt.pbyte, kt.nels
    d = tmp_path / "out"
    d.mkdir()
    name = str(d / "t")
    # abort after some ranges were placed and written, some records still held
    w = open_writer(name, kt, 3)
    place(w, kt, 0, n // 2)
    assert write_at(w, rec, pb, 0, n // 2) == 0
    L.hm_table_write_seal(w)
    assert L.hm_table_write_place(w, 0, 0, None, C.byref(C.c_int64())) == -1   # sealed: no range follows
    L.hm_table_write_abort(w)
    assert os.listdir(d) == []
    # records beyond what was placed: refused, and the writer is failed
    w = open_writer(name, kt, 3)
    place(w, kt, 0, n // 3)
    assert write_at(w, rec, pb, 0, n // 3 + 1) == -1
    assert L.hm_table_write_close(w) == -1
    assert os.listdir(d) == []
    # placed records never written: close refuses
    w = open_writer(name, kt, 3)
    place(w, kt, 0, n)
    L.hm_table_write_seal(w)
    assert write_at(w, rec, pb, 0, n - 1) == 0
    assert L.hm_table_write_close(w) == -1
    assert os.listdir(d) == []
    # one writer takes one mode
    w = open_writer(name, kt, 3)
    b0, cnt = bucket_counts(kt, 0, 10)
    _lib.check(L.hm_table_write_buckets(w, b0, len(cnt), cnt.ctypes.data))
    assert L.hm_table_write_place(w, b0, len(cnt), cnt.ctypes.data, C.byref(C.c_int64())) == -1
    L.hm_table_write_abort(w)
    w = open_writer(name, kt, 3)
    place(w, kt, 0, 10)
    assert L.hm_table_write_buckets(w, b0, len(cnt), cnt.ctypes.data) == -1
    assert L.hm_table_write_append(w, rec.ctypes.data, 10) == -1
    L.hm_table_write_abort(w)
    assert os.listdir(d) == []

"""CPU tests of the table writer's host-memory target (hm_table_write_open_host / _close_host, hm_host_table_free),
which hm_scan_condition_host writes through: the same place / at calls as the file target, in any order and from
several threads, give the records of the part files concatenated and the stub's index, byte for byte; records
beyond what was placed or what the table has room for are refused; an abort or a failed close frees everything."""
import ctypes as C
import os
import random
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from smudgeplot_b200 import _lib, fastk

from test_condition_files_host import random_table
from test_condition_files_positional_host import bucket_counts, open_writer, pieces, range_bounds, write_at


def open_host(kt, cap):
    w = C.c_void_p()
    _lib.check(_lib.lib().hm_table_write_open_host(kt.kmer, kt.ibyte, kt.minval, cap, C.byref(w)))
    return w


def close_host(w):
    t = C.POINTER(_lib.HostTable)()
    _lib.check(_lib.lib().hm_table_write_close_host(w, C.byref(t)))
    return t


def plan_calls(kt, rng, n_ranges):
    """the ranges (in table order) and, per range, its slices in shuffled order"""
    ranges = range_bounds(kt.nels, rng, n_ranges)
    slices = []
    for a, b in ranges:
        sl = pieces(a, b, rng)
        rng.shuffle(sl)
        slices.append(sl)
    return ranges, slices


def feed(w, kt, ranges, slices, seed):
    """place the ranges in order, write every range's slices on 4 threads as it is placed, seal"""
    L = _lib.lib()
    rec, pb = kt.all_records(), kt.pbyte
    with ThreadPoolExecutor(4) as pool:
        futures = []
        for (a, b), sl in zip(ranges, slices):
            b0, cnt = bucket_counts(kt, a, b)
            first = C.c_int64(-1)
            _lib.check(L.hm_table_write_place(w, b0, len(cnt), cnt.ctypes.data if len(cnt) else None, C.byref(first)))
            assert first.value == a
            futures += [pool.submit(write_at, w, rec, pb, x, y) for x, y in sl]
        random.Random(seed).shuffle(futures)
        L.hm_table_write_seal(w)
        assert all(f.result() == 0 for f in futures)


def host_arrays(t, kt):
    v = t.contents
    n = int(v.nels)
    assert (v.kmer, v.ibyte, v.nparts, v.minval) == (kt.kmer, kt.ibyte, 1, kt.minval)
    assert v.part_nels[0] == n and (v.part_fd is None or not v.part_fd)
    index = np.ctypeslib.as_array(v.index, shape=(1 << (8 * kt.ibyte),)).copy()
    rec = (np.ctypeslib.as_array(C.cast(v.part_rec[0], C.POINTER(C.c_uint8)), shape=(n * kt.pbyte,)).copy() if n
           else np.empty(0, dtype=np.uint8))
    return index, rec


def file_arrays(name):
    got = fastk.read_ktab(name)
    return np.asarray(got.index, dtype=np.int64), got.all_records(), got.nparts


CASES = [(12, 1), (21, 2), (31, 3), (40, 3), (64, 2)]


@pytest.mark.parametrize("k,ibyte", CASES)
@pytest.mark.parametrize("nparts", [1, 3])
def test_memory_target_matches_file_target(built, tmp_path, k, ibyte, nparts):
    """the same place / at calls, slices shuffled and written from 4 threads, into files of nparts parts and into
    memory with room above the count (the conditioning's histogram bound)"""
    L = _lib.lib()
    keys, cnt = random_table(k, 5000, seed=k * 10 + ibyte + nparts)
    kt = fastk.write_ktab(str(tmp_path / "src"), k, keys, cnt, ibyte=ibyte, nparts=nparts, minval=3)
    rng = np.random.default_rng(k + 100 * nparts)
    for trial, n_ranges in enumerate([1, 7, 25]):
        ranges, slices = plan_calls(kt, rng, n_ranges)
        name = str(tmp_path / f"files{trial}")
        w = open_writer(name, kt, nparts)
        feed(w, kt, ranges, slices, seed=trial)
        _lib.check(L.hm_table_write_close(w))
        want_index, want_rec, parts = file_arrays(name)
        assert parts == nparts
        w = open_host(kt, kt.nels + int(rng.integers(0, 500)))
        feed(w, kt, ranges, slices, seed=trial + 10)
        t = close_host(w)
        try:
            index, rec = host_arrays(t, kt)
        finally:
            L.hm_host_table_free(t)
        assert np.array_equal(index, want_index)
        assert rec.tobytes() == want_rec.tobytes()
        assert rec.tobytes() == kt.all_records().tobytes()


def test_memory_target_append_and_empty_table(built, tmp_path):
    """write_buckets + append into memory gives the source's records and index; an empty table closes to an empty
    one-part table"""
    from test_condition_files_host import c_write
    L = _lib.lib()
    keys, cnt = random_table(31, 4000, seed=2)
    kt = fastk.write_ktab(str(tmp_path / "src"), 31, keys, cnt, ibyte=3, nparts=2)
    c_write(str(tmp_path / "files"), kt, 2, [kt.nels // 3, kt.nels // 2])
    want_index, want_rec, _ = file_arrays(str(tmp_path / "files"))
    rec, n, pb = kt.all_records(), kt.nels, kt.pbyte
    w = open_host(kt, n)
    for a, b in [(0, n // 3), (n // 3, n // 2), (n // 2, n)]:
        b0, c = bucket_counts(kt, a, b)
        _lib.check(L.hm_table_write_buckets(w, b0, len(c), c.ctypes.data))
        chunk = np.ascontiguousarray(rec[a * pb:b * pb])
        _lib.check(L.hm_table_write_append(w, chunk.ctypes.data, b - a))
    t = close_host(w)
    index, got = host_arrays(t, kt)
    L.hm_host_table_free(t)
    assert np.array_equal(index, want_index) and got.tobytes() == want_rec.tobytes()
    w = open_host(kt, 0)
    L.hm_table_write_seal(w)
    t = close_host(w)
    index, got = host_arrays(t, kt)
    L.hm_host_table_free(t)
    assert t is not None and not index.any() and got.size == 0


def test_memory_target_refusals(built, tmp_path):
    L = _lib.lib()
    keys, cnt = random_table(21, 3000, seed=4)
    kt = fastk.write_ktab(str(tmp_path / "src"), 21, keys, cnt, ibyte=2, nparts=1)
    rec, pb, n = kt.all_records(), kt.pbyte, kt.nels
    out = C.POINTER(_lib.HostTable)()
    # a record beyond what was placed: refused, the writer failed, close refuses and returns no table
    w = open_host(kt, n)
    b0, c = bucket_counts(kt, 0, n // 3)
    _lib.check(L.hm_table_write_place(w, b0, len(c), c.ctypes.data, C.byref(C.c_int64())))
    assert write_at(w, rec, pb, 0, n // 3 + 1) == -1
    assert L.hm_table_write_close_host(w, C.byref(out)) == -1 and not out
    # more records than the table has room for: refused when announced
    w = open_host(kt, n - 1)
    b0, c = bucket_counts(kt, 0, n)
    assert L.hm_table_write_place(w, b0, len(c), c.ctypes.data, C.byref(C.c_int64())) == -1
    assert "room for" in L.hm_last_error().decode()
    L.hm_table_write_abort(w)
    # the targets' closes do not mix
    w = open_host(kt, n)
    assert L.hm_table_write_close(w) == -1
    d = tmp_path / "out"
    d.mkdir()
    w = open_writer(str(d / "t"), kt, 1)
    assert L.hm_table_write_close_host(w, C.byref(out)) == -1 and not out
    assert os.listdir(d) == []
    assert L.hm_table_write_open_host(21, 2, 0, -1, C.byref(C.c_void_p())) == -1


def rss_bytes():
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")


@pytest.mark.parametrize("end", ["abort", "failed_close", "free"])
def test_memory_target_leaves_nothing_allocated(built, end):
    """a writer with 64 MiB of records written, then aborted, closed with records missing, or closed and its table
    freed, five times over: the resident set does not grow by the buffers"""
    L = _lib.lib()
    k, ibyte = 21, 2
    pb = ((k + 3) >> 2) - ibyte + 2
    m = (64 << 20) // pb
    zeros = np.zeros(m * pb, dtype=np.uint8)
    cnt = np.array([m], dtype=np.int64)

    def one():
        w = C.c_void_p()
        _lib.check(L.hm_table_write_open_host(k, ibyte, 0, m, C.byref(w)))
        _lib.check(L.hm_table_write_place(w, 5, 1, cnt.ctypes.data, C.byref(C.c_int64())))
        upto = m - 1 if end == "failed_close" else m
        _lib.check(L.hm_table_write_at(w, 0, zeros.ctypes.data, upto))
        if end == "abort":
            L.hm_table_write_abort(w)
            return
        t = C.POINTER(_lib.HostTable)()
        rc = L.hm_table_write_close_host(w, C.byref(t))
        if end == "failed_close":
            assert rc == -1 and not t
        else:
            assert rc == 0 and t.contents.nels == m
            L.hm_host_table_free(t)

    one()
    base = rss_bytes()
    for _ in range(5):
        one()
    assert rss_bytes() - base < (32 << 20)

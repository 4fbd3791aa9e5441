"""CPU tests of the in-process pair files (hm_scan_write_pairs, DESIGN.md §6c): the C restatement of the window plan
(hm_pair_windows) against dist.pair_windows, and the new symbols and stats struct as _lib.py binds them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT


def c_plan(h, world, room):
    """hm_pair_windows -> (P, cuts), or raises HetmersError"""
    from smudgeplot_b200 import _lib
    L = _lib.lib()
    h = np.ascontiguousarray(h, dtype=np.int64)
    P = C.c_int64()
    _lib.check(L.hm_pair_windows(h.ctypes.data, h.size, world, room, C.byref(P), None))
    cuts = np.zeros(P.value * world + 1, dtype=np.int64)
    _lib.check(L.hm_pair_windows(h.ctypes.data, h.size, world, room, C.byref(P), cuts.ctypes.data))
    return P.value, [int(c) for c in cuts]


def histograms(seed):
    rng = np.random.default_rng(seed)
    n = 1 << int(rng.integers(4, 13))
    yield rng.integers(0, 30, size=n) * (rng.random(n) < 0.5)              # random, half empty
    skew = rng.zipf(1.6, size=n).clip(max=5000)                            # skewed: a few heavy prefixes
    yield skew
    one = np.zeros(n, dtype=np.int64)                                      # one prefix holds everything
    one[int(rng.integers(0, n))] = int(rng.integers(1, 1000))
    yield one


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("seed", range(5))
def test_c_plan_is_dist_pair_windows(world, seed, built):
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    for h in histograms(seed):
        big, total = int(h.max()), int(h.sum())
        for room in sorted({max(big - 1, 0), big, big + 7, max(total // 5, 1), total, 10 * total + 1}):
            try:
                want = hd.pair_windows(h, world, room)
            except _lib.HetmersError as e:
                assert e.code == -3
                with pytest.raises(_lib.HetmersError) as ei:
                    c_plan(h, world, room)
                assert ei.value.code == -3 and f"holds {big} records" in str(ei.value) and str(room) in str(ei.value)
                continue
            assert c_plan(h, world, room) == (want[0], list(want[1]))


def test_c_plan_edge_cases(built):
    from smudgeplot_b200 import _lib
    assert c_plan(np.zeros(16, dtype=np.int64), 3, 0) == (1, [0, 16, 16, 16])
    h = np.zeros(1 << 10, dtype=np.int64)
    h[77], h[3] = 500, 20
    with pytest.raises(_lib.HetmersError) as ei:
        c_plan(h, 2, 499)
    assert ei.value.code == -3 and "prefix 77 holds 500 records" in str(ei.value)
    assert c_plan(h, 2, 500)[0] == 1
    L = _lib.lib()
    P = C.c_int64()
    assert L.hm_pair_windows(h.ctypes.data, 0, 1, 10, C.byref(P), None) == -1
    assert L.hm_pair_windows(h.ctypes.data, h.size, 0, 10, C.byref(P), None) == -1


LAYOUT_PROBE = r"""
#include <stdio.h>
#include <stddef.h>
#include "hetmers_b200.h"
#define F(f) printf("%s %zu\n", #f, offsetof(hm_pairs_stats, f));
int main(void)
{ F(records) F(passes) F(windows) F(room) F(peak_bytes) F(budget) F(path) F(planned) F(ms_hist) F(ms_list)
  F(ms_sort) F(ms_format) F(ms_d2h) F(ms_write) F(ms_writer_busy) F(ms_total)
  printf("sizeof %zu\n", sizeof(hm_pairs_stats));
  return 0;
}
"""


def test_stats_struct_layout_and_symbols(built, tmp_path):
    """hm_pairs_stats as the header lays it out is what _lib.PairsStats binds; the new entry points are exported"""
    from smudgeplot_b200 import _lib
    src = tmp_path / "probe.c"
    src.write_text(LAYOUT_PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                       check=True).stdout.splitlines())
    names = [f for f, _ in _lib.PairsStats._fields_]
    assert names == [k for k in got if k != "sizeof"]
    for f in names:
        assert int(got[f]) == getattr(_lib.PairsStats, f).offset, f
    assert int(got["sizeof"]) == C.sizeof(_lib.PairsStats)
    L = _lib.lib()
    for sym in ("hm_scan_write_pairs", "hm_scan_pairs_hist", "hm_pair_windows"):
        assert sym in _lib.ABI_SYMBOLS and hasattr(L, sym)


def test_write_pairs_refuses_bad_arguments_without_a_device(built, tmp_path):
    """a NULL scan is refused before anything is looked at, and no file appears"""
    from smudgeplot_b200 import _lib
    L = _lib.lib()
    pm = np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)
    paths = (C.c_char_p * 1)(str(tmp_path / "o.1A1B.txt").encode())
    st = _lib.PairsStats()
    assert L.hm_scan_write_pairs(None, pm.ctypes.data, 1, paths, C.byref(st)) == -1
    assert st.planned == 0 and not os.listdir(tmp_path)

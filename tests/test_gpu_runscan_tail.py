"""Step 5 of the pass-1 kernels (csrc/hm_symm.cu runscan_kernel, runscan_dense_kernel): after a CTA barrier one
atomic per list reserves the CTA's range and every thread moves at most two staged records out.  Each table here
is scanned to the end, and pass 1's candidate list is read back: it holds no record twice (so `cand_n` equals the
number of distinct (key, lo, meta) records) and the plot equals the oracle's.  The tables put 1..255, 256..384 and
more than RS_STAGE = 384 records into a tile (the last spill to the list directly), list run heads for runs_kernel,
and take k = 40 (two key words) and the dense kernel."""
import numpy as np
import pytest
import torch

import oracle_util as ou
from smudgeplot_b200 import _lib, fastk
from smudgeplot_b200.device import DeviceTable
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _default_filter(monkeypatch):
    monkeypatch.delenv("HETMERS_BLOOM_BITS", raising=False)
    monkeypatch.delenv("HETMERS_RUNSCAN", raising=False)


def _rc(x, k):
    return synth.revcomp_left(torch.from_numpy(x.view(np.int64).copy()), k).numpy().view(np.uint64)


def _closure(vals, k, rng, cmax=60):
    """sorted unique keys = vals + their reverse complements; counts equal on both strands (k <= 32)"""
    keys = np.unique(np.concatenate([vals, _rc(vals, k)]))
    _, inv = np.unique(np.minimum(keys, _rc(keys, k)), return_inverse=True)
    return keys, rng.integers(1, cmax + 1, size=inv.max() + 1).astype(np.uint16)[inv]


def _pairs(npairs, seed, k=31):
    """npairs random keys, each with a mate one base apart in the back half (same run): a record per pair"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 1 << 62, size=npairs, dtype=np.int64).astype(np.uint64)
    base = (base >> np.uint64(64 - 2 * k)) << np.uint64(64 - 2 * k)
    pos = rng.integers(k // 2, k, size=npairs)
    mate = base ^ (rng.integers(1, 4, size=npairs).astype(np.uint64) << (np.uint64(62) - np.uint64(2) * pos.astype(np.uint64)))
    return _closure(np.concatenate([base, mate]), k, rng)


def _scan_records(k, khi, klo, cnt):
    """symmetric scan on cuda -> (plot, candidate records uint64[cand_n, 3] as (key, lo, meta), runs listed)"""
    t = DeviceTable(k, khi, cnt.to(torch.int16), keys_lo=klo).build_index(direct=False)
    assert t.check_symmetric()
    plot = t.scan("symm").cpu().numpy().copy()
    lay, w = t.symm_layout, t.symm_work
    hdr = w[lay.off_header: lay.off_header + 24].view(torch.int64).cpu().numpy()
    assert hdr[1] == 0, "status bits"
    nc = int(hdr[0])

    def words(off):
        return w[off: off + 8 * nc].view(torch.int64).cpu().numpy().view(np.uint64)
    lo = words(lay.off_cand_lo) if k > 32 else np.zeros(nc, np.uint64)
    return plot, np.stack([words(lay.off_cand_key), lo, words(lay.off_cand_meta)], axis=1), int(hdr[2])


def _check(k, keys, cnt):
    """keys uint64[n] (k <= 32) or uint64[n, 2], sorted; cnt uint16[n]"""
    kk = torch.from_numpy(np.ascontiguousarray(keys).view(np.int64)).cuda()
    khi = kk[:, 0].contiguous() if k > 32 else kk
    klo = kk[:, 1].contiguous() if k > 32 else None
    plot, rec, nr = _scan_records(k, khi, klo, torch.from_numpy(cnt.astype(np.int32)).cuda())
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    assert np.array_equal(plot.reshape(want.shape), want)
    assert len(np.unique(rec, axis=0)) == len(rec), "a candidate record was written twice"
    return len(rec), nr


@pytest.mark.parametrize("npairs", [1, 3, 121, 320])
def test_one_tile_stages_one_or_two_records_per_thread(npairs):
    """one CTA stages a few records, or more than 256 (a second record per thread): a pair gives one record,
    two when its mirror image differs at the first base after the run prefix too"""
    keys, cnt = _pairs(npairs, 500 + npairs)
    assert len(keys) <= 2048
    nc, _ = _check(31, keys, cnt)
    assert npairs <= nc <= 2 * npairs


def test_tables_of_pairs_spill_past_the_staging_area():
    """~1000 records per 2048-entry tile: the staged 384 leave in step 5, the rest went to the list directly"""
    keys, cnt = _pairs(30000, 4343)
    nc, _ = _check(31, keys, cnt)
    assert nc > (len(keys) // 2048) * 384


@pytest.mark.parametrize("route", ["sparse", "dense"])
def test_run_heads_and_records_leave_together(route, monkeypatch):
    """a run longer than the window: its head is listed for runs_kernel in step 5 next to the records"""
    monkeypatch.setenv("HETMERS_RUNSCAN", route)
    k, rng = 31, np.random.default_rng(77)
    tails = rng.choice(1 << 30, size=3000, replace=False).astype(np.uint64)
    run = ((np.uint64(int(rng.integers(0, 4 ** 15))) << np.uint64(32)) | tails) << np.uint64(64 - 2 * k)
    bk, _ = _pairs(2000, 78)
    keys, cnt = _closure(np.concatenate([run, bk]), k, rng)
    nc, nr = _check(k, keys, cnt)
    assert nc > 0 and nr > 0


def test_k40_records_carry_the_second_key_word():
    k = 40
    keys, cnt = synth.synth_table(k, 20000, 2, 0.02, 40, 4, 4040)
    nc, _ = _check(k, keys.numpy().view(np.uint64), cnt.numpy().astype(np.uint16))
    assert nc > 0


@pytest.mark.parametrize("route", ["auto", "dense"])
def test_crowded_small_k_table(route, monkeypatch):
    """a quarter of all 10-mers: the dense pass-1 kernel (auto picks it too), long runs left to runs_kernel"""
    monkeypatch.setenv("HETMERS_RUNSCAN", route)
    k, rng = 10, np.random.default_rng(1010)
    vals = rng.choice(4 ** k, size=4 ** k // 8, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _closure(vals, k, rng, 600)
    nc, _ = _check(k, keys, cnt)
    assert nc > 0

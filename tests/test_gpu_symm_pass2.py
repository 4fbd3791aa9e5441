"""Pass 2 of the symmetric scan (csrc/hm_symm.cu sweep, DESIGN.md §4a) at its edges: no candidate, fewer candidates
than one trip of the grid, many more than the grid takes at once (HETMERS_PASS2_CTAS caps the grid, so every
thread strides over many trips), extract slices whose first record is not 16-byte aligned, a crowded small-k
table where most candidates hit the Bloom filter and go through the exact check, at k <= 32 and k > 32 --
against the direct passes and the oracle."""
import numpy as np
import pytest
import torch

import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from smudgeplot_b200.device import DeviceTable
from tools import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _default_route(monkeypatch):
    monkeypatch.delenv("HETMERS_PATH", raising=False)
    monkeypatch.delenv("HETMERS_STREAM", raising=False)
    monkeypatch.delenv("HETMERS_PASS2_CTAS", raising=False)


def _scan_both(kt):
    with hetmers.Scan(kt) as sc:
        assert sc.is_symmetric()
        plot_s, st_s = sc.run("symm")
        plot_d, _ = sc.run("direct")
    assert st_s["path"] == 2
    return plot_s, plot_d


def test_a_table_without_candidates(tmp_path):
    """k-mers far apart from each other: no pair, no candidate record, an empty plot"""
    rng = np.random.default_rng(5)
    k = 31
    vals = rng.choice(1 << 40, size=300, replace=False).astype(np.uint64) << np.uint64(64 - 40)
    r = synth.revcomp_left(torch.from_numpy(vals.view(np.int64).copy()), k).numpy().view(np.uint64)
    keys = np.unique(np.concatenate([vals, r]))
    canon = np.minimum(keys, synth.revcomp_left(torch.from_numpy(keys.view(np.int64).copy()), k).numpy().view(np.uint64))
    _, inv = np.unique(canon, return_inverse=True)
    cnt = rng.integers(1, 50, size=inv.max() + 1).astype(np.uint16)[inv]
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=2, nparts=1)
    plot_s, plot_d = _scan_both(kt)
    assert plot_s.sum() == 0 and np.array_equal(plot_s, plot_d)


@pytest.mark.parametrize("ctas", [None, 1, 3])
@pytest.mark.parametrize("k,G", [(31, 1500), (21, 60_000), (40, 60_000)])
def test_plot_matches_direct_and_oracle_at_any_grid(k, G, ctas, tmp_path, monkeypatch):
    """G = 1500: fewer candidates than one trip of the grid; 60 000: tens of thousands, which one or three CTAs take
    in many trips (candidate counts are not multiples of a trip)"""
    if ctas is not None:
        monkeypatch.setenv("HETMERS_PASS2_CTAS", str(ctas))
    keys, cnt = synth.synth_table(k, G, 2, 0.02, 30.0, 4, 300 + k)
    kt = synth.write_table(str(tmp_path / "t"), k, keys, cnt, ibyte=2, nparts=2)
    kb, cn = fastk.unpack_host(kt)
    want, _ = ou.oracle_scan(kb, cn, k)
    plot_s, plot_d = _scan_both(fastk.read_ktab(str(tmp_path / "t")))
    assert np.array_equal(plot_d, want)
    assert np.array_equal(plot_s, want)


@pytest.mark.parametrize("ctas", [None, 2])
@pytest.mark.parametrize("k", [9, 10])
def test_crowded_small_k_table_mostly_bloom_hits(k, ctas, tmp_path, monkeypatch):
    """a quarter of all k-mers present: most reverse complements are in S, so nearly every trip queues exact
    checks, and the buckets they scan are long"""
    if ctas is not None:
        monkeypatch.setenv("HETMERS_PASS2_CTAS", str(ctas))
    rng = np.random.default_rng(900 + k)
    vals = rng.choice(4 ** k, size=4 ** k // 8, replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
    t = torch.from_numpy(vals.view(np.int64).copy())
    keys = np.unique(np.concatenate([vals, synth.revcomp_left(t, k).numpy().view(np.uint64)]))
    canon = np.minimum(keys, synth.revcomp_left(torch.from_numpy(keys.view(np.int64).copy()), k).numpy().view(np.uint64))
    _, inv = np.unique(canon, return_inverse=True)
    cnt = rng.integers(1, 600, size=inv.max() + 1).astype(np.uint16)[inv]
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=2, nparts=2)
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    plot_s, plot_d = _scan_both(kt)
    assert np.array_equal(plot_d, want)
    assert np.array_equal(plot_s, want)


def _records(out, count):
    n = int(count.item())
    rec = out[: n * 24].cpu().numpy().view(np.uint8).reshape(n, 24)
    return rec[np.lexsort(rec.T[::-1])]


@pytest.mark.parametrize("ctas", [None, 2])
def test_extract_slices_at_odd_starts(ctas, monkeypatch):
    """extract slices [c0, c1) with odd c0 (record arrays 8 bytes off 16-byte alignment) list together exactly
    what one slice over all candidates lists, and that is one record per unit of the plot"""
    if ctas is not None:
        monkeypatch.setenv("HETMERS_PASS2_CTAS", str(ctas))
    k = 31
    keys, cnt = synth.synth_table(k, 120_000, 2, 0.02, 30.0, 4, 77, device="cuda")
    t = DeviceTable(k, keys, cnt.to(torch.int16)).build_index(direct=False)
    assert t.check_symmetric()
    t.alloc_symm()
    t.plot.zero_()
    t.runscan()
    t.resolve()
    nc, st = t.symm_status()
    assert st == 0 and nc > 5000
    pix = torch.ones(_lib.PLOT_CELLS, dtype=torch.int16, device="cuda")
    cap = 2 * nc + 64

    def listed(c0, c1):
        out = torch.zeros(cap * 24, dtype=torch.uint8, device="cuda")
        count = torch.zeros(1, dtype=torch.int64, device="cuda")
        t.extract(pix, out, count, c0, c1)
        torch.cuda.synchronize()
        return _records(out, count)

    whole = listed(0, nc)
    assert len(whole) == int(t.plot.sum().item())
    cuts = [0, 1, 2, 3, 4098, 4099, 2049 + nc // 3, nc - 1, nc]          # odd and even starts, 1- and 2-record slices
    parts = np.concatenate([listed(a, b) for a, b in zip(cuts[:-1], cuts[1:])])
    parts = parts[np.lexsort(parts.T[::-1])]
    assert np.array_equal(parts, whole)

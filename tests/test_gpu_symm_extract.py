"""extract_kmer_pairs on the strand-symmetric scan (hm_k_symm_extract, DESIGN.md §4a): on a symmetric table
hm_scan_extract lists the pairs from the candidates of the symmetric run.  Its list must equal the direct
route's (HETMERS_PATH=direct) record for record, hold one record per labelled isolated pair of the plot, and
reproduce the golden and reference pair files.  The listing rule itself is pinned on the CPU in
test_symm_extract_rule.py."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from tools import synth

pytestmark = pytest.mark.gpu

SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _default_route_and_budget(monkeypatch):
    monkeypatch.delenv("HETMERS_PATH", raising=False)
    monkeypatch.delenv("HETMERS_STREAM", raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)


def _golden(name):
    return os.path.join(GOLDEN, name, name)


def read_sma(path):
    """pixel -> 1-based smudge index, smudges numbered in order of first appearance (as the executable does)"""
    pix = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    order = []
    with open(path) as f:
        next(f)
        for ln in f:
            m, rest, _, lab = ln.split()[:4]
            m, s = int(m), int(m) + int(rest)
            if lab not in order:
                order.append(lab)
            pix[s, m] = order.index(lab) + 1
    return pix


def direct_list(kt, pix, monkeypatch):
    monkeypatch.setenv("HETMERS_PATH", "direct")
    with hetmers.Scan(kt) as sc:
        plot, st = sc.run()
        rec = sc.extract(pix)
    monkeypatch.delenv("HETMERS_PATH")
    assert st["path"] == 1
    return plot, rec


def launches(sc):
    """kernels the scan has launched so far (a run reports the running total)"""
    return sc.run()[1]["kernel_launches"]


# ------------------------------------------------------------------ goldens ------------------------

@pytest.mark.parametrize("name", SMA_GOLDENS)
def test_golden_pair_list_is_the_same_on_both_routes(name, monkeypatch):
    kt = fastk.read_ktab(_golden(name))
    pix = read_sma(_golden(name) + ".sma")
    with hetmers.Scan(kt) as sc:
        plot, st = sc.run()
        rec = sc.extract(pix)
        assert st["path"] == 2 and sc.is_symmetric()                 # listed from the symmetric run
    _, want = direct_list(kt, pix, monkeypatch)
    assert len(rec) > 0 and len(rec) == int(plot[pix > 0].sum())
    assert np.array_equal(rec, want)


@pytest.mark.parametrize("route", ["auto", "direct", "symm"])
@pytest.mark.parametrize("name", SMA_GOLDENS)
def test_executable_writes_golden_pair_files_on_every_route(name, route, golden_meta, tmp_path, monkeypatch):
    if route != "auto":
        monkeypatch.setenv("HETMERS_PATH", route)
    out = str(tmp_path / "kp")
    hetmers.run_extract(_golden(name), _golden(name) + ".sma", o=out, t=4, e=golden_meta[name]["e"])
    d, pre = os.path.join(GOLDEN, name), name + ".pairs."
    want = {f[len(pre):-4]: open(os.path.join(d, f)).read().splitlines()
            for f in sorted(os.listdir(d)) if f.startswith(pre)}
    assert ou.sorted_pair_files(out) == want


# ------------------------------------------------------------------ seeded tables ------------------

def seeded_table(k, seed, path):
    """a symmetric table of >= 2e5 entries (both strands of a diploid genome); counts remapped by value, which
    keeps count(x) = count(rc x): many ties, and a third of the counts 498..502, so that pairs sum to 996..1004
    (999 / 1000 / 1001 among them)"""
    G = synth.calibrate_G(k, 250_000, 2, 0.02, 30.0, 4)
    keys, cnt = synth.synth_table(k, G, 2, 0.02, 30.0, 4, seed)
    c = cnt.numpy().astype(np.int64)
    c = np.where(c % 3 == 0, 498 + (c // 3) % 5, c)
    kt = fastk.write_ktab(path, k, synth.keys_to_u64_numpy(keys), c.astype(np.uint16), ibyte=2, nparts=2)
    assert kt.nels >= 200_000
    return kt


@pytest.mark.parametrize("k", [11, 16, 21, 31, 32, 33, 40, 64])
def test_seeded_tables_list_the_same_pairs_on_both_routes(k, tmp_path, monkeypatch):
    kt = seeded_table(k, 100 + k, str(tmp_path / "t"))
    rng = np.random.default_rng(k)
    with hetmers.Scan(kt) as sc:
        plot, st = sc.run()
        assert st["path"] == 2
        nz = np.flatnonzero(plot.reshape(-1) > 0)
        assert 0 < nz.size < 65535
        sums = set(np.nonzero(plot.sum(axis=1))[0].tolist())
        assert {999, 1000} <= sums                                    # (1001 is past SMAX: no pair)
        assert plot[np.arange(0, 1001, 2), np.arange(0, 1001, 2) // 2].sum() > 0     # count ties
        distinct = np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)
        distinct[nz] = np.arange(1, nz.size + 1)                     # a label per pixel: a swapped sum/min shows
        sparse = np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)
        pick = rng.random(_lib.PLOT_CELLS) < 0.3
        sparse[pick] = rng.integers(1, 6, size=int(pick.sum()))
        none = np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)
        pixmaps = [p.reshape(_lib.SMAX + 1, _lib.PLOT_W) for p in (distinct, sparse, none)]
        got = [sc.extract(p) for p in pixmaps]
        assert sc.is_symmetric()
    monkeypatch.setenv("HETMERS_PATH", "direct")
    with hetmers.Scan(kt) as sc:
        plot_d, _ = sc.run()
        want = [sc.extract(p) for p in pixmaps]
    assert np.array_equal(plot, plot_d)
    for p, a, b in zip(pixmaps, got, want):
        assert len(a) == int(plot[p > 0].sum())
        assert np.array_equal(a, b)
    assert len(got[0]) > 0 and len(got[2]) == 0
    if k % 2 == 1:                                                    # middle-base pairs: listed once
        assert np.any(got[0]["pos"] == k // 2)


@pytest.mark.parametrize("case", range(2))
def test_reference_pair_digests_on_the_symmetric_route(case, tmp_path, monkeypatch):
    from test_gpu_parity import EXTRACT_CASES, write_labelled_sma
    k, G, ploidy, seed, L = EXTRACT_CASES[case]
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed, device="cuda")
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
    sma = str(tmp_path / "ann.sma")
    with hetmers.Scan(kt) as sc:
        plot, st = sc.run("symm")
        pix, _ = write_labelled_sma(plot, sma)
    monkeypatch.setenv("HETMERS_PATH", "symm")
    out = str(tmp_path / "kp")
    hetmers.run_extract(name, sma, o=out, t=4, e=L)
    assert ou.pair_digests(ou.sorted_pair_files(out)) == ou.reference_pair_digests(k, seed)


# ------------------------------------------------------------------ scan states --------------------

@pytest.fixture(scope="module")
def state_table(tmp_path_factory):
    return seeded_table(31, 7, str(tmp_path_factory.mktemp("st") / "t"))


def test_extract_without_a_run_then_twice(state_table, monkeypatch):
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    _, want = direct_list(state_table, pix, monkeypatch)
    with hetmers.Scan(state_table) as sc:
        first = sc.extract(pix)                                      # no run: a symmetric run is done first
        second = sc.extract(pix)
        assert sc.is_symmetric()
    assert len(want) > 0 and np.array_equal(first, want) and np.array_equal(second, want)


def test_extract_after_a_direct_run(state_table, monkeypatch):
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    _, want = direct_list(state_table, pix, monkeypatch)
    with hetmers.Scan(state_table) as sc:
        sc.run("symm")
        sc.run("direct")
        assert np.array_equal(sc.extract(pix), want)
        assert sc.is_symmetric()


def test_extract_after_gpu_conditioning(golden_meta, monkeypatch):
    c = golden_meta["_conditioning"]["untrimmed"]
    kt = fastk.read_ktab(os.path.join(GOLDEN, "conditioning", "untrimmed"))
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    lists = {}
    for route in ("auto", "direct"):
        if route == "direct":
            monkeypatch.setenv("HETMERS_PATH", "direct")
        with hetmers.Scan(kt) as sc:
            sc.run()                                                 # results of the unconditioned table ...
            trim, symm = sc.examine(c["e"])
            assert not trim and symm
            sc.condition(c["e"], True, False)                        # ... are dropped by the conditioning
            plot, _ = sc.run()
            lists[route] = sc.extract(pix)
    assert len(lists["auto"]) == int(plot.sum()) > 0
    assert np.array_equal(lists["auto"], lists["direct"])


def test_a_small_budget_lists_in_many_slices(state_table, monkeypatch):
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    with hetmers.Scan(state_table) as sc:
        incore = sc.residency()[1]
        l0 = launches(sc)
        want = sc.extract(pix)
        assert launches(sc) - l0 == 3 + 1                            # a run, then one slice with the default budget
    with hetmers.Scan(state_table, device_budget=incore + _lib.EXTRACT_MIN_BYTES + 4096) as sc:
        assert not sc.residency()[0]
        l0 = launches(sc)
        got = sc.extract(pix)
        slices = launches(sc) - l0 - 3
    assert slices >= 5 and len(got) > 0
    assert np.array_equal(got, want)


def test_a_budget_below_the_floor_is_refused_before_any_launch(state_table):
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    with hetmers.Scan(state_table) as ref:
        incore = ref.residency()[1]
        want_plot, _ = ref.run()
    with hetmers.Scan(state_table, device_budget=incore + 4096) as sc:
        plot, _ = sc.run()
        l0 = launches(sc)
        with pytest.raises(_lib.HetmersError) as ei:
            sc.extract(pix)
        assert ei.value.code == -3 and "device budget" in str(ei.value)
        l1 = launches(sc)
        plot2, _ = sc.run()                                          # the table stays usable
    assert l1 - l0 == 3                                              # (only the run between: nothing was listed)
    assert np.array_equal(plot, want_plot) and np.array_equal(plot2, want_plot)


def test_forced_symmetric_route_on_an_asymmetric_table_is_refused(golden_meta, monkeypatch):
    kt = fastk.read_ktab(os.path.join(GOLDEN, "conditioning", "asymmetric"))
    monkeypatch.setenv("HETMERS_PATH", "symm")
    with hetmers.Scan(kt) as sc:
        assert not sc.is_symmetric()
        with pytest.raises(_lib.HetmersError) as run_err:
            sc.run()
        with pytest.raises(_lib.HetmersError) as ext_err:
            sc.extract(np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16))
    assert ext_err.value.code == run_err.value.code == -1
    assert str(ext_err.value) == str(run_err.value)

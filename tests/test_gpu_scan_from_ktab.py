"""GPU tests of Scan.from_ktab(src, L): a raw FastK table scanned in one process as hetmers -e<L> scans it, conditioned
on the way in -- in place when the source is in core and that fits the device budget, else into host memory
(hm_scan_condition_host) and scanned from there, in or out of core (DESIGN.md §4d, §6; run with -m gpu).  The plot
must be the reference binary's on the conditioned table, the host table the records and index condition_table
writes, and the pair list and files those of a scan over that written table."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import oracle_util as ou
from smudgeplot_b200 import _lib, fastk, hetmers
from test_gpu_condition_files import output_hist, table_u64
from test_gpu_condition_files_gpus import budget_for_ranges
from test_gpu_stream_condition_dist import CONDITIONING_CASES, raw_table

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch, built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"
    for var in ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK", "HETMERS_DEVICE_BUDGET", "HETMERS_GPUS"):
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)
    _lib.lib().hm_set_condition_gpus(1)


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def gives_back(cycle):
    cycle()
    before = free_bytes()
    cycle()
    assert free_bytes() == before


def host_table_equals_files(sc, written):
    """the scan's host table: the records and stub index condition_table wrote, as one part"""
    kt = fastk.read_ktab(written)
    assert sc.kt.nparts == 1 and sc.kt.nels == kt.nels and sc.kt.ibyte == kt.ibyte and sc.kt.minval == kt.minval
    assert sc.kt.records[0].tobytes() == kt.all_records().tobytes()
    assert np.array_equal(sc.kt.index, kt.index)


def file_digest(name):
    kt = fastk.read_ktab(name)
    paths = [fastk.stub_path(name)] + [fastk.part_path(name, p) for p in range(1, kt.nparts + 1)]
    return [hashlib.sha256(open(p, "rb").read()).hexdigest() for p in paths]


# ------------------------------------------------------------------ stored reference runs, streamed ---------------

@pytest.fixture(scope="module")
def reference_tables(tmp_path_factory, built):
    """the raw tables of the stored reference runs and a k = 17 one: (src, k, L, .smu wanted, condition_table's
    output)"""
    d = tmp_path_factory.mktemp("refs")
    out = []
    for k, G, ploidy, seed, L in CONDITIONING_CASES + [(17, 40000, 2, 36, 8)]:
        src = raw_table(d, k, G, ploidy, seed)
        if k == 17:
            smu = open(hetmers.hetmers(src, o=str(d / f"incore_k{k}"), L=L)).read()
        else:
            smu = ou.reference_smu("conditioned", k, seed)
        dst = str(d / f"cond_k{k}")
        assert hetmers.condition_table(src, dst, L) is not None
        out.append((src, k, L, smu, dst))
    return out


@pytest.mark.parametrize("config", ["dev0", "dev00", "gpus2"])
def test_stored_reference_runs_streamed(config, reference_tables, monkeypatch):
    if config == "gpus2" and _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    kw = {"dev0": {"devices": [0]}, "dev00": {"devices": [0, 0]}, "gpus2": {"gpus": 2}}[config]
    shards = 1 if config == "dev0" else 2
    monkeypatch.setenv("HETMERS_STREAM", "1")
    for src, k, L, smu, dst in reference_tables:
        n_out = fastk.read_ktab(dst).nels
        monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(max(32, n_out // (8 * shards))))
        with hetmers.Scan.from_ktab(src, L, **kw) as sc:
            st = sc.stats["condition"]
            assert st["route"] == "host" and st["steps"] == ["trim", "symmetrise"], st
            assert st["gpus"] == shards and st["nels_out"] == n_out
            assert st["host_bytes"] == st["bytes_written"] == sc.kt.records[0].nbytes + sc.kt.index.nbytes
            assert max(st["gpu_peak_bytes"]) == st["peak_bytes"] <= st["budget_bytes"]
            host_table_equals_files(sc, dst)
            plot, _ = sc.run()
            streamed, peak, chunks = sc.residency()
            assert hetmers.smu_text(plot) == smu, (k, config)
            assert streamed and chunks >= 4 * shards, (k, chunks)


# ------------------------------------------------------------------ raw goldens: the route, pairs and pair files ---

@pytest.mark.parametrize("name", ["untrimmed", "asymmetric"])
def test_raw_goldens_take_each_route(name, golden_meta, tmp_path, monkeypatch):
    from test_gpu_parity import write_labelled_sma
    from test_gpu_scan_write_pairs import files
    src = os.path.join(GOLDEN, "conditioning", name)
    e = golden_meta["_conditioning"][name]["e"]
    dst = str(tmp_path / "cond")
    hetmers.condition_table(src, dst, e)
    with hetmers.Scan(fastk.read_ktab(dst)) as ref:
        plot, _ = ref.run()
        sma = str(tmp_path / "x.sma")
        write_labelled_sma(plot, sma)
        pix, labels = hetmers.read_sma(sma)
        pairs = ref.extract(pix)
        ref.write_pairs(sma, str(tmp_path / "ref"))
    assert len(pairs) > 0
    hetmers.run_extract(dst, sma, o=str(tmp_path / "exe"))
    want_files = files(str(tmp_path / "exe"), labels)
    assert files(str(tmp_path / "ref"), labels) == want_files

    # a budget in-place conditioning fits: the pair list and files of a scan over condition_table's output
    with hetmers.Scan.from_ktab(src, e) as sc:
        st = sc.stats["condition"]
        assert st["route"] == "in_place" and st["host_bytes"] == 0 and st["nels_out"] == fastk.read_ktab(dst).nels
        assert np.array_equal(sc.run()[0], plot)
        assert sc.extract(pix).tobytes() == pairs.tobytes()
        sc.write_pairs(sma, str(tmp_path / "got"))
    assert files(str(tmp_path / "got"), labels) == want_files

    # streamed: into host memory, the same plot, and extraction refused as on any streamed scan
    monkeypatch.setenv("HETMERS_STREAM", "1")
    with hetmers.Scan.from_ktab(src, e) as sc:
        st = sc.stats["condition"]
        assert st["route"] == "host" and st["host_bytes"] > 0, st
        assert st["peak_bytes"] <= st["budget_bytes"]
        host_table_equals_files(sc, dst)
        assert np.array_equal(sc.run()[0], plot)
        assert sc.residency()[0]
        with pytest.raises(_lib.HetmersError) as ei:
            sc.extract(pix)
        assert ei.value.code == -6


# ------------------------------------------------------------------ the host route from an in-core source --------

def refused_in_place(src, L, b):
    """1 if under device budget b the source is in core and hm_scan_condition refuses it (the route rule's test)"""
    with hetmers.Scan(fastk.read_ktab(src), device_budget=b) as probe:
        if probe.residency()[0]:
            return False
        trim, symm = probe.examine(L)
        try:
            probe.condition(L, not trim, not symm)
        except _lib.HetmersError as e:
            assert e.code == -3
            return True
        return False


def test_in_core_source_that_in_place_does_not_fit_takes_the_host_route(tmp_path):
    """an in-core source under a device budget in-place conditioning does not fit: reopened streamed, conditioned
    into host memory with the whole budget, and scanned (streamed: the conditioned table's in-core scan is larger
    than the in-place working set whenever the source itself is in core, so no budget leaves it in core).  The
    table is large enough (2e6 entries) for that budget to hold the host route's fixed part and one range."""
    L = 8
    src = raw_table(tmp_path, 31, 1400000, 2, 41, ibyte=2)
    dst = str(tmp_path / "cond")
    hetmers.condition_table(src, dst, L)
    with hetmers.Scan(fastk.read_ktab(src)) as s0:
        incore_src = s0.residency()[1]
    with hetmers.Scan(fastk.read_ktab(dst)) as ref:
        plot, _ = ref.run()
    budget = None                       # the largest budget in-place conditioning does not fit (to 1 MiB)
    for b in range(incore_src, 3 * incore_src, 1 << 20):
        if refused_in_place(src, L, b):
            budget = b
        elif budget is not None:
            break
    _lib.lib().hm_set_device_budget(0)
    assert budget is not None, f"no budget from {incore_src} to {3 * incore_src} refuses in-place conditioning"
    with hetmers.Scan.from_ktab(src, L, device_budget=budget) as sc:
        st = sc.stats["condition"]
        assert st["route"] == "host" and st["steps"] == ["trim", "symmetrise"], st
        assert st["peak_bytes"] <= st["budget_bytes"] <= budget
        host_table_equals_files(sc, dst)
        assert np.array_equal(sc.run()[0], plot)
        streamed, peak, _ = sc.residency()
        assert 0 < peak <= budget


def test_in_core_scan_of_the_host_table(golden_meta, tmp_path, monkeypatch):
    """the table hm_scan_condition_host makes, scanned in core: the plot, pair list and pair files of a scan over
    condition_table's output and of extract_kmer_pairs on it; the table outlives close() while its arrays are held"""
    from test_gpu_parity import write_labelled_sma
    from test_gpu_scan_write_pairs import files
    for name in ("untrimmed", "asymmetric"):
        src = os.path.join(GOLDEN, "conditioning", name)
        e = golden_meta["_conditioning"][name]["e"]
        dst = str(tmp_path / f"cond_{name}")
        hetmers.condition_table(src, dst, e)
        with hetmers.Scan(fastk.read_ktab(dst)) as ref:
            plot, _ = ref.run()
            sma = str(tmp_path / f"{name}.sma")
            write_labelled_sma(plot, sma)
            pix, labels = hetmers.read_sma(sma)
            pairs = ref.extract(pix)
        hetmers.run_extract(dst, sma, o=str(tmp_path / f"exe_{name}"))
        monkeypatch.setenv("HETMERS_STREAM", "1")
        with hetmers.Scan(fastk.read_ktab(src)) as s0:
            trim, symm = s0.examine(e)
            ht, cs = C.POINTER(_lib.HostTable)(), _lib.ConditionStats()
            _lib.check(_lib.lib().hm_scan_condition_host(s0._h, e, int(not trim), int(not symm), -1, C.byref(ht),
                                                         C.byref(cs)))
        monkeypatch.delenv("HETMERS_STREAM")
        with hetmers.Scan(None, _owned=hetmers._OwnedTable(ht)) as sc:
            assert not sc.residency()[0]
            host_table_equals_files(sc, dst)
            assert np.array_equal(sc.run()[0], plot)
            assert sc.extract(pix).tobytes() == pairs.tobytes()
            sc.write_pairs(sma, str(tmp_path / f"got_{name}"))
            kt = sc.kt
        assert files(str(tmp_path / f"got_{name}"), labels) == files(str(tmp_path / f"exe_{name}"), labels)
        assert sc.kt is None
        want = fastk.read_ktab(dst)
        assert kt.records[0].tobytes() == want.all_records().tobytes() and np.array_equal(kt.index, want.index)


# ------------------------------------------------------------------ nothing to condition ---------------------------

def test_no_conditioning_scans_the_source(golden_meta):
    src = os.path.join(GOLDEN, "dip_k21", "dip_k21")
    want = open(src + ".smu").read()
    for L in (golden_meta["dip_k21"]["e"], None):
        with hetmers.Scan.from_ktab(src, L) as sc:
            st = sc.stats["condition"]
            assert st["route"] == "none" and st["steps"] == [] and st["host_bytes"] == 0
            assert sc.kt.name is not None
            assert hetmers.smu_text(sc.run()[0]) == want


# ------------------------------------------------------------------ several passes, budgets, refusals -------------

def test_small_device_budget_conditions_in_several_passes(tmp_path, monkeypatch):
    """a device budget leaving at least 3 range passes: the same host table and plot, the device peaks within it"""
    k, G, ploidy, seed, L = CONDITIONING_CASES[1]
    src = raw_table(tmp_path, k, G, ploidy, seed)
    dst = str(tmp_path / "cond")
    hetmers.condition_table(src, dst, L)
    smu = ou.reference_smu("conditioned", k, seed)
    ku, cn, kt = table_u64(src)
    b = budget_for_ranges(output_hist(ku, cn, k, L, True, True), kt.nels, k, kt.ibyte, 4, True)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    big = 8 << 30
    with hetmers.Scan.from_ktab(src, L, device_budget=big) as sc:
        held = big - sc.stats["condition"]["budget_bytes"]      # what the streamed source scan holds
        assert sc.stats["condition"]["ranges"] == 1
    for kw in ({"devices": [0]}, {"devices": [0, 0]}):
        with hetmers.Scan.from_ktab(src, L, device_budget=b + held, **kw) as sc:
            st = sc.stats["condition"]
            assert st["route"] == "host" and st["ranges"] >= 3 and st["budget_bytes"] == b, st
            assert max(st["gpu_peak_bytes"]) == st["peak_bytes"] <= st["budget_bytes"]
            host_table_equals_files(sc, dst)
            assert hetmers.smu_text(sc.run()[0]) == smu
            streamed, peak, chunks = sc.residency()
            assert streamed and 0 < peak <= b + held


def test_refusals_give_back_memory_and_leave_the_source(tmp_path, monkeypatch):
    """a host budget below the conditioned table: HetmersError -3 naming both sizes, before any range pass; device
    memory given back and the source files untouched; a scan conditioned in place is refused (HM_EINVAL)"""
    src = raw_table(tmp_path, 31, 80000, 3, 32)
    before = file_digest(src)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    tiny = 1 << 20

    def cycle():
        with pytest.raises(_lib.HetmersError) as ei:
            hetmers.Scan.from_ktab(src, 12, host_budget=tiny)
        msg = str(ei.value)
        assert ei.value.code == -3 and "host bytes" in msg and f"host budget of {tiny}" in msg, msg
        need = int(msg.split(" needs ")[1].split()[0])
        assert need > tiny
    gives_back(cycle)
    assert file_digest(src) == before

    # the refusal comes before any range pass
    with hetmers.Scan(fastk.read_ktab(src)) as sc:
        out, cs = C.POINTER(_lib.HostTable)(), _lib.ConditionStats()
        assert _lib.lib().hm_scan_condition_host(sc._h, 12, 1, 1, tiny, C.byref(out), C.byref(cs)) == -3 and not out
        assert cs.ranges == 0 and cs.nels_out == 0 and cs.bytes_written == 0

    monkeypatch.delenv("HETMERS_STREAM")
    with hetmers.Scan(fastk.read_ktab(src)) as sc:
        sc.condition(12, True, True)
        out = C.POINTER(_lib.HostTable)()
        assert _lib.lib().hm_scan_condition_host(sc._h, 12, 1, 1, -1, C.byref(out), None) == -1 and not out
    with hetmers.Scan.from_ktab(src, 12, host_budget=1 << 40) as sc:
        assert sc.stats["condition"]["route"] == "in_place"
    assert file_digest(src) == before

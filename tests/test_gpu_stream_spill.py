"""Streamed scans whose candidate records and S list go to host memory (hm_set_list_host_budget, DESIGN.md §4c,
*Lists in host memory*): pass 1 flushes the lists to host arrays when they run out of device room, pass 2 parks
every Bloom hit and answers the queries against S partitions uploaded from the host.  The plots must be what the
in-core scan, the goldens and the stored reference runs give.

Spilling is forced by the budget where a table's lists outgrow it (the list_table of test_gpu_memory.py), and on
the small goldens, whose lists fit any budget that holds a chunk, by HETMERS_LIST_ROOM (device bytes the lists may
take before a flush).  HETMERS_SPILL_ROOM shrinks pass 2's room, for many rounds, and HETMERS_SPILL_PART its
partitions: with one key each, every query found in S is a partition's first key."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import oracle_util as ou
from conftest import GOLDEN, golden_cases
from smudgeplot_b200 import _lib, fastk, hetmers
from test_gpu_stream import budget_for_chunk
from tools import synth

pytestmark = pytest.mark.gpu

CAP = 1 << 36                  # host bytes: far more than any table here needs
LIST_ROOM = 1                  # device list bytes before a flush: every chunk flushes
ENV = ("HETMERS_PATH", "HETMERS_STREAM", "HETMERS_STREAM_CHUNK", "HETMERS_LIST_ROOM", "HETMERS_SPILL_ROOM",
       "HETMERS_SPILL_PART", "HETMERS_NO_POOL")


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    yield
    _lib.lib().hm_set_device_budget(0)
    _lib.lib().hm_set_list_host_budget(0)


def _golden(name):
    return os.path.join(GOLDEN, name, name)


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def gives_back(cycle):
    cycle()
    before = free_bytes()
    cycle()
    assert free_bytes() == before


def incore_plot(kt):
    with hetmers.Scan(kt) as sc:
        assert not sc.residency()[0]
        return sc.run()[0]


def spilled_scan(kt, monkeypatch, chunks=8, devices=(0,), list_room=LIST_ROOM, spill_room=None, cap=CAP, part=None):
    """the streamed run of kt in about `chunks` chunks per shard with its lists in host memory
    -> (plot, spill_stats, residency, budget)"""
    chunk = max(256, -(-kt.nels // (chunks * len(devices))))
    budget = budget_for_chunk(kt.nels, kt.kmer, kt.ibyte, chunk) + (16 << 20)   # + pass 2's room
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    if list_room is not None:
        monkeypatch.setenv("HETMERS_LIST_ROOM", str(list_room))
    if spill_room is not None:
        monkeypatch.setenv("HETMERS_SPILL_ROOM", str(spill_room))
    if part is not None:
        monkeypatch.setenv("HETMERS_SPILL_PART", str(part))
    with hetmers.Scan(kt, devices=list(devices), device_budget=budget, list_host_budget=cap) as sc:
        plot, st = sc.run()
        sp, res = sc.spill_stats(), sc.residency()
    for var in ENV:
        monkeypatch.delenv(var, raising=False)
    assert st["path"] == 2 and res[0] and res[1] <= budget
    assert sp["spilled"] and sp["flushes"] >= len(devices) and sp["host_peak_bytes"] <= cap
    return plot, sp, res, budget


def floor_room(n_cand, n_s, k):
    """the smallest pass 2 room hm_spill_plan accepts for these list sizes"""
    lay, lo, hi = _lib.SpillLayout(), 1, 1 << 34
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.lib().hm_spill_plan(n_cand, n_s, k, mid, C.byref(lay)) == 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


# ------------------------------------------------------------------ the table one budget cannot hold ----------

@pytest.fixture(scope="module")
def list_table(tmp_path_factory, built):
    """test_gpu_memory's list_table: 1e6 entries at k = 31, chunks of nels / 32, and the budget at which run()
    refuses with "list needs" unless the lists may go to host memory"""
    keys, cnt = synth.synth_table(31, 1_000_000, 2, 0.01, 40, 8, 131, device="cuda")
    kt = synth.write_table(str(tmp_path_factory.mktemp("lt") / "t"), 31, keys, cnt, ibyte=2, nparts=2)
    chunk = -(-kt.nels // 32)
    os.environ["HETMERS_STREAM"], os.environ["HETMERS_STREAM_CHUNK"] = "1", str(chunk)
    try:
        with hetmers.Scan(kt, devices=[0] * 4, device_budget=1 << 34) as sc:
            sc.run()
            budget = int(sc.residency()[1] * 1.05)
    finally:
        del os.environ["HETMERS_STREAM"], os.environ["HETMERS_STREAM_CHUNK"]
        _lib.lib().hm_set_device_budget(0)
    return kt, chunk, budget, incore_plot(kt)


def test_list_table_spills_where_the_run_refuses(list_table, monkeypatch):
    kt, chunk, budget, want = list_table
    monkeypatch.setenv("HETMERS_NO_POOL", "1")
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    with hetmers.Scan(kt, devices=[0], device_budget=budget) as sc:
        with pytest.raises(_lib.HetmersError) as ei:
            sc.run()
        assert ei.value.code == -3 and "list needs" in str(ei.value)
    cap = 64 << 20
    seen = {}

    def cycle():
        with hetmers.Scan(kt, devices=[0], device_budget=budget, list_host_budget=cap) as sc:
            plot, st = sc.run()
            seen.update(plot=plot, sp=sc.spill_stats(), res=sc.residency())
    gives_back(cycle)
    assert np.array_equal(seen["plot"], want)
    sp, res = seen["sp"], seen["res"]
    assert res[0] and res[1] <= budget
    assert sp["spilled"] and sp["flushes"] >= 2 and 0 < sp["host_peak_bytes"] <= cap and sp["rounds"] >= 1
    assert sp["d2h_bytes"] == sp["host_peak_bytes"] and sp["h2d_bytes"] > 0 and sp["partitions"] >= 1


@pytest.mark.parametrize("k", [31, 40])
def test_many_rounds_and_partitions(k, tmp_path, monkeypatch):
    """pass 2 at the plan's floor (slices of ~HM_SPILL_MIN candidates: many rounds) with one S key per partition,
    so that every query found in S equals its partition's first key"""
    keys, cnt = synth.synth_table(k, 400_000, 4, 0.02, 60, 8, 150 + k, device="cuda")
    kt = synth.write_table(str(tmp_path / "t"), k, keys, cnt, ibyte=2, nparts=2)
    del keys, cnt
    want = incore_plot(kt)
    room = floor_room(kt.nels // 4, kt.nels // 2, k)
    plot, sp, _, _ = spilled_scan(kt, monkeypatch, chunks=16, list_room=1 << 20, spill_room=room, part=1)
    assert np.array_equal(plot, want)
    assert sp["rounds"] >= 3 and sp["partitions"] >= 3 and sp["first_key_queries"] >= 1, sp
    assert sp["slice"] <= 2 * _lib.SPILL_MIN and sp["part"] == 1


# ------------------------------------------------------------------ goldens and stored reference runs ---------

@pytest.mark.parametrize("name", golden_cases())
def test_goldens_spilled(name, monkeypatch):
    kt = fastk.read_ktab(_golden(name))
    plot, sp, _, _ = spilled_scan(kt, monkeypatch)
    assert hetmers.smu_text(plot) == open(_golden(name) + ".smu").read()
    assert sp["flushes"] >= 2 and sp["rounds"] >= 1, sp


from test_gpu_parity import MEDIUM_CASES  # noqa: E402


@pytest.mark.parametrize("k,target,ploidy,het,cov,L,seed,ref_threads", MEDIUM_CASES)
def test_stored_reference_runs_spilled(k, target, ploidy, het, cov, L, seed, ref_threads, tmp_path, monkeypatch):
    G = synth.calibrate_G(k, target, ploidy, het, cov, L)
    keys, cnt = synth.synth_table(k, G, ploidy, het, cov, L, seed, device="cuda")
    name = str(tmp_path / "t")
    synth.write_table(name, k, keys, cnt, ibyte=3, nparts=4)
    del keys, cnt
    plot, sp, _, _ = spilled_scan(fastk.read_ktab(name, mmap=True), monkeypatch, chunks=16, list_room=1 << 20)
    assert hetmers.smu_text(plot) == ou.reference_smu("medium", k, seed)
    assert sp["flushes"] >= 2 and sp["rounds"] >= 1, sp


# ------------------------------------------------------------------ shards ------------------------------------

@pytest.mark.parametrize("shards", [2, 3])
@pytest.mark.parametrize("name", ["dip_k21", "trip_k31", "dip_k40"])
def test_shards_spilled(name, shards, monkeypatch):
    kt = fastk.read_ktab(_golden(name))
    plot, sp, _, _ = spilled_scan(kt, monkeypatch, chunks=4, devices=[0] * shards)
    assert hetmers.smu_text(plot) == open(_golden(name) + ".smu").read()


def test_shards_spilled_with_empty_shards(tmp_path, monkeypatch):
    """k = 3, every k-mer: 4 runs of 16 entries, so of 5 shards one is empty"""
    from test_gpu_symm import _symmetric_closure
    k = 3
    rng = np.random.default_rng(5150)
    vals = np.arange(4 ** k, dtype=np.uint64) << np.uint64(64 - 2 * k)
    keys, cnt = _symmetric_closure(vals, k, rng, 300)
    kt = fastk.write_ktab(str(tmp_path / "t"), k, keys, cnt, ibyte=1, nparts=1)
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
    for G in (3, 5):
        plot, sp, _, _ = spilled_scan(kt, monkeypatch, chunks=1, devices=[0] * G)
        assert np.array_equal(plot, want), G


# ------------------------------------------------------------------ a cap that is not needed -----------------

def test_cap_set_and_lists_fit(monkeypatch):
    kt = fastk.read_ktab(_golden("trip_k31"))
    chunk = -(-kt.nels // 6)
    budget = budget_for_chunk(kt.nels, kt.kmer, kt.ibyte, chunk) + (16 << 20)
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    got = []
    for cap in (0, CAP):
        with hetmers.Scan(kt, device_budget=budget, list_host_budget=cap) as sc:
            plot, _ = sc.run()
            got.append((plot, sc.residency(), sc.spill_stats()))
    (p0, r0, s0), (p1, r1, s1) = got
    assert np.array_equal(p0, p1) and r0 == r1
    assert not s1["spilled"] and s1["flushes"] == 0 and s1["host_peak_bytes"] == 0


# ------------------------------------------------------------------ refusals ----------------------------------

def test_cap_too_small_is_refused_and_gives_back(list_table, monkeypatch):
    kt, chunk, budget, want = list_table
    monkeypatch.setenv("HETMERS_NO_POOL", "1")
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    tiny = 100_000

    def cycle():
        with hetmers.Scan(kt, devices=[0], device_budget=budget, list_host_budget=tiny) as sc:
            with pytest.raises(_lib.HetmersError) as ei:
                sc.run()
            msg = str(ei.value)
            assert ei.value.code == -3 and "host memory" in msg and f"list host budget is {tiny} bytes" in msg, msg
    gives_back(cycle)
    with hetmers.Scan(kt, devices=[0], device_budget=budget, list_host_budget=tiny) as sc:
        with pytest.raises(_lib.HetmersError):
            sc.run()
        _lib.lib().hm_set_list_host_budget(CAP)
        plot, _ = sc.run()
        assert sc.spill_stats()["spilled"]
    assert np.array_equal(plot, want)


def test_asymmetric_table_spilled_is_refused(tmp_path, monkeypatch):
    keys, cnt = synth.synth_table(31, 30000, 2, 0.02, 40, 4, 321)
    ku = synth.keys_to_u64_numpy(keys)
    cu = cnt.numpy().astype(np.uint16)
    keep = np.ones(len(ku), dtype=bool)
    keep[len(ku) // 3] = False
    kt = fastk.write_ktab(str(tmp_path / "asym"), 31, ku[keep], cu[keep], ibyte=3, nparts=2)
    with pytest.raises(_lib.HetmersError) as ei:
        spilled_scan(kt, monkeypatch)
    assert ei.value.code == -6 and "not strand-symmetric" in str(ei.value)


# ------------------------------------------------------------------ from_ktab and the executable --------------

@pytest.mark.parametrize("name", ["untrimmed", "asymmetric"])
def test_from_ktab_host_route_spilled(name, golden_meta, tmp_path, monkeypatch):
    src = os.path.join(GOLDEN, "conditioning", name)
    e = golden_meta["_conditioning"][name]["e"]
    dst = str(tmp_path / "cond")
    hetmers.condition_table(src, dst, e)
    with hetmers.Scan(fastk.read_ktab(dst)) as ref:
        want, _ = ref.run()
    monkeypatch.setenv("HETMERS_STREAM", "1")
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", "1024")
    monkeypatch.setenv("HETMERS_LIST_ROOM", str(LIST_ROOM))
    with hetmers.Scan.from_ktab(src, e, list_host_budget=CAP) as sc:
        assert sc.stats["condition"]["route"] == "host"
        plot, _ = sc.run()
        sp = sc.spill_stats()
        assert sc.residency()[0]
    assert sp["spilled"] and sp["flushes"] >= 2
    assert np.array_equal(plot, want)


@pytest.mark.parametrize("name", ["dip_k21", "dip_k40"])
def test_executable_spills_to_the_golden_smu(name, golden_meta, tmp_path):
    c = golden_meta[name]
    kt = fastk.read_ktab(_golden(name))
    chunk = -(-kt.nels // 8)
    budget = budget_for_chunk(kt.nels, kt.kmer, kt.ibyte, chunk) + (16 << 20)
    out = str(tmp_path / "out")
    env = dict(os.environ, HETMERS_STREAM="1", HETMERS_STREAM_CHUNK=str(chunk), HETMERS_DEVICE_BUDGET=str(budget),
               HETMERS_LIST_HOST_BUDGET=str(CAP), HETMERS_LIST_ROOM=str(LIST_ROOM), HETMERS_STATS="1")
    r = subprocess.run([_lib.BIN_PATH, f"-e{c['e']}", "-T4", f"-o{out}", _golden(name)],
                       input="n\n", capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    st = json.loads([ln for ln in r.stderr.splitlines() if ln.startswith("{")][0])
    assert st["streamed"] is True and st["device_bytes"] <= budget
    assert st["spill"]["flushes"] >= 2 and st["spill"]["rounds"] >= 1
    assert open(out + ".smu").read() == open(_golden(name) + ".smu").read()

"""GPU tests of a job whose ranks keep their candidate records and S lists in host memory (dist.StreamedShardedScan
with list_host_budget, hm_rank_scan_set_list_host_budget, DESIGN.md §4c, *Lists in host memory*; run with -m gpu).
World 1, 2 and 3 ranks are spawned with gloo, all on one H100.  HETMERS_LIST_ROOM makes the small tables' lists
flush in pass 1, HETMERS_SPILL_ROOM and HETMERS_SPILL_PART make pass 2 take several rounds over several S
partitions.  The plot must equal the goldens' .smu, the in-core scan and the oracle; extract() the in-core list
record for record; write_pairs() the files extract_kmer_pairs writes, byte for byte."""
import ctypes as C
import os
import re
import sys
import tempfile

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

CAP = 1 << 32                                   # host bytes a rank's lists may take
KNOBS = {"HETMERS_LIST_ROOM": "1", "HETMERS_SPILL_ROOM": str(4 << 20), "HETMERS_SPILL_PART": "700"}


def _worker(rank, world, port, cases, q, backend="gloo"):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    out = []
    try:
        from smudgeplot_b200 import _lib
        from smudgeplot_b200 import dist as hd
        for case in cases:
            for var in ("HETMERS_STREAM_CHUNK",) + tuple(KNOBS):
                os.environ.pop(var, None)
            env = case.get("env", {})
            if case.get("env_ranks") is not None and rank not in case["env_ranks"]:
                env = {v: x for v, x in env.items() if v != "HETMERS_LIST_ROOM"}
            os.environ.update(env)
            os.environ["HETMERS_STREAM_CHUNK"] = str(case["chunk"])
            res = {"name": case["name"]}
            try:
                if case.get("L") is not None:
                    sc = hd.StreamedShardedScan.from_ktab(case["path"], device=f"cuda:{dev}", L=case["L"],
                                                          budget=case["budget"], list_host_budget=case.get("cap"))
                else:
                    sc = hd.StreamedShardedScan(case["path"], device=f"cuda:{dev}", budget=case["budget"],
                                                list_host_budget=case.get("cap"))
            except _lib.HetmersError as e:
                out.append(dict(res, error=(e.code, str(e))))
                continue
            try:
                res["plot"] = sc.scan().cpu().numpy()
                res["scan_stats"] = dict(sc.stats)
                res["residency"] = sc.residency()
                if case.get("sma"):
                    from test_gpu_stream_dist_extract import read_sma
                    pix, _ = read_sma(case["sma"])
                    res["recs"] = sc.extract(pix, dst=0)
                    res["extract_stats"] = dict(sc.stats)
                    res["residency_extract"] = sc.residency()
                if case.get("pairs_out"):
                    sc.write_pairs(case["sma"], case["pairs_out"])
                    res["pairs_stats"] = dict(sc.stats)
            except _lib.HetmersError as e:
                res["error"] = (e.code, str(e))
            finally:
                sc.close()
            out.append(res)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """-> per rank, per case: a dict of what it gave (plot, stats, records, residency) or error = (code, message)"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36500 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, cases, q, backend)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=1800) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


def _budget(kt, world, chunk):
    from test_gpu_stream_dist import rank_budget
    return rank_budget(kt.nels, kt.kmer, kt.ibyte, world)


@pytest.fixture(scope="module")
def tables(built):
    """[(name, path, k, sma or None)]: the goldens at k = 21, 31, 32, 40 and seeded tables at k = 33 and 64"""
    from smudgeplot_b200 import _lib
    from tools import synth
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"
    with tempfile.TemporaryDirectory() as d:
        out = []
        for name in ("dip_k21", "trip_k31", "tet_k32", "dip_k40"):
            path = os.path.join(GOLDEN, name, name)
            out.append((name, path, path + ".sma" if os.path.exists(path + ".sma") else None))
        for k in (33, 64):
            keys, cnt = synth.synth_table(k, 40000, 2, 0.02, 40, 4, 900 + k, extra_hom_repeats=1)
            path = os.path.join(d, f"seed{k}")
            synth.write_table(path, k, keys, cnt, ibyte=2, nparts=3)
            out.append((f"seeded_k{k}", path, None))
        yield out, d


def _want(path):
    """the oracle's plot and the in-core Scan's plot of the table at path"""
    import oracle_util as ou
    from smudgeplot_b200 import fastk, hetmers
    kt = fastk.read_ktab(path)
    kb, cn = fastk.unpack_host(kt)
    plot, _ = ou.oracle_scan(kb, cn, kt.kmer)
    with hetmers.Scan(kt) as sc:
        got, _ = sc.run()
    assert np.array_equal(got, plot)
    return kt, plot


def _check_spill(st, world):
    sp = st["spill"]
    assert sp["spilled"] and sp["flushes"] >= 1 and sp["rounds"] >= 1 and sp["partitions"] >= 1, sp
    assert sp["host_peak_bytes"] <= CAP
    assert len(st["queries_sent_to"]) == world


def _in_process_spilled(kt, monkeypatch):
    """the plot of the in-process streamed scan with its lists in host memory"""
    from smudgeplot_b200 import _lib
    from test_gpu_stream_spill import spilled_scan
    try:
        return spilled_scan(kt, monkeypatch)[0]
    finally:                                            # (process-wide settings of hetmers.Scan)
        _lib.lib().hm_set_device_budget(0)
        _lib.lib().hm_set_list_host_budget(0)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_plots_lists_and_files(world, tables, tmp_path, monkeypatch):
    """every table spilled on every rank: plot = oracle (= .smu), extract() = the in-core list, write_pairs() = the
    golden pair files; several rounds and partitions, queries to every rank including itself, peak <= budget"""
    from smudgeplot_b200 import hetmers
    from test_gpu_stream_dist_extract import read_sma
    tabs, _ = tables
    cases, wants = [], {}
    for name, path, sma in tabs:
        kt, plot = _want(path)
        assert np.array_equal(_in_process_spilled(kt, monkeypatch), plot), name
        wants[name] = (kt, plot)
        chunk = max(256, -(-kt.nels // (4 * world)))
        case = {"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, world, chunk), "cap": CAP,
                "env": dict(KNOBS)}
        if sma is not None:
            case["sma"] = sma
            if os.path.exists(path + ".pairs.1A1B.txt"):
                case["pairs_out"] = str(tmp_path / f"{name}.w{world}")
        cases.append(case)
    res = run_ranks(world, cases)
    pairs = np.zeros((world, world), dtype=np.int64)        # queries rank r sent to rank q, over the tables
    fkq = 0                                                 # queries on a partition's first key, over the tables
    for i, (name, path, sma) in enumerate(tabs):
        kt, plot = wants[name]
        if os.path.exists(path + ".smu"):
            assert hetmers.smu_text(plot) == open(path + ".smu").read()
        for r in range(world):
            got = res[r][i]
            assert "error" not in got, (name, r, got.get("error"))
            assert np.array_equal(got["plot"], plot), (name, r)
            st = got["scan_stats"]
            _check_spill(st, world)
            fkq += st["spill"]["first_key_queries"]
            peak, _, budget = got["residency"]
            assert peak <= budget, (name, r, peak, budget)
            pairs[r] += np.array(st["queries_sent_to"])
            if sma is not None:
                es = got["extract_stats"]
                assert es["pass1_reused"]
                _check_spill(es, world)
                assert got["residency_extract"][0] <= budget
        if sma is not None:
            pix, _ = read_sma(sma)
            with hetmers.Scan(kt) as sc:
                sc.run()
                want = sc.extract(pix)
            recs = res[0][i]["recs"]
            assert recs is not None and recs.tobytes() == want.tobytes(), name
            assert all(res[r][i]["recs"] is None for r in range(1, world))
            if "pairs_out" in cases[i]:
                from smudgeplot_b200.hetmers import read_sma as labels_of
                from test_gpu_write_pairs import executable_files, label_files
                want = executable_files(path, sma, str(tmp_path / f"exe_{name}"))
                assert label_files(cases[i]["pairs_out"], labels_of(sma)[1]) == want, name
    assert (pairs > 0).all(), pairs
    assert fkq > 0


@pytest.mark.parametrize("world", [2, 3])
def test_one_rank_spilling_makes_every_rank_spill(world, tables):
    """only rank 0's lists flush (HETMERS_LIST_ROOM there alone): every rank runs the parked rounds, same plot"""
    tabs, _ = tables
    name, path, _ = tabs[0]
    kt, plot = _want(path)
    chunk = max(256, -(-kt.nels // (4 * world)))
    case = {"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, world, chunk), "cap": CAP,
            "env": dict(KNOBS), "env_ranks": [0]}
    res = run_ranks(world, [case])
    for r in range(world):
        got = res[r][0]
        assert "error" not in got, got.get("error")
        assert np.array_equal(got["plot"], plot)
        sp = got["scan_stats"]["spill"]
        assert sp["spilled"] and sp["rounds"] >= 1
        assert (sp["flushes"] > 1) if r == 0 else (sp["flushes"] == 1)


def test_lists_that_fit_stay_resident(tables):
    """a list host budget that is not needed: the resident routed pass, same plot"""
    tabs, _ = tables
    name, path, _ = tabs[0]
    kt, plot = _want(path)
    chunk = max(256, -(-kt.nels // 8))
    res = run_ranks(2, [{"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, 2, chunk), "cap": CAP}])
    for r in range(2):
        got = res[r][0]
        assert np.array_equal(got["plot"], plot)
        assert not got["scan_stats"]["spill"]["spilled"]


@pytest.mark.parametrize("world", [1, 3])
def test_tiny_list_host_budget_is_refused_on_every_rank(world, tables):
    tabs, _ = tables
    name, path, _ = tabs[0]
    from smudgeplot_b200 import fastk
    kt = fastk.read_ktab(path)
    chunk = max(256, -(-kt.nels // (4 * world)))
    res = run_ranks(world, [{"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, world, chunk),
                             "cap": 1000, "env": dict(KNOBS)}])
    for r in range(world):
        code, msg = res[r][0]["error"]
        assert code == -3, msg
        assert "list host budget is 1000 bytes" in msg and "list_host_budget" in msg, msg
        assert re.search(r"lists need \d+ bytes of host memory", msg), msg
        assert "HETMERS_LIST_HOST_BUDGET" not in msg


def test_one_rank_over_its_cap_raises_on_every_rank(tables):
    """rank 0 alone overflows (HETMERS_LIST_ROOM makes it flush, cap 1000): rank 1 raises naming rank 0"""
    tabs, _ = tables
    name, path, _ = tabs[0]
    from smudgeplot_b200 import fastk
    kt = fastk.read_ktab(path)
    chunk = max(256, -(-kt.nels // 8))
    res = run_ranks(2, [{"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, 2, chunk),
                         "cap": 1000, "env": dict(KNOBS), "env_ranks": [0]}])
    c0, m0 = res[0][0]["error"]
    c1, m1 = res[1][0]["error"]
    assert c0 == -3 and "list_host_budget" in m0
    assert c1 == -3 and "rank 0" in m1, m1


def test_from_ktab_with_host_lists(tables, tmp_path):
    """from_ktab(L=12) on a raw table with host lists: the conditioned table's plot, list and pair files"""
    from smudgeplot_b200 import hetmers
    from test_gpu_parity import write_labelled_sma
    from test_gpu_stream_condition_dist import raw_table
    from test_gpu_write_pairs import executable_files, label_files
    raw = raw_table(tmp_path, 31, 40000, 2, 77)
    cond = str(tmp_path / "cond")
    hetmers.condition_table(raw, cond, 12)
    kt, plot = _want(cond)
    sma = str(tmp_path / "cond.sma")
    write_labelled_sma(plot, sma)
    from test_gpu_stream_dist_extract import read_sma
    pix, _ = read_sma(sma)
    world = 2
    chunk = max(256, -(-kt.nels // 8))
    out = str(tmp_path / "ranks")
    res = run_ranks(world, [{"name": "raw", "path": raw, "L": 12, "chunk": chunk, "budget": None, "cap": CAP,
                             "env": dict(KNOBS), "sma": sma, "pairs_out": out}])
    for r in range(world):
        got = res[r][0]
        assert "error" not in got, got.get("error")
        assert np.array_equal(got["plot"], plot)
        assert got["scan_stats"]["spill"]["spilled"] and got["pairs_stats"]["spill"]["spilled"]
    with hetmers.Scan(kt) as sc:
        sc.run()
        want = sc.extract(pix)
    assert res[0][0]["recs"].tobytes() == want.tobytes()
    assert label_files(out, hetmers.read_sma(sma)[1]) == executable_files(cond, sma, str(tmp_path / "exe"))


# ------------------------------------------------------------------ many rounds, the default path, NCCL ---------

def _floor_room(k, world):
    """the smallest pass 2 room hm_rank_spill_plan accepts for a listing by `world` ranks with at least HM_SPILL_MIN
    candidates and S keys (slices of about HM_SPILL_MIN candidates)"""
    from smudgeplot_b200 import _lib
    lay, lo, hi = _lib.SpillLayout(), 1, 1 << 34
    while lo < hi:
        mid = (lo + hi) // 2
        if _lib.lib().hm_rank_spill_plan(1 << 30, 1 << 30, k, world, 1, mid, C.byref(lay)) == 0:
            hi = mid
        else:
            lo = mid + 1
    return lo


@pytest.fixture(scope="module")
def big_tables(built, tmp_path_factory):
    """seeded tables of a few hundred thousand entries at k = 31 and 40, with their .sma"""
    from smudgeplot_b200 import fastk
    from test_gpu_parity import write_labelled_sma
    from tools import synth
    d = tmp_path_factory.mktemp("big")
    out = []
    for k in (31, 40):
        keys, cnt = synth.synth_table(k, 200_000, 2, 0.02, 40, 8, 160 + k, device="cuda")
        path = str(d / f"big{k}")
        synth.write_table(path, k, keys, cnt, ibyte=2, nparts=2)
        kt, plot = _want(path)
        write_labelled_sma(plot, path + ".sma")
        from test_gpu_stream_dist_extract import read_sma
        out.append((path, kt, plot, read_sma(path + ".sma")[0]))
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_many_rounds_at_the_plan_floor(world, big_tables, tmp_path):
    """pass 2 at the room hm_rank_spill_plan needs at least: slices of about HM_SPILL_MIN candidates, so every rank
    takes three rounds or more in scan() and extract(), slices starting inside the host blocks of pass 1"""
    from smudgeplot_b200 import hetmers
    cases = []
    for path, kt, plot, pix in big_tables:
        chunk = max(256, -(-kt.nels // (8 * world)))
        cases.append({"name": path, "path": path, "chunk": chunk, "budget": _budget(kt, world, chunk), "cap": CAP,
                      "sma": path + ".sma",
                      "env": {"HETMERS_LIST_ROOM": "1", "HETMERS_SPILL_ROOM": str(_floor_room(kt.kmer, world))}})
    res = run_ranks(world, cases)
    for i, (path, kt, plot, pix) in enumerate(big_tables):
        with hetmers.Scan(kt) as sc:
            sc.run()
            want = sc.extract(pix)
        assert res[0][i]["recs"].tobytes() == want.tobytes(), path
        for r in range(world):
            got = res[r][i]
            assert "error" not in got, got.get("error")
            assert np.array_equal(got["plot"], plot), (path, r)
            for st in (got["scan_stats"], got["extract_stats"]):
                sp = st["spill"]
                assert sp["spilled"] and sp["rounds"] >= 3 and sp["flushes"] >= 3, (path, r, sp)
                assert sp["slice"] <= 2 * 1024, sp
            assert got["residency"][0] <= got["residency"][2]


def _list_budget(kt, world):
    """the largest budget whose plan leaves the resident lists at most 1.5 B per entry (they take about 3): the
    lists do not fit beside the chunk buffers -> (budget, the plan's chunk)"""
    from smudgeplot_b200 import _lib
    lay, lo, hi = _lib.StreamLayout(), 1 << 20, 1 << 36
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if _lib.lib().hm_stream_plan_shards(kt.nels, kt.kmer, kt.ibyte, mid, world, C.byref(lay)) != 0 or \
                lay.list_bytes <= 3 * kt.nels // 2:
            lo = mid
        else:
            hi = mid - 1
    assert _lib.lib().hm_stream_plan_shards(kt.nels, kt.kmer, kt.ibyte, lo, world, C.byref(lay)) == 0
    return lo, lay.chunk


def test_without_a_list_host_budget_the_overflow_still_refuses(big_tables):
    """one rank, a budget its lists outgrow: "list needs" without list_host_budget, as before; with it the lists
    go to host memory under the same budget and the plot is the in-core one"""
    path, kt, plot, _ = big_tables[0]
    budget, chunk = _list_budget(kt, 1)
    res = run_ranks(1, [{"name": "none", "path": path, "chunk": chunk, "budget": budget},
                        {"name": "cap", "path": path, "chunk": chunk, "budget": budget, "cap": CAP}])
    assert "error" in res[0][0], (budget, chunk, kt.nels, res[0][0].get("scan_stats"), res[0][0].get("residency"))
    code, msg = res[0][0]["error"]
    assert code == -3 and "list needs" in msg, msg
    got = res[0][1]
    assert "error" not in got, got.get("error")
    assert np.array_equal(got["plot"], plot)
    assert got["scan_stats"]["spill"]["spilled"] and got["residency"][0] <= budget


def test_one_rank_per_gpu_over_nccl(tables, tmp_path):
    """two ranks, a GPU each, NCCL collectives: the spilled job gives the oracle's plot and the in-core list"""
    import torch
    from smudgeplot_b200 import hetmers
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    tabs, _ = tables
    name, path, sma = tabs[0]
    kt, plot = _want(path)
    chunk = max(256, -(-kt.nels // 8))
    res = run_ranks(2, [{"name": name, "path": path, "chunk": chunk, "budget": _budget(kt, 2, chunk), "cap": CAP,
                         "env": dict(KNOBS), "sma": sma}], backend="nccl")
    from test_gpu_stream_dist_extract import read_sma
    with hetmers.Scan(kt) as sc:
        sc.run()
        want = sc.extract(read_sma(sma)[0])
    assert res[0][0]["recs"].tobytes() == want.tobytes()
    for r in range(2):
        assert np.array_equal(res[r][0]["plot"], plot)
        assert res[r][0]["scan_stats"]["spill"]["spilled"]

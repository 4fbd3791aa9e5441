"""GPU tests of conditioning a raw FastK table on the way into the one-process-per-GPU streamed scan
(dist.StreamedShardedScan.from_ktab(L=...), DESIGN.md §4c *Ranks* and §4f; run with -m gpu).  World 1, 2 and 3 ranks
are spawned with gloo, all on one H100; an NCCL case runs with a GPU per rank where there are two.  The plot must be
the reference binary's on the conditioned table and hetmers.hetmers(src, L=...)'s, the pair list and files the
in-core ones, and the ranks' host shares, concatenated in rank order, the records dist.condition_ktab writes."""
import datetime
import os
import sys
import traceback

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def _op(sc, case, op, dev):
    from smudgeplot_b200 import hetmers
    if op[0] == "smu":
        return hetmers.smu_text(sc.scan().cpu().numpy()), sc.residency(), sc.symm_ok()
    if op[0] == "extract":
        got = sc.extract(op[1], dst=0)
        return None if got is None else got.tobytes()
    if op[0] == "write_pairs":
        return sc.write_pairs(op[1], op[2])["records"]
    if op[0] == "share":
        sh = sc.share
        return None if sh is None else (sh.records[0].tobytes(), sh.index.copy(), sh.part_nels, sh.minval)
    raise ValueError(op)


def _worker(rank, world, port, backend, cases, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
    out = []
    try:
        from smudgeplot_b200 import _lib
        from smudgeplot_b200 import dist as hd
        for case in cases:
            os.environ["HETMERS_STREAM_CHUNK"] = str(case.get("chunk", 1 << 30))
            budget = case.get("budget")
            if isinstance(budget, list):
                budget = budget[rank]
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            res = {}
            if "condition_ktab" in case:                        # the files condition_ktab writes, for comparison
                res["stats"] = hd.condition_ktab(case["src"], case["condition_ktab"], case["L"], device=f"cuda:{dev}")
                out.append(res)
                continue
            try:
                sc = hd.StreamedShardedScan.from_ktab(case["src"], device=f"cuda:{dev}", L=case.get("L"),
                                                      budget=budget, host_budget=case.get("host_budget"))
            except _lib.HetmersError as e:
                torch.cuda.synchronize()
                out.append({"error": (e.code, str(e)), "memory": (before, torch.cuda.memory_allocated())})
                continue
            try:
                res["ops"] = [_op(sc, case, op, dev) for op in case.get("ops", [])]
                res["stats"] = sc.stats["condition"]
            finally:
                sc.close()
            out.append(res)
        q.put((rank, out))
    except BaseException:                                       # reported at once rather than by the timeout
        q.put((rank, {"crash": traceback.format_exc()}))
        raise
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{src, L, budget (or one per rank), host_budget, chunk, ops}] or [{src, L, condition_ktab: dst}] ->
    per rank, per case: {"stats": stats["condition"], "ops": results} | {"error": (code, message), "memory":
    (before, after)} | {"stats": condition_ktab's}"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 41600 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = {}
        for _ in range(world):
            r, v = q.get(timeout=360)
            assert not isinstance(v, dict), (r, v["crash"])
            res[r] = v
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    return [res[r] for r in range(world)]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    from smudgeplot_b200 import _lib
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _reset(monkeypatch):
    monkeypatch.delenv("HETMERS_PATH", raising=False)


def raw_table(d, k, G, ploidy, seed, ibyte=3, nparts=3):
    """a canonical untrimmed table, made as test_gpu_parity.test_gpu_conditioning_of_canonical_untrimmed_table
    makes it"""
    from smudgeplot_b200 import fastk
    from test_gpu_parity import canonical_mask
    from tools import synth
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 40, 1, seed)
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    path = str(d / f"raw_k{k}_s{seed}")
    fastk.write_ktab(path, k, ku[canon], cn[canon], ibyte=ibyte, nparts=nparts)
    return path


def chunk_for(src, world):
    """chunks small enough that every rank's share of the conditioned table takes at least 4"""
    from smudgeplot_b200 import fastk
    return max(32, fastk.read_ktab(src).nels // (16 * world))


def share_keys(share, k):
    """the keys of a host share (records, index, part_nels, minval) -> uint64 (k <= 32) or [n, 2]"""
    from smudgeplot_b200 import fastk
    rec, index, part_nels, minval = share
    kt = fastk.KtabFiles(kmer=k, nparts=1, minval=minval, ibyte=int(np.log2(len(index))) // 8, index=index,
                         part_nels=part_nels, records=[np.frombuffer(rec, dtype=np.uint8)])
    return fastk.keys_bytes_to_u64(fastk.unpack_host(kt)[0])


def check_shares(res, i, written, k):
    """the ranks' host shares concatenated = the records (and stub index) condition_ktab wrote; every non-empty
    share starts on a run (its first k//2 bases differ from those of the last entry before it); cuts agree"""
    from smudgeplot_b200 import fastk
    world = len(res)
    kt = fastk.read_ktab(written)
    shares = [res[r][i]["ops"][-1] for r in range(world)]
    assert b"".join(s[0] for s in shares) == kt.all_records().tobytes()
    assert np.array_equal(sum(s[1] for s in shares), kt.index)
    outs = [s[2][0] for s in shares]
    sts = [res[r][i]["stats"] for r in range(world)]
    assert all(st["cuts"] == [0] + np.cumsum(outs).tolist() for st in sts)
    assert [st["rank_entries_out"] for st in sts] == outs and sts[0]["entries_out"] == kt.nels
    for st, s in zip(sts, shares):
        assert st["host_bytes"] == len(s[0]) + s[1].nbytes
    sh = np.uint64(64 - 2 * (k >> 1))
    last = None
    for s in shares:
        keys = share_keys(s, k)
        first = keys if keys.ndim == 1 else keys[:, 0]
        if len(first):
            if last is not None:
                assert (first[0] >> sh) != (last >> sh)
            last = first[-1]
    return sts


def check_memory(res, i):
    for r in range(len(res)):
        st = res[r][i]["stats"]
        assert 0 < st["peak_bytes"] <= st["budget"], st
        for op in res[r][i]["ops"]:
            if isinstance(op, tuple) and len(op) == 3 and isinstance(op[1], tuple):     # ("smu", residency, ok)
                peak, chunks, budget = op[1]
                assert 0 < peak <= budget and op[2]


# ------------------------------------------------------------------ stored reference runs, small k, 1-3 ranks ----

CONDITIONING_CASES = [(21, 60000, 2, 31, 6), (31, 80000, 3, 32, 12), (32, 50000, 2, 33, 5),   # k, G, ploidy, seed, L
                      (40, 50000, 2, 34, 6), (12, 30000, 2, 35, 12)]


@pytest.fixture(scope="module")
def reference_tables(tmp_path_factory):
    """the raw tables of the stored reference runs and a k = 17 one: (src, k, L, .smu wanted)"""
    import oracle_util as ou
    from smudgeplot_b200 import hetmers
    d = tmp_path_factory.mktemp("refs")
    out = []
    for k, G, ploidy, seed, L in CONDITIONING_CASES + [(17, 40000, 2, 36, 8)]:
        src = raw_table(d, k, G, ploidy, seed)
        smu = open(hetmers.hetmers(src, o=str(d / f"incore_k{k}"), L=L)).read()
        if k != 17:
            assert smu == ou.reference_smu("conditioned", k, seed)
        assert len(smu) > 0
        out.append((src, k, L, smu))
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_stored_reference_runs(world, reference_tables, tmp_path):
    cases = []
    for src, k, L, _ in reference_tables:
        cases.append({"src": src, "L": L, "condition_ktab": str(tmp_path / f"ck{k}")})
        cases.append({"src": src, "L": L, "chunk": chunk_for(src, world), "ops": [("smu",), ("share",)]})
    res = run_ranks(world, cases)
    for j, (src, k, L, smu) in enumerate(reference_tables):
        i = 2 * j + 1
        for r in range(world):
            assert "error" not in res[r][i], res[r][i]
            got, (peak, chunks, budget), ok = res[r][i]["ops"][0]
            assert got == smu, (k, r)
            assert chunks >= 4 or res[r][i]["stats"]["rank_entries_out"] == 0, (k, r, chunks)
        sts = check_shares(res, i, str(tmp_path / f"ck{k}"), k)
        assert sts[0]["steps"] == ["trim", "symmetrise"]
        assert sts[0]["prefix_cuts"] == res[0][i - 1]["stats"]["prefix_cuts"] or k < 20
        check_memory(res, i)


# ------------------------------------------------------------------ raw goldens: plot, pairs, pair files ----------

@pytest.mark.parametrize("world", [2, 3])
def test_raw_goldens_list_and_write_the_in_core_pairs(world, golden_meta, tmp_path):
    from smudgeplot_b200 import fastk, hetmers
    from test_gpu_parity import write_labelled_sma
    from test_gpu_scan_write_pairs import conditioned_scan, files
    from test_gpu_stream_dist_extract import records
    cases, want = [], []
    for name in ("untrimmed", "asymmetric"):
        src = os.path.join(GOLDEN, "conditioning", name)
        e = golden_meta["_conditioning"][name]["e"]
        with conditioned_scan(fastk.read_ktab(src), e) as sc:
            plot, _ = sc.run()
            sma = str(tmp_path / f"{name}.sma")
            write_labelled_sma(plot, sma)
            pix, labels = hetmers.read_sma(sma)
            pairs = sc.extract(pix)
        hetmers.run_extract(src, sma, o=str(tmp_path / f"x_{name}"), e=e)
        assert len(pairs) > 0
        want.append((hetmers.smu_text(plot), pairs, files(str(tmp_path / f"x_{name}"), labels), labels, name))
        cases.append({"src": src, "L": e, "condition_ktab": str(tmp_path / f"ck_{name}")})
        cases.append({"src": src, "L": e, "chunk": chunk_for(src, world),
                      "ops": [("smu",), ("extract", pix), ("write_pairs", sma, str(tmp_path / f"w_{name}")),
                              ("share",)]})
    res = run_ranks(world, cases)
    for j, (smu, pairs, pair_files, labels, name) in enumerate(want):
        i = 2 * j + 1
        for r in range(world):
            assert "error" not in res[r][i], res[r][i]
            assert res[r][i]["ops"][0][0] == smu, (name, r)
            assert (res[r][i]["ops"][1] is None) == (r != 0)
            assert res[r][i]["ops"][2] == len(pairs)
        assert np.array_equal(records(res[0][i]["ops"][1]), pairs), name
        assert files(str(tmp_path / f"w_{name}"), labels) == pair_files, name
        check_shares(res, i, str(tmp_path / f"ck_{name}"), 21)
        check_memory(res, i)


# ------------------------------------------------------------------ nothing to condition ---------------------------

def test_no_conditioning_streams_the_source(golden_meta):
    """a table needing neither step, and L = None: the constructor's scan, no host share, the golden .smu"""
    src = os.path.join(GOLDEN, "dip_k21", "dip_k21")
    want = open(src + ".smu").read()
    e = golden_meta["dip_k21"]["e"]
    cases = [{"src": src, "L": e, "chunk": chunk_for(src, 2), "ops": [("smu",), ("share",)]},
             {"src": src, "L": None, "chunk": chunk_for(src, 2), "ops": [("smu",), ("share",)]}]
    res = run_ranks(2, cases)
    for r in range(2):
        for i in range(2):
            assert "error" not in res[r][i], res[r][i]
            st = res[r][i]["stats"]
            assert st["steps"] == [] and st["host_bytes"] == 0
            assert res[r][i]["ops"][0][0] == want and res[r][i]["ops"][1] is None
        assert (res[r][0]["stats"]["trimmed"], res[r][0]["stats"]["symmetric"]) == (True, True)


# ------------------------------------------------------------------ several passes, refusals -----------------------

def test_small_device_budgets_condition_in_several_passes(tmp_path):
    """budgets (found with the planning functions on numpy histograms) that leave every rank two sub-ranges or more:
    the same shares, and the peak within every rank's budget"""
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    from test_gpu_condition_files import output_hist
    from test_gpu_rank_condition_files import canonical, write
    k, L, world, ibyte = 31, 8, 2, 2
    ku, cn = canonical(k, 1_000_000, 78)
    src = write(str(tmp_path / "src"), k, ku, cn, ibyte=ibyte)
    n = len(cn)
    shares = [hd.share_range(n, world, r) for r in range(world)]
    locs = [np.stack([output_hist(ku[a:b], cn[a:b], k, L, True, False), output_hist(ku[a:b], cn[a:b], k, L, True, True)])
            for a, b in shares]
    h_all = sum(locs)
    hb = min(_lib.COND_HIST_BITS, 2 * k)
    cuts = hd.run_condition_cuts(h_all[1], world, hb, ibyte, k)
    Lb = _lib.lib()
    budget = Lb.hm_rank_condition_bytes(k, ibyte, world, n, n, 2 * n, n, 1)
    found = None
    while budget > 0 and found is None:
        budget = budget * 9 // 10
        try:
            subs = hd.rank_sub_cuts(k, ibyte, [b - a for a, b in shares], 1, [budget] * world, h_all[1], cuts)
        except _lib.HetmersError:
            break
        plans = [hd.rank_pass_counts(locs[r], h_all, subs, r) for r in range(world)]
        needs = [max(Lb.hm_rank_condition_bytes(k, ibyte, world, b - a, *c[:3], 1) for c in plans[r])
                 for r, (a, b) in enumerate(shares)]
        if min(len(s) - 1 for s in subs) >= 2 and max(needs) <= budget:
            found = budget
    assert found is not None
    res = run_ranks(world, [{"src": src, "L": L, "condition_ktab": str(tmp_path / "ck")},
                            {"src": src, "L": L, "budget": found, "ops": [("share",)]}])
    sts = check_shares(res, 1, str(tmp_path / "ck"), k)
    assert all(len(st["sub_ranges"]) - 1 >= 2 for st in sts) and sts[0]["passes"] >= 2
    assert all(0 < st["peak_bytes"] <= found for st in sts)


def test_refusals(tmp_path):
    """a host budget below one rank's share: HM_ENOMEM on every rank naming the sizes, before any pass; a device
    budget below one rank's share of the source: HM_ENOMEM; device memory returned either way, and the next call
    in the group succeeds"""
    from smudgeplot_b200 import fastk
    src = raw_table(tmp_path, 31, 80000, 3, 32)
    tiny = 1 << 20
    cases = [{"src": src, "L": 12, "host_budget": tiny},
             {"src": src, "L": 12, "budget": [None, tiny]},
             {"src": src, "L": 12, "host_budget": 1 << 40, "ops": [("share",)]}]
    res = run_ranks(2, cases)
    for r in range(2):
        code, msg = res[r][0]["error"]
        assert code == -3 and "host bytes" in msg and str(tiny) in msg, (r, msg)
        code, msg = res[r][1]["error"]
        assert code == -3 and "device bytes" in msg and str(tiny) in msg, (r, msg)
        for i in (0, 1):
            m0, m1 = res[r][i]["memory"]
            assert m0 == m1, (r, i, m0, m1)
        assert res[r][2]["stats"]["host_bytes"] > tiny
    assert sum(res[r][2]["stats"]["rank_entries_out"] for r in range(2)) > fastk.read_ktab(src).nels


def test_one_rank_per_gpu_over_nccl(tmp_path):
    from smudgeplot_b200 import _lib, hetmers
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    src = raw_table(tmp_path, 40, 50000, 2, 34)
    smu = open(hetmers.hetmers(src, o=str(tmp_path / "incore"), L=6)).read()
    res = run_ranks(2, [{"src": src, "L": 6, "condition_ktab": str(tmp_path / "ck")},
                        {"src": src, "L": 6, "chunk": chunk_for(src, 2), "ops": [("smu",), ("share",)]}],
                    backend="nccl")
    for r in range(2):
        assert res[r][1]["ops"][0][0] == smu
    check_shares(res, 1, str(tmp_path / "ck"), 40)
    check_memory(res, 1)

"""GPU tests of a job whose ranks stream their own shares (dist.StreamedShardedScan, hm_rank_scan_*, DESIGN.md §4c,
*Ranks*; run with -m gpu).  World 1, 2 and 3 ranks are spawned with gloo, all on one H100, each under its own
device budget; no rank holds the table, and a Bloom hit on a key another rank owns is settled by that rank.  The
plot must equal the goldens, the in-process streamed scan and the oracle."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT, golden_cases

pytestmark = pytest.mark.gpu


def route_bytes(slice_, k, world):
    """hm_scan.cu route_bytes: device bytes of pass 2's exchange buffers for slices of `slice_` candidates"""
    kw, q, o = (2 if k > 32 else 1), 2 * slice_, world - 1
    return 8 * slice_ + q * (8 * kw + 8 + (8 if kw == 2 else 0)) + q * (8 * kw + 4) + o * q * 8 * kw + o * q + q + \
        16 * 16 + 10 * 256


def rank_budget(n, k, ibyte, world):
    """a budget with room for each rank's share in a few chunks, its lists at their bound and the exchange"""
    from test_gpu_stream_shards import shard_budget
    return shard_budget(n, k, ibyte, world, max(256, -(-n // (3 * world)))) + route_bytes(n // 2 + 1024, k, world)


def _worker(rank, world, port, backend, cases, q):
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
        for name, path, budget, chunk in cases:
            os.environ["HETMERS_STREAM_CHUNK"] = str(chunk)
            try:
                sc = hd.StreamedShardedScan(path, device=f"cuda:{dev}", budget=budget)
            except _lib.HetmersError as e:
                out.append((name, "error", e.code, str(e)))
                continue
            try:
                plot = sc.scan().cpu().numpy()
                res = sc.residency()
                out.append((name, "ok", plot, dict(sc.stats, residency=res, cuts=sc.cuts, ok=sc.symm_ok())))
            except _lib.HetmersError as e:
                out.append((name, "error", e.code, str(e)))
            finally:
                sc.close()
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [(name, table path, budget, chunk)] -> per rank: [(name, "ok", plot, stats) | (name, "error", code, msg)]"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=1200) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


# ------------------------------------------------------------------ the tables -------------------------

def _tables(d):
    """[(name, path, k, keys_u64, cnt)] for the goldens and the tables test_gpu_stream.py / _shards use"""
    import test_gpu_symm as tg
    from smudgeplot_b200 import fastk
    from tools import synth
    out = []
    for name in golden_cases():
        path = os.path.join(GOLDEN, name, name)
        out.append((name, path, None, None, None))
    for k, seed in ((11, 1), (12, 2)):                                    # dense small k: runs of hundreds
        rng = np.random.default_rng(9300 + seed)
        vals = rng.choice(4 ** k, size=int(4 ** k * 0.05), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
        keys, cnt = tg._symmetric_closure(vals, k, rng, 700)
        fastk.write_ktab(os.path.join(d, f"dense{k}"), k, keys, cnt, ibyte=1, nparts=2)
        out.append((f"closure_k{k}", os.path.join(d, f"dense{k}"), k, keys, cnt))
    rng = np.random.default_rng(5150)                                    # runs longer than a share
    keys, cnt = tg._symmetric_closure(np.arange(64, dtype=np.uint64) << np.uint64(58), 3, rng, 300)
    fastk.write_ktab(os.path.join(d, "long3"), 3, keys, cnt, ibyte=1, nparts=1)
    out.append(("longrun_k3", os.path.join(d, "long3"), 3, keys, cnt))
    for k in (8, 10, 16):                                                 # even k with palindromes
        rng = np.random.default_rng(177 + k)
        vals = rng.choice(4 ** k, size=min(4 ** k // 20, 60000), replace=False).astype(np.uint64) << np.uint64(64 - 2 * k)
        keys, cnt = tg._symmetric_closure(vals, k, rng, 300)
        fastk.write_ktab(os.path.join(d, f"pal{k}"), k, keys, cnt, ibyte=1, nparts=2)
        out.append((f"pal_k{k}", os.path.join(d, f"pal{k}"), k, keys, cnt))
    for k in (32, 33, 40, 64):                                            # seeded, two-word keys above 32
        keys, cnt = synth.synth_table(k, 40000, 2, 0.02, 40, 4, 700 + k, extra_hom_repeats=1)
        path = os.path.join(d, f"seed{k}")
        synth.write_table(path, k, keys, cnt, ibyte=2, nparts=3)
        out.append((f"seeded_k{k}", path, k, None, None))
    return out


def _fixtures(d):
    """tables, what each must give (oracle or golden .smu), and the cases for the ranks"""
    import oracle_util as ou
    from smudgeplot_b200 import fastk, hetmers
    tables, want, kts = _tables(d), {}, {}
    for name, path, k, keys, cnt in tables:
        kt = fastk.read_ktab(path)
        kts[name] = kt
        if keys is None:
            kb, cn = fastk.unpack_host(kt)
            plot, _ = ou.oracle_scan(kb, cn, kt.kmer)
        else:
            plot, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, k), cnt, k)
        want[name] = plot
        if os.path.exists(path + ".smu"):
            assert hetmers.smu_text(plot) == open(path + ".smu").read()
    return tables, want, kts


@pytest.fixture(scope="module")
def fixtures(built):
    from smudgeplot_b200 import _lib
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"
    with tempfile.TemporaryDirectory() as d:
        yield _fixtures(d)


@pytest.fixture(autouse=True)
def _reset_budget():
    yield
    from smudgeplot_b200 import _lib
    _lib.lib().hm_set_device_budget(0)                                   # (_one_rank sets this process's budget)


SENT = {}


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ranks_stream_every_table_like_the_oracle(world, fixtures, monkeypatch):
    from smudgeplot_b200 import _lib, hetmers
    from test_gpu_stream_shards import sharded_scan
    tables, want, kts = fixtures
    cases = []
    for name, path, *_ in tables:
        kt = kts[name]
        cases.append((name, path, rank_budget(kt.nels, kt.kmer, kt.ibyte, world), max(256, -(-kt.nels // (3 * world)))))
    res = run_ranks(world, cases)
    for i, (name, path, *_) in enumerate(tables):
        kt = kts[name]
        inproc, _, _, _ = sharded_scan(kt, world, 3, monkeypatch)
        for rank in range(world):
            nm, what, plot, st = res[rank][i]
            assert nm == name and what == "ok", (name, rank, plot, st)
            assert np.array_equal(plot, want[name]), (name, world, rank)
            assert np.array_equal(plot, inproc), (name, world, rank)
            peak, chunks, budget = st["residency"]
            assert peak <= budget == cases[i][2], (name, rank, st)
            assert st["ok"]
            if os.path.exists(path + ".smu"):
                assert hetmers.smu_text(plot) == open(path + ".smu").read()
            for dst, c in enumerate(st["queries_sent_to"]):
                SENT[(world, rank, dst)] = SENT.get((world, rank, dst), 0) + c
    if world > 1:                                                          # routing really ran, both ways
        assert all(SENT.get((world, a, b), 0) > 0 for a in range(world) for b in range(world) if a != b), SENT
    print(f"world {world}: queries {SENT}")


def _one_rank(path, budget, chunk, monkeypatch):
    """a one-rank job in this process: -> (plot, stats)"""
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    with tempfile.TemporaryDirectory() as d:
        dist.init_process_group("gloo", init_method=f"file://{d}/store", rank=0, world_size=1)
        try:
            sc = hd.StreamedShardedScan(path, device="cuda:0", budget=budget)
            try:
                plot = sc.scan().cpu().numpy()
                return plot, dict(sc.stats, residency=sc.residency())
            finally:
                sc.close()
                torch.cuda.synchronize()
        finally:
            dist.destroy_process_group()


def test_a_tight_budget_slices_pass_2_into_rounds(monkeypatch):
    """the budget left beside the resident lists bounds the pending list and the queries: pass 2 then runs in
    several rounds over slices of the candidates, with the same plot, under a budget below the in-core scan's
    footprint; a budget without room for the smallest slice is HM_ENOMEM"""
    import oracle_util as ou
    from smudgeplot_b200 import _lib, fastk, hetmers
    from tools import synth
    keys, cnt = synth.synth_table(31, 200_000, 2, 0.01, 40, 4, 77)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "t")
        kt = synth.write_table(path, 31, keys, cnt, ibyte=2, nparts=2)
        kb, cn = fastk.unpack_host(kt)
        want, _ = ou.oracle_scan(kb, cn, 31)
        chunk = -(-kt.nels // 8)
        roomy = rank_budget(kt.nels, 31, 2, 1)
        plot, st = _one_rank(path, roomy, chunk, monkeypatch)
        assert np.array_equal(plot, want) and st["rounds"] == 1
        held = roomy - route_bytes(st["max_slice"], 31, 1)                 # what pass 2 holds beside the buffers
        tight = held + route_bytes(max(256, st["candidates"] // 4), 31, 1)
        plot, st2 = _one_rank(path, tight, chunk, monkeypatch)
        assert np.array_equal(plot, want)
        assert st2["rounds"] >= 2 and st2["residency"][0] <= tight, st2
        _lib.lib().hm_set_device_budget(0)
        with hetmers.Scan(kt) as sc:                                       # what the in-core scan would hold
            streamed, incore, _ = sc.residency()
        assert not streamed and tight < incore, (tight, incore)
        held = tight - route_bytes(st2["max_slice"], 31, 1)
        with pytest.raises(_lib.HetmersError) as ei:   # no room for the smallest slice: refused, with the sizes
            _one_rank(path, held + route_bytes(100, 31, 1), chunk, monkeypatch)
        assert ei.value.code == -3 and "bytes" in str(ei.value)           # (pass 1's lists may run out first)


def test_asymmetric_table_is_refused_on_every_rank(tmp_path):
    from smudgeplot_b200 import fastk
    from tools import synth
    keys, cnt = synth.synth_table(31, 30000, 2, 0.02, 40, 4, 421)
    ku = synth.keys_to_u64_numpy(keys)
    cu = cnt.numpy().astype(np.uint16)
    keep = np.ones(len(ku), dtype=bool)
    keep[len(ku) // 3] = False
    kt = fastk.write_ktab(str(tmp_path / "asym"), 31, ku[keep], cu[keep], ibyte=3, nparts=2)
    res = run_ranks(3, [("asym", str(tmp_path / "asym"), rank_budget(kt.nels, 31, 3, 3), 1024)])
    for rank in range(3):
        name, what, code, msg = res[rank][0]
        assert what == "error" and code == -6 and "not strand-symmetric" in msg, res[rank]


def test_one_rank_per_gpu_over_nccl():
    """world = every GPU of the box, NCCL collectives on the device buffers in place"""
    from smudgeplot_b200 import _lib, fastk
    ngpu = _lib.lib().hm_device_count()
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    name = "dip_k21"
    path = os.path.join(GOLDEN, name, name)
    kt = fastk.read_ktab(path)
    res = run_ranks(ngpu, [(name, path, rank_budget(kt.nels, kt.kmer, kt.ibyte, ngpu), 1024)], backend="nccl")
    from smudgeplot_b200 import hetmers
    for rank in range(ngpu):
        nm, what, plot, st = res[rank][0]
        assert what == "ok" and hetmers.smu_text(plot) == open(path + ".smu").read()

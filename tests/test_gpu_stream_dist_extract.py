"""GPU tests of extract_kmer_pairs' list in a job whose ranks stream their own shares (dist.StreamedShardedScan.extract,
hm_rank_scan_extract_*, DESIGN.md §4c, *Ranks*; run with -m gpu).  World 1, 2 and 3 ranks are spawned with gloo, all
on one H100, each under its own device budget; a Bloom hit on a key another rank owns is settled by that rank, and
the ranks' records are gathered on one rank.  That rank's list must be hetmers.Scan.extract's in-core list of the
table, record for record; the golden and reference-binary pair files follow from it."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]
PLOT_CELLS = 1001 * 501


def listing_bytes(slice_, k, world):
    """hm_scan.cu listing_bytes: the routed listing's buffers for slices of `slice_` candidates"""
    from test_gpu_stream_dist import route_bytes
    return route_bytes(slice_, k, world) + 8 * (2 if k > 32 else 1) * slice_ + 48 * slice_ + 3 * 256


LISTING_FIXED = 2 * PLOT_CELLS + 256                                       # the device pixmap and the record counter


def rank_budget(n, k, ibyte, world):
    """room for each rank's share in a few chunks, its lists at their bound and the listing of every candidate"""
    from test_gpu_stream_shards import shard_budget
    return shard_budget(n, k, ibyte, world, max(256, -(-n // (3 * world)))) + listing_bytes(n // 2 + 1024, k, world) + \
        LISTING_FIXED


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
        for case in cases:
            os.environ["HETMERS_STREAM_CHUNK"] = str(case["chunk"])
            res = []
            try:
                sc = hd.StreamedShardedScan(case["path"], device=f"cuda:{dev}", budget=case["budget"])
            except _lib.HetmersError as e:
                out.append([("error", e.code, str(e))])
                continue
            try:
                for op, pix, dst in case["ops"]:
                    if op == "scan":
                        sc.scan()
                        res.append(("scan", None, dict(sc.stats)))
                        continue
                    tm = {}
                    got = sc.extract(pix, dst=dst, timings=tm)
                    res.append(("extract", None if got is None else got.tobytes(),
                                dict(sc.stats, residency=sc.residency(), phases=sorted(tm))))
            except _lib.HetmersError as e:
                res.append(("error", e.code, str(e)))
            finally:
                sc.close()
            out.append(res)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{path, budget, chunk, ops: [("scan" | "extract", pixmap, dst)]}] -> per rank, per case, per op:
    ("scan", None, stats) | ("extract", record bytes or None, stats) | ("error", code, message)"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=1800) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


def records(b):
    from smudgeplot_b200.hetmers import PAIR_DTYPE
    return np.frombuffer(b, dtype=PAIR_DTYPE)


def read_sma(path):
    """pixel -> 1-based smudge index (order of first appearance, as the executable numbers them), and the names"""
    pix = np.zeros((1001, 501), dtype=np.uint16)
    order = []
    with open(path) as f:
        next(f)
        for ln in f:
            m, rest, _, lab = ln.split()[:4]
            if lab not in order:
                order.append(lab)
            pix[int(m) + int(rest), int(m)] = order.index(lab) + 1
    return pix, order


def pair_lines(recs, k, order):
    """{smudge name: sorted print_het lines} of a record list"""
    from test_symm_extract_rule import pair_line
    out = {}
    for r in recs:
        key = int(r["key_hi"]) if k <= 32 else (int(r["key_hi"]) << 64) | int(r["key_lo"])
        out.setdefault(order[int(r["smudge"]) - 1], []).append(pair_line(key, k, int(r["pos"]), int(r["alt"])))
    return {lab: sorted(v) for lab, v in out.items()}


def incore(kt, pixmaps):
    from smudgeplot_b200 import hetmers
    with hetmers.Scan(kt) as sc:
        plot, st = sc.run()
        assert st["path"] == 2
        return plot, [sc.extract(p) for p in pixmaps]


def check_dst(res, i, j, dst, want):
    """op j of case i: the list on dst equals want, the other ranks got None -> the ranks' stats"""
    stats = []
    for rank, per_case in enumerate(res):
        what, b, st = per_case[i][j]
        assert what == "extract", (rank, per_case[i][j])
        if rank == dst:
            assert np.array_equal(records(b), want), (i, j, len(records(b)), len(want))
        else:
            assert b is None
        stats.append(st)
    return stats


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    from smudgeplot_b200 import _lib
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.fixture(autouse=True)
def _reset(monkeypatch):
    monkeypatch.delenv("HETMERS_PATH", raising=False)
    yield
    from smudgeplot_b200 import _lib
    _lib.lib().hm_set_device_budget(0)


SENT = {}


def _count_queries(world, stats_per_rank):
    for rank, st in enumerate(stats_per_rank):
        for dst, c in enumerate(st["queries_sent_to"]):
            SENT[(world, rank, dst)] = SENT.get((world, rank, dst), 0) + c


# ------------------------------------------------------------------ goldens and seeded tables ---------------

@pytest.mark.parametrize("world", [1, 2, 3])
def test_golden_pair_lists(world):
    """the .sma goldens give on dst the in-core list: plot[pix > 0].sum() records, whose lines are the golden
    pair files"""
    from smudgeplot_b200 import fastk
    cases, wants = [], []
    for name in SMA_GOLDENS:
        path = os.path.join(GOLDEN, name, name)
        kt = fastk.read_ktab(path)
        pix, order = read_sma(path + ".sma")
        plot, (want,) = incore(kt, [pix])
        assert len(want) == int(plot[pix > 0].sum()) > 0
        d, pre = os.path.join(GOLDEN, name), name + ".pairs."
        files = {f[len(pre):-4]: sorted(open(os.path.join(d, f)).read().splitlines())
                 for f in sorted(os.listdir(d)) if f.startswith(pre)}
        assert pair_lines(want, kt.kmer, order) == {lab: v for lab, v in files.items() if v}
        cases.append({"path": path, "budget": rank_budget(kt.nels, kt.kmer, kt.ibyte, world),
                      "chunk": max(256, -(-kt.nels // (3 * world))), "ops": [("extract", pix, world - 1)]})
        wants.append(want)
    res = run_ranks(world, cases)
    for i, want in enumerate(wants):
        stats = check_dst(res, i, 0, world - 1, want)
        for st in stats:
            assert not st["pass1_reused"] and st["residency"][0] <= cases[i]["budget"]
        _count_queries(world, stats)


@pytest.mark.parametrize("world", [2, 3])
def test_seeded_tables_list_the_in_core_pairs(world, tmp_path):
    """for k in {11, 16, 21, 31, 32, 33, 40, 64} (test_gpu_symm_extract.seeded_table: ties, and pair sums around
    SMAX), a label per pixel of the plot: the in-core list record for record"""
    from smudgeplot_b200 import _lib, hetmers
    from test_gpu_symm_extract import seeded_table
    cases, wants = [], []
    for k in (11, 16, 21, 31, 32, 33, 40, 64):
        kt = seeded_table(k, 100 + k, str(tmp_path / f"t{k}"))
        with hetmers.Scan(kt) as sc:
            plot, _ = sc.run()
        nz = np.flatnonzero(plot.reshape(-1) > 0)
        pix = np.zeros(_lib.PLOT_CELLS, dtype=np.uint16)
        pix[nz] = np.arange(1, nz.size + 1)
        pix = pix.reshape(_lib.SMAX + 1, _lib.PLOT_W)
        _, (want,) = incore(kt, [pix])
        assert len(want) == int(plot[pix > 0].sum()) > 0
        cases.append({"path": str(tmp_path / f"t{k}"), "budget": rank_budget(kt.nels, k, kt.ibyte, world),
                      "chunk": max(256, -(-kt.nels // (3 * world))), "ops": [("extract", pix, 0)]})
        wants.append(want)
    res = run_ranks(world, cases)
    for i, want in enumerate(wants):
        _count_queries(world, check_dst(res, i, 0, 0, want))


@pytest.mark.parametrize("world", [2, 3])
def test_every_rank_asked_every_other(world):
    """(after the tests above) the extraction queries went between every ordered pair of ranks"""
    if not any(w == world for w, _, _ in SENT):
        pytest.skip("the golden and seeded listings did not run in this session")
    assert all(SENT.get((world, a, b), 0) > 0 for a in range(world) for b in range(world) if a != b), SENT


@pytest.mark.parametrize("case", range(2))
def test_reference_pair_digests_at_world_2(case, tmp_path):
    """test_gpu_parity.EXTRACT_CASES: the lines of the list on dst are the reference binary's pair files"""
    import oracle_util as ou
    from smudgeplot_b200 import hetmers
    from test_gpu_parity import EXTRACT_CASES, write_labelled_sma
    from tools import synth
    k, G, ploidy, seed, L = EXTRACT_CASES[case]
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed, device="cuda")
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
    with hetmers.Scan(kt) as sc:
        plot, _ = sc.run("symm")
    pix, order = write_labelled_sma(plot, str(tmp_path / "ann.sma"))
    res = run_ranks(2, [{"path": name, "budget": rank_budget(kt.nels, k, kt.ibyte, 2),
                         "chunk": max(256, -(-kt.nels // 6)), "ops": [("extract", pix, 0)]}])
    what, b, _ = res[0][0][0]
    assert what == "extract" and res[1][0][0][1] is None
    lines = pair_lines(records(b), k, order)
    assert ou.pair_digests(lines) == ou.reference_pair_digests(k, seed)


# ------------------------------------------------------------------ budgets, reuse, dst, refusal -----------

def _one_rank(path, budget, chunk, pix, monkeypatch, scan_first=False):
    """a one-rank job in this process: -> (records, stats)"""
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd
    monkeypatch.setenv("HETMERS_STREAM_CHUNK", str(chunk))
    with tempfile.TemporaryDirectory() as d:
        dist.init_process_group("gloo", init_method=f"file://{d}/store", rank=0, world_size=1)
        try:
            sc = hd.StreamedShardedScan(path, device="cuda:0", budget=budget)
            try:
                if scan_first:
                    sc.scan()
                got = sc.extract(pix)
                return got, dict(sc.stats, residency=sc.residency())
            finally:
                sc.close()
                torch.cuda.synchronize()
        finally:
            dist.destroy_process_group()


def test_a_tight_budget_lists_in_rounds(monkeypatch, tmp_path):
    """the room beside the resident lists bounds the slice: several rounds, the same list, the peak within the
    budget; a budget without room for a slice of 256 candidates is HM_ENOMEM with the sizes"""
    from smudgeplot_b200 import _lib
    from tools import synth
    keys, cnt = synth.synth_table(31, 200_000, 2, 0.01, 40, 4, 77)
    path = str(tmp_path / "t")
    kt = synth.write_table(path, 31, keys, cnt, ibyte=2, nparts=2)
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    _, (want,) = incore(kt, [pix])
    chunk = -(-kt.nels // 8)
    roomy = rank_budget(kt.nels, 31, 2, 1)
    got, st = _one_rank(path, roomy, chunk, pix, monkeypatch)
    assert np.array_equal(got, want) and st["rounds"] == 1 and len(want) > 0
    held = roomy - LISTING_FIXED - listing_bytes(st["max_slice"], 31, 1)   # what the listing holds beside its buffers
    tight = held + LISTING_FIXED + listing_bytes(max(256, st["candidates"] // 4), 31, 1)
    got, st2 = _one_rank(path, tight, chunk, pix, monkeypatch)
    assert np.array_equal(got, want)
    assert st2["rounds"] >= 2 and st2["residency"][0] <= tight, st2
    held = tight - LISTING_FIXED - listing_bytes(st2["max_slice"], 31, 1)
    with pytest.raises(_lib.HetmersError) as ei:   # no room for the smallest slice: refused, with the sizes
        _one_rank(path, held + LISTING_FIXED + listing_bytes(100, 31, 1), chunk, pix, monkeypatch)
    assert ei.value.code == -3 and "bytes" in str(ei.value)


def test_reuse_dst_and_an_empty_pixmap(tmp_path):
    """extract() after scan() runs no second pass 1 and lists what a fresh object lists; dst = 1 holds the list
    and the other ranks get None; an all-zero pixmap lists nothing"""
    from smudgeplot_b200 import _lib, fastk
    name = "dip_k21"
    path = os.path.join(GOLDEN, name, name)
    kt = fastk.read_ktab(path)
    pix, _ = read_sma(path + ".sma")
    zero = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    _, (want,) = incore(kt, [pix])
    base = {"path": path, "budget": rank_budget(kt.nels, kt.kmer, kt.ibyte, 3), "chunk": max(256, -(-kt.nels // 9))}
    cases = [dict(base, ops=[("scan", None, 0), ("extract", pix, 1), ("extract", zero, 1), ("extract", pix, 2)]),
             dict(base, ops=[("extract", pix, 1)])]
    res = run_ranks(3, cases)
    for st in check_dst(res, 0, 1, 1, want):                               # after scan(): pass 1 reused
        assert st["pass1_reused"] and "pass1" not in st["phases"], st
    check_dst(res, 0, 2, 1, want[:0])
    for st in check_dst(res, 0, 3, 2, want):                               # after extract(): reused again
        assert st["pass1_reused"] and "pass1" not in st["phases"]
    for st in check_dst(res, 1, 0, 1, want):                               # a fresh object runs pass 1
        assert not st["pass1_reused"] and "pass1" in st["phases"]


def test_asymmetric_table_is_refused_on_every_rank(tmp_path):
    from smudgeplot_b200 import _lib, fastk
    from tools import synth
    keys, cnt = synth.synth_table(31, 30000, 2, 0.02, 40, 4, 421)
    ku = synth.keys_to_u64_numpy(keys)
    cu = cnt.numpy().astype(np.uint16)
    keep = np.ones(len(ku), dtype=bool)
    keep[len(ku) // 3] = False
    kt = fastk.write_ktab(str(tmp_path / "asym"), 31, ku[keep], cu[keep], ibyte=3, nparts=2)
    pix = np.ones((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    res = run_ranks(3, [{"path": str(tmp_path / "asym"), "budget": rank_budget(kt.nels, 31, 3, 3), "chunk": 1024,
                         "ops": [("extract", pix, 0)]}])
    for rank in range(3):
        what, code, msg = res[rank][0][0]
        assert what == "error" and code == -6 and "not strand-symmetric" in msg, res[rank]


def test_one_rank_per_gpu_over_nccl():
    """world = every GPU of the box, the records staged through device tensors to dst"""
    from smudgeplot_b200 import _lib, fastk
    ngpu = _lib.lib().hm_device_count()
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    name = "dip_k21"
    path = os.path.join(GOLDEN, name, name)
    kt = fastk.read_ktab(path)
    pix, _ = read_sma(path + ".sma")
    _, (want,) = incore(kt, [pix])
    res = run_ranks(ngpu, [{"path": path, "budget": rank_budget(kt.nels, kt.kmer, kt.ibyte, ngpu), "chunk": 1024,
                            "ops": [("extract", pix, ngpu - 1)]}], backend="nccl")
    check_dst(res, 0, 0, ngpu - 1, want)

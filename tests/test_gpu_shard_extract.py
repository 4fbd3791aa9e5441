"""GPU tests of the in-core one-process-per-GPU job (dist.ShardedScan) loaded from FastK files and listing
extract_kmer_pairs' pairs (ShardedScan.from_ktab, ShardedScan.extract; DESIGN.md §6; run with -m gpu).  World 1, 2
and 3 ranks are spawned with gloo, all on one H100 (the collectives go through host copies, the direct route's
incidence arrays are mapped between the processes with CUDA IPC on the one device); an NCCL case runs with a GPU
per rank where there are two.  The replica must be the table's records, the plot the golden one, and the list on
dst hetmers.Scan.extract's in-core list of the table, record for record, on either route."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]
PLOT_CELLS = 1001 * 501
FIXED = 2 * PLOT_CELLS + 256                  # the listing's device pixmap and record counter
REC = 24                                      # bytes of one hm_pair_rec
# route of ShardedScan(path=...), and whether the direct route's incidence bytes are all-reduced (dense)
ROUTES = {"symm": ("symm", False), "direct": ("direct", False), "dense": ("direct", True)}


def _op(sc, op, rank):
    import torch
    from smudgeplot_b200 import fastk, hetmers
    what = op[0]
    info = {"exchange": sc.exchange, "path": sc.path}
    if what == "scan":
        sc.scan()
        return ("scan", None, info)
    if what == "replica":                     # the replica against the CPU unpack of the files
        kt = fastk.read_ktab(op[1])
        kb, wc = fastk.unpack_host(kt)
        want = fastk.keys_bytes_to_u64(kb)
        t = sc.table
        got = t.keys.cpu().numpy().view(np.uint64)
        if kt.kmer > 32:
            got = np.stack([got, t.keys_lo.cpu().numpy().view(np.uint64)], axis=1)
        ok = (got.shape == want.shape and np.array_equal(got, want) and
              np.array_equal(t.cnt.cpu().numpy().view(np.uint16), wc))
        return ("replica", ok, dict(info, load=[sc.load_lo, sc.load_hi], n=sc.n_total))
    if what == "smu":
        return ("smu", hetmers.smu_text(sc.scan().cpu().numpy()), info)
    if what == "dirty":                       # a non-zero status word on rank op[1] (header word 1)
        if rank == op[1]:
            lay = sc.table.symm_layout
            sc.table.symm_work[lay.off_header + 8] = 1
            torch.cuda.synchronize()
        return ("dirty", None, info)
    _, pix, dst, budget = op
    if isinstance(budget, list):
        budget = budget[rank]
    tm = {}
    got = sc.extract(pix, dst=dst, timings=tm, budget=budget)
    return ("extract", None if got is None else got.tobytes(), dict(sc.stats, phases=sorted(tm), **info))


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
            route, dense = ROUTES[case.get("route", "symm")]
            if dense:
                os.environ["HETMERS_DENSE_EXCHANGE"] = "1"
            else:
                os.environ.pop("HETMERS_DENSE_EXCHANGE", None)
            res = []
            try:
                sc = hd.ShardedScan.from_ktab(case["path"], device=f"cuda:{dev}", path=route)
            except (_lib.HetmersError, RuntimeError) as e:
                out.append([("error", getattr(e, "code", None), str(e))])
                continue
            try:
                for op in case["ops"]:
                    try:
                        res.append(_op(sc, op, rank))
                    except (_lib.HetmersError, RuntimeError) as e:
                        res.append(("error", getattr(e, "code", None), str(e)))
            finally:
                sc.close()
            out.append(res)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{path, route ("symm" | "direct" | "dense"), ops}] with ops ("scan",), ("replica", path), ("smu",),
    ("dirty", rank), ("extract", pixmap, dst, budget or [budget per rank] or None) -> per rank, per case, per op:
    (op name, result, stats) | ("error", code, message)"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36600 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=900) for _ in range(world))
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:                       # a rank that failed leaves nobody waiting behind
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    return [res[r] for r in range(world)]


def golden(name):
    from smudgeplot_b200 import fastk
    from test_gpu_stream_dist_extract import read_sma
    path = os.path.join(GOLDEN, name, name)
    pix, order = read_sma(path + ".sma")
    return path, fastk.read_ktab(path), pix, order


def incore_list(kt, pix):
    from test_gpu_stream_dist_extract import incore
    _, (want,) = incore(kt, [pix])
    return want


def check_dst(res, i, j, dst, want):
    """op j of case i: the list on dst equals want, the other ranks got None -> the ranks' stats"""
    from test_gpu_stream_dist_extract import records
    stats = []
    for rank, per_case in enumerate(res):
        what, b, st = per_case[i][j]
        assert what == "extract", (rank, per_case[i][j])
        if rank == dst:
            got = records(b)
            assert np.array_equal(got, want), (i, j, len(got), len(want))
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
    monkeypatch.delenv("HETMERS_DENSE_EXCHANGE", raising=False)


# ------------------------------------------------------------------ from_ktab ----------------------------------

REPLICA_TABLES = [  # k, ibyte, parts, seed
    (21, 1, 1, 501), (21, 3, 4, 502), (32, 2, 4, 503), (32, 1, 2, 504), (33, 3, 3, 505), (40, 2, 2, 506),
    (40, 1, 4, 507),
]


def replica_tables(tmp_path):
    from smudgeplot_b200 import fastk, hetmers
    from tools import synth
    out = []
    for k, ibyte, parts, seed in REPLICA_TABLES:
        keys, cnt = synth.synth_table(k, 20_000, 2, 0.02, 30, 4, seed)
        path = str(tmp_path / f"r{k}_{ibyte}_{parts}")
        kt = fastk.write_ktab(path, k, synth.keys_to_u64_numpy(keys), cnt.numpy().astype(np.uint16), ibyte=ibyte,
                              nparts=parts)
        with hetmers.Scan(kt) as sc:
            plot, _ = sc.run()
        out.append((path, kt, hetmers.smu_text(plot)))
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_from_ktab_replica_and_plot(world, tmp_path):
    """every rank's replica is fastk.unpack_host of the files (ibyte 1..3, 1..4 parts, k = 21, 32, 33, 40), whether
    a rank's share lies inside one part or spans a part boundary; the plot is the in-core one and, on the goldens,
    the golden .smu"""
    tables = replica_tables(tmp_path)
    spans = inside = 0
    for _, kt, _ in tables:
        ends = np.cumsum(kt.part_nels)[:-1].tolist()
        n = kt.nels
        for r in range(world):
            lo, hi = (n * r) // world, (n * (r + 1)) // world
            spans += any(lo < e < hi for e in ends)
            inside += r > 0 and lo not in ends
    if world > 1:
        assert spans and inside
    cases = [{"path": p, "ops": [("replica", p), ("smu",)]} for p, _, _ in tables]
    smus = [s for _, _, s in tables]
    for name in SMA_GOLDENS:
        path = os.path.join(GOLDEN, name, name)
        cases.append({"path": path, "ops": [("replica", path), ("smu",)]})
        smus.append(open(path + ".smu").read())
    res = run_ranks(world, cases)
    for rank in range(world):
        for i, smu in enumerate(smus):
            (w1, ok, st), (w2, got, _) = res[rank][i]
            assert w1 == "replica" and ok, (rank, cases[i]["path"], st)
            assert w2 == "smu" and got == smu and len(got) > 0, (rank, cases[i]["path"])


# ------------------------------------------------------------------ lists on both routes -------------------------

@pytest.mark.parametrize("world", [1, 2, 3])
def test_golden_pair_lists_on_every_route(world):
    """the .sma goldens, symmetric route, direct route over peer-mapped incidence arrays and over the all-reduced
    one: the list on dst is the in-core list, and its lines are the golden pair files"""
    from test_gpu_stream_dist_extract import pair_lines
    cases, wants = [], []
    for name in SMA_GOLDENS:
        path, kt, pix, order = golden(name)
        want = incore_list(kt, pix)
        d, pre = os.path.join(GOLDEN, name), name + ".pairs."
        files = {f[len(pre):-4]: sorted(open(os.path.join(d, f)).read().splitlines())
                 for f in sorted(os.listdir(d)) if f.startswith(pre)}
        assert len(want) > 0 and pair_lines(want, kt.kmer, order) == {lab: v for lab, v in files.items() if v}
        for route in ROUTES:
            cases.append({"path": path, "route": route, "ops": [("extract", pix, world - 1, None)]})
            wants.append(want)
    res = run_ranks(world, cases)
    for i, want in enumerate(wants):
        route = cases[i]["route"]
        for st in check_dst(res, i, 0, world - 1, want):
            assert st["route"] == ROUTES[route][0] and not st["scan_reused"], st
            assert {"scan", "listing", "gather_and_sort"} <= set(st["phases"]), st
            if world > 1 and route == "direct":         # CUDA IPC between processes on the one device
                assert "peer-memory" in st["exchange"], st
            if world > 1 and route == "dense":
                assert "all-reduce" in st["exchange"], st


@pytest.mark.parametrize("route", ["symm", "direct"])
@pytest.mark.parametrize("case", range(2))
def test_reference_pair_digests_at_world_2(case, route, tmp_path):
    """test_gpu_parity.EXTRACT_CASES (~1e6 entries): the lines of the list on dst are the reference binary's pair
    files"""
    import oracle_util as ou
    from smudgeplot_b200 import hetmers
    from test_gpu_parity import EXTRACT_CASES, write_labelled_sma
    from test_gpu_stream_dist_extract import pair_lines, records
    from tools import synth
    k, G, ploidy, seed, L = EXTRACT_CASES[case]
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed, device="cuda")
    name = str(tmp_path / "t")
    kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
    with hetmers.Scan(kt) as sc:
        plot, _ = sc.run("symm")
    pix, order = write_labelled_sma(plot, str(tmp_path / "ann.sma"))
    res = run_ranks(2, [{"path": name, "route": route, "ops": [("extract", pix, 0, None)]}])
    what, b, st = res[0][0][0]
    assert what == "extract" and res[1][0][0][1] is None, res[0][0][0]
    assert st["route"] == route
    assert ou.pair_digests(pair_lines(records(b), k, order)) == ou.reference_pair_digests(k, seed)


# ------------------------------------------------------------------ reuse, dst, budgets, refusal -----------------

@pytest.mark.parametrize("route", ["symm", "direct"])
def test_reuse_dst_and_scans_between(route):
    """extract() before any scan runs one; after scan() it reuses it; extract, scan, extract, extract again (the
    direct route alternates its two incidence buffers): the in-core list each time, on dst = 1 and 2"""
    path, kt, pix, _ = golden("dip_k21")
    want = incore_list(kt, pix)
    ops = [("extract", pix, 1, None), ("scan",), ("extract", pix, 2, None), ("scan",), ("extract", pix, 1, None),
           ("extract", pix, 2, None)]
    res = run_ranks(3, [{"path": path, "route": route, "ops": ops}])
    for j, dst, reused in ((0, 1, False), (2, 2, True), (4, 1, True), (5, 2, True)):
        for st in check_dst(res, 0, j, dst, want):
            assert st["scan_reused"] == reused and ("scan" in st["phases"]) != reused, (j, st)


@pytest.mark.parametrize("route", ["symm", "direct"])
def test_a_small_budget_lists_in_slices_and_too_small_is_refused(route):
    """a budget for 40 records: several slices, the same list; a budget below one slice on one rank: HM_ENOMEM with
    the sizes on every rank, before anything is listed"""
    path, kt, pix, _ = golden("dip_k21")
    want = incore_list(kt, pix)
    small = FIXED + 40 * REC
    ops = [("extract", pix, 0, small), ("extract", pix, 1, [None, FIXED + REC - 1]), ("extract", pix, 1, None)]
    res = run_ranks(2, [{"path": path, "route": route, "ops": ops}])
    for st in check_dst(res, 0, 0, 0, want):
        assert st["slices"] >= 2 and st["buffer_records"] <= 40, st
    for rank in range(2):
        what, code, msg = res[rank][0][1]
        assert what == "error" and code == -3 and "bytes" in msg and str(FIXED + 2 * REC if route == "symm" else
                                                                          FIXED + REC) in msg, (rank, msg)
    check_dst(res, 0, 2, 1, want)                                          # the job goes on after the refusal


def test_dirty_status_word_is_refused_on_every_rank():
    path, kt, pix, _ = golden("tet_k32")
    res = run_ranks(3, [{"path": path, "route": "symm", "ops": [("scan",), ("dirty", 1), ("extract", pix, 0, None)]}])
    for rank in range(3):
        what, _, msg = res[rank][0][2]
        assert what == "error" and "status word" in msg, (rank, res[rank][0][2])


def test_one_rank_per_gpu_over_nccl():
    """world = 2 GPUs of the box, each with its replica; both routes"""
    from smudgeplot_b200 import _lib
    ngpu = _lib.lib().hm_device_count()
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    path, kt, pix, _ = golden("dip_k40")
    want = incore_list(kt, pix)
    res = run_ranks(2, [{"path": path, "route": r, "ops": [("replica", path), ("extract", pix, 1, None)]}
                        for r in ("symm", "direct")], backend="nccl")
    for i in range(2):
        assert all(res[rank][i][0][1] for rank in range(2))
        check_dst(res, i, 1, 1, want)

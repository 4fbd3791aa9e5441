"""GPU tests of conditioning a FastK table across the ranks of the one-process-per-GPU job
(dist.ShardedScan.from_ktab(L=...), DESIGN.md §4e; run with -m gpu).  World 1, 2 and 3 ranks are spawned with gloo,
all on one H100; an NCCL case runs with a GPU per rank where there are two.  The verdicts must be
hetmers.Scan.examine's, the replica entry for entry what hetmers.Scan.condition + download give in one process (and
the numpy restatement of trim + symmetrise), the plot the reference binary's on the conditioned table."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def _op(sc, op):
    import torch
    from smudgeplot_b200 import hetmers
    if op[0] == "replica":
        t = sc.table
        keys = t.keys.cpu().numpy().view(np.uint64)
        if sc.kmer > 32:
            keys = np.stack([keys, t.keys_lo.cpu().numpy().view(np.uint64)], axis=1)
        return keys, t.cnt.cpu().numpy().view(np.uint16)
    if op[0] == "smu":
        return hetmers.smu_text(sc.scan().cpu().numpy()), sc.path
    if op[0] == "extract":
        got = sc.extract(op[1], dst=0)
        return None if got is None else got.tobytes()
    if op[0] == "memory":
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()
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
    dist.init_process_group(backend, rank=rank, world_size=world)
    out = []
    try:
        from smudgeplot_b200 import _lib
        from smudgeplot_b200 import dist as hd
        for case in cases:
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            budget = case.get("budget")
            if isinstance(budget, list):
                budget = budget[rank]
            try:
                sc = hd.ShardedScan.from_ktab(case["path"], device=f"cuda:{dev}", L=case.get("L"), budget=budget)
            except _lib.HetmersError as e:
                torch.cuda.synchronize()
                out.append({"error": (e.code, str(e)), "memory": (before, torch.cuda.memory_allocated())})
                continue
            try:
                res = {"stats": sc.stats.get("condition"), "ops": [_op(sc, op) for op in case.get("ops", [])]}
            finally:
                sc.close()
            out.append(res)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{path, L, budget (or one per rank), ops: ("replica",) | ("smu",) | ("extract", pixmap)}] -> per rank,
    per case: {"stats": stats["condition"], "ops": results} or {"error": (code, message), "memory": (before, after)}"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 38600 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=300) for _ in range(world))
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


def incore(path, L, scan=True):
    """hetmers.Scan on one GPU: (examine verdicts, conditioned keys, counts, .smu, scan path)"""
    from smudgeplot_b200 import fastk, hetmers
    with hetmers.Scan(fastk.read_ktab(path)) as sc:
        trim, symm = sc.examine(L)
        sc.condition(L, not trim, not symm)
        keys, cnt, _ = sc.download(deg=False)
        smu = path_ = None
        if scan:
            plot, st = sc.run()
            smu, path_ = hetmers.smu_text(plot), st["path"]
    return (trim, symm), keys, cnt, smu, path_


def numpy_conditioned(path, L, verdicts):
    from smudgeplot_b200 import fastk
    from test_gpu_parity import _condition_numpy
    kt = fastk.read_ktab(path)
    kb, cn = fastk.unpack_host(kt)
    return _condition_numpy(fastk.keys_bytes_to_u64(kb), cn, kt.kmer, L, not verdicts[0], not verdicts[1])


def check_case(res, i, path, L, want_verdicts=None, smu=None):
    """every rank: verdicts, replica = in core = numpy, stats consistent; -> the in-core result"""
    verdicts, keys, cnt, smu_in, path_in = incore(path, L, scan=smu is not None)
    if want_verdicts is not None:
        assert verdicts == want_verdicts, (path, verdicts)
    nk, nc = numpy_conditioned(path, L, verdicts)
    assert np.array_equal(keys, nk) and np.array_equal(cnt, nc), path
    world = len(res)
    for rank in range(world):
        r = res[rank][i]
        assert "error" not in r, (rank, path, r)
        st = r["stats"]
        assert (st["trimmed"], st["symmetric"]) == verdicts, (rank, path, st)
        assert st["steps"] == (["trim"] if not verdicts[0] else []) + (["symmetrise"] if not verdicts[1] else [])
        assert st["entries_out"] == len(cnt)
        assert set(st["ms"]) >= {"load", "gather"} and ("route" in st["ms"]) == bool(st["steps"])
        if st["steps"]:
            assert set(st["ms"]) >= {"examine", "hist_and_plan", "route", "exchange"}
            assert 0 < st["peak_bytes"] <= st["working_set_bytes"] <= st["budget"], st
        got_k, got_c = r["ops"][0]
        assert np.array_equal(got_k, keys) and np.array_equal(got_c, cnt), (rank, path, len(got_c), len(cnt))
        if smu is not None:
            got_smu, route = r["ops"][1]
            assert got_smu == smu == smu_in and len(smu) > 0, (rank, path)
            assert route == {1: "direct", 2: "symm"}[path_in], (rank, path, route, path_in)
        assert sum(st["received"]) == sum(res[q][i]["stats"]["sent"][rank] for q in range(world))
    return keys, cnt


def write(tmp_path, tag, k, ku, cn, ibyte=3, nparts=3):
    from smudgeplot_b200 import fastk
    path = str(tmp_path / tag)
    fastk.write_ktab(path, k, ku, cn, ibyte=ibyte, nparts=nparts)
    return path


def canonical_untrimmed(tmp_path, k, G, ploidy, seed, ibyte=3, nparts=3, cov=40):
    """a FastK-style table: canonical k-mers only, counts from 1 (test_gpu_parity's conditioning input)"""
    from test_gpu_parity import canonical_mask
    from tools import synth
    keys, cnt = synth.synth_table(k, G, ploidy, 0.02, cov, 1, seed)
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    return write(tmp_path, f"c{k}_{seed}_{ibyte}_{nparts}", k, ku[canon], cn[canon], ibyte, nparts)


# ------------------------------------------------------------------ the parity cases -----------------------------

@pytest.mark.parametrize("world", [1, 2, 3])
def test_conditioning_cases_match_in_core_numpy_and_reference(world, tmp_path):
    """test_gpu_parity.CONDITIONING_CASES: untrimmed and not symmetric; the replica is the in-core conditioned table,
    the plot the reference binary's on it, and k = 12 takes the in-core scan's route"""
    import oracle_util as ou
    from test_gpu_parity import CONDITIONING_CASES
    cases, meta = [], []
    for k, G, ploidy, seed, L in CONDITIONING_CASES:
        path = canonical_untrimmed(tmp_path, k, G, ploidy, seed)
        cases.append({"path": path, "L": L, "ops": [("replica",), ("smu",)]})
        meta.append((path, L, ou.reference_smu("conditioned", k, seed)))
    res = run_ranks(world, cases)
    for i, (path, L, smu) in enumerate(meta):
        check_case(res, i, path, L, (False, False), smu)


# ------------------------------------------------------------------ goldens, verdicts, edges ----------------------

def _golden_cases(golden_meta):
    out = []
    for name, verdicts in (("untrimmed", (False, True)), ("asymmetric", (True, False))):
        out.append((os.path.join(GOLDEN, "conditioning", name), golden_meta["_conditioning"][name]["e"], verdicts))
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_golden_conditioning_tables_and_a_table_needing_nothing(world, golden_meta):
    """golden conditioning/untrimmed (trim only), conditioning/asymmetric (symmetrise only), and dip_k21 at the L it
    already satisfies: no step, the replica the table's own entries"""
    from smudgeplot_b200 import fastk
    gold = _golden_cases(golden_meta)
    dip = os.path.join(GOLDEN, "dip_k21", "dip_k21")
    e = golden_meta["dip_k21"]["e"]
    cases = [{"path": p, "L": L, "ops": [("replica",)]} for p, L, _ in gold]
    cases.append({"path": dip, "L": e, "ops": [("replica",), ("smu",)]})
    res = run_ranks(world, cases)
    for i, (p, L, verdicts) in enumerate(gold):
        check_case(res, i, p, L, verdicts)
    keys, cnt = check_case(res, len(gold), dip, e, (True, True), open(dip + ".smu").read())
    kb, wc = fastk.unpack_host(fastk.read_ktab(dip))
    assert np.array_equal(keys, fastk.keys_bytes_to_u64(kb)) and np.array_equal(cnt, wc)
    for rank in range(world):
        st = res[rank][len(gold)]["stats"]
        assert st["steps"] == [] and st["sent"] == [0] * world


def edge_tables(tmp_path):
    """(path, L): palindromes at k = 8 and 64, both strands held with different counts, everything under one 20-bit
    prefix, L above every count, k = 33/40/64 over ibyte 1..3 and 1..4 parts"""
    from smudgeplot_b200 import fastk
    rng = np.random.default_rng(11)
    out = []

    def pack(strs, k):
        words = []
        for s in strs:
            v = 0
            for ch in s:
                v = (v << 2) | "ACGT".index(ch)
            v <<= (128 if k > 32 else 64) - 2 * k
            words.append((v >> 64, v & ((1 << 64) - 1)) if k > 32 else (v,))
        a = np.array(words, dtype=np.uint64)
        return a if k > 32 else a[:, 0]

    def rc(s):
        return s[::-1].translate(str.maketrans("ACGT", "TGCA"))

    def table(tag, k, strs, counts, ibyte=2, nparts=2):
        order = sorted(range(len(strs)), key=lambda i: strs[i])
        ku = pack([strs[i] for i in order], k)
        cn = np.array([counts[i] for i in order], dtype=np.uint16)
        return write(tmp_path, tag, k, ku, cn, ibyte, nparts)

    every8 = ["".join("ACGT"[(v >> (2 * (7 - j))) & 3] for j in range(8)) for v in range(1 << 16)]
    canon8 = sorted({min(s, rc(s)) for s in every8})                      # holds all 136 palindromes
    out.append((table("all8", 8, canon8, rng.integers(1, 30, len(canon8)).tolist(), 1, 1), 10))
    half = ["".join(rng.choice(list("ACGT"), 32)) for _ in range(300)]
    pal64 = sorted({h + rc(h) for h in half} | {min(s, rc(s)) for s in ("".join(rng.choice(list("ACGT"), 64))
                                                                           for _ in range(3000))})
    out.append((table("pal64", 64, pal64, rng.integers(1, 30, len(pal64)).tolist(), 3, 4), 5))
    base = sorted({"".join(rng.choice(list("ACGT"), 31)) for _ in range(4000)})
    both = {}
    for j, s in enumerate(base):                                          # some k-mers with both strands, the
        both[s] = int(rng.integers(1, 40))                                #   reverse complement's count different
        if j % 3 == 0 and rc(s) not in both:
            both[rc(s)] = int(rng.integers(1, 40))
    ks = sorted(both)
    out.append((table("both31", 31, ks, [both[s] for s in ks], 3, 3), 6))
    pre = "ACGTACGTAC"                                                    # one 20-bit prefix, symmetric: trim only
    mids = sorted({"".join(rng.choice(list("ACGT"), 11)) for _ in range(2000)})
    one = {}
    for mid in mids:
        s = pre + mid + rc(pre)
        one[s] = one.get(rc(s), int(rng.integers(1, 40)))
        one[rc(s)] = one[s]
    ks = sorted(one)
    out.append((table("oneprefix", 31, ks, [one[s] for s in ks], 3, 2), 12))
    out.append((table("oneprefix_symm", 31, [pre + m + "A" * 10 for m in mids], [20] * len(mids), 3, 2), 4))
    out.append((table("tiny", 31, ["C" * 31, "G" * 30 + "T"], [3, 5], 3, 1), 2))
    out.append((out[2][0], 1000))                                         # L above every count: empty
    for k, ibyte, nparts, seed in ((33, 1, 1, 41), (40, 2, 4, 42), (64, 3, 2, 43), (64, 1, 3, 44)):
        out.append((canonical_untrimmed(tmp_path, k, 20_000, 2, seed, ibyte, nparts, cov=30), 4))
    assert fastk.read_ktab(out[1][0]).kmer == 64
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_edge_tables_and_verdicts(world, tmp_path):
    tables = edge_tables(tmp_path)
    res = run_ranks(world, [{"path": p, "L": L, "ops": [("replica",)]} for p, L in tables])
    for i, (p, L) in enumerate(tables):
        keys, cnt = check_case(res, i, p, L)
        if L == 1000:
            assert len(cnt) == 0
    if world > 1:                                                        # everything under one prefix: one rank
        assert sum(sum(res[r][3]["stats"]["received"]) > 0 for r in range(world)) == 1   # owns it, the others none


def test_examine_probe_moves_past_a_palindrome_and_handles_tiny_tables(tmp_path):
    """entry 1 a palindrome at even k: the probe goes on to entry 2; tables of 0 and 1 entries"""
    from smudgeplot_b200 import fastk
    k = 32
    pal = "A" * 15 + "C" + "G" + "T" * 15
    strs = ["A" * 32, pal, "C" * 32]
    pack = lambda s: int("".join(str("ACGT".index(c)) for c in s), 4)   # noqa: E731
    p1 = write(tmp_path, "pal", k, np.array(sorted(pack(s) for s in strs), dtype=np.uint64), np.array([4, 4, 4], np.uint16),
               1, 1)
    p0 = write(tmp_path, "empty", 21, np.zeros(0, dtype=np.uint64), np.zeros(0, dtype=np.uint16), 1, 1)
    pone = write(tmp_path, "one", 21, np.array([7 << 40], dtype=np.uint64), np.array([3], np.uint16), 1, 1)
    cases = [(p1, 2), (p0, 2), (pone, 2), (pone, 5)]
    res = run_ranks(3, [{"path": p, "L": L, "ops": [("replica",)]} for p, L in cases])
    for i, (p, L) in enumerate(cases):
        check_case(res, i, p, L)
    assert fastk.read_ktab(p1).nels == 3


# ------------------------------------------------------------------ extract, budget, NCCL -------------------------

def test_extract_on_a_conditioned_job(tmp_path):
    """extract(pixmap) of the conditioned job = hetmers.Scan.extract of the in-core conditioned table"""
    from smudgeplot_b200 import fastk, hetmers
    from test_gpu_parity import write_labelled_sma
    from test_gpu_stream_dist_extract import records
    path = canonical_untrimmed(tmp_path, 31, 80_000, 3, 32)
    with hetmers.Scan(fastk.read_ktab(path)) as sc:
        sc.condition(12, True, True)
        plot, _ = sc.run()
        pix, _ = write_labelled_sma(plot, str(tmp_path / "ann.sma"))
        want = sc.extract(pix)
    assert len(want) > 0
    res = run_ranks(2, [{"path": path, "L": 12, "ops": [("extract", pix)]}])
    assert np.array_equal(records(res[0][0]["ops"][0]), want) and res[1][0]["ops"][0] is None


def test_a_budget_below_the_working_set_is_refused_on_every_rank(tmp_path):
    """HM_ENOMEM with the sizes on every rank, before anything is routed; the device memory of the call is
    returned, and the next from_ktab in the same group succeeds"""
    path = canonical_untrimmed(tmp_path, 21, 60_000, 2, 31)
    cases = [{"path": path, "L": 6, "budget": [None, 1 << 20]},
             {"path": path, "L": 6, "budget": 1 << 20},
             {"path": path, "L": 6, "ops": [("replica",), ("memory",)]}]
    res = run_ranks(2, cases)
    for rank in range(2):
        for i in (0, 1):
            code, msg = res[rank][i]["error"]
            before, after = res[rank][i]["memory"]
            assert code == -3 and "device bytes" in msg and str(1 << 20) in msg, (rank, msg)
            assert after == before, (rank, i, before, after)
    check_case([[r[2]] for r in res], 0, path, 6, (False, False))


def test_one_rank_per_gpu_over_nccl(tmp_path):
    from smudgeplot_b200 import _lib
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    path = canonical_untrimmed(tmp_path, 40, 50_000, 2, 34)
    res = run_ranks(2, [{"path": path, "L": 6, "ops": [("replica",)]}], backend="nccl")
    check_case(res, 0, path, 6, (False, False))

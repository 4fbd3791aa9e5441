"""GPU tests of conditioning a FastK table into new table files across the ranks of the one-process-per-GPU job
(dist.condition_ktab, DESIGN.md §4f; run with -m gpu).  World 1, 2 and 3 ranks are spawned with gloo, all on one
H100; an NCCL case runs with a GPU per rank where there are two.  The table written must hold what
hetmers.condition_table writes (stub index, kmer, ibyte, minval, and the records of all parts concatenated) and the
numpy restatement of trim + symmetrise; its parts are the ranks' with a non-empty output, each starting on a stub
bucket; the readers (the reference binary, the ranks' scans, extract) must see the table condition_table wrote."""
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def parts_on_buckets(kt):
    starts = set(np.concatenate([[0], kt.index]).tolist())
    return all(c in starts for c in np.cumsum(kt.part_nels).tolist())


def _op(op, dst, dev):
    from smudgeplot_b200 import dist as hd
    from smudgeplot_b200 import hetmers
    if op[0] in ("streamed_smu", "sharded_smu"):
        if op[0] == "streamed_smu":
            sc = hd.StreamedShardedScan(dst, device=f"cuda:{dev}")
        else:
            sc = hd.ShardedScan.from_ktab(dst, device=f"cuda:{dev}")
        try:
            return hetmers.smu_text(sc.scan().cpu().numpy())
        finally:
            sc.close()
    if op[0] == "streamed_extract":
        sc = hd.StreamedShardedScan(dst, device=f"cuda:{dev}")
        try:
            got = sc.extract(op[1], dst=0)
        finally:
            sc.close()
        return None if got is None else got.tobytes()
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
            budget = case.get("budget")
            if isinstance(budget, list):
                budget = budget[rank]
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            res = {}
            try:
                res["stats"] = hd.condition_ktab(case["src"], case["dst"], case["L"], device=f"cuda:{dev}",
                                                 budget=budget)
            except _lib.HetmersError as e:
                res["error"] = (e.code, str(e))
            torch.cuda.synchronize()
            res["memory"] = (before, torch.cuda.memory_allocated())
            res["ops"] = [] if "error" in res else [_op(op, case["dst"], dev) for op in case.get("ops", [])]
            out.append(res)
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{src, dst, L, budget (or one per rank), ops: ("streamed_smu",) | ("sharded_smu",) |
    ("streamed_extract", pixmap)}] -> per rank, per case: {"stats": condition_ktab's result, or "error": (code,
    message), "memory": (before, after), "ops": results}"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 39600 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(q.get(timeout=600) for _ in range(world))
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


def write(path, k, ku, cn, ibyte=3, nparts=3):
    from smudgeplot_b200 import fastk
    os.makedirs(os.path.dirname(path), exist_ok=True)
    fastk.write_ktab(path, k, ku, cn, ibyte=ibyte, nparts=nparts)
    return path


def canonical(k, target, seed, cov=40):
    """a canonical untrimmed table of about `target` entries (counts from 1): (uint64 keys, counts)"""
    from test_gpu_parity import canonical_mask
    from tools import synth
    G = synth.calibrate_G(k, 2 * target, 2, 0.02, cov, 1) if target > 100_000 else target
    keys, cnt = synth.synth_table(k, G, 2, 0.02, cov, 1, seed, device="cuda")
    keys, cnt = keys.cpu(), cnt.cpu()
    ku = synth.keys_to_u64_numpy(keys)
    cn = cnt.numpy().astype(np.uint16)
    canon = canonical_mask(keys, ku, k)
    return ku[canon], cn[canon]


def reference(src, dst, L):
    """condition_table's table, or None when the table needs neither step"""
    from smudgeplot_b200 import hetmers
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    return None if hetmers.condition_table(src, dst, L) is None else dst


def temporaries(d):
    return [f for f in os.listdir(d) if "tmp" in f]


def check(res, i, src, dst, ref, L, budget_bound=True):
    """every rank: the same result; the files = condition_table's = the numpy restatement, parts per non-empty rank
    on buckets, peak device bytes within the planned working set and the budget -> the stats of rank 0"""
    from smudgeplot_b200 import fastk
    from test_gpu_parity import _condition_numpy
    world = len(res)
    sts = [res[r][i]["stats"] for r in range(world)]
    assert all("error" not in res[r][i] for r in range(world)), [res[r][i].get("error") for r in range(world)]
    want, got = fastk.read_ktab(ref), fastk.read_ktab(dst)
    assert (got.kmer, got.ibyte, got.minval) == (want.kmer, want.ibyte, want.minval), dst
    assert np.array_equal(got.index, want.index), dst
    assert np.array_equal(got.all_records(), want.all_records()), dst
    kt = fastk.read_ktab(src)
    kb, cn = fastk.unpack_host(kt)
    ck, cc = _condition_numpy(fastk.keys_bytes_to_u64(kb), cn, kt.kmer, L, not sts[0]["trimmed"],
                              not sts[0]["symmetric"])
    gb, gc = fastk.unpack_host(got)
    assert np.array_equal(fastk.keys_bytes_to_u64(gb), ck) and np.array_equal(gc, cc), dst
    outs = [st["rank_entries_out"] for st in sts]
    assert sum(outs) == got.nels == sts[0]["entries_out"]
    if got.nels:
        assert got.nparts == sum(1 for x in outs if x > 0) and got.part_nels == [x for x in outs if x > 0]
        assert [st["part"] for st in sts] == [sum(1 for x in outs[:r + 1] if x > 0) if outs[r] else None
                                              for r in range(world)]
    assert parts_on_buckets(got)
    for st in sts:
        assert st["passes"] == sts[0]["passes"] and st["prefix_cuts"] == sts[0]["prefix_cuts"]
        assert len(st["ms"]["passes"]) == st["passes"]
        assert set(st["ms"]) >= {"load", "examine", "hist_and_plan", "commit", "writer_busy"}
        assert 0 < st["peak_bytes"] <= st["working_set_bytes"] <= st["budget"] or not budget_bound, st
    assert temporaries(os.path.dirname(dst)) == []
    return sts


# ------------------------------------------------------------------ three modes, 1-3 ranks -----------------------

L_MODES = 12


@pytest.fixture(scope="module")
def mode_tables(tmp_path_factory):
    """canonical untrimmed (trim + symmetrise), trimmed canonical (symmetrise), untrimmed symmetric (trim), at k = 31
    and 40, ibyte 3, 3 parts, each with condition_table's output"""
    from test_gpu_parity import _condition_numpy
    d = tmp_path_factory.mktemp("modes")
    out = []
    for k in (31, 40):
        ku, cn = canonical(k, 2_500_000, 60 + k)
        assert len(cn) > 2_000_000
        keep = cn >= L_MODES
        sk, sc = _condition_numpy(ku, cn, k, 1, False, True)
        for tag, (tk, tc), steps in (("raw", (ku, cn), ["trim", "symmetrise"]),
                                     ("trimmed", (ku[keep], cn[keep]), ["symmetrise"]),
                                     ("symmetric", (sk, sc), ["trim"])):
            src = write(str(d / f"{tag}{k}" / "src"), k, tk, tc)
            out.append((src, reference(src, str(d / f"{tag}{k}" / "ref"), L_MODES), steps))
    return out


@pytest.mark.parametrize("world", [1, 2, 3])
def test_three_modes_write_condition_tables_table(world, mode_tables):
    cases = [{"src": s, "dst": os.path.join(os.path.dirname(s), f"w{world}"), "L": L_MODES} for s, _, _ in mode_tables]
    res = run_ranks(world, cases)
    for i, (src, ref, steps) in enumerate(mode_tables):
        sts = check(res, i, src, cases[i]["dst"], ref, L_MODES)
        assert sts[0]["steps"] == steps


def test_small_budgets_take_three_passes_or_more(tmp_path):
    """budgets (found with the planning functions on numpy histograms) that leave every rank three sub-ranges or
    more: the same table, and the peak within every rank's budget"""
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    from test_gpu_condition_files import output_hist
    k, L, world, ibyte = 31, 8, 2, 2
    ku, cn = canonical(k, 2_000_000, 77)
    src = write(str(tmp_path / "src"), k, ku, cn, ibyte=ibyte)
    ref = reference(src, str(tmp_path / "ref"), L)
    n = len(cn)
    shares = [hd.share_range(n, world, r) for r in range(world)]
    locs = [np.stack([output_hist(ku[a:b], cn[a:b], k, L, True, False), output_hist(ku[a:b], cn[a:b], k, L, True, True)])
            for a, b in shares]
    h_all = sum(locs)
    hb = min(_lib.COND_HIST_BITS, 2 * k)
    cuts = hd.bucket_condition_cuts(h_all[1], world, hb, ibyte)
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
        if min(len(s) - 1 for s in subs) >= 3 and max(needs) <= budget:
            found = budget
    assert found is not None
    res = run_ranks(world, [{"src": src, "dst": str(tmp_path / "small"), "L": L, "budget": found},
                            {"src": src, "dst": str(tmp_path / "big"), "L": L}])
    small = check(res, 0, src, str(tmp_path / "small"), ref, L)
    big = check(res, 1, src, str(tmp_path / "big"), ref, L)
    assert all(len(st["sub_ranges"]) - 1 >= 3 for st in small) and small[0]["passes"] >= 3
    assert all(st["peak_bytes"] <= found for st in small) and big[0]["passes"] < small[0]["passes"]


# ------------------------------------------------------------------ edge tables -----------------------------------

def _pack(strs, k):
    words = []
    for s in strs:
        v = 0
        for ch in s:
            v = (v << 2) | "ACGT".index(ch)
        v <<= (128 if k > 32 else 64) - 2 * k
        words.append((v >> 64, v & ((1 << 64) - 1)) if k > 32 else (v,))
    a = np.array(words, dtype=np.uint64)
    return a if k > 32 else a[:, 0]


def _rc(s):
    return s[::-1].translate(str.maketrans("ACGT", "TGCA"))


def edge_tables(d):
    """(src, L): palindromes at k = 16, k = 12 at ibyte 1 and 2, k = 32 / 33 / 64, both strands held, one 20-bit
    prefix holding the output, L above every count"""
    rng = np.random.default_rng(17)
    out = []

    def table(tag, k, strs, counts, ibyte=2, nparts=2):
        order = sorted(range(len(strs)), key=lambda i: strs[i])
        ku = _pack([strs[i] for i in order], k)
        cn = np.array([counts[i] for i in order], dtype=np.uint16)
        return write(str(d / tag / "src"), k, ku, cn, ibyte, nparts)

    half = {"".join(rng.choice(list("ACGT"), 8)) for _ in range(3000)}
    pal16 = sorted({h + _rc(h) for h in half} | {min(s, _rc(s)) for s in ("".join(rng.choice(list("ACGT"), 16))
                                                                         for _ in range(20000))})
    out.append((table("pal16", 16, pal16, rng.integers(1, 30, len(pal16)).tolist(), 2, 3), 5))
    k12 = sorted({min(s, _rc(s)) for s in ("".join(rng.choice(list("ACGT"), 12)) for _ in range(60000))})
    for ibyte in (1, 2):
        out.append((table(f"k12_{ibyte}", 12, k12, rng.integers(1, 40, len(k12)).tolist(), ibyte, 2), 6))
    for k, ibyte, nparts, seed in ((32, 2, 3, 51), (33, 1, 2, 52), (64, 3, 2, 53)):
        ku, cn = canonical(k, 20_000, seed, cov=30)
        out.append((write(str(d / f"k{k}" / "src"), k, ku, cn, ibyte, nparts), 4))
    base = sorted({"".join(rng.choice(list("ACGT"), 31)) for _ in range(6000)})
    both = {}
    for j, s in enumerate(base):                                          # some k-mers with both strands, the
        both[s] = int(rng.integers(1, 40))                                #   reverse complement's count different
        if j % 3 == 0 and _rc(s) not in both:
            both[_rc(s)] = int(rng.integers(1, 40))
    ks = sorted(both)
    while _rc(ks[1]) in both:                                             # entry 1 without its reverse complement,
        del both[_rc(ks[1])]                                              #   so that the table is not symmetric
        ks = sorted(both)
    out.append((table("both31", 31, ks, [both[s] for s in ks], 3, 3), 6))
    pre = "ACGTACGTAC"                                                    # one 20-bit prefix, symmetric: trim only
    one = {}
    for mid in sorted({"".join(rng.choice(list("ACGT"), 11)) for _ in range(3000)}):
        s = pre + mid + _rc(pre)
        one[s] = one.get(_rc(s), int(rng.integers(1, 40)))
        one[_rc(s)] = one[s]
    ks = sorted(one)
    out.append((table("oneprefix", 31, ks, [one[s] for s in ks], 3, 2), 12))
    out.append((out[-2][0], 1000))                                        # L above every count: empty
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_edge_tables(world, tmp_path):
    from smudgeplot_b200 import fastk
    tables = edge_tables(tmp_path)
    cases, refs = [], []
    for j, (src, L) in enumerate(tables):
        cases.append({"src": src, "dst": str(tmp_path / f"out{j}" / "t"), "L": L})
        os.makedirs(os.path.dirname(cases[-1]["dst"]))
        refs.append(reference(src, str(tmp_path / f"ref{j}" / "t"), L))
    res = run_ranks(world, cases)
    for j, (src, L) in enumerate(tables):
        sts = check(res, j, src, cases[j]["dst"], refs[j], L)
        if L == 1000:                                                     # empty everywhere: condition_table's
            assert sts[0]["entries_out"] == 0 and all(st["part"] is None for st in sts)   # files, byte for byte
            want, got = fastk.read_ktab(refs[j]), fastk.read_ktab(cases[j]["dst"])
            assert got.nparts == want.nparts == fastk.read_ktab(src).nparts
            for p in range(1, want.nparts + 1):
                assert open(fastk.part_path(refs[j], p), "rb").read() == \
                    open(fastk.part_path(cases[j]["dst"], p), "rb").read()
            assert open(fastk.stub_path(refs[j]), "rb").read() == open(fastk.stub_path(cases[j]["dst"]), "rb").read()
        if "oneprefix" in src and L == 12:                                # one rank owns the output: one part
            assert fastk.read_ktab(cases[j]["dst"]).nparts == 1
            assert sum(st["rank_entries_out"] > 0 for st in sts) == 1
        if "both31" in src:
            assert sts[0]["steps"] == ["trim", "symmetrise"]


# ------------------------------------------------------------------ readers ---------------------------------------

def test_readers_see_condition_tables_table(tmp_path):
    """the reference binary, StreamedShardedScan / ShardedScan.from_ktab's scans and StreamedShardedScan.extract on
    the new table give what they give on condition_table's"""
    import oracle_util as ou
    from smudgeplot_b200 import fastk, hetmers
    from test_gpu_parity import write_labelled_sma
    from test_gpu_stream_dist_extract import records
    L = 12
    ku, cn = canonical(31, 80_000, 32)
    src = write(str(tmp_path / "src"), 31, ku, cn)
    ref = reference(src, str(tmp_path / "ref"), L)
    with hetmers.Scan(fastk.read_ktab(ref)) as sc:
        plot, _ = sc.run()
        pix, _ = write_labelled_sma(plot, str(tmp_path / "ann.sma"))
        want_pairs = sc.extract(pix)
    smu = hetmers.smu_text(plot)
    assert len(want_pairs) > 0 and len(smu) > 0
    dst = str(tmp_path / "dst")
    res = run_ranks(2, [{"src": src, "dst": dst, "L": L,
                         "ops": [("streamed_smu",), ("sharded_smu",), ("streamed_extract", pix)]}])
    check(res, 0, src, dst, ref, L)
    for rank in range(2):
        got_stream, got_sharded, got_pairs = res[rank][0]["ops"]
        assert got_stream == smu and got_sharded == smu, rank
        assert (got_pairs is None) == (rank != 0)
    assert np.array_equal(records(res[0][0]["ops"][2]), want_pairs)
    if ou.have_ref():
        a = ou.run_ref(dst, str(tmp_path / "a"), L)
        b = ou.run_ref(ref, str(tmp_path / "b"), L)
        assert a.returncode == 0 and b.returncode == 0, (a.stderr, b.stderr)
        assert open(str(tmp_path / "a.smu")).read() == open(str(tmp_path / "b.smu")).read() == smu


# ------------------------------------------------------------------ refusals, NCCL --------------------------------

def test_refusals(tmp_path, golden_meta):
    """a table needing neither step: None everywhere, nothing written; a dst naming the source: HM_EINVAL everywhere
    before anything is written; one rank's budget below its working set: HM_ENOMEM everywhere with the sizes, no file
    under dst's names, no temporary, device memory returned, and the next call in the group succeeds"""
    import shutil
    from smudgeplot_b200 import fastk
    dip = os.path.join(GOLDEN, "dip_k21", "dip_k21")
    L = 6
    ku, cn = canonical(21, 60_000, 31)
    d = tmp_path / "t"
    src = write(str(d / "src"), 21, ku, cn)
    ref = reference(src, str(tmp_path / "ref"), L)
    before = sorted(os.listdir(d))
    tiny = 1 << 20
    nothing = str(d / "nothing")
    shutil.copy(fastk.stub_path(dip), str(d / "dip.ktab"))
    for p in range(1, fastk.read_ktab(dip).nparts + 1):
        shutil.copy(fastk.part_path(dip, p), fastk.part_path(str(d / "dip"), p))
    before = sorted(os.listdir(d))
    cases = [{"src": str(d / "dip"), "dst": nothing, "L": golden_meta["dip_k21"]["e"]},
             {"src": src, "dst": src, "L": L},
             {"src": src, "dst": str(d / "src.ktab"), "L": L},
             {"src": src, "dst": str(d / "dst"), "L": L, "budget": [None, tiny]},
             {"src": src, "dst": str(d / "dst"), "L": L}]
    res = run_ranks(2, cases)
    for rank in range(2):
        assert res[rank][0]["stats"] is None and "error" not in res[rank][0]
        for i in (1, 2):
            code, msg = res[rank][i]["error"]
            assert code == -1 and "names the source" in msg, (rank, msg)
        code, msg = res[rank][3]["error"]
        assert code == -3 and "device bytes" in msg and str(tiny) in msg, (rank, msg)
        for i in (1, 2, 3):
            m0, m1 = res[rank][i]["memory"]
            assert m0 == m1, (rank, i, m0, m1)
    assert sorted(f for f in os.listdir(d) if not f.startswith(("dst", ".dst"))) == before
    check(res, 4, src, str(d / "dst"), ref, L)
    assert fastk.read_ktab(src).nels == len(cn)


def test_one_rank_per_gpu_over_nccl(tmp_path):
    from smudgeplot_b200 import _lib
    if _lib.lib().hm_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ku, cn = canonical(40, 50_000, 34)
    src = write(str(tmp_path / "src"), 40, ku, cn)
    ref = reference(src, str(tmp_path / "ref"), 6)
    res = run_ranks(2, [{"src": src, "dst": str(tmp_path / "dst"), "L": 6}], backend="nccl")
    check(res, 0, src, str(tmp_path / "dst"), ref, 6)

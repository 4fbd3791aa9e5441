"""GPU tests of extract_kmer_pairs' pair files written by the ranks of a one-process-per-GPU job
(dist.ShardedScan.write_pairs, dist.StreamedShardedScan.write_pairs, csrc/hm_pairs.cu, DESIGN.md §6b; run with -m gpu).
World 1, 2 and 3 ranks are spawned with gloo, all on one H100; every label file must be byte for byte the file
`extract_kmer_pairs -o<o> <table> <sma>` writes, and the seeded tables' files must carry the reference binary's
sorted-line digests (tests/golden/reference_runs/extract.json)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

from conftest import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

SMA_GOLDENS = ["dip_k21", "dip_k40", "tet_k32"]


def _run_case(hd, case, dev):
    """one write_pairs call (and the ops around it) on this rank -> what the test compares"""
    kind = case["kind"]
    if kind == "streamed":
        os.environ["HETMERS_STREAM_CHUNK"] = str(case["chunk"])
        sc = hd.StreamedShardedScan(case["path"], device=f"cuda:{dev}", budget=case["scan_budget"])
    else:
        sc = hd.ShardedScan.from_ktab(case["path"], device=f"cuda:{dev}", path=kind)
    try:
        tm = {}
        st = sc.write_pairs(case["sma"], case["out"], timings=tm, budget=case.get("budget"))
        st["phases"] = sorted(tm)
        after = None
        if case.get("extract_after"):
            from smudgeplot_b200.hetmers import read_sma
            got = sc.extract(read_sma(case["sma"])[0], dst=0)
            after = None if got is None else got.tobytes()
        return ("ok", st, after)
    finally:
        sc.close()


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
            try:
                out.append(_run_case(hd, case, dev))
            except (_lib.HetmersError, RuntimeError, ValueError, OSError) as e:
                out.append(("error", type(e).__name__, str(e)))
        q.put((rank, out))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def run_ranks(world, cases, backend="gloo"):
    """cases: [{kind: symm | direct | streamed, path, sma, out, budget, ...}] -> per rank, per case:
    ("ok", stats, extract-after bytes or None) | ("error", exception type, message)"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 36500 + (os.getpid() % 2000) + 10 * world + (5 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=1800) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


def executable_files(table, sma, out, e=None):
    """{label name: bytes} of what extract_kmer_pairs writes"""
    from smudgeplot_b200 import hetmers
    hetmers.run_extract(table, sma, o=out, e=e)
    return label_files(out, hetmers.read_sma(sma)[1])


def label_files(out, labels):
    got = {}
    for a, b in labels:
        with open(f"{out}.{a}A{b}B.txt", "rb") as f:
            got[f"{a}A{b}B"] = f.read()
    return got


def stream_budget(kt, world):
    from test_gpu_stream_dist_extract import rank_budget
    return rank_budget(kt.nels, kt.kmer, kt.ibyte, world)


def golden_cases(tmp_path, world, kinds=("symm", "direct", "streamed")):
    from smudgeplot_b200 import fastk
    cases, wants = [], []
    for name in SMA_GOLDENS:
        path = os.path.join(GOLDEN, name, name)
        kt = fastk.read_ktab(path)
        want = executable_files(path, path + ".sma", str(tmp_path / f"exe_{name}"))
        for kind in kinds:
            cases.append({"kind": kind, "path": path, "sma": path + ".sma", "out": str(tmp_path / f"{kind}_w{world}_{name}"),
                          "scan_budget": stream_budget(kt, world), "chunk": max(256, -(-kt.nels // (3 * world)))})
            wants.append(want)
    return cases, wants


def check_files(res, cases, wants):
    from smudgeplot_b200.hetmers import read_sma
    for i, (case, want) in enumerate(zip(cases, wants)):
        for rank, per_case in enumerate(res):
            assert per_case[i][0] == "ok", (rank, case["kind"], per_case[i])
        got = label_files(case["out"], read_sma(case["sma"])[1])
        assert got == want, (case["kind"], case["path"], {k: (len(got[k]), len(want[k])) for k in want})
        st = res[0][i][1]
        assert st["lines"] == {k: v.count(b"\n") for k, v in want.items()}
        assert st["records"] == sum(st["lines"].values())


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(built):
    from smudgeplot_b200 import _lib
    assert _lib.lib().hm_device_count() >= 1, "these tests need a CUDA device (no CPU fallback exists)"


@pytest.mark.parametrize("world", [1, 2, 3])
def test_golden_files_are_the_executables(world, tmp_path):
    """both ShardedScan routes and StreamedShardedScan: every label file of the three .sma goldens byte for byte"""
    cases, wants = golden_cases(tmp_path, world)
    res = run_ranks(world, cases)
    check_files(res, cases, wants)
    for per_case in res:
        for what, st, _ in per_case:
            assert st["passes"] == 1 and st["windows"] == world
            assert {"hist_and_plan", "route", "all_to_all", "sort", "format", "text_d2h", "write"} <= set(st["phases"])


@pytest.mark.parametrize("world", [2, 3])
def test_seeded_tables_carry_the_reference_digests(world, tmp_path):
    """test_gpu_parity.EXTRACT_CASES (k = 31 and 40): the files are the executable's, and their sorted lines carry
    the reference binary's digests"""
    import oracle_util as ou
    from smudgeplot_b200 import hetmers
    from test_gpu_parity import EXTRACT_CASES, write_labelled_sma
    from tools import synth
    cases, wants, digests = [], [], []
    for k, G, ploidy, seed, L in EXTRACT_CASES:
        keys, cnt = synth.synth_table(k, G, ploidy, 0.02, 20 * ploidy, L, seed, device="cuda")
        name = str(tmp_path / f"t{k}")
        kt = synth.write_table(name, k, keys, cnt, ibyte=3, nparts=3)
        with hetmers.Scan(kt) as sc:
            plot, _ = sc.run("symm")
        sma = str(tmp_path / f"ann{k}.sma")
        write_labelled_sma(plot, sma)
        want = executable_files(name, sma, str(tmp_path / f"exe{k}"), e=L)
        for kind in ("symm", "direct", "streamed"):
            cases.append({"kind": kind, "path": name, "sma": sma, "out": str(tmp_path / f"{kind}{k}"),
                          "scan_budget": stream_budget(kt, world), "chunk": max(256, -(-kt.nels // (3 * world)))})
            wants.append(want)
            digests.append(ou.reference_pair_digests(k, seed))
    res = run_ranks(world, cases)
    check_files(res, cases, wants)
    for case, want, dg in zip(cases, wants, digests):
        lines = {lab: sorted(b.decode().splitlines()) for lab, b in want.items()}
        assert ou.pair_digests(lines) == dg


def test_a_small_budget_takes_three_passes(tmp_path):
    """a file-phase budget with room for about a sixth of the records per window: three or more passes at world 2,
    the same bytes, and every rank's peak within the budget"""
    from smudgeplot_b200 import _lib, fastk
    from smudgeplot_b200 import dist as hd
    name = "dip_k40"
    path = os.path.join(GOLDEN, name, name)
    kt = fastk.read_ktab(path)
    want = executable_files(path, path + ".sma", str(tmp_path / "exe"))
    total = sum(v.count(b"\n") for v in want.values())
    budget = int(_lib.lib().hm_pairs_bytes(kt.kmer, max(total // 6, 1)))
    assert hd.pairs_room(kt.kmer, budget) >= total // 6
    cases = [{"kind": kind, "path": path, "sma": path + ".sma", "out": str(tmp_path / kind), "budget": budget,
              "scan_budget": stream_budget(kt, 2), "chunk": max(256, -(-kt.nels // 6))}
             for kind in ("symm", "streamed")]
    res = run_ranks(2, cases)
    check_files(res, cases, [want, want])
    for per_case in res:
        for _, st, _ in per_case:
            assert st["passes"] >= 3 and st["windows"] == 2 * st["passes"], st
            assert 0 < st["peak_bytes"] <= budget, st


def test_empty_label_truncation_refusals_and_extract_after(tmp_path):
    """a label with no pair gets an empty file, an existing longer file is truncated, extract() after write_pairs
    lists the in-core records; a malformed .sma and an oversized prefix raise on every rank and leave no file"""
    from smudgeplot_b200 import _lib, fastk, hetmers
    name = "dip_k21"
    path = os.path.join(GOLDEN, name, name)
    kt = fastk.read_ktab(path)
    sma = str(tmp_path / "extra.sma")
    with open(path + ".sma") as f:
        text = f.read()
    with open(sma, "w") as f:                                  # a smudge on a pixel no pair reaches
        f.write(text + "490\t500\t0\t9A1B\n")
    out = str(tmp_path / "o")
    with open(out + ".1A1B.txt", "w") as f:
        f.write("x" * 10_000_000)
    want = executable_files(path, sma, str(tmp_path / "exe"))
    assert want["9A1B"] == b""
    with hetmers.Scan(kt) as sc:
        sc.run()
        incore = sc.extract(hetmers.read_sma(sma)[0])
    bad = str(tmp_path / "bad.sma")
    with open(bad, "w") as f:
        f.write("covB\tcovA\tfreq\tsmudge\n3 4 5 1A2B\n")
    cases = [{"kind": "symm", "path": path, "sma": sma, "out": out, "extract_after": True},
             {"kind": "symm", "path": path, "sma": bad, "out": str(tmp_path / "b")},
             {"kind": "symm", "path": path, "sma": path + ".sma", "out": str(tmp_path / "c"),
              "budget": int(_lib.lib().hm_pairs_bytes(kt.kmer, 0))}]                # room for no record
    res = run_ranks(2, cases)
    check_files(res, cases[:1], [want])
    assert np.array_equal(np.frombuffer(res[0][0][2], dtype=incore.dtype), incore) and res[1][0][2] is None
    for rank in range(2):
        assert res[rank][1][:2] == ("error", "ValueError") and "not a valid smudge label" in res[rank][1][2]
        assert res[rank][2][:2] == ("error", "HetmersError") and "beyond the 0 records" in res[rank][2][2], res[rank][2]
    left = sorted(os.listdir(tmp_path))
    assert not any(f.startswith("b.") or f.startswith("c.") for f in left), left


def test_device_sort_and_format_in_one_process():
    """hm_k_pairs_sort against hm_sort_pair_records on records with many ties, and hm_k_pairs_format against
    pair_line at k = 2, 31, 32, 33 and 64"""
    import torch
    from smudgeplot_b200 import _lib
    from smudgeplot_b200 import dist as hd
    from smudgeplot_b200.device import _ptr, _stream
    from test_dist_extract import records
    from test_symm_extract_rule import pair_line
    L = _lib.lib()
    for n in (1, 2, 1000, 300_000):
        r = records(3, n, 5)
        want = hd.sort_pair_records(r.copy())
        a = torch.from_numpy(r.view(np.uint8).copy()).cuda()
        b = torch.empty_like(a)
        scratch = torch.empty(max(L.hm_pairs_sort_scratch_bytes(n), 1), dtype=torch.uint8, device="cuda")
        in_alt = C.c_int()
        _lib.check(L.hm_k_pairs_sort(_ptr(a), _ptr(b), n, _ptr(scratch), scratch.numel(), C.byref(in_alt), _stream()))
        got = (b if in_alt.value else a).cpu().numpy().view(want.dtype)
        assert np.array_equal(got, want), n
        assert L.hm_pairs_sort_scratch_bytes(n) <= L.hm_pairs_bytes(64, n) - 2 * 24 * n
    rng = np.random.default_rng(11)
    for k in (2, 31, 32, 33, 64):
        n = 1000 + k
        r = records(0, n, k)
        W = 64 if k <= 32 else 128
        mask = ((1 << (2 * k)) - 1) << (W - 2 * k)
        keys = [int(x) & mask for x in rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * 2 + 1] if k <= 32 else \
            [((int(h) << 64) | int(lo)) & mask for h, lo in zip(rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * 2,
                                                                rng.integers(0, 1 << 63, size=n, dtype=np.uint64) * 2 + 1)]
        r["key_hi"] = [x >> 64 if k > 32 else x for x in keys]
        r["key_lo"] = [x & ((1 << 64) - 1) if k > 32 else 0 for x in keys]
        r["pos"] = rng.integers(0, k, size=n)
        d = torch.from_numpy(r.view(np.uint8).copy()).cuda()
        text = torch.empty(n * (k + 5), dtype=torch.uint8, device="cuda")
        _lib.check(L.hm_k_pairs_format(_ptr(d), n, k, _ptr(text), _stream()))
        want = "".join(pair_line(x, k, int(p), int(a)) + "\n" for x, p, a in zip(keys, r["pos"], r["alt"]))
        assert text.cpu().numpy().tobytes().decode() == want, k


def test_one_rank_per_gpu_over_nccl(tmp_path):
    from smudgeplot_b200 import _lib
    ngpu = _lib.lib().hm_device_count()
    if ngpu < 2:
        pytest.skip("needs 2 GPUs")
    cases, wants = golden_cases(tmp_path, ngpu)
    res = run_ranks(ngpu, cases, backend="nccl")
    check_files(res, cases, wants)

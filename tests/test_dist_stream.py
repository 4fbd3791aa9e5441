"""world-size 2 and 3 gloo tests (CPU) of the host logic of a job whose ranks stream their own shares
(dist.StreamedShardedScan, DESIGN.md §4c, *Ranks*): the cuts every rank computes from the table files, the
fingerprint verdict, the Bloom segment all-gather, the per-round all_to_all of the query keys and of the answers
with per-owner splits, and the plot all-reduce.  The per-rank compute is stood in for by the restatement in
test_stream_route_rule.py; the summed plot must equal the oracle's."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K, N0, CMAX, SEED, SEG_BITS, SLICE = 21, 1500, 40, 1, 61, 64


def _fp(keys, cnt, k, lo, hi):
    """stand-in for the fingerprint sums: {(x, c)} and {(rc x, c)} summed mod 2^64 over [lo, hi)"""
    import oracle_util as ou
    m, a, b = (1 << 64) - 1, 0, 0
    for x, c in zip(keys[lo:hi].tolist(), cnt[lo:hi].tolist()):
        a = (a + (x * 0x9E3779B97F4A7C15 + c) * 0xC2B2AE3D27D4EB4F) & m
        b = (b + (ou._rc(x, k) * 0x9E3779B97F4A7C15 + c) * 0xC2B2AE3D27D4EB4F) & m
    s = lambda v: v - (1 << 64) if v >= (1 << 63) else v       # noqa: E731
    return torch.tensor([s(a), 0, s(b), 0], dtype=torch.int64)


def _worker(rank, world, port, table, drop, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from smudgeplot_b200 import dist as hd
        from smudgeplot_b200 import fastk
        from test_stream_route_rule import Rank
        kt = fastk.read_ktab(table)
        cuts = hd.file_run_aligned_cuts(kt, world)
        every = [torch.empty(world + 1, dtype=torch.int64) for _ in range(world)]
        dist.all_gather(every, torch.tensor(cuts, dtype=torch.int64))
        assert all(e.tolist() == cuts for e in every)
        kb, cnt = fastk.unpack_host(kt)                  # (the restated pass 1 reads the entries it scans)
        keys = fastk.keys_bytes_to_u64(kb)
        if not hd.fingerprint_verdict(_fp(keys, cnt, K, cuts[rank], cuts[rank + 1])):
            q.put((rank, "asymmetric", None, None))
            return
        rk = Rank(keys, cnt, K, cuts, rank, SEG_BITS)
        seg = torch.zeros((world, SEG_BITS), dtype=torch.uint8)
        seg[rank] = torch.from_numpy(rk.seg)
        hd.exchange_segments(seg, rank)
        segs = [s.numpy() for s in seg]
        lim = torch.tensor([SLICE, -len(rk.cand)], dtype=torch.int64)
        dist.all_reduce(lim, op=dist.ReduceOp.MIN)
        slice_ = max(1, min(int(lim[0]), -int(lim[1])))
        rounds = torch.tensor([(len(rk.cand) + slice_ - 1) // slice_])
        dist.all_reduce(rounds, op=dist.ReduceOp.MAX)
        sent = [0] * world
        for rd in range(int(rounds)):
            c0, c1 = min(rd * slice_, len(rk.cand)), min((rd + 1) * slice_, len(rk.cand))
            pend, queries = rk.resolve(c0, c1, segs)
            out_c = [len(queries.get(o, [])) for o in range(world)]
            send = torch.tensor([x - (1 << 64) if x >= (1 << 63) else x for o in range(world)
                                 for x, _ in queries.get(o, [])], dtype=torch.int64)
            slots = [s for o in range(world) for _, s in queries.get(o, [])]
            rc = torch.empty(world, dtype=torch.int64)
            dist.all_to_all_single(rc, torch.tensor(out_c, dtype=torch.int64))
            in_c = rc.tolist()
            recv = torch.empty(sum(in_c), dtype=torch.int64)
            hd._all_to_all(recv, send, in_c, out_c, None)
            ans = torch.tensor(rk.answer([v & ((1 << 64) - 1) for v in recv.tolist()]), dtype=torch.uint8)
            back = torch.empty(sum(out_c), dtype=torch.uint8)
            hd._all_to_all(back, ans, out_c, in_c, None)
            rk.settle(pend, {s for s, a in zip(slots, back.tolist()) if a})
            for o, c in enumerate(out_c):
                sent[o] += c
        plot = torch.from_numpy(rk.plot.reshape(-1).copy())
        hd.allreduce_plot(plot)
        q.put((rank, "ok", plot.numpy().copy(), sent))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _run(world, table, drop=False):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000) + world + 7 * drop
    procs = [ctx.Process(target=_worker, args=(r, world, port, table, drop, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(world)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return res


@pytest.mark.parametrize("world", [2, 3])
def test_streamed_ranks_host_logic_gloo(world, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_util as ou
    from smudgeplot_b200 import fastk
    from test_symm_identity import _symmetric_table
    keys, cnt = _symmetric_table(K, N0, CMAX, SEED)
    fastk.write_ktab(str(tmp_path / "t"), K, keys, cnt, ibyte=2, nparts=2)
    want, _ = ou.oracle_scan(fastk.keys_u64_to_bytes(keys, K), cnt, K)
    res = _run(world, str(tmp_path / "t"))
    for rank, what, plot, sent in res:
        assert what == "ok"
        assert np.array_equal(plot.reshape(want.shape), want)
        assert all(c > 0 for o, c in enumerate(sent) if o != rank), sent     # the filter is full of false hits


def test_asymmetric_table_is_refused_on_every_rank(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from smudgeplot_b200 import fastk
    from test_symm_identity import _symmetric_table
    keys, cnt = _symmetric_table(K, N0, CMAX, SEED)
    keep = np.ones(len(keys), dtype=bool)
    keep[len(keys) // 3] = False
    fastk.write_ktab(str(tmp_path / "a"), K, keys[keep], cnt[keep], ibyte=2, nparts=2)
    assert [r[1] for r in _run(3, str(tmp_path / "a"), drop=True)] == ["asymmetric"] * 3

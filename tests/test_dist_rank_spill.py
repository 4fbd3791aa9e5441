"""world-size 2 and 3 gloo tests (CPU) of the agreement a job whose ranks may keep their lists in host memory runs
(dist.pass1_agreement, dist.raise_on_any_rank; DESIGN.md §4c, *Lists in host memory*): one all-gather after pass 1
gives every rank the fingerprint verdict and whether any rank spilled, and a rank that failed at any of the points
where the mode can fail makes every rank raise, naming it, with no rank left waiting in a later collective."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, spill_ranks, fail_at, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out = []
    try:
        from smudgeplot_b200 import _lib
        from smudgeplot_b200 import dist as hd
        cpu = torch.device("cpu")
        fp = [(rank + 1) * 7, 0, (rank + 1) * 7, 0]           # symmetric sums
        err = None
        if fail_at == ("pass1", rank):
            err = _lib.HetmersError(-3, f"rank {rank}'s lists need 6000 bytes of host memory")
        try:
            sym, spilled = hd.pass1_agreement(fp, rank in spill_ranks, err, cpu)
            out.append(("pass1", sym, spilled))
            err = _lib.HetmersError(-3, "plan refused") if fail_at == ("prepare", rank) else None
            hd.raise_on_any_rank(err, "preparing pass 2", cpu)
            out.append(("prepare", True))
            err = _lib.HetmersError(-2, "status") if fail_at == ("status", rank) else None
            hd.raise_on_any_rank(err, "the rounds", cpu)
            out.append(("done", True))
        except _lib.HetmersError as e:
            out.append(("raised", e.code, str(e)))
        x = torch.tensor([1])                                   # the next collective: nobody is left behind
        dist.all_reduce(x)
        out.append(("after", int(x)))
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def _run(world, spill_ranks=(), fail_at=None):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 34700 + (os.getpid() % 2000) + 10 * world
    procs = [ctx.Process(target=_worker, args=(r, world, port, tuple(spill_ranks), fail_at, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


@pytest.mark.parametrize("world", [2, 3])
def test_one_rank_spilling_is_every_ranks_mode(world):
    for spill in ((), (world - 1,)):
        res = _run(world, spill)
        for r in range(world):
            assert res[r][0] == ("pass1", True, bool(spill))
            assert res[r][-1] == ("after", world)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("where", ["pass1", "prepare", "status"])
def test_a_failing_rank_raises_on_every_rank(world, where):
    bad = world - 1
    res = _run(world, (0,), (where, bad))
    for r in range(world):
        raised = [x for x in res[r] if x[0] == "raised"]
        assert len(raised) == 1, res[r]
        _, code, msg = raised[0]
        assert code == (-2 if where == "status" else -3)
        if r != bad:
            assert f"on rank {bad}" in msg, msg
        assert res[r][-1] == ("after", world)

"""world-size 2 and 3 gloo tests (CPU) of dist.gather_pairs, which moves the ranks' pair records to one rank of a
job whose ranks list extract_kmer_pairs' pairs of their own shares (dist.StreamedShardedScan.extract, DESIGN.md
§4c, *Ranks*).  The gathered list must hold every rank's records, in the order hm_scan_extract returns
(hm_sort_pair_records: smudge, key, position, alternative base), on the chosen rank only."""
import os
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORDER = ["smudge", "key_hi", "key_lo", "pos", "alt"]


def records(rank, n, seed=0):
    """n random records of rank `rank` (few labels, keys with repeats, so that every sort field matters)"""
    from smudgeplot_b200.hetmers import PAIR_DTYPE
    rng = np.random.default_rng(1000 * seed + rank)
    r = np.zeros(n, dtype=PAIR_DTYPE)
    r["smudge"] = rng.integers(1, 6, size=n)
    r["key_hi"] = rng.integers(0, 1 << 62, size=n, dtype=np.uint64) << np.uint64(2)   # (all 64 bits, top ones too)
    r["key_hi"][: n // 3] = r["key_hi"][:1]
    r["key_lo"] = rng.integers(0, 3, size=n)
    r["pos"] = rng.integers(0, 40, size=n)
    r["alt"] = rng.integers(0, 4, size=n)
    return r


def _worker(rank, world, port, sizes, dst, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from smudgeplot_b200 import dist as hd
        got = hd.gather_pairs(records(rank, sizes[rank], len(sizes)), dst)
        q.put((rank, None if got is None else got.tobytes()))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _run(world, sizes, dst):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 32700 + (os.getpid() % 2000) + 10 * world + dst
    procs = [ctx.Process(target=_worker, args=(r, world, port, sizes, dst, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [res[r] for r in range(world)]


@pytest.mark.parametrize("world,sizes,dst", [(2, [300, 0], 0), (2, [0, 500], 1), (2, [70000, 1000], 1),
                                             (3, [200, 0, 400], 2), (3, [0, 0, 0], 1), (3, [50, 60, 0], 0)])
def test_gather_pairs_over_gloo(world, sizes, dst, built):
    from smudgeplot_b200.hetmers import PAIR_DTYPE
    res = _run(world, sizes, dst)
    every = np.concatenate([records(r, sizes[r], world) for r in range(world)])
    want = np.sort(every, order=ORDER)
    for rank, got in enumerate(res):
        if rank != dst:
            assert got is None
            continue
        got = np.frombuffer(got, dtype=PAIR_DTYPE)
        assert len(got) == sum(sizes)
        assert np.array_equal(got, want)


def test_sort_pair_records_is_hm_scan_extracts_order(built):
    """past 2^16 records hm_sort_pair_records buckets by (smudge, first 8 bases) before its qsort; either way the
    order is (smudge, key_hi, key_lo, pos, alt)"""
    from smudgeplot_b200 import dist as hd
    for n in (1, 1000, 70000):
        r = records(0, n, 7)
        want = np.sort(r, order=ORDER)
        assert np.array_equal(hd.sort_pair_records(r.copy()), want)

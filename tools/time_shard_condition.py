#!/usr/bin/env python3
"""Conditioning across the ranks of the one-process-per-GPU job (dist.ShardedScan.from_ktab(L=...), DESIGN.md §4e)
against the in-core hm_scan_condition (hetmers.Scan.condition, rank 0) and against condition_kmer_table's route
(hetmers.Scan.condition_files on rank 0, then from_ktab of the new table on every rank), on the canonical untrimmed
k = 31 table of tools/time_condition.py (~2e8 entries, L = bench.py's LCUT = 12).  The table is written once as FastK
files to a temporary directory.  The arms alternate in every round after `warmup` rounds; per rank the conditioning's
phases (load, examine, histogram and plan, route, exchange, sort and merge, gather).  Prints one JSON line on rank 0
with the card name and power limit; exits 3 unless every rank's replica equals the in-core conditioned table.
Writes nothing to the tree.

    torchrun --nproc-per-node W tools/time_shard_condition.py [--nels 2e8] [--steps 2] [--warmup 1]

Several ranks run NCCL when there is a GPU per rank, else gloo with every rank on GPU 0 (the ranks then share the
card and their collectives go through host memory).
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_stream import power_limit  # noqa: E402


def _digest(keys, cnt):
    import hashlib
    h = hashlib.sha256(np.ascontiguousarray(keys).tobytes())
    h.update(np.ascontiguousarray(cnt).tobytes())
    return len(cnt), h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8, help="entries of the canonical untrimmed table")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd, fastk, hetmers
    if not torch.cuda.is_available():
        raise SystemExit("time_shard_condition.py needs a CUDA device: conditioning has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_shard_condition.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29747")
    nccl = world > 1 and torch.cuda.device_count() >= world
    dev = torch.device("cuda", rank if nccl else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=world)
    tmp = tempfile.TemporaryDirectory() if rank == 0 else None

    def say(msg):
        sys.stderr.write(f"time_shard_condition[{rank}]: {msg}\n")
        sys.stderr.flush()

    def free():
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        dist.barrier()

    try:
        names = [None, None]
        if rank == 0:                                          # the table files (setup, untimed)
            G = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
            keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, 1, SEED, device=dev)
            keep = keys <= synth.revcomp_left(keys, K)
            names = [os.path.join(tmp.name, "raw"), os.path.join(tmp.name, "cond")]
            synth.write_table(names[0], K, keys[keep].contiguous(), cnt[keep].contiguous(), ibyte=3, nparts=4)
            del keys, cnt, keep
            torch.cuda.empty_cache()
        dist.broadcast_object_list(names, src=0)
        raw, cond = names
        n = fastk.read_ktab(raw).nels
        rounds = {"shard": [], "in_core": [], "files": []}
        ok = True
        for i in range(a.warmup + a.steps):
            r = {}
            free()
            t0 = time.perf_counter()
            sc = hd.ShardedScan.from_ktab(raw, L=LCUT)
            torch.cuda.synchronize(dev)
            dist.barrier()
            r["shard"] = {"ms": (time.perf_counter() - t0) * 1e3, "phases": sc.stats["condition"]["ms"],
                          "stats": {k: v for k, v in sc.stats["condition"].items() if k not in ("ms", "prefix_cuts")}}
            if i == 0:                                          # every replica against the in-core table
                digest = [None]
                if rank == 0:
                    with hetmers.Scan(fastk.read_ktab(raw)) as s:
                        s.condition(LCUT, True, True)
                        digest[0] = _digest(*s.download(deg=False)[:2])
                dist.broadcast_object_list(digest, src=0)
                mine = _digest(sc.table.keys.cpu().numpy().view(np.uint64), sc.table.cnt.cpu().numpy().view(np.uint16))
                eq = torch.tensor([int(mine == digest[0])], device=dev if nccl else "cpu")
                dist.all_reduce(eq, op=dist.ReduceOp.MIN)
                ok = bool(eq.item())
            sc.close()
            del sc
            free()
            if rank == 0:                                       # in core, one process
                kt = fastk.read_ktab(raw)
                t0 = time.perf_counter()
                with hetmers.Scan(kt) as s:
                    t1 = time.perf_counter()
                    s.condition(LCUT, True, True)
                    t2 = time.perf_counter()
                r["in_core"] = {"ms_create": (t1 - t0) * 1e3, "ms_condition": (t2 - t1) * 1e3}
            free()
            t0 = time.perf_counter()                            # condition_kmer_table, then from_ktab of its table
            if rank == 0:
                with hetmers.Scan(fastk.read_ktab(raw)) as s:
                    st = s.condition_files(cond, LCUT, True, True)
            dist.barrier()
            t1 = time.perf_counter()
            sc = hd.ShardedScan.from_ktab(cond)
            torch.cuda.synchronize(dev)
            dist.barrier()
            t2 = time.perf_counter()
            r["files"] = {"ms_condition_files": (t1 - t0) * 1e3, "ms_from_ktab": (t2 - t1) * 1e3,
                          "ms": (t2 - t0) * 1e3}
            if rank == 0:
                r["files"]["condition_files"] = {k: st[k] for k in ("ms_total", "ms_write", "peak_bytes", "nels_out")}
            sc.close()
            del sc
            say(f"round {i}: {json.dumps(r)}")
            if i >= a.warmup:
                for k, v in r.items():
                    rounds[k].append(v)
        every = [None] * world
        dist.all_gather_object(every, rounds)
        if rank == 0:
            line = {"metric": "conditioning a canonical untrimmed table across the ranks vs in core vs to files",
                    "unit": "ms", "nels_in": n, "k": K, "L": LCUT, "world": world,
                    "backend": "nccl" if nccl else "gloo (ranks share GPU 0)", "steps": a.steps, "warmup": a.warmup,
                    "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
                    "per_rank": [{"shard": rr["shard"], "files": rr["files"]} for rr in every],
                    "in_core": rounds["in_core"], "replicas_equal_in_core": ok}
            print(json.dumps(line), flush=True)
    finally:
        dist.barrier()
        dist.destroy_process_group()
        if tmp is not None:
            tmp.cleanup()
    if not ok:
        sys.stderr.write("time_shard_condition.py: a replica differs from the in-core conditioned table\n")
        sys.exit(3)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Conditioning into new table files across the ranks of the one-process-per-GPU job (dist.condition_ktab, DESIGN.md
§4f) against condition_kmer_table's route in the same job (hetmers.condition_table on rank 0, one GPU), on the
canonical untrimmed k = 31 table of tools/time_condition.py (~2e8 entries, L = bench.py's LCUT = 12).  The table is
written once as FastK files to a temporary directory, and so are both outputs.  The arms alternate in every round
after `warmup` rounds; per rank: ms of each phase (load, examine, histograms and plan, per pass route / exchange /
settle / pack, writer busy, commit), the passes, peak device bytes against the planned working set, and the bytes
written.  Prints one JSON line on rank 0 with the card name and power limit; exits 3 unless both outputs have equal
content (stub index, kmer, ibyte, minval, records of all parts concatenated).  Writes nothing to the tree.

    torchrun --nproc-per-node W tools/time_rank_condition.py [--nels 2e8] [--steps 1] [--warmup 1] [--gloo]

Several ranks run NCCL when there is a GPU per rank (unless --gloo), else gloo with every rank on GPU 0 (the ranks
then share the card and their collectives go through host memory).
"""
import argparse
import hashlib
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


def content(name):
    """(kmer, ibyte, minval, entries, digest of the stub index and of the records of all parts in order)"""
    from smudgeplot_b200 import fastk
    kt = fastk.read_ktab(name, mmap=True)
    h = hashlib.sha256(np.ascontiguousarray(kt.index, dtype="<i8").tobytes())
    step = kt.pbyte * (1 << 22)
    for rec in kt.records:
        for o in range(0, rec.size, step):
            h.update(np.asarray(rec[o:o + step]).tobytes())
    return kt.kmer, kt.ibyte, kt.minval, kt.nels, h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8, help="entries of the canonical untrimmed table")
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gloo", action="store_true", help="gloo with every rank on GPU 0 even with a GPU per rank")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd, fastk, hetmers
    if not torch.cuda.is_available():
        raise SystemExit("time_rank_condition.py needs a CUDA device: conditioning has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_rank_condition.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29749")
    nccl = world > 1 and torch.cuda.device_count() >= world and not a.gloo
    dev = torch.device("cuda", rank if nccl else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=world)
    tmp = tempfile.TemporaryDirectory() if rank == 0 else None

    def say(msg):
        sys.stderr.write(f"time_rank_condition[{rank}]: {msg}\n")
        sys.stderr.flush()

    def free():
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        dist.barrier()

    try:
        names = [None, None, None]
        if rank == 0:                                          # the table files (setup, untimed)
            G = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
            keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, 1, SEED, device=dev)
            keep = keys <= synth.revcomp_left(keys, K)
            names = [os.path.join(tmp.name, x) for x in ("raw", "ranks", "one")]
            synth.write_table(names[0], K, keys[keep].contiguous(), cnt[keep].contiguous(), ibyte=3, nparts=4)
            del keys, cnt, keep
            torch.cuda.empty_cache()
        dist.broadcast_object_list(names, src=0)
        raw, ranks_out, one_out = names
        n = fastk.read_ktab(raw).nels
        rounds = {"ranks": [], "one": []}
        for i in range(a.warmup + a.steps):
            r = {}
            free()
            t0 = time.perf_counter()
            st = hd.condition_ktab(raw, ranks_out, LCUT)
            dist.barrier()
            r["ranks"] = {"ms": (time.perf_counter() - t0) * 1e3, "phases": st["ms"],
                          "stats": {k: v for k, v in st.items() if k not in ("ms", "prefix_cuts", "sub_ranges")}}
            free()
            t0 = time.perf_counter()
            if rank == 0:                                       # condition_kmer_table's route: one GPU, one writer
                one = hetmers.condition_table(raw, one_out, LCUT)
                r["one"] = {"ms": (time.perf_counter() - t0) * 1e3,
                            "stats": {k: one[k] for k in ("ms_total", "ms_write", "peak_bytes", "ranges", "nels_out",
                                                          "bytes_written")}}
            dist.barrier()
            say(f"round {i}: {json.dumps(r)}")
            if i >= a.warmup:
                for k, v in r.items():
                    rounds[k].append(v)
        every = [None] * world
        dist.all_gather_object(every, rounds)
        ok = True
        if rank == 0:
            got, want = content(ranks_out), content(one_out)
            ok = got == want
            line = {"metric": "conditioning a canonical untrimmed table into files across the ranks vs on one GPU",
                    "unit": "ms", "nels_in": n, "k": K, "L": LCUT, "world": world,
                    "backend": "nccl" if nccl else "gloo (ranks share GPU 0)", "steps": a.steps, "warmup": a.warmup,
                    "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
                    "per_rank": [rr["ranks"] for rr in every], "condition_table": rounds["one"],
                    "nparts": fastk.read_ktab(ranks_out).nparts, "entries_out": got[3], "outputs_equal": ok}
            print(json.dumps(line), flush=True)
        flag = [ok]
        dist.broadcast_object_list(flag, src=0)
        ok = flag[0]
    finally:
        dist.barrier()
        dist.destroy_process_group()
        if tmp is not None:
            tmp.cleanup()
    if not ok:
        sys.stderr.write("time_rank_condition.py: the two outputs differ\n")
        sys.exit(3)


if __name__ == "__main__":
    main()

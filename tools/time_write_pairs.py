#!/usr/bin/env python3
"""extract_kmer_pairs' pair files written by the ranks of a job that streams bench.py's workload (BASELINE.json
configs[1]) under a device budget (dist.StreamedShardedScan.write_pairs, DESIGN.md §6b), next to the two other ways of
getting the same files in the same job: extract() on dst followed by the executable's writer (the records formatted
and written per label on dst's host, vectorised with numpy), and the extract_kmer_pairs executable on the table's
files (--exe).  Three quarters of the plot's pixels carry one of three labels (time_extract.label_pixels).

Per rank: write_pairs phase by phase (the listing's phases, hist_and_plan, route, all_to_all, sort, format, text_d2h,
write).  Prints one JSON line on rank 0 with the card name and power limit; exits 3 unless every way wrote the same
bytes.  Writes only under a temporary directory (--dir, default the system's).

    torchrun --nproc-per-node W tools/time_write_pairs.py --budget-gb 8 [--nels 2e8] [--exe]

Several ranks run NCCL when there is a GPU per rank, else gloo with every rank on GPU 0 (then the budget is per
rank and the ranks share the card).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED, workload_name  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_extract import label_pixels  # noqa: E402
from tools.time_stream import host_records, power_limit  # noqa: E402

LABELS = [(1, 1), (2, 1), (2, 2)]


def write_sma(pix, path):
    """the labelled pixels as a .sma (labels 1..3 -> LABELS, in order of first appearance = label order here)"""
    s, m = np.nonzero(pix)
    order = np.argsort(pix[s, m], kind="stable")
    with open(path, "w") as f:
        f.write("covB\tcovA\tfreq\tsmudge\n")
        for i in order:
            a, b = LABELS[int(pix[s[i], m[i]]) - 1]
            f.write(f"{m[i]}\t{s[i] - m[i]}\t1\t{a}A{b}B\n")


def executable_writer(recs, k, out):
    """what extract_kmer_pairs writes for a sorted record list, one file per label: print_het lines"""
    dna = np.frombuffer(b"acgt", dtype=np.uint8)
    for lab, (a, b) in enumerate(LABELS, 1):
        mine = recs[recs["smudge"] == lab]
        with open(f"{out}.{a}A{b}B.txt", "wb") as f:
            for c in range(0, len(mine), 1 << 20):
                f.write(_lines(mine[c:c + (1 << 20)], k, dna))


def _lines(r, k, dna):
    n = len(r)
    txt = np.empty((n, k + 5), dtype=np.uint8)
    p = np.arange(k)
    hi = (r["key_hi"][:, None] >> (62 - 2 * np.minimum(p, 31)).astype(np.uint64)) & np.uint64(3)
    lo = (r["key_lo"][:, None] >> (62 - 2 * (np.maximum(p, 32) - 32)).astype(np.uint64)) & np.uint64(3)
    base = dna[np.where(p < 32, hi, lo).astype(np.int64)]
    pos = r["pos"].astype(np.int64)
    col = p[None, :] + 4 * (p[None, :] > pos[:, None])        # the varying base takes 5 columns
    txt[np.arange(n)[:, None], col] = base
    i = np.arange(n)
    txt[i, pos] = ord("(")
    txt[i, pos + 1] = base[i, pos]
    txt[i, pos + 2] = ord("/")
    txt[i, pos + 3] = dna[r["alt"].astype(np.int64) & 3]
    txt[i, pos + 4] = ord(")")
    txt[:, k + 4] = ord("\n")
    return txt.tobytes()


def files_of(out):
    got = {}
    for a, b in LABELS:
        with open(f"{out}.{a}A{b}B.txt", "rb") as f:
            got[f"{a}A{b}B"] = f.read()
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget-gb", type=float, required=True, help="device budget of each rank (GB)")
    ap.add_argument("--nels", type=float, default=2e8)
    ap.add_argument("--exe", action="store_true", help="also run extract_kmer_pairs on the table's files")
    ap.add_argument("--dir", default=None, help="directory for the temporary files (every rank must see it)")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from smudgeplot_b200 import dist as hd
    from smudgeplot_b200 import hetmers
    if not torch.cuda.is_available():
        raise SystemExit("time_write_pairs.py needs a CUDA device: the hetmers path has no CPU fallback")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if "MASTER_ADDR" not in os.environ:                       # plain `python tools/time_write_pairs.py`: one rank
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29737")
    nccl = world > 1 and torch.cuda.device_count() >= world
    dev = torch.device("cuda", rank if nccl else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl" if nccl else "gloo", rank=rank, world_size=world)
    tmp = tempfile.mkdtemp(prefix="time_write_pairs.", dir=a.dir) if rank == 0 else None
    shared = [tmp]
    dist.broadcast_object_list(shared, src=0)
    tmp = shared[0]
    try:
        G = synth.calibrate_G(K, int(a.nels), PLOIDY, HET, COV, LCUT)
        keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, LCUT, SEED, device=dev)
        n = keys.numel()
        if a.exe and rank == 0:
            synth.write_table(os.path.join(tmp, "t"), K, keys, cnt, ibyte=3, nparts=4)
        ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
        del keys, cnt
        torch.cuda.empty_cache()
        budget = int(a.budget_gb * 1e9)
        sma = os.path.join(tmp, "ann.sma")

        sc = hd.StreamedShardedScan(ht, device=dev, budget=budget)
        try:
            plot = sc.scan().cpu().numpy()
            pix = label_pixels(plot)
            if rank == 0:
                write_sma(pix, sma)
            dist.barrier()
            assert np.array_equal(hetmers.read_sma(sma)[0], pix)
            tm = {}
            dist.barrier()
            t0 = time.perf_counter()
            st = sc.write_pairs(sma, os.path.join(tmp, "w"), timings=tm)
            ms_write_pairs = (time.perf_counter() - t0) * 1e3
            dist.barrier()
            tx = {}
            t0 = time.perf_counter()
            recs = sc.extract(pix, dst=0, timings=tx)
            ms_extract = (time.perf_counter() - t0) * 1e3
        finally:
            sc.close()
        mine = {"rank": rank, "device": str(dev), "write_pairs_ms": tm, "write_pairs_total_ms": ms_write_pairs,
                "stats": st, "extract_ms": tx, "extract_total_ms": ms_extract}
        every = [None] * world
        dist.all_gather_object(every, mine)
        dist.barrier()
        if rank == 0:
            t0 = time.perf_counter()
            executable_writer(recs, K, os.path.join(tmp, "x"))
            ms_writer = (time.perf_counter() - t0) * 1e3
            got, want = files_of(os.path.join(tmp, "w")), files_of(os.path.join(tmp, "x"))
            same = {"write_pairs_equals_extract_then_writer": got == want}
            ms_exe = None
            if a.exe:
                t0 = time.perf_counter()
                subprocess.run([hetmers.get_binary_path("extract_kmer_pairs"), f"-e{LCUT}",
                                f"-o{os.path.join(tmp, 'e')}", os.path.join(tmp, "t"), sma], check=True)
                ms_exe = (time.perf_counter() - t0) * 1e3
                same["write_pairs_equals_executable"] = got == files_of(os.path.join(tmp, "e"))
            ok = all(same.values())
            line = {"metric": "ms to write extract_kmer_pairs' files: write_pairs on the ranks, extract() on dst + the "
                              "executable's writer, and the executable",
                    "unit": "ms", "workload": workload_name(1), "nels": n, "world": world,
                    "backend": "nccl" if nccl else "gloo", "gpu": torch.cuda.get_device_name(dev),
                    "power_limit": power_limit(), "budget_bytes": budget, "records": int(st["records"]),
                    "file_bytes": sum(len(v) for v in got.values()),
                    "write_pairs_ms": max(r["write_pairs_total_ms"] for r in every),
                    "extract_then_writer_ms": max(r["extract_total_ms"] for r in every) + ms_writer,
                    "writer_ms": ms_writer, "executable_ms": ms_exe, "ranks": every, "parity": same, "ok": ok}
            print(json.dumps(line), flush=True)
            if not ok:
                sys.stderr.write("time_write_pairs.py: the ways wrote different files\n")
                sys.exit(3)
    finally:
        dist.barrier()
        if rank == 0:
            import shutil
            shutil.rmtree(tmp, ignore_errors=True)
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

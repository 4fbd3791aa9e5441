#!/usr/bin/env python3
"""BASELINE configs[3] / configs[4] at full size (run under torchrun, one rank per GPU).

  --mode files   configs[3]: the synthetic triploid 2e9-k-mer k=31 table (cov 60, L=12, seed 4) is generated in
                 shards on the GPUs, written as a FastK table with one part file per rank to /dev/shm, and
                 then scanned files -> .smu by our drop-in executable (HETMERS_GPUS=N and 1) and by the
                 unmodified reference binary (-T min(cores,64)) on the same files; .smu compared byte-wise.
  --mode device  configs[4]: the tetraploid 4.4e9-k-mer table (het 2 %, cov 80, L=10, seed 5; >= 2^32 entries:
                 64-bit offsets everywhere) is generated on the GPUs and scanned device-resident with the
                 sharded symmetric scan over all N ranks, again over an independent second sharding (the
                 first N/2 ranks), and with the direct passes when their buffers fit beside the replica
                 (on 80 GB GPUs they do not at the default size: the record then says so and all_equal
                 covers the two symmetric scans); the plots must be equal.
Rank 0 prints one JSON record (and writes it to --out)."""
import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smudgeplot_b200 import _lib, fastk, hetmers  # noqa: E402
from smudgeplot_b200 import dist as hd  # noqa: E402
from tools import synth  # noqa: E402


def write_shard_files(name, k, keys, cnt, rank, world, dev):
    """this rank's sorted shard -> part file rank+1; rank 0 also writes the stub (index = all-reduced bucket counts)"""
    kb, ib = (k + 3) // 4, 3
    hb = kb - ib
    pre = (keys >> 40) & 0xFFFFFF
    counts = torch.bincount(pre, minlength=1 << 24)
    dist.all_reduce(counts)
    n = keys.numel()
    t0 = time.perf_counter()
    rec = torch.empty((n, hb + 2), dtype=torch.uint8, device=dev)
    for j in range(ib, kb):
        rec[:, j - ib] = ((keys >> (56 - 8 * j)) & 0xFF).to(torch.uint8)
    rec[:, hb] = (cnt & 0xFF).to(torch.uint8)
    rec[:, hb + 1] = ((cnt >> 8) & 0xFF).to(torch.uint8)
    h = rec.cpu().numpy()
    del rec
    with open(fastk.part_path(name, rank + 1), "wb") as f:
        f.write(struct.pack("<iq", k, n))
        h.tofile(f)
    if rank == 0:
        index = torch.cumsum(counts, 0).cpu().numpy().astype("<i8")
        with open(fastk.stub_path(name), "wb") as f:
            f.write(struct.pack("<4i", k, world, 1, ib))
            index.tofile(f)
    dist.barrier()
    return time.perf_counter() - t0


def timed(cmd, env=None, stdin="n\n"):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, input=stdin, capture_output=True, text=True, env=env)
    return time.perf_counter() - t0, r


def stats_of(r):
    for ln in r.stderr.splitlines():
        if ln.startswith("{"):
            try:
                return json.loads(ln)
            except Exception:
                pass
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["files", "device"], required=True)
    ap.add_argument("--nels", type=float, default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-reference", action="store_true")
    ap.add_argument("--dir", default="/dev/shm")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
    cpu_group = dist.new_group(backend="gloo")      # waits that must not occupy the GPUs (executables run meanwhile)
    rec = {"mode": a.mode, "n_gpus": world}
    if a.mode == "files":
        k, P, het, cov, L, seed = 31, 3, 0.01, 60.0, 12, 4
        target = int(a.nels or 2e9)
    else:
        k, P, het, cov, L, seed = 31, 4, 0.02, 80.0, 10, 5
        target = int(a.nels or 4.4e9)
    G = synth.calibrate_G(k, target, P, het, cov, L)
    rec["config"] = {"k": k, "ploidy": P, "het": het, "cov": cov, "L": L, "seed": seed, "target_nels": target, "G": G}
    t0 = time.perf_counter()
    rng = hd.prefix_partition(world)[rank]
    keys, cnt = synth.synth_table(k, G, P, het, cov, L, seed, device=dev, key_range=rng)
    torch.cuda.synchronize()
    rec["gen_s"] = time.perf_counter() - t0

    if a.mode == "files":
        d = os.path.join(a.dir, f"hetmers_full_{os.getpid() if rank == 0 else 0}")
        box = [d]
        dist.broadcast_object_list(box, src=0)
        d = box[0]
        if rank == 0:
            os.makedirs(d, exist_ok=True)
        dist.barrier()
        name = os.path.join(d, "c3")
        rec["write_s"] = write_shard_files(name, k, keys, cnt, rank, world, dev)
        nloc = torch.tensor([keys.numel()], dtype=torch.int64, device=dev)
        dist.all_reduce(nloc)
        rec["nels"] = int(nloc.item())
        del keys, cnt
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        dist.barrier(cpu_group)
        if rank == 0:
            threads = min(len(os.sched_getaffinity(0)), 64)
            exe = hetmers.get_binary_path("hetmers")
            runs = {}
            for g in (world, 1):
                for rep in range(2):
                    out = os.path.join(d, f"gpu{g}")
                    if os.path.exists(out + ".smu"):
                        os.remove(out + ".smu")
                    env = dict(os.environ, HETMERS_STATS="1", HETMERS_GPUS=str(g))
                    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "CUDA_VISIBLE_DEVICES"):
                        env.pop(v, None)
                    dt, r = timed([exe, f"-e{L}", f"-T{threads}", f"-o{out}", name], env)
                    runs.setdefault(f"ours_{g}gpu", []).append({"wall_s": dt, "rc": r.returncode, "stats": stats_of(r),
                                                                 "err": r.stderr[-300:] if r.returncode else ""})
            rec["runs"] = runs
            rec["smu_1gpu_vs_ngpu"] = open(os.path.join(d, "gpu1.smu")).read() == open(os.path.join(d, f"gpu{world}.smu")).read()
            ref = os.path.join(ROOT, "oracle", "_ref", "hetmers")
            if os.path.exists(ref) and not a.skip_reference:
                out = os.path.join(d, "ref")
                dt, r = timed([ref, f"-e{L}", f"-T{threads}", f"-o{out}", name])
                rec["reference"] = {"wall_s": dt, "rc": r.returncode, "threads": threads, "err": r.stderr[-300:] if r.returncode else ""}
                if r.returncode == 0:
                    rec["smu_identical_to_reference"] = open(out + ".smu").read() == open(os.path.join(d, f"gpu{world}.smu")).read()
                    best = min(x["wall_s"] for x in runs[f"ours_{world}gpu"])
                    rec["speedup_wall_ngpu"] = dt / best
                    rec["speedup_wall_1gpu"] = dt / min(x["wall_s"] for x in runs["ours_1gpu"])
            import shutil
            shutil.rmtree(d, ignore_errors=True)
    else:
        cnt16 = cnt.to(torch.int16)
        del cnt
        kf, cf, lo, hi = hd.gather_table(keys, cnt16)
        del keys, cnt16
        torch.cuda.empty_cache()
        rec["nels"] = int(kf.numel())
        rec["idx64"] = bool(kf.numel() >= 0xFFFFFFF0)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def run_job(job, reps=3):
            ms = []
            for _ in range(reps):
                torch.cuda.synchronize()
                dist.barrier(job.group)
                ev[0].record()
                p = job.scan()
                ev[1].record()
                torch.cuda.synchronize()
                ms.append(ev[0].elapsed_time(ev[1]))
            ok = job.symm_ok()
            return p.clone(), ms, ok

        job = hd.ShardedScan(k, kf, cf, lo, hi)
        rec["symmetric"] = bool(job.symmetric)
        pa, ms, ok = run_job(job)
        t = torch.tensor([min(ms)], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        rec["scan_all_ranks"] = {"path": job.path, "ms": float(t.item()), "status_clean": ok, "pairs": int(pa.sum()),
                                 "kmers_per_s": kf.numel() / (float(t.item()) * 1e-3), "offsets": job.offsets}
        job.close()
        del job
        torch.cuda.empty_cache()
        # independent second sharding: the first world/2 ranks (every rank holds the full replica)
        half = max(world // 2, 1)
        g2 = dist.new_group(list(range(half)))
        same2 = True
        if rank < half:
            n = kf.numel()
            j2 = hd.ShardedScan(k, kf, cf, (n * rank) // half, (n * (rank + 1)) // half, group=g2)
            pb, ms2, ok2 = run_job(j2)
            same2 = bool(torch.equal(pa, pb)) and ok2
            rec["scan_half_ranks"] = {"path": j2.path, "ranks": half, "ms": min(ms2), "equal_to_all_ranks": same2}
            j2.close()
            del j2, pb
            torch.cuda.empty_cache()
        dist.barrier()
        # the direct passes on the same replica (uint64 instantiations of pass 1 / pass 2)
        os.environ["HETMERS_PATH"] = "direct"
        try:
            j3 = hd.ShardedScan(k, kf, cf, lo, hi)
            pc, ms3, _ = run_job(j3, reps=2)
            t3 = torch.tensor([min(ms3)], dtype=torch.float64, device=dev)
            dist.all_reduce(t3, op=dist.ReduceOp.MAX)
            rec["scan_direct_all_ranks"] = {"path": j3.path, "ms": float(t3.item()), "exchange": j3.exchange,
                                            "equal_to_symmetric": bool(torch.equal(pa, pc))}
            j3.close()
        except Exception as e:                       # noqa: BLE001
            oom = isinstance(e, torch.cuda.OutOfMemoryError) or "out of memory" in str(e)
            rec["scan_direct_all_ranks"] = {"skipped" if oom else "error": repr(e)[:300]}
        flag = torch.tensor([int(same2)], dtype=torch.int32, device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        direct = rec["scan_direct_all_ranks"]
        rec["all_equal"] = bool(flag.item()) and ("skipped" in direct or bool(direct.get("equal_to_symmetric", False)))
    if rank == 0:
        print(json.dumps(rec), flush=True)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(rec, f, indent=1)
    dist.barrier(cpu_group)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

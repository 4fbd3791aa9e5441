#!/usr/bin/env python3
"""Conditioning to table files on one GPU against G GPUs of one process (hm_set_condition_gpus, DESIGN.md §4d), on
the canonical untrimmed k = 31 table of tools/time_condition.py (~2e8 entries), at the default budget and at
--budget-gb (from a streamed scan).  With G GPUs visible the G arm scans and conditions on devices 0..G-1 (in core at
the default budget, streamed at --budget-gb); on a one-GPU box it runs --shards streamed shards on device 0 listed
that many times, which exercises the split and the positional writes but not several GPUs.
Per arm: histogram pass, range passes, writer threads busy (summed and the slowest), peak device bytes per GPU, the
whole call.  The arms alternate after --warmup rounds; in the first round every arm's files are hashed, and the run
exits 3 unless all arms wrote the same bytes.  Prints one JSON line with the card, its power limit and the
filesystem of --dir; the table files go to a temporary directory there, removed afterwards.

    python tools/time_condition_gpus.py [--nels 2e8] [--budget-gb 1.6] [--shards 2] [--steps 2] [--warmup 1] [--dir /tmp]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import COV, HET, K, LCUT, PLOIDY, SEED  # noqa: E402
from smudgeplot_b200 import _lib  # noqa: E402
from tools import synth  # noqa: E402
from tools.time_stream import host_records, power_limit  # noqa: E402


def filesystem(path):
    """the type and device of the mount holding path (/proc/mounts)"""
    path, best = os.path.realpath(path), ("?", "?", "")
    try:
        for line in open("/proc/mounts"):
            dev, mnt, typ = line.split()[:3]
            if (path == mnt or path.startswith(mnt.rstrip("/") + "/")) and len(mnt) >= len(best[2]):
                best = (typ, dev, mnt)
    except OSError:
        pass
    return {"type": best[0], "device": best[1], "mount": best[2]}


def digest(work):
    h = hashlib.sha256()
    for f in sorted(os.listdir(work)):
        h.update(f.encode())
        with open(os.path.join(work, f), "rb") as fh:
            for block in iter(lambda: fh.read(1 << 24), b""):
                h.update(block)
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8, help="entries of the canonical untrimmed table")
    ap.add_argument("--budget-gb", type=float, default=1.6)
    ap.add_argument("--shards", type=int, default=2, help="streamed shards on device 0 when one GPU is visible")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_condition_gpus.py needs a CUDA device: conditioning has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    G = torch.cuda.device_count()
    G = min(G, _lib.COND_MAX_GPUS)
    genome = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
    keys, cnt = synth.synth_table(K, genome, PLOIDY, HET, COV, 1, SEED, device=dev)
    keep = keys <= synth.revcomp_left(keys, K)
    keys, cnt = keys[keep].contiguous(), cnt[keep].contiguous()
    n = keys.numel()
    ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
    del keys, cnt, keep
    torch.cuda.empty_cache()
    L = _lib.lib()
    work = tempfile.mkdtemp(prefix="time_condition_gpus.", dir=a.dir)
    budget = int(a.budget_gb * 1e9)
    several = list(range(G)) if G > 1 else [0] * a.shards
    # (name, devices, condition GPUs, budget, streamed)
    arms = [("1gpu_default", [0], 1, 0, False), (f"{len(several)}gpu_default", several, len(several), 0, G == 1),
            (f"1gpu_{a.budget_gb:g}GB", [0], 1, budget, True),
            (f"{len(several)}gpu_{a.budget_gb:g}GB", several, len(several), budget, True)]

    def run(devices, gpus, b, streamed, check):
        h = C.c_void_p()
        arr = (C.c_int * len(devices))(*devices)
        if streamed:
            os.environ["HETMERS_STREAM"] = "1"
        try:
            _lib.check(L.hm_scan_create(C.byref(ht), arr, len(devices), C.byref(h)))
        finally:
            os.environ.pop("HETMERS_STREAM", None)
        st = _lib.ConditionStats()
        t0 = time.perf_counter()
        try:
            L.hm_set_device_budget(b)
            L.hm_set_condition_gpus(gpus)
            _lib.check(L.hm_scan_condition_files(h, LCUT, 1, 1, os.path.join(work, "cond").encode(), C.byref(st)))
        finally:
            t1 = time.perf_counter()
            L.hm_set_device_budget(0)
            L.hm_set_condition_gpus(1)
            L.hm_scan_destroy(h)
        d = st.as_dict()
        d["ms_call_host"] = (t1 - t0) * 1e3
        d["sha256"] = digest(work) if check else None
        for f in os.listdir(work):
            os.remove(os.path.join(work, f))
        return d

    def say(msg):
        sys.stderr.write(f"time_condition_gpus: {msg}\n")
        sys.stderr.flush()

    say(f"{n} canonical entries, {G} GPUs visible, arms {[x[0] for x in arms]}")
    runs = {x[0]: [] for x in arms}
    digests = {}
    try:
        for i in range(a.warmup + a.steps):
            for name, devices, gpus, b, streamed in arms:
                r = run(devices, gpus, b, streamed, i == 0)
                say(f"round {i}: {name}: {r}")
                if i == 0:
                    digests[name] = r["sha256"]
                if i >= a.warmup:
                    runs[name].append(r)
    finally:
        shutil.rmtree(work, ignore_errors=True)

    def mean(rs, key):
        return sum(x[key] for x in rs) / len(rs)

    line = {"metric": "conditioning to table files: one GPU against several", "unit": "ms", "nels_in": n, "k": K,
            "L": LCUT, "steps": a.steps, "warmup": a.warmup, "gpu": torch.cuda.get_device_name(0),
            "gpus_visible": G, "power_limit": power_limit(), "filesystem": filesystem(work),
            "record_bytes": int(h_rec.numel()), "stub_index_bytes": int(h_idx.numel()) * 8,
            "several_gpus_measured": G > 1}
    for name, devices, gpus, b, streamed in arms:
        rs = runs[name]
        last = rs[-1]
        line[name] = {"devices": devices, "streamed": streamed, "ms_hist": mean(rs, "ms_hist"),
                      "ms_ranges": mean(rs, "ms_ranges"), "ms_writer_busy_sum": mean(rs, "ms_write"),
                      "ms_writer_busy_max": mean(rs, "ms_write_max"), "ms_total": mean(rs, "ms_total"),
                      "ms_total_each": [x["ms_total"] for x in rs], "ranges": last["ranges"],
                      "gpu_peak_bytes": last["gpu_peak_bytes"], "budget_bytes": last["budget_bytes"],
                      "gb_read_pcie": last["bytes_read"] / 1e9, "gb_written": last["bytes_written"] / 1e9,
                      "nels_out": last["nels_out"]}
    ok = len(set(digests.values())) == 1
    line["same_files"] = ok
    print(json.dumps(line), flush=True)
    if not ok:
        sys.stderr.write(f"time_condition_gpus.py: the arms wrote different files: {digests}\n")
        sys.exit(3)


if __name__ == "__main__":
    main()

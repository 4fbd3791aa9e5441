#!/usr/bin/env python3
"""Conditioning to table files (hm_scan_condition_files, DESIGN.md §4d) against the in-core hm_scan_condition, on a
canonical untrimmed synthetic table the size of bench.py's workload (BASELINE.json configs[1]: ~2e8 entries, k = 31):
wall clock per phase, ranges and passes, GB read over PCIe and GB written, at the default budget (from an in-core scan)
and at --budget-gb (from a streamed scan, as for a table larger than the GPU: an explicit budget also covers what the
scan holds, which for a streamed scan is a few MB).
Runs alternate between the arms after --warmup rounds.  Prints one JSON line with the card name and power limit;
exits 3 unless the written table has as many entries as the in-core result.  The table files go to a temporary
directory (--dir), removed afterwards.

    python tools/time_condition.py [--nels 2e8] [--budget-gb 1.6] [--steps 2] [--warmup 1] [--dir /tmp]
"""
import argparse
import ctypes as C
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nels", type=float, default=2e8, help="entries of the canonical untrimmed table")
    ap.add_argument("--budget-gb", type=float, default=1.6)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dir", default=None, help="where the table files are written (a temporary directory)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_condition.py needs a CUDA device: conditioning has no CPU fallback")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    # untrimmed (counts from 1), canonical strand only: what FastK writes
    G = synth.calibrate_G(K, int(2 * a.nels), PLOIDY, HET, COV, 1)
    keys, cnt = synth.synth_table(K, G, PLOIDY, HET, COV, 1, SEED, device=dev)
    keep = keys <= synth.revcomp_left(keys, K)
    keys, cnt = keys[keep].contiguous(), cnt[keep].contiguous()
    n = keys.numel()
    ht, h_rec, h_idx = host_records(torch, dev, keys, cnt)
    del keys, cnt, keep
    torch.cuda.empty_cache()
    L = _lib.lib()
    devs = (C.c_int * 1)(0)
    work = tempfile.mkdtemp(prefix="time_condition.", dir=a.dir)
    budgets = {"default": 0, f"{a.budget_gb:g}GB": int(a.budget_gb * 1e9)}

    def in_core():
        h = C.c_void_p()
        t0 = time.perf_counter()
        _lib.check(L.hm_scan_create(C.byref(ht), devs, 1, C.byref(h)))
        t1 = time.perf_counter()
        m = C.c_int64()
        try:
            _lib.check(L.hm_scan_condition(h, LCUT, 1, 1, C.byref(m)))
        finally:
            L.hm_scan_destroy(h)
        t2 = time.perf_counter()
        return {"ms_create": (t1 - t0) * 1e3, "ms_condition": (t2 - t1) * 1e3, "nels_out": m.value}

    def to_files(budget):
        h = C.c_void_p()
        dst = os.path.join(work, "cond")
        t0 = time.perf_counter()
        if budget:
            os.environ["HETMERS_STREAM"] = "1"
        try:
            _lib.check(L.hm_scan_create(C.byref(ht), devs, 1, C.byref(h)))
        finally:
            os.environ.pop("HETMERS_STREAM", None)
        t1 = time.perf_counter()
        st = _lib.ConditionStats()
        try:
            L.hm_set_device_budget(budget)
            _lib.check(L.hm_scan_condition_files(h, LCUT, 1, 1, dst.encode(), C.byref(st)))
        finally:
            L.hm_set_device_budget(0)
            L.hm_scan_destroy(h)
        d = st.as_dict()
        d["ms_create"] = (t1 - t0) * 1e3
        for f in os.listdir(work):
            os.remove(os.path.join(work, f))
        return d

    def say(msg):
        sys.stderr.write(f"time_condition: {msg}\n")
        sys.stderr.flush()

    say(f"{n} canonical entries, {len(budgets)} budgets")
    runs = {"in_core": []}
    runs.update({k: [] for k in budgets})
    try:
        for i in range(a.warmup + a.steps):
            r = {"in_core": in_core()}
            say(f"round {i}: in core {r['in_core']}")
            for name, b in budgets.items():
                r[name] = to_files(b)
                say(f"round {i}: files at {name}: {r[name]}")
            if i >= a.warmup:
                for k, v in r.items():
                    runs[k].append(v)
    finally:
        shutil.rmtree(work, ignore_errors=True)

    def mean(rs, key):
        return sum(x[key] for x in rs) / len(rs)

    ic = runs["in_core"]
    line = {"metric": "conditioning a canonical untrimmed table: in core vs to table files", "unit": "ms",
            "nels_in": n, "k": K, "L": LCUT, "steps": a.steps, "warmup": a.warmup,
            "gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(),
            "record_bytes": int(h_rec.numel()), "stub_index_bytes": int(h_idx.numel()) * 8,
            "in_core": {"ms_create": mean(ic, "ms_create"), "ms_condition": mean(ic, "ms_condition"),
                        "nels_out": ic[-1]["nels_out"]}}
    ok = True
    for name in budgets:
        rs = runs[name]
        last = rs[-1]
        ok = ok and last["nels_out"] == ic[-1]["nels_out"]
        line[f"files_{name}"] = {
            "ms_create": mean(rs, "ms_create"), "ms_hist": mean(rs, "ms_hist"), "ms_ranges": mean(rs, "ms_ranges"),
            "ms_write_thread": mean(rs, "ms_write"), "ms_total": mean(rs, "ms_total"),
            "ranges": last["ranges"], "passes": last["passes"], "peak_device_bytes": last["peak_bytes"],
            "budget_bytes": last["budget_bytes"],
            "gb_read_pcie": last["bytes_read"] / 1e9, "gb_written": last["bytes_written"] / 1e9,
            "nels_out": last["nels_out"]}
    line["ok"] = ok
    print(json.dumps(line), flush=True)
    if not ok:
        sys.stderr.write("time_condition.py: the written table's size differs from the in-core result\n")
        sys.exit(3)


if __name__ == "__main__":
    main()
